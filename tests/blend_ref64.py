"""Float64 reference of the blend stage (forward and backward), with its contribution decisions as an input.

The reference takes a view's projected and sorted state as given (tile `ranges`, `point_list`, `means2D`, `conic_opacity`,
colours, depth, features) and re-does only the blend:

* `decide` evaluates the reference's rule in float64 for every (tile-list entry, pixel of the tile): `power <= 0`,
  `alpha = min(0.99, o G) >= 1/255`, stop when `T (1 - alpha) < 1e-4`.  A decision that lies inside the band the fp32
  evaluation can move (a few ulp of the quadratic's terms, of `expf` and of the running product) is *borderline*; a pixel's
  decisions after its first borderline one are unknown.  `decide_fp32` restates the C oracle's fp32 decisions instead.
* `blend` computes, from a given set of contributor masks, the images (colour, features, depth, final_T, alpha, n_contrib)
  and the blend-stage gradients in the reference's conventions (the 0.99 clamp is gradient-transparent; dL_dmeans2D carries
  the 0.5 W / 0.5 H factors; dL_dconic.y is the reference's half-weight off-diagonal term), each with a per-element bound
  from a first-order model of the reference's fp32 arithmetic.  The bounds are in units of u = 2^-24; a checked value is
  within bound when |value - ref| <= KAPPA u B + tiny.

Per tile everything is a (256 pixels x L entries) array: transmittances come from cumulative products, the suffix sums of
the backward from reversed cumulative sums.

Extra columns (columns 4..7 of the kernels' {r,g,b,depth} tile): `st["quad"]` [P,4] per-Gaussian quads blended as four more
channels without a background term and without `cot_scale`.  With `st["planar"]` false (the normal plane, the flow plane) the
cotangent planes are `st["g_quad"]` [3 or 4,H,W]; `blend` returns the plane `quad` [4,H,W] and `dL_dquad` [P,4] = w^T g_quad.
With `st["planar"]` true the quad is {a, b, e, 0} and each pair's depth is per pixel, D = z + a px + b py + e: the depth
plane is col3 + px col4 + py col5 + col6, the cotangent columns are {g px, g py, g, 0} with g the depth cotangent, so dot,
S and dL/dalpha are those of the planar depth, and `dL_dquad` = {sum w g (px - mu_x), sum w g (py - mu_y), sum w g, 0}:
dL/d(a, b) with the share of e = -(a mu_x + b mu_y) folded in, the kernels' gn, whose terms are footprint-sized wherever the
pixels lie (its bound: |px - mu_x| + 16 per term, the block-local columns and the mean's offset from the block origin).
`median_planar` adds the planar median depth and its gradient.
"""
import numpy as np

ALPHA_MAX = np.float64(np.float32(0.99))
ALPHA_MIN = np.float64(np.float32(1.0) / np.float32(255.0))
T_STOP = np.float64(np.float32(0.0001))
U = 2.0 ** -24
# Bound scale per checked quantity: 4x the largest |x - ref| / (u B) measured for that quantity over the C oracle and the
# stored outputs of the compiled reference on the four golden scenes (tests/test_blend_ref64_cpu.py) and both blend
# kernels on every scene of tests/test_blend_pairs_gpu.py (H100 SXM).  The measured ratios are in those tests' docstrings.
# dL_ddepth (w^T g_depth, the per-Gaussian depth cotangent), which the kernels keep in their blend-stage record only, is
# measured against the C oracle's blend with the depth as a feature channel (test_depth_cotangent_matches_oracle_per_element).
KAPPA = dict(color=14.5, feature=24.0, depth=11.1, final_T=7.1, alpha=2.0,
             dL_dmeans2D=0.23, dL_dconic=0.012, dL_dopacity=0.7, dL_dcolors=1.6, dL_ddepth=0.26, dL_dfeature=5.3)
# the extra columns (tests/test_blend_planes_gpu.py, measured on the near-origin scenes); planar_depth covers the planar depth
# plane, median_planar the planar median depth
KAPPA.update(normal=9.0, planar_depth=8.7, median_planar=2.6, dL_dquad=1.0)
# dL_dconic with the depth / mask heads folded into the cotangents (their term64 case: 0.0151, past the plain scenes' 0.003)
KAPPA["dL_dconic_heads"] = 0.061


def tile_pixels(W, H, tile):
    """Pixel coordinates of a 16x16 tile in (ly, lx) order, and which of them lie inside the image."""
    gx = (W + 15) // 16
    tx, ty = tile % gx, tile // gx
    ly, lx = np.divmod(np.arange(256), 16)
    px, py = tx * 16 + lx, ty * 16 + ly
    return px, py, (px < W) & (py < H)


def pixel_block_bit(lx, ly):
    """(8x4 block of the tile, bit of the pixel in that block's 32-bit mask) for tile-local pixel coordinates."""
    s = (ly // 4) * 2 + lx // 8
    return s, (lx % 8) * 4 + ly % 4


def _pairs(st, tile):
    r0, r1 = (int(v) for v in st["ranges"][tile])
    ids = st["point_list"][r0:r1].astype(np.int64)
    px, py, inside = tile_pixels(st["W"], st["H"], tile)
    m = st["means2D"][ids].astype(np.float64)
    co = st["conic_opacity"][ids].astype(np.float64)
    dx = m[None, :, 0] - px[:, None]
    dy = m[None, :, 1] - py[:, None]
    a, b, c, o = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
    mag = 0.5 * (np.abs(a) * dx * dx + np.abs(c) * dy * dy) + np.abs(b * dx * dy)
    G = np.exp(power)
    alpha = np.minimum(ALPHA_MAX, o * G)
    # relative error of the fp32 alpha, in u: dx rounding + five operations on the quadratic's terms, expf, the product
    ea = 8.0 * mag + np.where(power != 0, 2.0, 0.0) + np.where(o * G < ALPHA_MAX, 1.0, 0.0)
    return dict(ids=ids, px=px, py=py, inside=inside, dx=dx, dy=dy, a=a, b=b, c=c, o=o, power=power, mag=mag, G=G,
                alpha=alpha, ea=ea)


def decide(st, tile, band=4.0):
    """Float64 decisions of one tile.  Returns dict(mask [256,L] bool, first_border [256] (L where none),
    foot_in [256,L] (surely inside the alpha >= 1/255 footprint, whatever T does), pairs)."""
    p = _pairs(st, tile)
    L = len(p["ids"])
    alpha, power, ea = p["alpha"], p["power"], p["ea"]
    pw_band = band * 8.0 * U * p["mag"]
    al_band = band * U * ea * alpha
    pos_in = power <= -pw_band
    pos_out = power > pw_band
    a_in = alpha >= ALPHA_MIN + al_band
    a_out = alpha < ALPHA_MIN - al_band
    foot_in = pos_in & a_in
    foot_out = pos_out | a_out
    foot_border = ~(foot_in | foot_out)
    # transmittance: running product over the footprint contributors; the fp32 product drifts by (1 + ea alpha/(1-alpha)) u per step
    om = np.where(foot_in, 1.0 - alpha, 1.0)
    cp = np.cumprod(om, axis=1)
    rel = np.cumsum(np.where(foot_in, 2.0 + ea * alpha / (1.0 - alpha), 0.0), axis=1) * U * band
    stop = foot_in & (cp < T_STOP)
    t_border = foot_in & (np.abs(cp - T_STOP) <= rel * cp)
    idx = np.arange(L)[None, :]
    first_stop = np.where(stop.any(1), np.argmax(stop, 1), L)
    border = foot_border | t_border
    first_border = np.where(border.any(1), np.argmax(border, 1), L)
    # a border pair behind the stop does not matter
    first_border = np.where(first_border > first_stop, L, first_border)
    mask = foot_in & (idx < first_stop[:, None])
    mask &= p["inside"][:, None]
    first_border = np.where(p["inside"], first_border, L)
    return dict(mask=mask, first_border=first_border, foot_in=foot_in & p["inside"][:, None], pairs=p)


def decide_fp32(st, tile):
    """The C oracle's own decisions (gs_oracle.c gso_render_forward, built with -ffp-contract=off), restated in numpy float32:
    same operation order, expf correctly rounded."""
    r0, r1 = (int(v) for v in st["ranges"][tile])
    ids = st["point_list"][r0:r1].astype(np.int64)
    px, py, inside = tile_pixels(st["W"], st["H"], tile)
    f = np.float32
    m = st["means2D"][ids].astype(f)
    co = st["conic_opacity"][ids].astype(f)
    dx = m[None, :, 0] - px[:, None].astype(f)
    dy = m[None, :, 1] - py[:, None].astype(f)
    power = f(-0.5) * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy
    G = np.exp(power.astype(np.float64)).astype(f)
    alpha = np.minimum(f(0.99), co[:, 3] * G)
    ok = ~(power > 0) & ~(alpha < f(1.0) / f(255.0))
    om = np.where(ok, f(1) - alpha, f(1)).astype(f)
    cp = np.cumprod(om, axis=1, dtype=f)
    stop = ok & (cp < f(0.0001))
    L = len(ids)
    first_stop = np.where(stop.any(1), np.argmax(stop, 1), L)
    return ok & (np.arange(L)[None, :] < first_stop[:, None]) & inside[:, None]


def _nfeat(st):
    return st["feature"].shape[1] if (st.get("feature") is not None and st["feature"].ndim == 2) else 0


def _channels(st, ids):
    """[L, C] channel rows {r, g, b, depth?, features..., quad?} of the entries."""
    cols = [st["colors"][ids].astype(np.float64)]
    if st.get("depth") is not None:
        cols.append(st["depth"][ids].astype(np.float64)[:, None])
    if st.get("feature") is not None and st["feature"].ndim == 2 and st["feature"].shape[1]:
        cols.append(st["feature"][ids].astype(np.float64))
    if st.get("quad") is not None:
        cols.append(st["quad"][ids].astype(np.float64))
    return np.concatenate(cols, 1)


def _cot(st, px, py, inside):
    """[256, C] cotangents of the tile's pixels in the order of _channels, and [256] alpha cotangents."""
    x, y = np.where(inside, px, 0), np.where(inside, py, 0)
    g = [st["g_color"][:, y, x].T.astype(np.float64)]
    if st.get("depth") is not None:
        gd = st.get("g_depth")
        g.append((gd[y, x] if gd is not None else np.zeros(256))[:, None].astype(np.float64))
    if st.get("feature") is not None and st["feature"].ndim == 2 and st["feature"].shape[1]:
        g.append(st["g_feature"][:, y, x].T.astype(np.float64))
    if st.get("quad") is not None:
        if st.get("planar"):
            gd = g[1][:, 0]
            g.append(np.stack([gd * px, gd * py, gd, np.zeros(256)], 1))
        else:
            gq = np.zeros((256, 4))
            gq[:, :st["g_quad"].shape[0]] = st["g_quad"][:, y, x].T
            g.append(gq)
    ga = st.get("g_alpha")
    h = ga[y, x].astype(np.float64) if ga is not None else np.zeros(256)
    g = np.concatenate(g, 1)
    g[~inside] = 0
    h[~inside] = 0
    return g, h


def blend(st, masks, backward=True):
    """Images and blend-stage gradients in float64 from `masks` (per tile, [256, L] bool), with bounds.

    Returns dict: per pixel `color` [3,H,W], `feature` [F,H,W], `depth` [H,W], `final_T`, `alpha` [H,W], `n_contrib` [H,W]
    (1-based tile-list position of the last contributor) and `*_B` the matching bound magnitudes; per Gaussian
    `dL_dmeans2D` [P,2], `dL_dconic` [P,3] (a, b, c slots), `dL_dopacity` [P], `dL_dcolors` [P,3], `dL_dfeature` [P,F],
    and their `*_B`."""
    out = new_out(st)
    for tile in range(st["ranges"].shape[0]):
        blend_tile(st, tile, masks[tile], out, backward)
    return out


def new_out(st):
    """Zeroed result arrays of blend() for the state `st`."""
    W, H, P = st["W"], st["H"], st["means2D"].shape[0]
    F = st["feature"].shape[1] if (st.get("feature") is not None and st["feature"].ndim == 2) else 0
    out = {k: np.zeros(s) for k, s in (("color", (3, H, W)), ("color_B", (3, H, W)), ("feature", (F, H, W)),
                                       ("feature_B", (F, H, W)), ("depth", (H, W)), ("depth_B", (H, W)),
                                       ("final_T", (H, W)), ("final_T_B", (H, W)), ("alpha", (H, W)), ("alpha_B", (H, W)))}
    if st.get("quad") is not None:
        for k, s in (("quad", (4, H, W)), ("dL_dquad", (P, 4))):
            out[k] = np.zeros(s)
            out[k + "_B"] = np.zeros(s)
    out["n_contrib"] = np.zeros((H, W), np.int64)
    for k, s in (("dL_dmeans2D", (P, 2)), ("dL_dconic", (P, 3)), ("dL_dopacity", (P,)), ("dL_dcolors", (P, 3)),
                 ("dL_ddepth", (P,)), ("dL_dfeature", (P, F))):
        out[k] = np.zeros(s)
        out[k + "_B"] = np.zeros(s)
    return out


def blend_tile(st, tile, m, out, backward=True):
    """Adds one tile's pixels and per-Gaussian gradient terms (contributor mask m [256, L]) into `out` (see blend)."""
    W, H = st["W"], st["H"]
    F = st["feature"].shape[1] if (st.get("feature") is not None and st["feature"].ndim == 2) else 0
    has_d = st.get("depth") is not None
    bg = np.asarray(st["bg"], np.float64)
    nch = 3 + int(has_d)
    if m.shape[1] == 0:
        px, py, inside = tile_pixels(W, H, tile)
        x, y = px[inside], py[inside]
        out["final_T"][y, x] = 1.0
        out["color"][:, y, x] = bg[:, None]
        out["color_B"][:, y, x] = np.abs(bg)[:, None]
        return
    p = _pairs(st, tile)
    inside, px, py = p["inside"], p["px"], p["py"]
    x, y = px[inside], py[inside]
    a = np.where(m, p["alpha"], 0.0)
    ea = np.where(m, p["ea"], 0.0)
    om = 1.0 - a
    cp = np.cumprod(om, axis=1)
    Tf = cp[:, -1]
    Tb = np.concatenate([np.ones((256, 1)), cp[:, :-1]], 1)
    w = a * Tb
    step = np.where(m, 2.0 + ea * a / om, 0.0)
    relT = np.cumsum(step, 1)                 # relative error of T after each entry (u)
    relTb = relT - step
    relTf = relT[:, -1]
    C = _channels(st, p["ids"])
    vals = w @ C
    ew = ea + relTb + 2.0
    vB = (np.abs(w) * ew) @ np.abs(C)
    col = vals[:, :3] + Tf[:, None] * bg[None, :]
    colB = vB[:, :3] + Tf[:, None] * np.abs(bg)[None, :] * (relTf[:, None] + 1.0)
    out["color"][:, y, x] = col[inside].T
    out["color_B"][:, y, x] = colB[inside].T
    if has_d:
        out["depth"][y, x] = vals[inside, 3]
        out["depth_B"][y, x] = vB[inside, 3]
    if F:
        out["feature"][:, y, x] = vals[inside, nch:nch + F].T
        out["feature_B"][:, y, x] = vB[inside, nch:nch + F].T
    if st.get("quad") is not None:
        q0 = nch + F
        out["quad"][:, y, x] = vals[inside, q0:q0 + 4].T
        out["quad_B"][:, y, x] = vB[inside, q0:q0 + 4].T
        if st.get("planar"):
            # col3 + px col4 + py col5 + col6: each term's bound, plus the magnitude of every term for the products and the
            # three fp32 additions
            terms = (vals[:, 3], px * vals[:, q0], py * vals[:, q0 + 1], vals[:, q0 + 2])
            mag = sum(np.abs(t) for t in terms)
            out["depth"][y, x] = sum(terms)[inside]
            out["depth_B"][y, x] = (vB[:, 3] + px * vB[:, q0] + py * vB[:, q0 + 1] + vB[:, q0 + 2] + 4.0 * mag)[inside]
    out["final_T"][y, x] = Tf[inside]
    out["final_T_B"][y, x] = (Tf * (relTf + 1.0))[inside]
    out["alpha"][y, x] = 1.0 - Tf[inside]
    out["alpha_B"][y, x] = (Tf * (relTf + 1.0) + (1.0 - Tf))[inside]
    L = m.shape[1]
    last = np.where(m.any(1), L - np.argmax(m[:, ::-1], 1), 0)
    out["n_contrib"][y, x] = last[inside]
    if not backward:
        return
    g, h = _cot(st, px, py, inside)
    dot = g @ C.T                                   # [256, L]  c_k . g
    dabs = np.abs(g) @ np.abs(C).T
    wd = w * dot
    S = np.cumsum(wd[:, ::-1], 1)[:, ::-1] - wd     # sum over the contributors behind k
    Sabs = np.cumsum((np.abs(w) * dabs)[:, ::-1], 1)[:, ::-1] - np.abs(w) * dabs
    Bp = Tf * (g[:, :3] @ bg - h)
    Babs = Tf * (np.abs(g[:, :3]) @ np.abs(bg) + np.abs(h))
    dA = np.where(m, Tb * dot - (S + Bp[:, None]) / om, 0.0)
    dAabs = np.where(m, Tb * dabs + (Sabs + Babs[:, None]) / om, 0.0)
    # the backward rebuilds T_k from T_final: its relative error is the pixel's whole product drift; 1/(1-alpha)
    # amplifies alpha's own error by 1/(1-alpha)
    e = np.where(m, 4.0 + ea / om + relTf[:, None], 0.0)
    G, o, dx, dy = p["G"], p["o"], p["dx"], p["dy"]
    ids = p["ids"]
    dG = o * dA
    qabs = o * G * dAabs * e
    gx_ = -G * (dx * p["a"] + dy * p["b"])
    gy_ = -G * (dy * p["c"] + dx * p["b"])
    mx = np.abs(dx) + 8.0
    my = np.abs(dy) + 8.0
    acc = [("dL_dmeans2D", 0, (dG * gx_ * (0.5 * W)).sum(0), (qabs * (np.abs(p["a"]) * mx + np.abs(p["b"]) * my) * (0.5 * W)).sum(0)),
           ("dL_dmeans2D", 1, (dG * gy_ * (0.5 * H)).sum(0), (qabs * (np.abs(p["c"]) * my + np.abs(p["b"]) * mx) * (0.5 * H)).sum(0)),
           ("dL_dconic", 0, (-0.5 * G * dx * dx * dG).sum(0), (0.5 * qabs * mx * mx).sum(0)),
           ("dL_dconic", 1, (-0.5 * G * dx * dy * dG).sum(0), (0.5 * qabs * mx * my).sum(0)),
           ("dL_dconic", 2, (-0.5 * G * dy * dy * dG).sum(0), (0.5 * qabs * my * my).sum(0)),
           ("dL_dopacity", None, (G * dA).sum(0), (G * dAabs * e).sum(0))]
    for k, c, v, vb in acc:
        if c is None:
            np.add.at(out[k], ids, v)
            np.add.at(out[k + "_B"], ids, vb)
        else:
            np.add.at(out[k][:, c], ids, v)
            np.add.at(out[k + "_B"][:, c], ids, vb)
    ge = np.abs(w) * e
    np.add.at(out["dL_dcolors"], ids, w.T @ g[:, :3])
    np.add.at(out["dL_dcolors_B"], ids, ge.T @ np.abs(g[:, :3]))
    if has_d:
        np.add.at(out["dL_ddepth"], ids, w.T @ g[:, 3])
        np.add.at(out["dL_ddepth_B"], ids, ge.T @ np.abs(g[:, 3]))
    if F:
        np.add.at(out["dL_dfeature"], ids, w.T @ g[:, nch:nch + F])
        np.add.at(out["dL_dfeature_B"], ids, ge.T @ np.abs(g[:, nch:nch + F]))
    if st.get("quad") is not None:
        gq = g[:, nch + F:nch + F + 4]
        dq, dqB = w.T @ gq, ge.T @ np.abs(gq)
        if st.get("planar"):
            # relative to each pair's mean: dx = mu_x - px
            gd = np.abs(gq[:, 2])[:, None]
            dq[:, 0] = (w * gq[:, 2][:, None] * -dx).sum(0)
            dq[:, 1] = (w * gq[:, 2][:, None] * -dy).sum(0)
            dqB[:, 0] = (ge * gd * (np.abs(dx) + 16.0)).sum(0)
            dqB[:, 1] = (ge * gd * (np.abs(dy) + 16.0)).sum(0)
        np.add.at(out["dL_dquad"], ids, dq)
        np.add.at(out["dL_dquad_B"], ids, dqB)


def median_planar(st, median_id, g_median, out):
    """The median depth of each pixel's median contributor (`median_id` [H,W], -1: none) with its bound -- z, or with
    st["planar"] z + a px + b py + e -- and its gradient: `g_median` [H,W] (or None) added to that Gaussian's dL_ddepth and,
    planar, as g {px - mu_x, py - mu_y, 1, 0} to its dL_dquad in `out`.  The kernels add one term per pixel into the blend's sums with
    fp32 atomics, each rounding its running sum: n terms on a Gaussian add n (|its blend sum| + sum |g|) to the bound.
    Returns (plane, bound)."""
    H, W = median_id.shape
    py, px = np.mgrid[0:H, 0:W].astype(np.float64)
    has = median_id >= 0
    ids = np.where(has, median_id, 0)
    z = st["depth"][ids].astype(np.float64)
    planar = bool(st.get("planar"))
    q = st["quad"][ids].astype(np.float64) if planar else None
    terms = (z, q[..., 0] * px, q[..., 1] * py, q[..., 2]) if planar else (z,)
    plane = np.where(has, sum(terms), 0.0)
    B = np.where(has, 4.0 * sum(np.abs(t) for t in terms), 0.0)
    if g_median is not None:
        g = np.where(has, g_median.astype(np.float64), 0.0)
        i = ids[has]
        n = np.bincount(i, minlength=out["dL_ddepth"].shape[0]).astype(np.float64)
        cols = [(out["dL_ddepth"], out["dL_ddepth_B"], g)]
        if planar:
            mu = st["means2D"][ids].astype(np.float64)
            cols += [(out["dL_dquad"][:, c], out["dL_dquad_B"][:, c], g * f)
                     for c, f in enumerate((px - mu[..., 0], py - mu[..., 1], np.ones_like(px)))]
        for v, vB, x in cols:
            sabs = np.bincount(i, np.abs(x[has]), minlength=len(n))
            vB += n * (np.abs(v) + sabs) + sabs
            np.add.at(v, i, x[has])
    return plane, B


def masks_from_blocks(st, block_lists, pixel_masks, block_nwalk):
    """Contributor masks per tile from the kernels' per-block work lists and pixel masks (entries up to block_nwalk)."""
    out = []
    for tile in range(st["ranges"].shape[0]):
        r0, r1 = (int(v) for v in st["ranges"][tile])
        m = np.zeros((256, r1 - r0), bool)
        px, py, inside = tile_pixels(st["W"], st["H"], tile)
        for s in range(8):
            k = int(block_nwalk[tile, s])
            # a block with no pixel inside the image is never blended: its block_nwalk is not written
            if k == 0 or not inside[pixel_block_bit(np.arange(256) % 16, np.arange(256) // 16)[0] == s].any():
                continue
            pos = block_lists[s, r0:r0 + k].astype(np.int64)
            bits = pixel_masks[s, r0:r0 + k].astype(np.uint64)
            for b in range(32):
                xx, yy = b >> 2, b & 3
                lx, ly = (s & 1) * 8 + xx, (s >> 1) * 4 + yy
                m[ly * 16 + lx, pos] = ((bits >> np.uint64(b)) & np.uint64(1)).astype(bool)
        out.append(m)
    return out


def ratio(got, ref, B, quantity, kappa=None):
    """|got - ref| / (kappa u B + tiny), elementwise; kappa defaults to KAPPA[quantity] (kappa = 1: the raw ratio)."""
    k = KAPPA[quantity] if kappa is None else kappa
    return np.abs(np.asarray(got, np.float64) - ref) / (k * U * B + 1e-30)
