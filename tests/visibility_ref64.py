"""Float64 restatement of point visibility (include/mgs_rasterizer.h, mgs_visibility_views).

* `project`: (u, v), depth t.z and the cull of each point under a view, with flow_ref64's map of a mean (planar_ref64's
  screen_mean, every camera model) and its cull; `in_view` adds the image bounds [-0.5, W - 0.5) x [-0.5, H - 0.5).
* `transmittance`: T = prod (1 - alpha_i) over the instances of the point's 16x16 tile with depth z_i < d, in the view's
  tile-list order, with blend_ref64's constants (0.99 clamp, 1/255 cut, 1e-4 stop) and its alpha expression evaluated at the
  continuous (u, v).  The view's projected and sorted state (ranges, point_list, means2D, conic_opacity, depths) is an input,
  as in blend_ref64.  Each point also gets a `border` flag where fp32 may decide differently: alpha within a band of 1/255,
  power within a band of 0, z_i within a band of d, T within a band of 1e-4, or u + 0.5 / v + 0.5 within a band of a tile
  edge.
"""
import numpy as np
import torch

import blend_ref64 as R64
import flow_ref64 as F64

BAND = 1e-5    # relative width of the alpha, power and depth decision bands (fp32 rounding of a few operations and expf)
T_BAND = 1e-4  # relative width of the stop's band (the running product drifts by about one rounding per factor)


def project(points, view):
    """(uv [Q,2], depth [Q], ok [Q]) of float64 points [Q,3] under a planar_ref64 view dict; uv and depth NaN where the cull
    fails"""
    p = torch.as_tensor(np.asarray(points, np.float64))
    ok = F64.valid(p, view).numpy()
    uv = F64.screen_mean(p, view).detach().numpy()
    z = F64.view_space(p, view)[:, 2].detach().numpy()
    uv[~ok] = np.nan
    z = np.where(ok, z, np.nan)
    return uv, z, ok


def in_view(uv, ok, W, H):
    u, v = uv[:, 0], uv[:, 1]
    with np.errstate(invalid="ignore"):
        return ok & (u >= -0.5) & (u < W - 0.5) & (v >= -0.5) & (v < H - 0.5)


def tile_of(uv, W, H):
    """the tile of pixel (floor(u + 0.5), floor(v + 0.5)), the pixel clamped into the image"""
    gx = (W + 15) // 16
    ix = np.minimum(np.floor(uv[:, 0] + 0.5), W - 1).astype(np.int64)
    iy = np.minimum(np.floor(uv[:, 1] + 0.5), H - 1).astype(np.int64)
    return (iy // 16) * gx + ix // 16


def transmittance(st, uv, d, inside):
    """(T [Q], border [Q]) of points at uv [Q,2] with depth d [Q]; T = 1 where `inside` is False"""
    Q = len(d)
    T = np.ones(Q)
    border = np.zeros(Q, bool)
    W, H = st["W"], st["H"]
    tiles = tile_of(np.where(inside[:, None], uv, 0.0), W, H)
    for q in np.nonzero(inside)[0]:
        u, v = float(uv[q, 0]), float(uv[q, 1])
        for c in (u + 0.5, v + 0.5):
            r = c % 16.0
            border[q] |= min(r, 16.0 - r) <= 1e-3
        r0, r1 = (int(x) for x in st["ranges"][tiles[q]])
        ids = st["point_list"][r0:r1].astype(np.int64)
        z = st["depths"][ids].astype(np.float64)
        border[q] |= bool(np.isfinite(d[q]) and np.any(np.abs(z - d[q]) <= BAND * abs(d[q])))
        ids = ids[z < d[q]]
        m = st["means2D"][ids].astype(np.float64)
        co = st["conic_opacity"][ids].astype(np.float64)
        dx, dy = m[:, 0] - u, m[:, 1] - v
        a, b, c, o = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
        power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
        mag = 0.5 * (np.abs(a) * dx * dx + np.abs(c) * dy * dy) + np.abs(b * dx * dy)
        alpha = np.minimum(R64.ALPHA_MAX, o * np.exp(power))
        ok = (power <= 0) & (alpha >= R64.ALPHA_MIN)
        near = (np.abs(power) <= BAND * mag) | (np.abs(alpha - R64.ALPHA_MIN) <= BAND * R64.ALPHA_MIN)
        # the running product over the accepted pairs; the walk ends at the first one that would take it below 1e-4
        cp = np.cumprod(np.where(ok, 1.0 - alpha, 1.0))
        stop = ok & (cp < R64.T_STOP)
        end = int(np.argmax(stop)) if stop.any() else len(ids)
        T[q] = cp[end - 1] if end > 0 else 1.0
        walked = np.arange(len(ids)) <= end
        border[q] |= bool(np.any(walked & (near | (ok & (np.abs(cp - R64.T_STOP) <= T_BAND * R64.T_STOP)))))
    return T, border



# ------------------------------------------------------------------------------------------------ bounded restatement
# `bounded` restates visibility.cu pair by pair in closed form (numpy float64, no autograd), in the kernels' operation
# order, and gives every value a first-order bound B of its fp32 evaluation in units of u = 2^-24 (project_ref64.E's
# convention: each fp32 operation adds |result| to its operands' propagated bounds).
#
# * Decisions replayed exactly in fp32 from the kernel's own uv and depth: the tile of pixel (min(floor(u + 0.5f), W - 1),
#   min(floor(v + 0.5f), H - 1)), and the cut, vis_query_kernel's lower-bound binary search of d over the fp32 depths of
#   the tile's list.  No point is excluded for a seam, the last-column clamp or a depth tie.
# * Decisions kept in a band: alpha within BAND u B of 1/255, power within BAND u B of 0, and the running product within
#   BAND u B of T_STOP (an interval over the either-side pairs' factors).  The reference takes the float64 outcome, and a
#   pair that may go either way is an either-side pair: its whole term enters an absolute bound D that KAPPA does not
#   scale (field_ref64.bounded's rule), and its rounding enters B.  For T, D spans the products over every consistent set.
# * Values: T_out (the product up to, not including, the pair that takes it below T_STOP); per point duv = -sum m dpower/dmu
#   summed in lane (list) order; per Gaussian the six blend-stage terms {dmx W/2, dmy H/2, -m dx^2 / 2, -m dx dy / 2,
#   -m dy^2 / 2, dL/do} with m = o dL/dG and dL/dalpha = -g_T T_out / (1 - alpha) (the 0.99 clamp passes the gradient;
#   under AA the opacity slot is dL/do_eff), each summed over the warp by 5 halving levels and then by one red.global.add
#   per warp item that reaches the record (items of 32 points of a tile, in id order), charged (5 + items) u |term|.
import project_ref64 as PR

f32 = np.float32
U = R64.U
BAND_U = 4.0          # a decision is either-side when its argument is within BAND_U u B of the threshold
EXP_ULP = 2.0         # expf, CUDA's bound
WARP_LEVELS = 5       # vis_halve's additions per term
GB_SLOTS = 6          # {dmx, dmy, dca, dcb, dcc, dop}
MUTATIONS = ("T_with_stop", "cut_le", "tile_floor_u", "no_inv_1ma", "clamp_masks", "b_unhalved", "duv_sign", "no_half_W")
# an element is within bound when |x - v| <= KAPPA[q] u B + D: 4x the largest (|x - v| - D) / (u B) measured against the
# kernels over every case of tests/test_visibility_ref64_gpu.py (the measured worsts are in its docstring)
KAPPA = dict(T=1.21, duv=1.24, gb=1.62)


def tile_of32(uv, W, H, mutate=()):
    """vis_points_kernel's tile of fp32 points uv [n,2] (in view): min(floor(u + 0.5f), W - 1) in fp32 arithmetic"""
    u = np.asarray(uv, f32)
    h = f32(0.0) if "tile_floor_u" in mutate else f32(0.5)
    ix = np.minimum(np.floor(u[:, 0] + h), f32(W - 1)).astype(np.int64)
    iy = np.minimum(np.floor(u[:, 1] + h), f32(H - 1)).astype(np.int64)
    return (iy // 16) * ((W + 15) // 16) + ix // 16


def cut_of(st, tiles, d, mutate=()):
    """(list start, cut) per point: vis_query_kernel's binary search for the first list entry whose fp32 depth is not < d"""
    rg = np.asarray(st["ranges"], np.int64)[tiles]
    lo, l, h = rg[:, 0], rg[:, 0].copy(), rg[:, 1].copy()
    dep = np.asarray(st["depths"], f32)
    pl = np.asarray(st["point_list"]).astype(np.int64)
    d = np.asarray(d, f32)
    while True:
        act = l < h
        if not act.any():
            break
        m = (l + h) >> 1
        z = dep[pl[np.where(act, m, 0)]]
        go = (z <= d) if "cut_le" in mutate else (z < d)
        l = np.where(act & go, m + 1, l)
        h = np.where(act & ~go, m, h)
    return lo, l - lo


def _items(tiles, q):
    """each point's warp item, numbered densely: its tile and its rank among the tile's points (ascending id) over 32"""
    order = np.lexsort((q, tiles))
    ts = tiles[order]
    rank = np.empty(len(q), np.int64)
    rank[order] = np.arange(len(q)) - np.searchsorted(ts, ts, "left")
    per = int(rank.max()) // 32 + 1 if len(q) else 1
    return np.unique(tiles * per + rank // 32, return_inverse=True)[1].reshape(-1)


def _gate(t, live, either):
    z = np.zeros_like(t.v)
    return np.where(live, t.v, z), np.where(live | either, t.e + z, z), np.where(either, np.abs(t.v), z)


def bounded(st, uv, d, inside, g_T=None, T_out=None, sel=None, mutate=(), chunk=512):
    """The visibility forward and, with a cotangent g_T [Q], the T path's backward of one view, each entry (value, B, D):
    an element x is within bound when |x - value| <= KAPPA u B + D.  `st`: the view's projected and sorted state (W, H,
    ranges, point_list, means2D, conic_opacity, depths); uv [Q,2], d [Q], inside [Q]: the kernel's fp32 outputs.  T_out
    [Q]: the forward's T the backward reads (default the reference's own).  `sel`: the points to evaluate (default every
    in-view point; the others still count in the warp items).  Returns T [Q] (1 outside the view, NaN in view but not
    evaluated), duv [Q,2], gb [P,6], `checked` (points evaluated), `pairs` (pairs walked), `either` (either-side pairs),
    `accepted` (per point the Gaussian ids of its live pairs), and per point its `cut` (0 where not evaluated), `tile` (-1
    outside the view) and
    `stop` (the list index of the pair that ends its walk below T_STOP, -1 where none does) [Q]."""
    mutate = set(mutate)
    W, H = int(st["W"]), int(st["H"])
    Q, P = len(d), len(st["means2D"])
    inside = np.asarray(inside, bool)
    uv32, d32 = np.asarray(uv, f32), np.asarray(d, f32)
    qs = np.nonzero(inside)[0]
    tiles = tile_of32(uv32[qs], W, H, mutate)
    ev = np.isin(qs, np.asarray(sel)) if sel is not None else np.ones(len(qs), bool)
    r0, cut = np.zeros(len(qs), np.int64), np.zeros(len(qs), np.int64)
    r0[ev], cut[ev] = cut_of(st, tiles[ev], d32[qs[ev]], mutate)
    item = _items(tiles, qs)
    NI = int(item.max()) + 1 if len(item) else 1
    pl = np.asarray(st["point_list"]).astype(np.int64)
    mu = np.asarray(st["means2D"], np.float64)
    co = np.asarray(st["conic_opacity"], np.float64)
    Tv, TB, TD = np.ones(Q), np.zeros(Q), np.zeros(Q)
    Tv[qs[~ev]] = np.nan
    grads = g_T is not None
    z3 = lambda *s: (np.zeros(s), np.zeros(s), np.zeros(s))  # noqa: E731
    duv, gb = z3(Q, 2), z3(P, GB_SLOTS)
    gabs = np.zeros((P, GB_SLOTS))
    keys, accepted = [], [np.zeros(0, np.int64)] * Q
    out = dict(checked=int(ev.sum()), pairs=0, either=0, cut=np.zeros(Q, np.int64), tile=np.full(Q, -1, np.int64),
               stop=np.full(Q, -1, np.int64))
    out["cut"][qs] = cut
    out["tile"][qs] = tiles
    todo = np.nonzero(ev)[0]
    for a in range(0, len(todo), chunk):
        ix = todo[a:a + chunk]
        q = qs[ix]
        L = int(cut[ix].max()) if len(ix) else 0
        if L == 0:
            continue
        k = np.arange(L)[None]
        valid = k < cut[ix][:, None]
        gid = pl[np.where(valid, r0[ix][:, None] + k, 0)]
        E = PR.E
        u, v = E(uv32[q, 0].astype(np.float64)[:, None]), E(uv32[q, 1].astype(np.float64)[:, None])
        ca, cb, cc, op = (E(co[gid, i]) for i in range(4))
        dx, dy = E(mu[gid, 0]) - u, E(mu[gid, 1]) - v
        power = (ca * dx * dx + cc * dy * dy) * -0.5 - cb * dx * dy
        ex = np.exp(power.v)
        G = E(ex, ex * (power.e + EXP_ULP))
        araw = op * G
        alpha = np.minimum(R64.ALPHA_MAX, araw.v)
        clamped = araw.v > R64.ALPHA_MAX
        ok = valid & (power.v <= 0) & (alpha >= R64.ALPHA_MIN)
        band = valid & ((np.abs(araw.v - R64.ALPHA_MIN) <= BAND_U * U * araw.e) |
                        ((np.abs(power.v) <= BAND_U * U * power.e) & (power.e > 0)))
        passes = ok | band
        onem = 1.0 - alpha
        cp = np.cumprod(np.where(ok, onem, 1.0), 1)
        r = np.cumsum(np.where(passes, araw.e / onem + 2.0, 0.0), 1)
        lower = np.cumprod(np.where(passes, onem, 1.0), 1) * (1.0 - BAND_U * U * r)
        upper = np.cumprod(np.where(ok & ~band, onem, 1.0), 1) * (1.0 + BAND_U * U * r)
        stopped = upper < R64.T_STOP                    # past the stop whatever the either-side pairs do
        live = ok & (cp >= R64.T_STOP)
        either = passes & ~stopped & (band | ~(lower >= R64.T_STOP))
        liveT = ok & (cp / np.where(ok, onem, 1.0) >= R64.T_STOP) if "T_with_stop" in mutate else live
        Tv[q] = np.prod(np.where(liveT, onem, 1.0), 1)
        hi = np.prod(np.where(live & ~either, onem, 1.0), 1)
        lo = np.prod(np.where(live | either, onem, 1.0), 1)
        TD[q] = np.maximum(np.maximum(hi - Tv[q], Tv[q] - lo), 0.0)
        TB[q] = Tv[q] * np.sum(np.where(live | either, araw.e / onem + 2.0, 0.0), 1)
        out["pairs"] += int(valid.sum())
        out["either"] += int(either.sum())
        stop = ok & (cp < R64.T_STOP)
        out["stop"][q] = np.where(stop.any(1), np.argmax(stop, 1), -1)
        for j, qq in enumerate(q):
            accepted[qq] = gid[j][live[j]]
        if not grads:
            continue
        gT = np.asarray(g_T, f32)[q].astype(np.float64)[:, None]
        Tk = (np.asarray(T_out, f32)[q].astype(np.float64) if T_out is not None else Tv[q])[:, None]
        s = E(-gT * Tk, np.abs(gT * Tk))
        dLda = s if "no_inv_1ma" in mutate else s / E(onem, araw.e + onem)
        dop = G * dLda
        m = op * dop
        gx = -(ca * dx + cb * dy)
        gy = -(cc * dy + cb * dx)
        lv = live & ~clamped if "clamp_masks" in mutate else live
        le = live | either
        # duv: the lane's running sum over its pairs in list order
        for c, gc in enumerate((gx, gy)):
            t = m * gc
            tv, te, td = _gate(t, lv, either)
            S = -np.cumsum(tv, 1)
            run = np.abs(S) + np.cumsum(td, 1)
            duv[0][q, c] = -S[:, -1] if "duv_sign" in mutate else S[:, -1]
            duv[1][q, c] = np.sum(te + np.where(le, run, 0.0), 1)
            duv[2][q, c] = np.sum(td, 1)
        hm = m * -0.5
        hb = m * -1.0 if "b_unhalved" in mutate else hm
        terms = [m * gx if "no_half_W" in mutate else E(0.5 * W) * m * gx,
                 m * gy if "no_half_W" in mutate else E(0.5 * H) * m * gy,
                 hm * dx * dx, hb * dx * dy, hm * dy * dy, dop]
        gl = gid[le]
        sent = le & (s.v != 0)                          # a lane with s = 0 walks nothing and sends nothing
        for i, t in enumerate(terms):
            tv, te, td = _gate(t, lv, either)
            gb[0][:, i] += np.bincount(gl, tv[le], P)
            gb[1][:, i] += np.bincount(gl, te[le], P)
            gb[2][:, i] += np.bincount(gl, td[le], P)
            gabs[:, i] += np.bincount(gl, np.abs(t.v)[le], P)
        keys.append(np.unique(gid[sent] * NI + np.broadcast_to(item[ix][:, None], le.shape)[sent]))
    out["T"] = (Tv, TB, TD)
    out["accepted"] = accepted
    if grads:
        nitems = np.zeros(P)
        if keys:
            g_of = np.unique(np.concatenate(keys)) // NI
            nitems = np.bincount(g_of, minlength=P).astype(np.float64)
        gb = (gb[0], gb[1] + (WARP_LEVELS + nitems)[:, None] * gabs, gb[2])
        out["duv"], out["gb"] = duv, gb
    return out


def ratio(got, ref, quantity=None):
    """|got - value| / (KAPPA[quantity] u B + D) elementwise for ref = (value, B, D): within bound when <= 1.  Without a
    quantity, the measured ratio max(|got - value| - D, 0) / (u B) from which KAPPA is set.  A zero bound asks for an
    exact element; a non-finite got is inf."""
    v, B, D = (np.asarray(x, np.float64) for x in ref)
    got = np.asarray(got, np.float64)
    err = np.abs(got - v)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.maximum(err - D, 0.0) / (U * B) if quantity is None else err / (KAPPA[quantity] * U * B + D)
    r = np.where(err == 0, 0.0, r)
    return np.where(np.isfinite(got), r, np.inf)
