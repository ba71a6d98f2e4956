"""The pointwise heads on the GPU, element by element against the float64 reference with bounds (tests/heads_ref64.py):
mgs_activate / mgs_activate_backward (DESIGN row f2), mgs_loss_heads (f4), mgs_ssim / mgs_ssim_backward (f9), and the heads
fused into rasterize_views_raw / rasterize_views_backward_raw, evaluated on the kernels' own read-back images.

Every checked element must satisfy |x - v| <= KAPPA[q] u e; the per-view accumulators are checked view by view.  Worst
|x - v| / (u e) per quantity over every case of this file (H100 80GB HBM3); KAPPA (heads_ref64.KAPPA) is 4x these:
  activations  means 1.0, scales 0.99, rot 0.58, opac 0.72, feature 0.42,
               dL_scales 0.74, dL_rot 0.49, dL_opac 0.72, dL_feature 0.35
  loss heads   cot_color 0.75, cot_feature 0.38, S_rgb 0.15, S_cos 0.015
  L1 + SSIM    dS_dmu 0.16, dS_dxx 0.17, dS_dxg 0.18, sum_l1 0.097, sum_S 0.022, ssim_cot 0.48
(the largest of three runs: the accumulators are float atomics, whose order changes from run to run).  `-s` prints this run's.
"""
import numpy as np
import pytest

import heads_ref64 as R

pytestmark = pytest.mark.gpu

f32 = np.float32
WORST = {}
FS = [0, 1, 3, 4, 5, 31, 32, 33, 64, 128, 129, 130, 512]
SUB_EPS = [0.0, 1e-12, 5e-9, 1e-8 * (1 - 1e-6), 1e-8 * (1 + 1e-6)]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |x - v| / (u e): " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def _check(q, got, ref, skip=None, what=""):
    got = np.asarray(got, np.float64)
    assert np.isfinite(got).all(), (q, what)
    r = R.ratio(got, ref)
    if skip is not None:
        r = np.where(np.broadcast_to(skip, r.shape), 0.0, r)
    WORST[q] = max(WORST.get(q, 0.0), float(r.max(initial=0.0)))
    bad = r > R.KAPPA[q]
    if bad.any():
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        raise AssertionError(f"{q} {what}: {int(bad.sum())} of {r.size} past {R.KAPPA[q]} u e; worst {r.max():.3g} at {i}: "
                             f"got {got[i]!r}, want {R._arr(ref).v[i]!r} +- u e = {R.U * R._arr(ref).e[i]!r}")


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, f32)).cuda()


def _misaligned(a):
    """a device copy of a whose data starts 4 bytes past a 16-byte boundary (the feature rows take the scalar path)"""
    import torch
    buf = torch.empty(a.size + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(np.ascontiguousarray(a, f32).ravel()).cuda()
    return buf[1:].view(a.shape)


def _empty_like(a, off):
    import torch
    if off:
        return torch.empty(a.size + 1, dtype=torch.float32, device="cuda")[1:].view(a.shape)
    return torch.empty(a.shape, dtype=torch.float32, device="cuda")


def _ptr(t):
    return None if t is None else t.data_ptr()


# --------------------------------------------------------------------------- f2 activations
def _act_inputs(P, F, seed):
    rng = np.random.default_rng(seed)
    g = dict(means=rng.standard_normal((P, 3)), d_means=rng.standard_normal((P, 3)) * 0.1,
             rot=rng.standard_normal((P, 4)) * rng.uniform(0.2, 3, (P, 1)), d_rot=rng.standard_normal((P, 4)) * 0.1,
             scales=np.log(0.05) + rng.uniform(-0.3, 0.3, (P, 3)), d_scales=rng.standard_normal((P, 3)) * 0.01,
             opac=rng.standard_normal((P, 1)) * 3,
             feature=rng.standard_normal((P, F)) * rng.uniform(0.1, 10, (P, 1)))
    # row 0: a zero quaternion and a zero feature row; row 1: opacity +100 and a feature row of norm ~1e-7; row 2: opacity
    # -100 and log-scales at ln 0.05 (exp lands within an ulp or two of scale_max: border, unchecked)
    g["rot"][:1] = g["d_rot"][:1] = g["feature"][:1] = 0.0
    g["opac"][1:2], g["opac"][2:3] = 100.0, -100.0
    g["feature"][1:2] *= 1e-7
    g["scales"][2:3], g["d_scales"][2:3] = np.log(0.05), 0.0
    g = {k: np.asarray(v, f32) for k, v in g.items()}
    gr = dict(g_means=rng.standard_normal((P, 3)), g_rot=rng.standard_normal((P, 4)), g_scales=rng.standard_normal((P, 3)),
              g_opac=rng.standard_normal((P, 1)), g_feature=rng.standard_normal((P, F)))
    return g, {k: np.asarray(v, f32) for k, v in gr.items()}


def _run_activate(g, gr, F, off=False, scale_mode=1, opacity_mode=1, smax=0.05):
    """both kernels; -> (forward outputs, backward outputs) as numpy dicts"""
    import torch
    from manigaussian_b200 import _binding as B
    P = (g["means"] if g["means"] is not None else g["feature"]).shape[0]
    d = {k: (None if v is None else _dev(v)) for k, v in g.items()}
    gd = {k: (None if v is None else _dev(v)) for k, v in gr.items()}
    feat = gfeat = None
    if F:
        feat = _misaligned(g["feature"]) if off else d["feature"]
        gfeat = _misaligned(gr["g_feature"]) if off else gd["g_feature"]
    o = {k: torch.full(g[k].shape, float("nan"), device="cuda") for k in ("means", "rot", "scales", "opac") if g[k] is not None}
    o_feat = _empty_like(g["feature"], off) if F else None
    L, st = B.lib(), torch.cuda.current_stream().cuda_stream
    B.check(L.mgs_activate(P, F, _ptr(d["means"]), _ptr(d["d_means"]), _ptr(d["rot"]), _ptr(d["d_rot"]), _ptr(d["scales"]),
                           _ptr(d["d_scales"]), _ptr(d["opac"]), _ptr(feat), scale_mode, smax, opacity_mode, 1, 1,
                           _ptr(o.get("means")), _ptr(o.get("rot")), _ptr(o.get("scales")), _ptr(o.get("opac")), _ptr(o_feat), st),
            "mgs_activate")
    names = ("means", "d_means", "rot", "d_rot", "scales", "d_scales", "opac", "feature")
    like = ("means", "means", "rot", "rot", "scales", "scales", "opac", None)
    b = {n: (torch.full(g[lk].shape, float("nan"), device="cuda") if lk and g[lk] is not None else None)
         for n, lk in zip(names, like)}
    b["feature"] = _empty_like(g["feature"], off) if F else None
    B.check(L.mgs_activate_backward(P, F, _ptr(d["means"]), _ptr(d["d_means"]), _ptr(d["rot"]), _ptr(d["d_rot"]), _ptr(d["scales"]),
                                    _ptr(d["d_scales"]), _ptr(d["opac"]), _ptr(feat), scale_mode, smax, opacity_mode, 1, 1,
                                    _ptr(gd["g_means"]), _ptr(gd["g_rot"]), _ptr(gd["g_scales"]), _ptr(gd["g_opac"]), _ptr(gfeat),
                                    *[_ptr(b[n]) for n in names], st), "mgs_activate_backward")
    torch.cuda.synchronize()
    fw = {k: v.cpu().numpy() for k, v in o.items()}
    if F:
        fw["feature"] = o_feat.cpu().numpy()
    return fw, {k: v.cpu().numpy() for k, v in b.items() if v is not None}


def _check_activate(g, gr, F, fw, bw, what, scale_mode=1, opacity_mode=1):
    kw = dict(scale_mode=scale_mode, opacity_mode=opacity_mode)
    ref = R.activate(**g, **kw)
    rb = R.activate_backward(**g, **gr, **kw)
    if g["means"] is not None:
        _check("means", fw["means"], ref["means"], what=what)
        _check("scales", fw["scales"], ref["scales"], ref.get("border_scales"), what)
        _check("rot", fw["rot"], R.E(np.stack([q.v for q in ref["rot"]], 1), np.stack([q.e + 0 * q.v for q in ref["rot"]], 1)),
               ref["border_rot"][:, None], what)
        _check("opac", fw["opac"], ref["opac"], what=what)
        assert np.array_equal(bw["means"], gr["g_means"]) and np.array_equal(bw["d_means"], gr["g_means"]), what
        for n, q in (("scales", "dL_scales"), ("d_scales", "dL_scales"), ("opac", "dL_opac")):
            if n in bw:
                _check(q, bw[n], rb[q], rb.get("border_scales") if "scales" in n else None, what)
        rr = R.E(np.stack([q.v for q in rb["dL_rot"]], 1), np.stack([q.e + 0 * q.v for q in rb["dL_rot"]], 1))
        _check("dL_rot", bw["rot"], rr, rb["border_rot"][:, None], what)
        _check("dL_rot", bw["d_rot"], rr, rb["border_rot"][:, None], what)
    if F:
        _check("feature", fw["feature"], ref["feature"], what=what)
        _check("dL_feature", bw["feature"], rb["dL_feature"], what=what)


@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "offset4"])
@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("P", [1, 127, 128, 129])
def test_activate(P, F, off):
    g, gr = _act_inputs(P, F, P * 1000 + F)
    if not F:
        g["feature"], gr["g_feature"] = None, None
    fw, bw = _run_activate(g, gr, F, off)
    _check_activate(g, gr, F, fw, bw, f"P={P} F={F} off={off}")


@pytest.mark.parametrize("mask", range(9), ids=[f"offsets{m:03b}" for m in range(8)] + ["next_frame"])
def test_activate_offsets_and_modes(mask):
    """each of d_means, d_rot, d_scales present and absent; and the next frame's call (offsets on means and rotations,
    scales and opacities carried over: both modes 0)"""
    P, F = 129, 33
    g, gr = _act_inputs(P, F, 77 + mask)
    modes = dict(scale_mode=1, opacity_mode=1)
    if mask == 8:
        g["d_scales"] = None
        modes = dict(scale_mode=0, opacity_mode=0)
    else:
        for bit, k in enumerate(("d_means", "d_rot", "d_scales")):
            if not (mask >> bit) & 1:
                g[k] = None
    fw, bw = _run_activate(g, gr, F, **modes)
    _check_activate(g, gr, F, fw, bw, f"mask={mask}", **modes)


@pytest.mark.parametrize("P,F,off", [(600_000, 32, 0), (150_000, 128, 0), (40_000, 130, 0), (40_000, 32, 1)],
                         ids=["vec4_F32", "vec4_F128", "scalar_F130", "scalar_F32_offset4"])
def test_feature_rows_over_several_grid_stride_trips(P, F, off):
    """the feature grid is capped at 132 * 16 * 4 blocks of 128 threads: vec4 rows per trip = 8448 * 4 warps * (32 / G4) * 4,
    scalar rows per trip = 8448 * 4 warps * (32 / G); every case here takes at least two trips"""
    G = 1
    while G < (F // 4 if (F % 4 == 0 and not off) else F) and G < 32:
        G <<= 1
    per_trip = 8448 * 4 * (32 // G) * (4 if (F % 4 == 0 and not off) else 1)
    assert P > per_trip, (P, per_trip)
    rng = np.random.default_rng(P + F)
    x = (rng.standard_normal((P, F)) * rng.uniform(0.1, 10, (P, 1))).astype(f32)
    x[::1000] = 0.0
    gf = rng.standard_normal((P, F)).astype(f32)
    g = dict(means=None, d_means=None, rot=None, d_rot=None, scales=None, d_scales=None, opac=None, feature=x)
    gr = dict(g_means=None, g_rot=None, g_scales=None, g_opac=None, g_feature=gf)
    fw, bw = _run_activate(g, gr, F, off)
    for lo in range(0, P, 50_000):
        s = slice(lo, min(P, lo + 50_000))
        _check("feature", fw["feature"][s], R.activate(feature=x[s])["feature"], what=f"rows {lo}+")
        _check("dL_feature", bw["feature"][s], R.activate_backward(feature=x[s], g_feature=gf[s])["dL_feature"], what=f"rows {lo}+")


# --------------------------------------------------------------------------- f4 colour L2 + cosine embedding
def _head_inputs(V, F, N, seed, norm=1.0):
    rng = np.random.default_rng(seed)
    col = rng.uniform(-0.2, 1.2, (V, 3, N))
    tgt = rng.uniform(0, 1, (V, 3, N))
    x = rng.standard_normal((V, F, N)) * norm
    y = rng.standard_normal((V, F, N))
    special = [(0, None), (1, "zero_target"), (2, "zero_both")] + [(3 + i, n) for i, n in enumerate(SUB_EPS)]
    for i, kind in special:
        if i >= N:
            break
        if kind == "zero_target":
            y[:, :, i] = 0.0
            tgt[:, :, i] = 0.0
        elif kind == "zero_both":
            x[:, :, i] = y[:, :, i] = 0.0
            col[:, :, i] = tgt[:, :, i] = 0.0
        elif kind is None:
            x[:, :, i] = 0.0   # zero render
            col[:, :, i] = 0.0
        else:
            d = rng.standard_normal((V, F))
            x[:, :, i] = d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-30) * kind
    return [a.astype(f32) for a in (col, tgt, x, y)]


def _run_heads(col, tgt, x, y, with_feature=True):
    import torch
    from manigaussian_b200 import _binding as B
    V, F, N = x.shape
    d = [_dev(a) for a in (col, tgt, x, y)]
    cc = torch.full((V, 3, N), float("nan"), device="cuda")
    cf = torch.full((V, F, N), float("nan"), device="cuda")
    acc = torch.full((V, 2), float("nan"), device="cuda")
    emb = with_feature and F > 0
    B.check(B.lib().mgs_loss_heads(V, F, N, d[0].data_ptr(), d[2].data_ptr() if emb else None, d[1].data_ptr(),
                                   d[3].data_ptr() if emb else None, cc.data_ptr(), cf.data_ptr() if emb else None,
                                   acc.data_ptr(), torch.cuda.current_stream().cuda_stream), "mgs_loss_heads")
    torch.cuda.synchronize()
    return cc.cpu().numpy(), cf.cpu().numpy(), acc.cpu().numpy()


def _check_heads(ref, cc, cf, acc, F, what):
    _check("cot_color", cc, ref["cot_color"], what=what)
    for v in range(acc.shape[0]):
        _check("S_rgb", acc[v, 0], R.E(ref["S_rgb"].v[v], ref["S_rgb"].e[v]), what=f"{what} view {v}")
    if F:
        _check("cot_feature", cf, ref["cot_feature"], what=what)
        for v in range(acc.shape[0]):
            _check("S_cos", acc[v, 1], R.E(ref["S_cos"].v[v], ref["S_cos"].e[v]), what=f"{what} view {v}")


@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("N", [1, 255, 256, 257, 61 * 37])
@pytest.mark.parametrize("V", [1, 3])
def test_loss_heads(V, N, F):
    col, tgt, x, y = _head_inputs(V, F, N, V * 100000 + N * 10 + F)
    cc, cf, acc = _run_heads(col, tgt, x, y)
    ref = R.loss_heads(col, tgt, x if F else None, y if F else None)
    _check_heads(ref, cc, cf, acc, F, f"V={V} N={N} F={F}")
    if F and N > 8:
        # the sub-eps pixels on their own: above eps the gradient is the same under either rule
        _check("cot_feature", cf[:, :, 3:8], R.E(ref["cot_feature"].v[:, :, 3:8], ref["cot_feature"].e[:, :, 3:8]),
               what=f"V={V} N={N} F={F} sub-eps pixels")


@pytest.mark.parametrize("N", [1, 257, 61 * 37])
def test_loss_heads_without_features(N):
    col, tgt, x, y = _head_inputs(3, 8, N, N)
    cc, _, acc = _run_heads(col, tgt, x, y, with_feature=False)
    ref = R.loss_heads(col, tgt)
    _check_heads(ref, cc, None, acc, 0, f"N={N} no features")
    assert (acc[:, 1] == 0).all()


# --------------------------------------------------------------------------- f9 L1 + SSIM
SIZES = [(1, 1), (5, 7), (11, 11), (16, 32), (17, 33), (48, 96), (37, 61), (1, 300), (300, 1), (256, 256)]
SSIM_CASES = [(V, hw, "random") for hw in SIZES for V in (1, 4)] + \
             [(4, hw, k) for hw in ((1, 1), (5, 7), (17, 33), (37, 61)) for k in ("constant", "equal", "outside")]


def _ssim_images(V, H, W, kind, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-0.1, 1.1, (V, 3, H, W))
    g = rng.uniform(0, 1, (V, 3, H, W))
    if kind == "constant":
        x[:] = 0.3
        g[:] = 0.7
    elif kind == "equal":
        g = x.copy()
    elif kind == "outside":
        x = rng.uniform(-2, 3, (V, 3, H, W))
    x, g = x.astype(f32), g.astype(f32)
    if kind == "random":
        x[:, 0, ::2, ::3] = g[:, 0, ::2, ::3]
    return x, g


def seams(H, W):
    """pixels on either side of a tile seam: x = 32 k - 1, 32 k or y = 16 k - 1, 16 k (k >= 1)"""
    ys, xs = np.arange(H), np.arange(W)
    col = ((xs % R.SS_TW == 0) | (xs % R.SS_TW == R.SS_TW - 1)) & (xs > 0) & (xs < W - 1)
    row = ((ys % R.SS_TH == 0) | (ys % R.SS_TH == R.SS_TH - 1)) & (ys > 0) & (ys < H - 1)
    return row[:, None] | col[None, :]


def _check_ssim_fwd(fw, terms, acc, V, what, depth_acc=None):
    H, W = terms.shape[-2:]
    sm = seams(H, W)
    for t, q in enumerate(("dS_dmu", "dS_dxx", "dS_dxg")):
        _check(q, terms[:, t], fw[q], what=what)
        if sm.any():
            _check(q, terms[:, t][..., sm], R.E(R._arr(fw[q]).v[..., sm], R._arr(fw[q]).e[..., sm]), what=f"{what} seams")
    for v in range(V):
        _check("sum_l1", acc[v, 0], R.E(fw["sum_l1"].v[v], fw["sum_l1"].e[v]), what=f"{what} view {v}")
        _check("sum_S", acc[v, 1], R.E(fw["sum_S"].v[v], fw["sum_S"].e[v]), what=f"{what} view {v}")


@pytest.mark.parametrize("V,hw,kind", SSIM_CASES, ids=[f"V{v}-{h}x{w}-{k}" for v, (h, w), k in SSIM_CASES])
def test_ssim(V, hw, kind):
    import torch
    from manigaussian_b200 import _binding as B
    H, W = hw
    x, g = _ssim_images(V, H, W, kind, V * 7919 + H * 31 + W)
    rng = np.random.default_rng(H + W)
    scale = rng.uniform(-2, 2, (V, 2)).astype(f32)
    cot_in = rng.uniform(-1e-4, 1e-4, (V, 3, H, W)).astype(f32)
    xd, gd, sd, cd = _dev(x), _dev(g), _dev(scale), _dev(cot_in)
    terms = torch.full((V, 9, H, W), float("nan"), device="cuda")
    acc = torch.full((V, 2), float("nan"), device="cuda")
    cot = [torch.full((V, 3, H, W), float("nan"), device="cuda") for _ in range(2)]
    L, st = B.lib(), torch.cuda.current_stream().cuda_stream
    B.check(L.mgs_ssim(V, 3, H, W, xd.data_ptr(), gd.data_ptr(), terms.data_ptr(), acc.data_ptr(), st), "mgs_ssim")
    for c, ci in zip(cot, (None, cd)):
        B.check(L.mgs_ssim_backward(V, 3, H, W, xd.data_ptr(), gd.data_ptr(), terms.data_ptr(), sd.data_ptr(), _ptr(ci),
                                    c.data_ptr(), st), "mgs_ssim_backward")
    torch.cuda.synchronize()
    terms = terms.cpu().numpy().reshape(V, 3, 3, H, W)
    what = f"V={V} {H}x{W} {kind}"
    _check_ssim_fwd(R.ssim_forward(x, g), terms, acc.cpu().numpy(), V, what)
    sm = seams(H, W)
    for c, ci in zip(cot, (None, cot_in)):
        ref = R.ssim_backward(x, g, terms, scale, ci)
        got = c.cpu().numpy()
        _check("ssim_cot", got, ref, what=f"{what} cot_in={ci is not None}")
        if sm.any():
            _check("ssim_cot", got[..., sm], R.E(R._arr(ref).v[..., sm], R._arr(ref).e[..., sm]), what=f"{what} seams")


# --------------------------------------------------------------------------- the heads fused into the render
FUSED_F = [0, 1, 3, 8, 31, 32, 33, 40, 67]


def _fused(F, seed, feat_scale=None):
    """forward with the loss heads and the L1 + SSIM head, then the backward with per-view scales; -> numpy dict"""
    import torch
    from manigaussian_b200 import rasterizer as Rz
    from manigaussian_b200.gaussian_renderer import _ssim_head
    from test_clouds_gpu import _leaves
    from test_render_gpu import _cams
    V, W, H = 3, 61, 37
    host = _leaves(6000, F, seed, "sh")
    # the cloud drawn in to 40 % about the cameras' target, so that every view keeps uncovered pixels (|x| = 0) at its border
    host["xyz"] = (np.array([0.2, 0.0, 1.1]) + 0.4 * (host["xyz"] - np.array([0.2, 0.0, 1.1]))).astype(f32)
    host["scale"] = (0.4 * host["scale"]).astype(f32)
    if F and feat_scale is not None:
        host["feat"] = (host["feat"] / np.linalg.norm(host["feat"], axis=1, keepdims=True) * feat_scale).astype(f32)
    L = {k: _dev(v) for k, v in host.items()}
    cams = _cams(V, W, H)
    views = [cams.settings(i, torch.zeros(3, device="cuda"), 1, F > 0) for i in range(V)]
    rng = np.random.default_rng(seed)
    tg_rgb = _dev(rng.uniform(0, 1, (V, 3, H, W)))
    tg_emb = _dev(rng.standard_normal((V, F, H, W))) if F else None
    opts = dict(dtype=torch.float32, device="cuda")
    color = torch.empty((V, 3, H, W), **opts)
    feat = torch.empty((V, F, H, W), **opts) if F else None
    cot_rgb = torch.full((V, 3, H, W), float("nan"), **opts)
    cot_emb = torch.full((V, F, H, W), float("nan"), **opts) if F else None
    acc = torch.full((V, 2), float("nan"), **opts)
    head = _ssim_head(V, H, W, torch.device("cuda"))
    args = (views, L["xyz"], None, L.get("feat"), L["opac"], L["scale"], L["rot"], 1.0, None, L["col"], 1, F > 0)
    outs, streams = Rz.rasterize_views_raw(*args, out_buffers=(color, feat, None), loss_heads=(tg_rgb, tg_emb, cot_rgb, cot_emb, acc),
                                           ssim=head)
    torch.cuda.synchronize()
    out = dict(color=color.cpu().numpy(), tg_rgb=tg_rgb.cpu().numpy(), cot_rgb=cot_rgb.cpu().numpy(), acc=acc.cpu().numpy(),
               terms=head[0].cpu().numpy().reshape(V, 3, 3, H, W), ssim_acc=head[1].cpu().numpy()[:, :2])
    if F:
        out.update(feat=feat.cpu().numpy(), tg_emb=tg_emb.cpu().numpy(), cot_emb=cot_emb.cpu().numpy())
    cot_scale = rng.uniform(0.5, 2, (V, 2)).astype(f32)
    ssim_scale = rng.uniform(-2, 2, (V, 2)).astype(f32)
    Rz.rasterize_views_backward_raw(views, outs, streams, cot_rgb, cot_emb, L["xyz"], None, L.get("feat"), L["scale"], L["rot"], 1.0,
                                    None, L["col"], 1, F > 0, cot_scale=_dev(cot_scale), ssim=head + (color, tg_rgb),
                                    ssim_scale=_dev(ssim_scale))
    torch.cuda.synchronize()
    out.update(cot_scale=cot_scale, ssim_scale=ssim_scale, combined=head[2].cpu().numpy())
    return out


def _check_fused(o, F, what):
    V, _, H, W = o["color"].shape
    N = H * W
    flat = lambda a: a.reshape(a.shape[0], a.shape[1], -1)  # noqa: E731
    # the epilogue's warps and the loss_heads pass reduce in orders this file does not restate: any order of the view's
    # terms (3 N colour terms, N cosines) is within the bound
    ref = R.loss_heads(flat(o["color"]), flat(o["tg_rgb"]), flat(o["feat"]) if F else None, flat(o["tg_emb"]) if F else None,
                       depth=3 * N)
    _check_heads(ref, flat(o["cot_rgb"]), flat(o["cot_emb"]) if F else None, o["acc"], F, what)
    _check_ssim_fwd(R.ssim_forward(o["color"], o["tg_rgb"]), o["terms"], o["ssim_acc"], V, what)
    ref = R.ssim_backward(o["color"], o["tg_rgb"], o["terms"], o["ssim_scale"], o["cot_rgb"], o["cot_scale"][:, 0])
    _check("ssim_cot", o["combined"], ref, what=f"{what} combined colour cotangent")
    if F:
        return np.linalg.norm(o["feat"].astype(np.float64), axis=1)
    return None


@pytest.mark.parametrize("F", FUSED_F)
def test_fused_heads(F):
    """F <= 32: the heads run in the forward blend's epilogue; F > 32: the colour head there, the embedding head in a
    loss_heads pass behind the grouped blend"""
    o = _fused(F, 300 + F)
    nx = _check_fused(o, F, f"fused F={F}")
    if F:
        assert (nx == 0).any(), "no uncovered pixel (|x| = 0)"


def test_fused_heads_with_pixels_below_eps():
    """unnormalised features of norm 1e-7: faint pixels render into the (0, eps) band of the cosine head"""
    o = _fused(8, 400, feat_scale=1e-7)
    nx = _check_fused(o, 8, "fused F=8 features 1e-7")
    band = (nx > 0) & (nx <= R.COS_EPS)
    assert band.sum() >= 10, int(band.sum())
    assert (nx == 0).any()
