"""The alpha plane (accumulated opacity 1 - final_T) on the GPU: the plane itself, its gradient, and every public path that
returns it.  The gradient checks need no oracle: an alpha cotangent h alone drives the kernels exactly like the "bg trick",
a render with zero colours on a background (1, 0, 0) and colour cotangent (-h, 0, 0), because per pair both evaluate
dL/da_k = T_final h / (1 - a_k); the two differ only in the order of the float atomics."""
import numpy as np
import pytest

import util
from test_clouds_gpu import _leaves, _mk
from test_render_gpu import _cams, _cloud, _t

pytestmark = pytest.mark.gpu

GEOM = ("xyz", "rot", "scale", "opac")  # the per-Gaussian leaves an alpha gradient reaches
GRAD_NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dfeature", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
              "dL_drotations")


def _settings(cams, i, bg, sh_degree, include):
    import torch
    return cams.settings(i, torch.tensor(bg, dtype=torch.float32, device="cuda"), sh_degree, include)


def test_alpha_plane_is_one_minus_final_T_everywhere():
    """Ragged 70x45 image (partial tiles and blocks), an alpha buffer prefilled with NaN: every pixel is written, bit-identical
    to 1 - final_T of the image state, within [0, 1 - 1e-4].  A cloud that is entirely culled (empty tile lists) gives 0."""
    import torch
    from manigaussian_b200 import rasterizer as R
    W, H, V, F = 70, 45, 2, 3
    cams = _cams(V, W, H)
    for culled in (False, True):
        g = _cloud(2000, F, 61)
        xyz = _t(g["means3D"])
        if culled:  # every Gaussian far above the scene: behind both cameras, which look slightly downwards
            xyz = torch.tensor([[0.2, 0.0, 100.0]], device="cuda").expand(2000, 3).contiguous()
        views = [_settings(cams, v, (0.2, 0.4, 0.6), 1, True) for v in range(V)]
        alpha = torch.full((V, H, W), float("nan"), device="cuda")
        color = torch.empty((V, 3, H, W), device="cuda")
        feat = torch.empty((V, F, H, W), device="cuda")
        outs, _ = R.rasterize_views_raw(views, xyz, None, _t(g["feature"]), _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]), 1.0,
                                        None, _t(g["shs"]), 1, True, out_buffers=(color, feat, None, alpha), return_alpha=True)
        torch.cuda.synchronize()
        for v, o in enumerate(outs):
            assert len(o) == 8 and o[7].data_ptr() == alpha[v].data_ptr()
            addr = R.state_array("image", "final_T", o[6], W, H)
            off = addr - o[6].data_ptr()
            fT = o[6][off:off + 4 * W * H].view(torch.float32).reshape(H, W)
            a = alpha[v]
            assert torch.isfinite(a).all(), (culled, v)
            assert torch.equal(a, 1 - fT), (culled, v)
            assert float(a.min()) >= 0 and float(a.max()) <= float(np.float32(1) - np.float32(1e-4))
            if culled:
                assert not a.any()
            else:
                assert float(a.max()) > 0.5
        # the layout without alpha keeps depth at o[7]; with both, alpha follows depth
        o2, _ = R.rasterize_views_raw(views, xyz, None, _t(g["feature"]), _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]), 1.0,
                                      None, _t(g["shs"]), 1, True, return_depth=True, return_alpha=True)
        o3, _ = R.rasterize_views_raw(views, xyz, None, _t(g["feature"]), _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]), 1.0,
                                      None, _t(g["shs"]), 1, True, return_depth=True)
        assert len(o2[0]) == 9 and len(o3[0]) == 8
        for v in range(V):
            assert torch.equal(o2[v][8], alpha[v]) and torch.equal(o2[v][7], o3[v][7]) and torch.equal(o2[v][1], color[v])


def test_alpha_equals_the_red_channel_of_a_white_render():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, W, H, V = 20000, 96, 72, 3
    g = _cloud(P, 3, 62)
    cams = _cams(V, W, H)
    L = {k: _t(g[k]) for k in ("means3D", "rotations", "scales", "opacities", "shs")}
    o = render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], (0.3, 0.5, 0.7), features_color=L["shs"],
                     return_alpha=True)
    white = render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], (0.0, 0.0, 0.0),
                         pts_rgb=torch.ones(P, 3, device="cuda"))
    assert o["alpha"].shape == (V, H, W)
    assert util.rel_l2(o["alpha"].detach().cpu().numpy(), white["render"][:, 0].detach().cpu().numpy()) < 1e-5


def _alpha_only_vs_bg_trick(monkeypatch, P, F, W, H, V, seed):
    """Gradients of sum(alpha h) (SH colours, features, a coloured background) against those of the bg trick, <= 1e-6.
    The views run one after another on one stream: overlapping view streams schedule the two different workloads'
    blend CTAs differently, and at 500k Gaussians over 4 views that reordering of the atomics alone moved the scale and
    rotation gradients by up to 1.2e-6 on an H100 (serialised: 1.7e-7, the spread of two runs of one workload)."""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    monkeypatch.setenv("MGS_ONE_STREAM", "1")
    cams = _cams(V, W, H)
    host = _leaves(P, F, seed, "sh")
    h = torch.randn(V, H, W, device="cuda")
    A = _mk(host)
    oa = render_views(cams, A["xyz"], A["rot"], A["scale"], A["opac"], (0.3, 0.6, 0.9), features_color=A["col"],
                      features_language=A.get("feat"), return_alpha=True)
    (oa["alpha"] * h).sum().backward()
    B = _mk(host)
    zero = torch.zeros(P, 3, device="cuda", requires_grad=True)
    ob = render_views(cams, B["xyz"], B["rot"], B["scale"], B["opac"], (1.0, 0.0, 0.0), pts_rgb=zero, features_language=B.get("feat"))
    (ob["render"][:, 0] * -h).sum().backward()
    for k in GEOM:
        assert A[k].grad is not None and A[k].grad.abs().sum() > 0, k
        err = util.rel_l2(A[k].grad.cpu().numpy(), B[k].grad.cpu().numpy())
        assert err <= 1e-6, (k, err)
    err = util.rel_l2(oa["viewspace_points"].grad.cpu().numpy(), ob["viewspace_points"].grad.cpu().numpy())
    assert err <= 1e-6, ("means2D", err)
    # nothing but the geometry sees an alpha cotangent
    assert not A["col"].grad.any()
    if F:
        assert not A["feat"].grad.any()


@pytest.mark.parametrize("F", [0, 3, 32, 40, 64])
def test_alpha_gradient_equals_the_bg_trick(monkeypatch, F):
    """F = 40 and 64 run in channel groups of 32 (only group 0 carries the background and alpha terms)."""
    _alpha_only_vs_bg_trick(monkeypatch, 8000, F, 72, 56, 2, 70 + F)


def test_alpha_gradient_equals_the_bg_trick_at_baseline_size(monkeypatch):
    """BASELINE.json configs[2] size: 500k Gaussians, 4 views 256x256, 32 feature channels."""
    _alpha_only_vs_bg_trick(monkeypatch, 500_000, 32, 256, 256, 4, 1234)


def _views_run(inp, with_ct=True, h=None, depth=False):
    """One view through rasterize_views_raw / rasterize_views_backward_raw with the alpha plane on."""
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings as S
    from manigaussian_b200 import rasterizer as R
    cam, g, ct = inp["cam"], inp["g"], inp["ct"]
    W, H, F = inp["W"], inp["H"], inp["F"]
    view = S(H, W, cam["tanfovx"], cam["tanfovy"], _t(inp["bg"]), 1.0, _t(cam["viewmatrix"]), _t(cam["projmatrix"]), g["sh_degree"],
             _t(cam["campos"]), False, False, F > 0)
    u = util._t
    args = (u(g["means3D"]), u(g["colors_precomp"]), u(g["feature"]) if F else None, u(g["opacities"]), u(g["scales"]), u(g["rotations"]),
            1.0, u(g["cov3D_precomp"]), u(g["shs"]), g["sh_degree"], F > 0)
    outs, sts = R.rasterize_views_raw([view], *args, return_depth=depth, return_alpha=True)
    o = outs[0]
    s = 1.0 if with_ct else 0.0
    gc = _t(ct["dL_dcolor"]) * s
    gf = [_t(ct["dL_dfeature"]) * s] if F else None
    gd = [_t(ct["dL_ddepth"]) * s] if depth else None
    m3, col, feat, op, sc, rot, smod, cov, sh, deg, inc = args
    grads = R.rasterize_views_backward_raw([view], outs, sts, [gc], gf, m3, col, feat, sc, rot, smod, cov, sh, deg, inc, grads_depth=gd,
                                           grads_alpha=[_t(h)] if h is not None else None)
    torch.cuda.synchronize()
    return o, {n: (t.cpu().numpy() if t is not None else None) for n, t in zip(GRAD_NAMES, grads)}


CASES = {  # test_parity_gpu.CASES
    "tiny_f3": dict(P=300, W=32, H=32, F=3, seed=1),
    "mg_real_f3": dict(P=16384, W=128, H=128, F=3, seed=2),
    "ragged_f32": dict(P=5000, W=200, H=120, F=32, seed=3, bg=(0.3, 0.6, 0.9)),
    "rgb_only_precomp": dict(P=4000, W=96, H=96, F=0, seed=4, precomp_colors=True, precomp_cov=True),
    "sh3_big": dict(P=1500, W=128, H=96, F=8, seed=5, sh_degree=3, scale0=0.04, bg=(1.0, 1.0, 1.0)),
    "c1_like": dict(P=50000, W=128, H=128, F=0, seed=6),
    "f16": dict(P=3000, W=64, H=64, F=16, seed=7),
    "f5_odd": dict(P=2000, W=64, H=80, F=5, seed=8),
}


@pytest.mark.parametrize("name", list(CASES))
def test_alpha_vs_oracle(name):
    """Colour, feature and alpha cotangents together against the C oracle (alpha expectations of tests/alpha_oracle.py), at the
    stage-wise bars of test_parity_gpu (images 1e-4, gradients 1e-3)."""
    import alpha_oracle as O
    inp = util.make_inputs(**CASES[name])
    g, cam, ct = inp["g"], inp["cam"], inp["ct"]
    h = np.random.default_rng(inp["P"]).standard_normal((inp["H"], inp["W"])).astype(np.float32)
    o, gr = _views_run(inp, h=h)
    kw = dict(scales=g["scales"], rotations=g["rotations"], cov3D_precomp=g["cov3D_precomp"], shs=g["shs"], sh_degree=g["sh_degree"],
              colors_precomp=g["colors_precomp"], feature=g["feature"])
    fw = O.forward(g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], inp["W"], inp["H"], cam["tanfovx"],
                   cam["tanfovy"], inp["bg"], **kw)
    bw = O.backward(fw, ct["dL_dcolor"], ct["dL_dfeature"], g["means3D"], cam["viewmatrix"], cam["projmatrix"], cam["campos"],
                    cam["tanfovx"], cam["tanfovy"], inp["bg"], dL_dalpha=h, **kw)
    assert util.rel_l2(o[7].cpu().numpy(), fw["alpha"]) < 1e-4
    assert util.rel_l2(o[1].cpu().numpy(), fw["out_color"]) < 1e-4
    for k in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dsh", "dL_dscales", "dL_drotations", "dL_dfeature", "dL_dcolors"):
        if gr[k] is None or (k == "dL_dfeature" and not inp["F"]) or (k == "dL_dsh" and g["shs"] is None):
            continue
        if k in ("dL_dscales", "dL_drotations") and g["scales"] is None:
            continue
        if k == "dL_dcolors" and g["colors_precomp"] is None:
            continue
        err = util.rel_l2(gr[k].reshape(bw[k].shape), bw[k])
        assert err < 1e-3, (k, err)


def test_backward_is_linear_in_the_alpha_cotangent():
    """Colour, feature, depth and alpha cotangents in one backward == the colour/feature/depth backward + the alpha-only one."""
    inp = util.make_inputs(P=6000, W=80, H=64, F=32, seed=9, bg=(0.2, 0.3, 0.4), depth=True)
    h = np.random.default_rng(9).standard_normal((inp["H"], inp["W"])).astype(np.float32)
    _, both = _views_run(inp, h=h, depth=True)
    _, cfd = _views_run(inp, depth=True)
    _, alpha = _views_run(inp, with_ct=False, h=h, depth=True)
    for k in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dsh", "dL_dscales", "dL_drotations", "dL_dfeature"):
        err = util.rel_l2(both[k], cfd[k] + alpha[k])
        assert err <= 1e-5, (k, err)


def _data(cams):
    return {"novel_view": cams.as_novel_view()}


def test_paths_agree():
    """The single-view operator (also with debug=True), render, render_views against a loop of render, and render_clouds
    against render_views: alpha planes bit-identical, gradients within the spread of the atomics' order."""
    import torch
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import normalize_features, render, render_clouds, render_views
    P, F, W, H, V = 7000, 32, 72, 56, 4
    cams = _cams(V, W, H)
    host = _leaves(P, F, 81, "sh")
    cts = [(torch.randn(3, H, W, device="cuda"), torch.randn(F, H, W, device="cuda"), torch.randn(H, W, device="cuda"))
           for _ in range(V)]

    def obj(img, emb, alpha, v):
        return (img * cts[v][0]).sum() + (emb * cts[v][1]).sum() + (alpha * cts[v][2]).sum()

    # render_views (V = 4) against a loop of render
    A = _mk(host)
    ov = render_views(cams, A["xyz"], A["rot"], A["scale"], A["opac"], (0.1, 0.2, 0.3), features_color=A["col"],
                      features_language=A["feat"], return_alpha=True)
    assert ov["alpha"].shape == (V, H, W) and "depth" not in ov
    sum(obj(ov["render"][v], ov["render_embed"][v], ov["alpha"][v], v) for v in range(V)).backward()
    B = _mk(host)
    data = _data(cams)
    for v in range(V):
        o = render(data, v, B["xyz"], B["rot"], B["scale"], B["opac"], [0.1, 0.2, 0.3], features_color=B["col"], features_language=B["feat"],
                   return_alpha=True)
        assert o["alpha"].shape == (H, W) and torch.equal(o["alpha"], ov["alpha"][v]), v
        obj(o["render"], o["render_embed"], o["alpha"], v).backward()
    for k in A:
        assert util.rel_l2(A[k].grad.cpu().numpy(), B[k].grad.cpu().numpy()) < 1e-6, k

    # the single-view operator, plain and debug, with depth and alpha (depth before alpha) against one view of render
    for debug in (False, True):
        C = _mk(host)
        s = cams.settings(1, torch.tensor([0.1, 0.2, 0.3], device="cuda"), 1, True, debug=debug)
        m2 = torch.zeros_like(C["xyz"], requires_grad=True)
        img, emb, radii, depth, alpha = GaussianRasterizer(s, return_depth=True, return_alpha=True)(
            means3D=C["xyz"], means2D=m2, opacities=C["opac"], shs=C["col"], language_feature_precomp=normalize_features(C["feat"]),
            scales=C["scale"],
            rotations=C["rot"])
        assert torch.equal(alpha, ov["alpha"][1]), debug
        (obj(img, emb, alpha, 1) + depth.sum() * 0).backward()
        D = _mk(host)
        o = render(data, 1, D["xyz"], D["rot"], D["scale"], D["opac"], [0.1, 0.2, 0.3], features_color=D["col"], features_language=D["feat"],
                   return_alpha=True)
        obj(o["render"], o["render_embed"], o["alpha"], 1).backward()
        for k in C:
            assert util.rel_l2(C[k].grad.cpu().numpy(), D[k].grad.cpu().numpy()) < 1e-6, (debug, k)
        assert util.rel_l2(m2.grad.cpu().numpy(), o["viewspace_points"].grad.cpu().numpy()) < 1e-6, debug

    # render_clouds: two clouds of different P and image size against render_views per cloud
    spec = [(P, cams, host), (3000, _cams(2, 48, 40), _leaves(3000, F, 82, "sh"))]
    cts2 = [torch.randn(len(c), c.height, c.width, device="cuda") for _, c, _ in spec]
    E = [_mk(hh) for _, _, hh in spec]
    oc = render_clouds([dict(cameras=c, pts_xyz=L["xyz"], rotations=L["rot"], scales=L["scale"], opacity=L["opac"], features_color=L["col"],
                             features_language=L["feat"]) for L, (_, c, _) in zip(E, spec)], bg_color=(0.1, 0.2, 0.3), return_alpha=True,
                       return_depth=True)
    sum((o["alpha"] * t).sum() + o["render"].sum() + o["depth"].sum() for o, t in zip(oc, cts2)).backward()
    for b, (_, c, hh) in enumerate(spec):
        G = _mk(hh)
        r = render_views(c, G["xyz"], G["rot"], G["scale"], G["opac"], (0.1, 0.2, 0.3), features_color=G["col"], features_language=G["feat"],
                         return_alpha=True, return_depth=True)
        ((r["alpha"] * cts2[b]).sum() + r["render"].sum() + r["depth"].sum()).backward()
        assert set(oc[b]) == set(r) and torch.equal(oc[b]["alpha"], r["alpha"]) and torch.equal(oc[b]["depth"], r["depth"]), b
        for k in G:
            assert util.rel_l2(E[b][k].grad.cpu().numpy(), G[k].grad.cpu().numpy()) < 1e-6, (b, k)
        assert util.rel_l2(oc[b]["viewspace_points"].grad.cpu().numpy(), r["viewspace_points"].grad.cpu().numpy()) < 1e-6, b


def test_no_gaussians_and_targets():
    import torch
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    cams = _cams(2, 40, 24)
    s = cams.settings(0, torch.zeros(3, device="cuda"), 1, False)
    e = torch.zeros((0, 3), device="cuda")
    img, _, radii, alpha = GaussianRasterizer(s, return_alpha=True)(means3D=e, means2D=e, opacities=torch.zeros((0, 1), device="cuda"),
                                                                    shs=torch.zeros((0, 4, 3), device="cuda"), scales=e,
                                                                    rotations=torch.zeros((0, 4), device="cuda"))
    assert alpha.shape == (24, 40) and not alpha.any() and not img.any()
    g = _cloud(500, 3, 83)
    L = {k: _t(g[k]) for k in ("means3D", "rotations", "scales", "opacities", "shs")}
    tg = {"rgb": torch.rand(2, 3, 24, 40, device="cuda")}
    with pytest.raises(ValueError, match="return_alpha"):
        render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"], targets=tg, return_alpha=True)
    with pytest.raises(ValueError, match="return_alpha"):
        render_clouds([dict(cameras=cams, pts_xyz=L["means3D"], rotations=L["rotations"], scales=L["scales"], opacity=L["opacities"],
                            features_color=L["shs"], targets=tg)], return_alpha=True)


def test_cuda_graph_capture_with_alpha():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, F, W, H, V = 12000, 32, 80, 64, 3
    g = _cloud(P, F, 84)
    cams = _cams(V, W, H)
    names = ("means3D", "rotations", "scales", "opacities", "shs", "feature")
    L = {k: _t(np.asarray(g[k], np.float32)).requires_grad_(True) for k in names}
    cts = (torch.randn(V, 3, H, W, device="cuda"), torch.randn(V, F, H, W, device="cuda"), torch.randn(V, H, W, device="cuda"))
    keep = {}

    def fwd_bwd():
        o = render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L["feature"], return_alpha=True)
        loss = (o["render"] * cts[0]).sum() + (o["render_embed"] * cts[1]).sum() + (o["alpha"] * cts[2]).sum()
        loss.backward()
        keep["alpha"] = o["alpha"].detach()
        return loss

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for v in L.values():
                v.grad = None
            fwd_bwd()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eager = {k: v.grad.clone() for k, v in L.items()}
    eager_alpha = keep["alpha"].clone()
    for v in L.values():
        v.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fwd_bwd()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(keep["alpha"], eager_alpha)
    for k in names:
        assert util.rel_l2(L[k].grad.cpu().numpy(), eager[k].cpu().numpy()) < 1e-5, k


@pytest.mark.parametrize("path", ["module", "render", "render_views", "render_clouds"])
def test_steps_with_alpha_do_not_accumulate_device_memory(path):
    import gc
    import torch
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import render, render_clouds, render_views
    P, F, W, H, V = 6000, 32, 64, 48, 2
    g = _cloud(P, F, 85)
    cams = _cams(V, W, H)
    data = _data(cams)
    host = {k: np.asarray(g[k], np.float32) for k in ("means3D", "rotations", "scales", "opacities", "shs", "feature")}
    h = torch.randn(V, H, W, device="cuda")

    def step():
        L = {k: _t(v).requires_grad_(True) for k, v in host.items()}
        if path == "module":
            s = cams.settings(0, torch.zeros(3, device="cuda"), 1, True)
            img, _, _, alpha = GaussianRasterizer(s, return_alpha=True)(
                means3D=L["means3D"], means2D=torch.zeros_like(L["means3D"]), opacities=L["opacities"], shs=L["shs"],
                language_feature_precomp=L["feature"], scales=L["scales"], rotations=L["rotations"])
            loss = img.sum() + (alpha * h[0]).sum()
        elif path == "render":
            o = render(data, 0, L["means3D"], L["rotations"], L["scales"], L["opacities"], [0, 0, 0], features_color=L["shs"],
                       features_language=L["feature"], return_alpha=True)
            loss = o["render"].sum() + (o["alpha"] * h[0]).sum()
        else:
            kw = dict(pts_xyz=L["means3D"], rotations=L["rotations"], scales=L["scales"], opacity=L["opacities"], features_color=L["shs"],
                      features_language=L["feature"])
            o = render_views(cams, return_alpha=True, **kw) if path == "render_views" else \
                render_clouds([dict(cameras=cams, **kw)], return_alpha=True)[0]
            loss = o["render"].sum() + (o["alpha"] * h).sum()
        loss.backward()
        return float(loss)

    gc.disable()
    try:
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        for _ in range(4):
            step()
        torch.cuda.synchronize()
        grown = torch.cuda.memory_allocated() - base
    finally:
        gc.enable()
    assert grown == 0, f"{grown} bytes stayed allocated after 4 more steps"


def test_expected_depth_loss_reaches_every_leaf():
    """ManiGaussian's depth supervision: expected depth = depth / alpha, an L1 loss against a target depth plus a mask loss on
    alpha, through render_views(return_depth=True, return_alpha=True)."""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, F, W, H, V = 8000, 32, 64, 64, 2
    host = _leaves(P, F, 86, "sh")
    cams = _cams(V, W, H)
    L = _mk(host)
    o = render_views(cams, L["xyz"], L["rot"], L["scale"], L["opac"], features_color=L["col"], features_language=L["feat"],
                     return_depth=True, return_alpha=True)
    d = o["depth"] / o["alpha"].clamp_min(1e-4)
    gt = torch.full((V, H, W), 1.5, device="cuda")
    mask = (torch.rand(V, H, W, device="cuda") > 0.5).float()
    valid = (o["alpha"] > 0.5).detach()
    loss = (d - gt).abs()[valid].mean() + torch.nn.functional.binary_cross_entropy(o["alpha"].clamp(1e-4, 1 - 1e-4), mask)
    loss = loss + o["render"].square().mean() + o["render_embed"].square().mean()  # the colour and embedding losses beside it
    loss.backward()
    assert torch.isfinite(loss)
    for k in L:
        assert L[k].grad is not None and torch.isfinite(L[k].grad).all() and L[k].grad.abs().sum() > 0, k
    assert torch.isfinite(o["viewspace_points"].grad).all()
