"""The depth and mask loss heads (expected-depth L1, alpha BCE) fused into the blend epilogue, on the GPU: against the
unfused recipe of INTEGRATION.md §4 (render_views(return_depth=True, return_alpha=True) + PyTorch), against the numpy
oracle (tests/depth_heads_oracle.py) on the cotangent planes, through render_clouds, at the edges (no valid pixel, no
Gaussian), under CUDA-graph capture and over repeated steps."""
import numpy as np
import pytest

import util
from test_clouds_gpu import _leaves, _mk
from test_render_gpu import _cams
import depth_heads_oracle as O

pytestmark = pytest.mark.gpu

W, H = 61, 37  # ragged: partial tiles and blocks
LEAVES = ("xyz", "rot", "scale", "opac", "col", "feat")


def _kw(L):
    return dict(pts_xyz=L["xyz"], rotations=L["rot"], scales=L["scale"], opacity=L["opac"], features_color=L["col"],
                features_language=L.get("feat"))


def _targets(cams, L, F, heads, seed):
    """rgb / embed targets, and depth / mask targets drawn from an unfused render: the depth target sits at least 1e-3 away
    from the rendered expected depth, so that no pixel's sign depends on the last ulp; 30 % of it is 0 (unknown)"""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    V = len(cams)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, device="cuda", generator=gen)
    tg = {"rgb": rnd(V, 3, H, W)}
    if F:
        tg["embed"] = rnd(V, F, H, W) - 0.5
    with torch.no_grad():
        o = render_views(cams, **_kw(L), return_depth=True, return_alpha=True)
        d = o["depth"] / o["alpha"].clamp_min(1e-4)
    if "depth" in heads:
        sign = torch.where(rnd(V, H, W) < 0.5, -1.0, 1.0)
        g = (d + sign * (1e-3 + 0.3 * rnd(V, H, W))).clamp_min(0)
        g[rnd(V, H, W) < 0.3] = 0
        tg["depth"] = g
    if "mask" in heads:
        m = (rnd(V, H, W) > 0.4).float()
        soft = rnd(V, H, W) < 0.2
        m[soft] = rnd(V, H, W)[soft]
        tg["mask"] = m
    return tg


def _recipe(o, tg):
    """INTEGRATION.md §4 per view, on an unfused render_views(return_depth=True, return_alpha=True) result -> dict of [V]"""
    import torch
    V = o["render"].shape[0]
    out = {"loss_rgb": ((o["render"] - tg["rgb"]) ** 2).flatten(1).mean(1)}
    if "embed" in tg:
        cos = torch.nn.functional.cosine_similarity(o["render_embed"], tg["embed"], dim=1)
        out["loss_embed"] = 1 - cos.flatten(1).mean(1)
    if "depth" in tg:
        d = o["depth"] / o["alpha"].clamp_min(1e-4)
        valid = (tg["depth"] > 0) & (o["alpha"] > 0.5).detach()
        per = []
        for v in range(V):
            per.append((d[v] - tg["depth"][v]).abs()[valid[v]].mean() if bool(valid[v].any()) else (d[v] * 0).sum())
        out["loss_depth"] = torch.stack(per)
        out["depth_pixels"] = valid.flatten(1).sum(1).float()
    if "mask" in tg:
        a = o["alpha"].clamp(1e-4, 1 - 1e-4)
        out["loss_mask"] = torch.stack([torch.nn.functional.binary_cross_entropy(a[v], tg["mask"][v]) for v in range(V)])
    return out


LOSSES = ("loss_rgb", "loss_embed", "loss_depth", "loss_mask")


def _weights(V, seed):
    rng = np.random.default_rng(seed)
    return {k: rng.uniform(0.5, 2.0, V).astype(np.float32) for k in LOSSES}


def _step(L, losses, wts):
    import torch
    for x in L.values():
        x.grad = None
    total = sum((losses[k] * torch.from_numpy(wts[k]).cuda()).sum() for k in LOSSES if k in losses)
    total.backward()
    return {k: x.grad.detach().clone() for k, x in L.items()}


@pytest.mark.parametrize("heads", ["depth", "mask", "depth+mask"])
@pytest.mark.parametrize("F", [0, 3, 32, 40, 67])
def test_fused_heads_match_the_unfused_recipe(F, heads):
    """losses within 1e-5 relative, every leaf gradient and viewspace_points.grad within 2e-5 rel-L2"""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    V = 3
    cams = _cams(V, W, H)
    L = _mk(_leaves(6000, F, 90 + F, "sh"))
    if not F:
        L.pop("feat", None)
    tg = _targets(cams, L, F, heads, 7 + F)
    wts = _weights(V, F)
    fused = render_views(cams, **_kw(L), targets=tg)
    g_f = _step(L, fused, wts)
    vsp_f = fused["viewspace_points"].grad.clone()
    unf = render_views(cams, **_kw(L), return_depth=True, return_alpha=True)
    ref = _recipe(unf, tg)
    g_u = _step(L, ref, wts)
    vsp_u = unf["viewspace_points"].grad.clone()
    for k, want in ref.items():
        got = fused[k].detach().cpu().numpy()
        want = want.detach().cpu().numpy()
        assert np.allclose(got, want, rtol=1e-5, atol=1e-7), (k, got, want)
    for k in ("loss_depth", "depth_pixels", "loss_mask"):
        assert (k in fused) == (k in ref), k
    if "depth" in heads:
        assert not fused["depth_pixels"].requires_grad and fused["depth_pixels"].dtype == torch.float32
        assert float(fused["depth_pixels"].min()) > 0
    for k in L:
        err = util.rel_l2(g_f[k].cpu().numpy(), g_u[k].cpu().numpy())
        assert err < 2e-5, (k, err)
    assert util.rel_l2(vsp_f.cpu().numpy(), vsp_u.cpu().numpy()) < 2e-5


@pytest.mark.parametrize("F", [3, 40])
def test_cotangent_planes_equal_the_oracle_on_the_unfused_images(F):
    import torch
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200.gaussian_renderer import _depth_mask_heads, render_views
    V = 2
    cams = _cams(V, W, H)
    L = _mk(_leaves(6000, F, 95, "sh"))
    tg = _targets(cams, L, F, "depth+mask", 11)
    tg["depth"][1] = 0  # a view with no valid pixel
    views = [cams.settings(i, torch.zeros(3, device="cuda"), 1, True) for i in range(V)]
    opts = dict(dtype=torch.float32, device="cuda")
    args = (views, L["xyz"].detach(), None, L["feat"].detach(), L["opac"].detach(), L["scale"].detach(), L["rot"].detach(), 1.0, None,
            L["col"].detach(), 1, True)
    heads = (tg["rgb"], tg["embed"], torch.empty((V, 3, H, W), **opts), torch.empty((V, F, H, W), **opts), torch.empty((V, 2), **opts))
    dm = _depth_mask_heads(tg["depth"], tg["mask"], V, H, W, torch.device("cuda"))
    for p in dm[2:5]:
        p.fill_(float("nan"))  # every in-image pixel is written
    R.rasterize_views_raw(*args, loss_heads=heads, depth_mask=dm)
    with torch.no_grad():
        unf = render_views(cams, **_kw({k: v.detach() for k, v in L.items()}), return_depth=True, return_alpha=True)
    torch.cuda.synchronize()
    acc = dm[5].cpu().numpy()
    for v in range(V):
        D, A = unf["depth"][v].cpu().numpy(), unf["alpha"][v].cpu().numpy()
        g, m = tg["depth"][v].cpu().numpy(), tg["mask"][v].cpu().numpy()
        loss_d, n, cd, ca = O.depth_head(D, A, g)
        loss_m, cm = O.mask_head(A, m)
        for name, got, want in (("cot_depth", dm[2][v], cd), ("cot_alpha_depth", dm[3][v], ca), ("cot_alpha_mask", dm[4][v], cm)):
            got = got.cpu().numpy()
            assert np.isfinite(got).all(), (name, v)
            assert np.allclose(got, want, rtol=1e-6, atol=1e-12), (name, v, np.abs(got - want).max())
        assert acc[v, 1] == n
        assert abs(acc[v, 0] / max(acc[v, 1], 1) - loss_d) <= 1e-5 * max(loss_d, 1e-6)
        assert abs(acc[v, 2] / (H * W) - loss_m) <= 1e-5 * loss_m
    assert acc[1, 0] == 0 and acc[1, 1] == 0


def test_render_clouds_matches_render_views_per_cloud():
    """2 clouds x 2 views, the second cloud with detached features as in the dyna step"""
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    F, V = 32, 2
    cams = [_cams(V, W, H), _cams(V, W, H)]
    L0 = _mk(_leaves(6000, F, 97, "sh"))
    host1 = _leaves(5000, F, 98, "sh")
    L1 = _mk(host1)
    L1["feat"] = L1["feat"].detach()
    tgs = [_targets(cams[0], L0, F, "depth+mask", 21), _targets(cams[1], L1, F, "depth+mask", 22)]
    tgs[1].pop("mask")  # per cloud: the second has a depth head only
    wts = [_weights(len(cams[b]), 1 + b) for b in range(2)]
    Ls = (L0, L1)
    outs = render_clouds([dict(cameras=cams[b], targets=tgs[b], **_kw(Ls[b])) for b in range(2)])
    for x in list(L0.values()) + list(L1.values()):
        x.grad = None
    total = sum((o[k] * torch.from_numpy(w[k]).cuda()).sum() for o, w in zip(outs, wts) for k in LOSSES if k in o)
    total.backward()
    g_c = [{k: x.grad.clone() for k, x in Lb.items() if x.grad is not None} for Lb in Ls]
    assert L1["feat"].grad is None and "loss_mask" not in outs[1] and "loss_depth" in outs[1]
    for b in range(2):
        ref = render_views(cams[b], **_kw(Ls[b]), targets=tgs[b])
        g_v = _step({k: x for k, x in Ls[b].items() if x.requires_grad}, ref, wts[b])
        for k in ("loss_rgb", "loss_embed", "loss_depth", "depth_pixels", "loss_mask"):
            assert (k in ref) == (k in outs[b]), (b, k)
            if k in ref:
                assert torch.allclose(outs[b][k], ref[k], rtol=1e-5, atol=0), (b, k)
        for k, gv in g_v.items():
            assert util.rel_l2(g_c[b][k].cpu().numpy(), gv.cpu().numpy()) < 1e-5, (b, k)


def test_no_valid_pixel_gives_zero_and_leaves_the_gradients_alone():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    F, V = 32, 2
    cams = _cams(V, W, H)
    L = _mk(_leaves(6000, F, 99, "sh"))
    tg = _targets(cams, L, F, "depth+mask", 31)
    tg["depth"][0] = 0  # view 0: no valid pixel
    o = render_views(cams, **_kw(L), targets=tg)
    assert float(o["loss_depth"][0].detach()) == 0 and float(o["depth_pixels"][0]) == 0 and float(o["depth_pixels"][1]) > 0
    assert torch.isfinite(o["loss_depth"]).all()
    # with every depth target zero the depth head adds nothing: the gradients are those without it
    tg["depth"][:] = 0
    wts = _weights(V, 5)
    with_d = render_views(cams, **_kw(L), targets=tg)
    g_d = _step(L, with_d, wts)
    assert not with_d["loss_depth"].any() and not with_d["depth_pixels"].any()
    without = render_views(cams, **_kw(L), targets={k: v for k, v in tg.items() if k != "depth"})
    g_0 = _step(L, without, wts)
    for k in L:
        assert util.rel_l2(g_d[k].cpu().numpy(), g_0[k].cpu().numpy()) < 1e-5, k


def test_no_gaussians():
    """P = 0: the fused path needs Gaussians, with or without the depth / mask heads (the same error), and depth / mask
    targets still cannot be combined with returned depth or alpha images"""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    V = 2
    cams = _cams(V, W, H)
    e = torch.zeros((0, 3), device="cuda")
    kw = dict(pts_xyz=e, rotations=torch.zeros((0, 4), device="cuda"), scales=e, opacity=torch.zeros((0, 1), device="cuda"),
              features_color=torch.zeros((0, 4, 3), device="cuda"))
    base = {"rgb": torch.rand(V, 3, H, W, device="cuda")}
    errs = []
    for extra in ({}, {"depth": torch.rand(V, H, W, device="cuda"), "mask": torch.rand(V, H, W, device="cuda")}):
        with pytest.raises(RuntimeError) as ex:
            render_views(cams, targets=dict(base, **extra), **kw)
        errs.append(str(ex.value))
    assert errs[0] == errs[1]
    with pytest.raises(ValueError, match="return_depth"):
        render_views(cams, targets=dict(base, depth=torch.rand(V, H, W, device="cuda")), return_depth=True, **kw)


def test_cuda_graph_capture_with_depth_and_mask_heads():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    F, V = 32, 3
    cams = _cams(V, W, H)
    L = _mk(_leaves(8000, F, 100, "sh"))
    tg = _targets(cams, L, F, "depth+mask", 41)
    wts = {k: torch.from_numpy(v).cuda() for k, v in _weights(V, 6).items()}
    keep = {}

    def fwd_bwd():
        o = render_views(cams, **_kw(L), targets=tg)
        total = sum((o[k] * wts[k]).sum() for k in LOSSES)
        total.backward()
        keep["losses"] = torch.stack([o[k].detach() for k in LOSSES] + [o["depth_pixels"]])

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for x in L.values():
                x.grad = None
            fwd_bwd()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eager = {k: x.grad.clone() for k, x in L.items()}
    eager_losses = keep["losses"].clone()
    for x in L.values():
        x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fwd_bwd()
    graph.replay()
    torch.cuda.synchronize()
    # the loss sums are float atomics, whose order differs from run to run; the valid-pixel counts are exact
    assert torch.equal(keep["losses"][-1], eager_losses[-1])
    assert torch.allclose(keep["losses"], eager_losses, rtol=1e-5, atol=0)
    for k in L:
        assert util.rel_l2(L[k].grad.cpu().numpy(), eager[k].cpu().numpy()) < 1e-5, k


@pytest.mark.parametrize("path", ["render_views", "render_clouds"])
def test_steps_with_depth_and_mask_heads_do_not_accumulate_device_memory(path):
    import gc
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    F, V = 32, 2
    cams = _cams(V, W, H)
    host = _leaves(6000, F, 101, "sh")
    tg = _targets(cams, _mk(host), F, "depth+mask", 51)

    def step():
        L = _mk(host)
        o = render_views(cams, **_kw(L), targets=tg) if path == "render_views" else \
            render_clouds([dict(cameras=cams, targets=tg, **_kw(L))])[0]
        total = sum(o[k].sum() for k in LOSSES)
        total.backward()
        return float(total)

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
