"""The L1 + SSIM photometric loss on the GPU: the standalone kernels (mgs_ssim / mgs_ssim_backward) against the float64
oracle (tests/ssim_oracle.py), the fused render_views(targets, ssim=True) against the unfused recipe (render_views, then the
reference's PyTorch l1_loss + ssim in float32 with TF32 off), render_clouds against render_views, the standalone
losses.ssim against the recipe, CUDA-graph capture and device memory over repeated steps."""
import contextlib
import math

import numpy as np
import pytest

import util
from test_clouds_gpu import _leaves, _mk
from test_render_gpu import _cams
import ssim_oracle as O

pytestmark = pytest.mark.gpu

W, H = 61, 37  # ragged: partial tiles


def _kw(L):
    return dict(pts_xyz=L["xyz"], rotations=L["rot"], scales=L["scale"], opacity=L["opac"], features_color=L["col"],
                features_language=L.get("feat"))


@contextlib.contextmanager
def _no_tf32():
    import torch
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _ref_ssim(img1, img2):
    """the reference's _ssim (window 11, sigma 1.5), per image of a [B,C,H,W] batch: [B]"""
    import torch
    import torch.nn.functional as F
    C = img1.shape[1]
    gauss = torch.tensor([math.exp(-(i - 5) ** 2 / 4.5) for i in range(11)], dtype=torch.float32)
    gauss = gauss / gauss.sum()
    w = (gauss[:, None] @ gauss[None, :]).expand(C, 1, 11, 11).contiguous().to(img1.device)
    mu1, mu2 = F.conv2d(img1, w, padding=5, groups=C), F.conv2d(img2, w, padding=5, groups=C)
    s1 = F.conv2d(img1 * img1, w, padding=5, groups=C) - mu1 ** 2
    s2 = F.conv2d(img2 * img2, w, padding=5, groups=C) - mu2 ** 2
    s12 = F.conv2d(img1 * img2, w, padding=5, groups=C) - mu1 * mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    smap = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 ** 2 + mu2 ** 2 + c1) * (s1 + s2 + c2))
    return smap.flatten(1).mean(1)


def _targets(V, F, seed):
    import torch
    gen = torch.Generator(device="cuda").manual_seed(seed)
    tg = {"rgb": torch.rand(V, 3, H, W, device="cuda", generator=gen)}
    if F:
        tg["embed"] = torch.rand(V, F, H, W, device="cuda", generator=gen) - 0.5
    return tg


def _weights(V, seed):
    """per-view loss weights, on the device (a CUDA-graph capture cannot copy from pageable host memory)"""
    import torch
    rng = np.random.default_rng(seed)
    return {k: torch.from_numpy(rng.uniform(0.5, 2.0, V).astype(np.float32)).cuda() for k in ("loss_rgb", "loss_embed", "loss_l1", "ssim")}


def _objective(o, w):
    """0.8 l1 + 0.2 (1 - ssim) per view, plus the L2 colour and embedding heads, with per-view weights"""
    total = (w["loss_l1"] * 0.8 * o["loss_l1"]).sum() + (w["ssim"] * 0.2 * (1 - o["ssim"])).sum()
    total = total + (w["loss_rgb"] * o["loss_rgb"]).sum()
    if "loss_embed" in o:
        total = total + (w["loss_embed"] * o["loss_embed"]).sum()
    return total


def _recipe(o, tg):
    """the unfused recipe on a render_views result: dict of [V]"""
    import torch
    out = {"loss_rgb": ((o["render"] - tg["rgb"]) ** 2).flatten(1).mean(1),
           "loss_l1": (o["render"] - tg["rgb"]).abs().flatten(1).mean(1)}
    with _no_tf32():
        out["ssim"] = _ref_ssim(o["render"], tg["rgb"])
    if "embed" in tg:
        out["loss_embed"] = 1 - torch.nn.functional.cosine_similarity(o["render_embed"], tg["embed"], dim=1).flatten(1).mean(1)
    return out


def _grads(L, total):
    for x in L.values():
        x.grad = None
    total.backward()
    return {k: x.grad.detach().clone() for k, x in L.items() if x.grad is not None}


@pytest.mark.parametrize("V", [1, 4])
@pytest.mark.parametrize("hw", [(1, 1), (5, 7), (16, 16), (37, 61), (128, 128), (256, 256)])
def test_standalone_kernels_match_the_float64_oracle(hw, V):
    import torch
    from manigaussian_b200 import _binding as B
    h, w = hw
    rng = np.random.default_rng(h * 1000 + w + V)
    x = rng.uniform(-0.1, 1.1, (V, 3, h, w)).astype(np.float32)
    g = rng.uniform(0, 1, (V, 3, h, w)).astype(np.float32)
    xf, gf = x.reshape(V, 3, -1), g.reshape(V, 3, -1)
    xf[:, 0, ::3] = gf[:, 0, ::3]  # sign(0) pixels for L1 (every image keeps pixels with x != g)
    scale = rng.uniform(-2, 2, (V, 2)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    xd, gd, sd = t(x), t(g), t(scale)
    terms = torch.full((V, 9, h, w), float("nan"), device="cuda")
    acc = torch.full((V, 2), float("nan"), device="cuda")
    cot = torch.full((V, 3, h, w), float("nan"), device="cuda")
    L = B.lib()
    st = torch.cuda.current_stream().cuda_stream
    B.check(L.mgs_ssim(V, 3, h, w, xd.data_ptr(), gd.data_ptr(), terms.data_ptr(), acc.data_ptr(), st), "mgs_ssim")
    B.check(L.mgs_ssim_backward(V, 3, h, w, xd.data_ptr(), gd.data_ptr(), terms.data_ptr(), sd.data_ptr(), None, cot.data_ptr(), st),
            "mgs_ssim_backward")
    cot_in = t(rng.uniform(-1e-4, 1e-4, (V, 3, h, w)).astype(np.float32))
    cot2 = torch.empty_like(cot)
    B.check(L.mgs_ssim_backward(V, 3, h, w, xd.data_ptr(), gd.data_ptr(), terms.data_ptr(), sd.data_ptr(), cot_in.data_ptr(),
                                cot2.data_ptr(), st), "mgs_ssim_backward")
    torch.cuda.synchronize()
    N = 3 * h * w
    acc, terms, cot, cot2 = acc.cpu().numpy(), terms.cpu().numpy(), cot.cpu().numpy(), cot2.cpu().numpy()
    for v in range(V):
        l1, ss = O.losses(x[v], g[v])
        assert abs(acc[v, 0] / N - l1) <= 1e-5 * l1, (v, acc[v, 0] / N, l1)
        assert abs(acc[v, 1] / N - ss) <= 1e-5 * abs(ss), (v, acc[v, 1] / N, ss)
        assert util.rel_l2(terms[v], O.terms(x[v], g[v])) < 1e-4
        want = O.grad(x[v], g[v], float(scale[v, 0]), float(scale[v, 1]))
        assert np.isfinite(cot[v]).all()
        assert util.rel_l2(cot[v], want) < 1e-5, (v, util.rel_l2(cot[v], want))
    assert np.allclose(cot2, cot + cot_in.cpu().numpy(), rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("F", [0, 3, 32, 40])
def test_fused_ssim_matches_the_unfused_recipe(F):
    """losses within 1e-5, every leaf gradient and viewspace_points.grad within 2e-5 rel-L2"""
    from manigaussian_b200.gaussian_renderer import render_views
    V = 3
    cams = _cams(V, W, H)
    L = _mk(_leaves(6000, F, 110 + F, "sh"))
    tg = _targets(V, F, 3 + F)
    wts = _weights(V, F)
    fused = render_views(cams, **_kw(L), targets=tg, ssim=True)
    g_f = _grads(L, _objective(fused, wts))
    vsp_f = fused["viewspace_points"].grad.clone()
    unf = render_views(cams, **_kw(L))
    ref = _recipe(unf, tg)
    g_u = _grads(L, _objective(ref, wts))
    vsp_u = unf["viewspace_points"].grad.clone()
    for k, want in ref.items():
        got, want = fused[k].detach().cpu().numpy(), want.detach().cpu().numpy()
        assert np.allclose(got, want, rtol=1e-5, atol=1e-7), (k, got, want)
    assert fused["loss_l1"].requires_grad and fused["ssim"].requires_grad
    for k in g_u:
        err = util.rel_l2(g_f[k].cpu().numpy(), g_u[k].cpu().numpy())
        assert err < 2e-5, (k, err)
    assert util.rel_l2(vsp_f.cpu().numpy(), vsp_u.cpu().numpy()) < 2e-5


def test_other_heads_are_unchanged_with_ssim_on_and_off():
    """the images and the colour / embedding heads' cotangent planes are bit-identical with the SSIM head on and off; the
    loss sums are float atomics, whose order differs from run to run, so they agree to rounding"""
    import torch
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200.gaussian_renderer import _ssim_head, render_views
    F, V = 32, 2
    cams = _cams(V, W, H)
    L = _mk(_leaves(6000, F, 120, "sh"))
    tg = _targets(V, F, 9)
    off = render_views(cams, **_kw(L), targets=tg)
    on = render_views(cams, **_kw(L), targets=tg, ssim=True)
    assert "loss_l1" not in off and "ssim" not in off
    for k in ("render", "render_embed", "radii"):
        assert torch.equal(off[k], on[k]), k
    for k in ("loss_rgb", "loss_embed"):
        assert torch.allclose(off[k], on[k], rtol=1e-6, atol=0), k
    views = [cams.settings(i, torch.zeros(3, device="cuda"), 1, True) for i in range(V)]
    opts = dict(dtype=torch.float32, device="cuda")
    args = (views, L["xyz"].detach(), None, L["feat"].detach(), L["opac"].detach(), L["scale"].detach(), L["rot"].detach(), 1.0, None,
            L["col"].detach(), 1, True)
    planes = []
    for head in (None, _ssim_head(V, H, W, torch.device("cuda"))):
        heads = (tg["rgb"], tg["embed"], torch.empty((V, 3, H, W), **opts), torch.empty((V, F, H, W), **opts), torch.empty((V, 2), **opts))
        color = torch.empty((V, 3, H, W), **opts)
        R.rasterize_views_raw(*args, out_buffers=(color, torch.empty((V, F, H, W), **opts), None), loss_heads=heads, ssim=head)
        planes.append((color, heads[2], heads[3]))
    torch.cuda.synchronize()
    for a, b in zip(*planes):
        assert torch.equal(a, b)


def test_render_clouds_matches_render_views_with_depth_mask_and_antialiasing():
    """2 clouds x 2 views with the depth and mask heads and the anti-aliased projection"""
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    F, V = 32, 2
    cams = [_cams(V, W, H), _cams(V, W, H)]
    Ls = (_mk(_leaves(6000, F, 121, "sh")), _mk(_leaves(5000, F, 122, "sh")))
    tgs = []
    for b in range(2):
        tg = _targets(V, F, 30 + b)
        gen = torch.Generator(device="cuda").manual_seed(40 + b)
        tg["depth"] = torch.rand(V, H, W, device="cuda", generator=gen) * 3
        tg["mask"] = (torch.rand(V, H, W, device="cuda", generator=gen) > 0.4).float()
        tgs.append(tg)
    wts = [_weights(V, 50 + b) for b in range(2)]

    def total(o, w):
        return _objective(o, w) + o["loss_depth"].sum() + o["loss_mask"].sum()

    outs = render_clouds([dict(cameras=cams[b], targets=tgs[b], **_kw(Ls[b])) for b in range(2)], ssim=True, antialiasing=True)
    all_leaves = {f"{b}{k}": x for b in range(2) for k, x in Ls[b].items()}
    g_c = _grads(all_leaves, total(outs[0], wts[0]) + total(outs[1], wts[1]))
    for b in range(2):
        ref = render_views(cams[b], **_kw(Ls[b]), targets=tgs[b], ssim=True, antialiasing=True)
        g_v = _grads(Ls[b], total(ref, wts[b]))
        for k in ("loss_rgb", "loss_embed", "loss_depth", "loss_mask", "loss_l1", "ssim"):
            assert torch.allclose(outs[b][k], ref[k], rtol=1e-5, atol=0), (b, k)
        for k, gv in g_v.items():
            assert util.rel_l2(g_c[f"{b}{k}"].cpu().numpy(), gv.cpu().numpy()) < 1e-5, (b, k)


@pytest.mark.parametrize("shape", [(3, 37, 61), (2, 3, 16, 16), (4, 1, 5, 7)])
def test_losses_ssim_matches_the_recipe(shape):
    import torch
    from manigaussian_b200 import losses
    gen = torch.Generator(device="cuda").manual_seed(sum(shape))
    a = torch.rand(*shape, device="cuda", generator=gen).requires_grad_()
    b = torch.rand(*shape, device="cuda", generator=gen)
    got = losses.ssim(a, b)
    (ga,) = torch.autograd.grad(got, a)
    a2 = a.detach().clone().requires_grad_()
    with _no_tf32():
        x, y = (a2, b) if len(shape) == 4 else (a2.unsqueeze(0), b.unsqueeze(0))
        want = _ref_ssim(x, y).mean()
    (gw,) = torch.autograd.grad(want, a2)
    assert got.shape == () and abs(float(got.detach()) - float(want.detach())) <= 1e-5 * abs(float(want.detach()))
    assert util.rel_l2(ga.cpu().numpy(), gw.cpu().numpy()) < 2e-5


def _graph_vs_eager(fwd_bwd, L):
    import torch
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for x in L.values():
                x.grad = None
            out = fwd_bwd()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eager = {k: x.grad.clone() for k, x in L.items()}
    eager_losses = out.clone()
    for x in L.values():
        x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fwd_bwd()
    graph.replay()
    torch.cuda.synchronize()
    # the loss sums are float atomics, whose order differs from run to run
    assert torch.allclose(out, eager_losses, rtol=1e-5, atol=0)
    for k in L:
        assert util.rel_l2(L[k].grad.cpu().numpy(), eager[k].cpu().numpy()) < 1e-5, k


@pytest.mark.parametrize("path", ["render_views", "render_clouds"])
def test_cuda_graph_capture_with_ssim(path):
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    F, V = 32, 3
    cams = _cams(V, W, H)
    L = _mk(_leaves(8000, F, 130, "sh"))
    tg = _targets(V, F, 61)
    wts = _weights(V, 7)

    def fwd_bwd():
        o = render_views(cams, **_kw(L), targets=tg, ssim=True) if path == "render_views" else \
            render_clouds([dict(cameras=cams, targets=tg, **_kw(L))], ssim=True)[0]
        _objective(o, wts).backward()
        return torch.stack([o[k].detach() for k in ("loss_rgb", "loss_embed", "loss_l1", "ssim")])

    _graph_vs_eager(fwd_bwd, L)


@pytest.mark.parametrize("path", ["render_views", "render_clouds"])
def test_steps_with_ssim_do_not_accumulate_device_memory(path):
    import gc
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    F, V = 32, 2
    cams = _cams(V, W, H)
    host = _leaves(6000, F, 131, "sh")
    tg = _targets(V, F, 71)
    wts = _weights(V, 8)

    def step():
        L = _mk(host)
        o = render_views(cams, **_kw(L), targets=tg, ssim=True) if path == "render_views" else \
            render_clouds([dict(cameras=cams, targets=tg, **_kw(L))], ssim=True)[0]
        total = _objective(o, wts)
        total.backward()
        return float(total.detach())

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
