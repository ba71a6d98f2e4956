"""Control-graph deformation on the GPU (deform.cu, mgs_deform, gaussian_renderer.deform_gaussians).

1. Against the float64 reference (tests/deform_ref64.py): outputs within 1e-5 relative, the six gradients within 1e-4
   relative L2, for k = 1, 4, 8, 20, 32 on knn lists over uniform and rendered-surface clouds, on hand-built lists with -1
   padding, out-of-range indices and a node repeated in a row, with weights that do not sum to 1 and negative ones, node
   quaternions with a negative real part, unnormalised and zero, P = 0 and N = 0, the forward at c3 size (500k Gaussians,
   4,096 nodes, k = 8) and the gradients at 50k, and rigid segments (500k Gaussians on 3 nodes, k = 1: the contended
   reduction).
2. A learnable weight built in torch from node_xyz and a radius per node: end-to-end gradients match float64.
3. Next-frame only (node_rot and node_t requiring grad): the same gradients as the all-grad call, None for the rest.
4. deform_gaussians then render_views: node gradients equal those of the float32 torch restatement through the same render.
5. Forward outputs bitwise identical across calls; CUDA-graph capture of forward + backward replayed on new values; no
   device-memory growth over repeated calls; a call on a non-current device.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import deform_ref64 as D64
import util

pytestmark = pytest.mark.gpu

_NAMES = ("xyz", "rot", "node_xyz", "node_rot", "node_t", "weight")


def _surface_points():
    """the scene's depth image unprojected, as tests/test_knn_gpu.py builds it (16,384 points, some on the camera centre)"""
    from test_knn_gpu import _surface
    return torch.from_numpy(_surface())


def _cloud(kind, P=None, N=64, seed=0):
    """xyz [P,3] (the 16,384 surface points for "surface"), unit rot, and N nodes subsampled from the cloud with random
    rotations and small translations"""
    g = torch.Generator().manual_seed(seed)
    xyz = _surface_points() if kind == "surface" else torch.rand(P, 3, generator=g)
    P = xyz.shape[0]
    rot = F.normalize(torch.randn(P, 4, generator=g), dim=-1)
    node_xyz = xyz[torch.randperm(P, generator=g)[:N]].clone() if N > 0 else torch.zeros(0, 3)
    node_rot = torch.randn(N, 4, generator=g)
    node_t = 0.05 * torch.randn(N, 3, generator=g)
    return xyz, rot, node_xyz, node_rot, node_t


def _knn_lists(xyz, node_xyz, k, sigma=0.1):
    from manigaussian_b200 import gaussian_renderer as GR
    nn = GR.knn(node_xyz.cuda(), k, queries=xyz.cuda())
    w = torch.softmax(torch.where(nn["index"] >= 0, -nn["dist2"] / (2 * sigma ** 2), torch.full_like(nn["dist2"], -1e30)), 1)
    return nn["index"].cpu(), torch.where(nn["index"] >= 0, w, torch.zeros_like(w)).cpu()


def _cot(P, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(P, 3, generator=g), torch.randn(P, 4, generator=g)


def _run_gpu(inputs, needs=(True,) * 6, cot=None):
    from manigaussian_b200 import gaussian_renderer as GR
    xyz, rot, node_xyz, node_rot, node_t, index, weight = inputs
    ins = [t.cuda().requires_grad_(n) for t, n in zip((xyz, rot, node_xyz, node_rot, node_t, weight), needs)]
    out = GR.deform_gaussians(*ins[:5], index.cuda(), ins[5])
    gx, gr = cot if cot is not None else _cot(xyz.shape[0])
    if any(needs):
        ((out["xyz"] * gx.cuda()).sum() + (out["rot"] * gr.cuda()).sum()).backward()
    return [out["xyz"].detach().cpu(), out["rot"].detach().cpu()], [t.grad.cpu() if t.grad is not None else None for t in ins]


def _run_ref(inputs, grads=True, cot=None):
    xyz, rot, node_xyz, node_rot, node_t, index, weight = inputs
    ins = [t.double().requires_grad_(grads) for t in (xyz, rot, node_xyz, node_rot, node_t, weight)]
    out = D64.deform_ref64(*ins[:5], index, ins[5])
    if not grads:
        return [o.detach() for o in out], None
    gx, gr = cot if cot is not None else _cot(xyz.shape[0])
    ((out[0] * gx.double()).sum() + (out[1] * gr.double()).sum()).backward()
    return [o.detach() for o in out], [t.grad for t in ins]


def _check(inputs, grads=True, rtol_out=1e-5, rtol_grad=1e-4):
    og, gg = _run_gpu(inputs, needs=(grads,) * 6)
    orf, gr = _run_ref(inputs, grads=grads)
    for name, a, b in zip(("xyz'", "rot'"), og, orf):
        err = (a.double() - b).abs().max() / max(b.abs().max().item(), 1e-30)
        assert err <= rtol_out, (name, float(err))
    if grads:
        for name, a, b in zip(_NAMES, gg, gr):
            if b.numel() == 0:
                assert a.shape == b.shape
                continue
            err = util.rel_l2(a.numpy(), b.numpy())
            assert err < rtol_grad, (name, err)
    return og, gg


@pytest.mark.parametrize("kind", ["uniform", "surface"])
@pytest.mark.parametrize("k", [1, 4, 8, 20, 32])
def test_knn_lists_match_the_reference(kind, k):
    xyz, rot, node_xyz, node_rot, node_t = _cloud(kind, 6000, N=256, seed=k)
    index, weight = _knn_lists(xyz, node_xyz, k)
    _check((xyz, rot, node_xyz, node_rot, node_t, index, weight))


def test_hand_built_lists_with_padding_out_of_range_and_repeats():
    P, N, k = 3000, 40, 12
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", P, N=N, seed=3)
    g = torch.Generator().manual_seed(4)
    index = torch.randint(0, N, (P, k), generator=g)
    index[:, 1] = index[:, 0]                         # one node twice in a row
    index[::3, 2] = -1                                # knn's padding
    index[::5, 3] = N                                 # out of range
    index[::7, 4] = 2 ** 40
    index[::11, 5] = -(2 ** 35)
    index[:, 10:] = -1                                # padded tails
    index[:50] = -1                                   # rows with no valid slot
    weight = 0.15 * torch.rand(P, k, generator=g) - 0.03  # negative weights; rows do not sum to 1
    weight[50:80] = 0.0                               # rows with zero weights
    og, _ = _check((xyz, rot, node_xyz, node_rot, node_t, index, weight))
    assert torch.equal(og[0][:80], xyz[:80]) and torch.equal(og[1][:80], rot[:80])


@pytest.mark.parametrize("case", ["negative_real", "unnormalised", "zero"])
def test_node_quaternions(case):
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 4000, N=128, seed=5)
    index, weight = _knn_lists(xyz, node_xyz, 8)
    if case == "negative_real":
        node_rot[:, 0] = -node_rot[:, 0].abs()
        node_rot[::2] *= -1
    elif case == "unnormalised":
        node_rot[::3] *= 37.0
        node_rot[1::3] *= 1e-3
    else:
        node_rot[::9] = 0.0
    _check((xyz, rot, node_xyz, node_rot, node_t, index, weight))


def test_negated_nodes_give_the_same_output():
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 4000, N=128, seed=6)
    index, weight = _knn_lists(xyz, node_xyz, 8)
    a, _ = _run_gpu((xyz, rot, node_xyz, node_rot, node_t, index, weight), needs=(False,) * 6)
    b, _ = _run_gpu((xyz, rot, node_xyz, -node_rot, node_t, index, weight), needs=(False,) * 6)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_no_gaussians_and_no_nodes():
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 100, N=8, seed=7)
    e3, e4 = torch.zeros(0, 3), torch.zeros(0, 4)
    out, g = _run_gpu((e3, e4, node_xyz, node_rot, node_t, torch.zeros(0, 4, dtype=torch.int64), torch.zeros(0, 4)),
                      cot=(e3, e4))
    assert [tuple(t.shape) for t in out] == [(0, 3), (0, 4)]
    assert [tuple(t.shape) for t in g] == [(0, 3), (0, 4), (8, 3), (8, 4), (8, 3), (0, 4)]
    assert all((t == 0).all() for t in g[2:5])
    index = torch.full((100, 4), -1, dtype=torch.int64)
    index[::2, 0] = 3  # out of range of N = 0
    inputs = (xyz, rot, e3, e4, e3, index, torch.rand(100, 4))
    out, g = _run_gpu(inputs)
    assert torch.equal(out[0], xyz) and torch.equal(out[1], rot)
    gx, gr = _cot(100)
    assert torch.equal(g[0], gx) and torch.equal(g[1], gr)
    assert [tuple(t.shape) for t in g[2:5]] == [(0, 3), (0, 4), (0, 3)]
    assert (g[5] == 0).all()


def test_c3_size_forward():
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 500_000, N=4096, seed=8)
    index, weight = _knn_lists(xyz, node_xyz, 8, sigma=0.03)
    _check((xyz, rot, node_xyz, node_rot, node_t, index, weight), grads=False)


def test_fifty_thousand_gaussians_gradients():
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 50_000, N=1024, seed=9)
    index, weight = _knn_lists(xyz, node_xyz, 8, sigma=0.05)
    _check((xyz, rot, node_xyz, node_rot, node_t, index, weight))


def test_rigid_segments():
    """500k Gaussians on 3 nodes, k = 1: a moving gripper and object with weight 1, the table with weight 0"""
    P = 500_000
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", P, N=3, seed=10)
    g = torch.Generator().manual_seed(11)
    index = torch.randint(0, 3, (P, 1), generator=g)
    weight = (index != 2).float()
    _check((xyz, rot, node_xyz, node_rot, node_t, index, weight))


def test_learnable_weight_from_node_radii():
    """SC-GS's weights softmax(-d^2 / 2 sigma_j^2), with a learnable radius per node, built in torch: the gradients to
    node_xyz (through both the motion and the weight) and sigma match float64"""
    from manigaussian_b200 import gaussian_renderer as GR
    xyz, rot, node_xyz, node_rot, node_t = _cloud("surface", N=256, seed=12)
    index, _ = _knn_lists(xyz, node_xyz, 8)
    sigma = 0.05 + 0.1 * torch.rand(256, generator=torch.Generator().manual_seed(13))
    gx, gr = _cot(xyz.shape[0], seed=14)

    def run(dev, dtype, fn):
        nx = node_xyz.to(dev, dtype).requires_grad_()
        sg = sigma.to(dev, dtype).requires_grad_()
        idx = index.to(dev)
        valid = idx >= 0
        j = idx.clamp(min=0)
        d2 = ((xyz.to(dev, dtype)[:, None] - nx[j]) ** 2).sum(-1)
        logit = torch.where(valid, -d2 / (2 * sg[j] ** 2), torch.full_like(d2, -1e30))
        w = torch.where(valid, torch.softmax(logit, 1), torch.zeros_like(d2))
        out = fn(xyz.to(dev, dtype), rot.to(dev, dtype), nx, node_rot.to(dev, dtype), node_t.to(dev, dtype), idx, w)
        ((out[0] * gx.to(dev, dtype)).sum() + (out[1] * gr.to(dev, dtype)).sum()).backward()
        return nx.grad.double().cpu(), sg.grad.double().cpu()

    def fused(*a):
        o = GR.deform_gaussians(*a)
        return o["xyz"], o["rot"]
    got = run("cuda", torch.float32, fused)
    want = run("cpu", torch.float64, D64.deform_ref64)
    for name, a, b in zip(("node_xyz", "sigma"), got, want):
        assert util.rel_l2(a.numpy(), b.numpy()) < 1e-4, name


def test_next_frame_only_gradients_equal_the_all_grad_call():
    xyz, rot, node_xyz, node_rot, node_t = _cloud("surface", N=256, seed=15)
    index, weight = _knn_lists(xyz, node_xyz, 8)
    inputs = (xyz, rot, node_xyz, node_rot, node_t, index, weight)
    o_all, g_all = _run_gpu(inputs)
    o_next, g_next = _run_gpu(inputs, needs=(False, False, False, True, True, False))
    assert torch.equal(o_all[0], o_next[0]) and torch.equal(o_all[1], o_next[1])
    assert all(g_next[n] is None for n in (0, 1, 2, 5))
    for n in (3, 4):
        assert util.rel_l2(g_next[n].numpy(), g_all[n].numpy()) < 1e-6


def test_deform_then_render_matches_the_torch_restatement():
    from manigaussian_b200 import gaussian_renderer as GR
    from test_planar_depth_gpu import _inputs, _settings, _t
    P, W, H = 2000, 96, 64
    inps, g = _inputs(P, W, H, 0, 2, seed=16)
    views = [_settings(i, 0) for i in inps]
    means = torch.from_numpy(np.asarray(g["means3D"], np.float32))
    rot = torch.from_numpy(np.asarray(g["rotations"], np.float32))
    gen = torch.Generator().manual_seed(17)
    node_xyz = means[torch.randperm(P, generator=gen)[:32]].clone()
    node_rot = torch.tensor([1.0, 0.0, 0.0, 0.0]) + 0.05 * torch.randn(32, 4, generator=gen)
    node_t = 0.02 * torch.randn(32, 3, generator=gen)
    index, weight = _knn_lists(means, node_xyz, 4, sigma=0.3)
    gc = torch.randn((2, 3, H, W), device="cuda", generator=torch.Generator("cuda").manual_seed(18))
    cloud = dict(scales=_t(g["scales"]), opacity=_t(g["opacities"]).reshape(-1, 1), features_color=_t(g["shs"]))

    def run(fn):
        nr = node_rot.cuda().requires_grad_()
        nt = node_t.cuda().requires_grad_()
        xyz2, rot2 = fn(means.cuda(), rot.cuda(), node_xyz.cuda(), nr, nt, index.cuda(), weight.cuda())
        res = GR.render_views(views, xyz2, rot2, cloud["scales"], cloud["opacity"], features_color=cloud["features_color"])
        (res["render"] * gc).sum().backward()
        return nr.grad.cpu(), nt.grad.cpu()

    def fused(*a):
        o = GR.deform_gaussians(*a)
        return o["xyz"], o["rot"]
    got = run(fused)
    want = run(D64.deform_ref64)  # the restatement in float32 on the GPU
    for name, a, b in zip(("node_rot", "node_t"), got, want):
        assert util.rel_l2(a.numpy(), b.numpy()) < 1e-4, name


def test_forward_outputs_are_bitwise_identical_across_calls():
    from manigaussian_b200 import gaussian_renderer as GR
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 100_000, N=512, seed=19)
    index, weight = _knn_lists(xyz, node_xyz, 8)
    args = [t.cuda() for t in (xyz, rot, node_xyz, node_rot, node_t, index, weight)]
    a = GR.deform_gaussians(*args)
    b = GR.deform_gaussians(*args)
    for n in ("xyz", "rot"):
        assert torch.equal(a[n].view(torch.int32), b[n].view(torch.int32))


def test_cuda_graph_replay_on_new_values():
    from manigaussian_b200 import gaussian_renderer as GR
    P, N, k = 5000, 128, 8
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", P, N=N, seed=20)
    index, weight = _knn_lists(xyz, node_xyz, k)
    static = [t.cuda().requires_grad_() for t in (xyz, rot, node_xyz, node_rot, node_t, weight)]
    s_index = index.cuda()
    gx, gr = (t.cuda() for t in _cot(P, seed=21))

    def step():
        for t in static:
            t.grad = None
        out = GR.deform_gaussians(*static[:5], s_index, static[5])
        ((out["xyz"] * gx).sum() + (out["rot"] * gr).sum()).backward()
        return out["xyz"].detach(), out["rot"].detach()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for t in static:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = step()
    new = _cloud("uniform", P, N=N, seed=22)
    new_index, new_weight = _knn_lists(new[0], new[2], k)
    with torch.no_grad():
        for t, v in zip(static, list(new) + [new_weight]):
            t.copy_(v.cuda())
        s_index.copy_(new_index.cuda())
    graph.replay()
    torch.cuda.synchronize()
    out, grads = _run_ref(tuple(new) + (new_index, new_weight), cot=(gx.cpu(), gr.cpu()))
    for a, b in zip(cap, out):
        np.testing.assert_allclose(a.cpu().numpy(), b.numpy(), rtol=1e-5, atol=1e-6)
    for t, b in zip(static, grads):
        assert util.rel_l2(t.grad.cpu().numpy(), b.numpy()) < 1e-4


def test_repeated_calls_do_not_grow_device_memory():
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 20_000, N=256, seed=23)
    index, weight = _knn_lists(xyz, node_xyz, 8)
    inputs = (xyz, rot, node_xyz, node_rot, node_t, index, weight)
    for _ in range(3):
        _run_gpu(inputs)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for _ in range(20):
        _run_gpu(inputs)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= before


def test_a_call_on_a_non_current_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import gaussian_renderer as GR
    xyz, rot, node_xyz, node_rot, node_t = _cloud("uniform", 3000, N=64, seed=24)
    index, weight = _knn_lists(xyz, node_xyz, 8)
    d1 = torch.device("cuda:1")
    ins = [t.to(d1).requires_grad_() for t in (xyz, rot, node_xyz, node_rot, node_t, weight)]
    out = GR.deform_gaussians(*ins[:5], index.to(d1), ins[5])
    assert out["xyz"].device == d1
    gx, gr = _cot(3000)
    ((out["xyz"] * gx.to(d1)).sum() + (out["rot"] * gr.to(d1)).sum()).backward()
    o, grads = _run_ref((xyz, rot, node_xyz, node_rot, node_t, index, weight))
    np.testing.assert_allclose(out["xyz"].detach().cpu().numpy(), o[0].numpy(), rtol=1e-5, atol=1e-6)
    for t, b in zip(ins, grads):
        assert t.grad.device == d1
        assert util.rel_l2(t.grad.cpu().numpy(), b.numpy()) < 1e-4
