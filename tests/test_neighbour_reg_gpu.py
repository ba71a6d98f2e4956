"""Neighbour regularisers on the GPU (neighbour_reg.cu, mgs_neighbour_reg, gaussian_renderer.neighbour_regularisers).

1. Against the float64 reference (tests/neighbour_reg_ref64.py): losses within 1e-5 relative, the four gradients within
   1e-4 relative L2, for k = 1, 3, 8, 20, 32 on knn lists over uniform and rendered-surface clouds, on hand-built lists with
   -1 padding, out-of-range indices, j = i and duplicate points, with unnormalised, near-zero and zero quaternions, P = 0,
   the losses at c3 size (500k Gaussians) and the gradients at 50k.
2. Only xyz_next and rot_next requiring grad (ManiGaussian's next-frame pass): the same gradients, none for xyz and rot.
3. Forward losses bitwise identical across calls; CUDA-graph capture of forward + backward replayed on new values; no
   device-memory growth over repeated calls; a call on a non-current device.
"""
import numpy as np
import pytest
import torch

import neighbour_reg_ref64 as N64
import util

pytestmark = pytest.mark.gpu

_COT = (1.0, 0.7, 1.3)  # upstream gradients of rigid, rotation, isometry


def _surface_points():
    """the scene's depth image unprojected, as tests/test_knn_gpu.py builds it (16,384 points, some on the camera centre)"""
    from test_knn_gpu import _surface
    return torch.from_numpy(_surface())


def _cloud(kind, P=None, seed=0):
    """xyz [P,3] (the 16,384 surface points for "surface") and a small deformation of it for the next frame"""
    g = torch.Generator().manual_seed(seed)
    xyz = _surface_points() if kind == "surface" else torch.rand(P, 3, generator=g)
    P = xyz.shape[0]
    rot = torch.randn(P, 4, generator=g)
    xyz_next = xyz + 0.01 * torch.randn(P, 3, generator=g)
    rot_next = rot + 0.05 * torch.randn(P, 4, generator=g)
    return xyz, rot, xyz_next, rot_next


def _knn_lists(xyz, k, lam=2000.0):
    from manigaussian_b200 import gaussian_renderer as GR
    nn = GR.knn(xyz.cuda(), k)
    w = torch.exp(-lam * nn["dist2"])
    return nn["index"].cpu(), torch.where(nn["index"] >= 0, w, torch.zeros_like(w)).cpu()


def _run_gpu(xyz, rot, xyz_next, rot_next, index, weight, needs=(True,) * 4):
    from manigaussian_b200 import gaussian_renderer as GR
    ins = [t.cuda().requires_grad_(n) for t, n in zip((xyz, rot, xyz_next, rot_next), needs)]
    out = GR.neighbour_regularisers(*ins, index.cuda(), weight.cuda())
    loss = [out[n] for n in ("rigid", "rotation", "isometry")]
    sum(c * o for c, o in zip(_COT, loss)).backward()
    return [float(o.detach()) for o in loss], [t.grad.cpu() if t.grad is not None else None for t in ins]


def _run_ref(xyz, rot, xyz_next, rot_next, index, weight, grads=True):
    ins = [t.double().requires_grad_(grads) for t in (xyz, rot, xyz_next, rot_next)]
    out = N64.neighbour_reg_ref64(*ins, index, weight.double())
    if not grads:
        return [float(o) for o in out], None
    sum(c * o for c, o in zip(_COT, out)).backward()
    return [float(o) for o in out], [t.grad for t in ins]


def _check(inputs, grads=True, rtol_loss=1e-5, rtol_grad=1e-4):
    lg, gg = _run_gpu(*inputs)
    lr, gr = _run_ref(*inputs, grads=grads)
    for name, a, b in zip(("rigid", "rotation", "isometry"), lg, lr):
        assert abs(a - b) <= rtol_loss * abs(b) + 1e-30, (name, a, b)
    if grads:
        for name, a, b in zip(("xyz", "rot", "xyz_next", "rot_next"), gg, gr):
            err = util.rel_l2(a.numpy(), b.numpy())
            assert err < rtol_grad, (name, err)
    return lg, gg


@pytest.mark.parametrize("kind", ["uniform", "surface"])
@pytest.mark.parametrize("k", [1, 3, 8, 20, 32])
def test_knn_lists_match_the_reference(kind, k):
    xyz, rot, xyz_next, rot_next = _cloud(kind, 6000, seed=k)
    index, weight = _knn_lists(xyz, k)
    _check((xyz, rot, xyz_next, rot_next, index, weight))


def test_hand_built_lists_with_padding_out_of_range_self_and_duplicates():
    P, k = 3000, 12
    xyz, rot, xyz_next, rot_next = _cloud("uniform", P, seed=3)
    xyz[1:40] = xyz[0]           # duplicate points (o = 0 between them)
    xyz_next[1:20] = xyz_next[0]  # and some also coincide in the next frame (o' = 0)
    g = torch.Generator().manual_seed(4)
    index = torch.randint(0, P, (P, k), generator=g)
    index[:, 0] = torch.arange(P)                      # j = i
    index[:40, 1] = torch.arange(40).flip(0)           # the duplicates point at each other
    index[::3, 2] = -1                                 # knn's padding
    index[::5, 3] = P                                  # out of range
    index[::7, 4] = 2 ** 40
    index[::11, 5] = -(2 ** 35)
    index[:, 10:] = -1                                 # padded tails
    weight = torch.rand(P, k, generator=g)
    _check((xyz, rot, xyz_next, rot_next, index, weight))


@pytest.mark.parametrize("case", ["unnormalised", "near_zero", "below_clamp", "zero"])
def test_quaternions_far_from_unit_length(case):
    xyz, rot, xyz_next, rot_next = _cloud("uniform", 4000, seed=5)
    index, weight = _knn_lists(xyz, 8)
    sel = slice(0, 4000, 9)
    scale = {"unnormalised": 37.0, "near_zero": 1e-6, "below_clamp": 1e-14, "zero": 0.0}[case]
    rot[sel] *= scale
    rot_next[1::13] *= scale
    if case == "unnormalised":
        rot_next *= 0.02
    _check((xyz, rot, xyz_next, rot_next, index, weight))


def test_no_gaussians_give_zeros_and_empty_gradients():
    e3, e4 = torch.zeros(0, 3), torch.zeros(0, 4)
    loss, g = _run_gpu(e3, e4, e3, e4, torch.zeros(0, 20, dtype=torch.int64), torch.zeros(0, 20))
    assert loss == [0.0, 0.0, 0.0]
    assert [tuple(t.shape) for t in g] == [(0, 3), (0, 4), (0, 3), (0, 4)]


def test_c3_size_losses():
    xyz, rot, xyz_next, rot_next = _cloud("uniform", 500_000, seed=7)
    index, weight = _knn_lists(xyz, 20, lam=1e5)
    _check((xyz, rot, xyz_next, rot_next, index, weight), grads=False)


def test_fifty_thousand_gaussians_gradients():
    xyz, rot, xyz_next, rot_next = _cloud("uniform", 50_000, seed=8)
    index, weight = _knn_lists(xyz, 20, lam=1e4)
    _check((xyz, rot, xyz_next, rot_next, index, weight))


def test_next_frame_only_gradients_equal_the_all_grad_call():
    xyz, rot, xyz_next, rot_next = _cloud("surface", seed=9)
    index, weight = _knn_lists(xyz, 20)
    inputs = (xyz, rot, xyz_next, rot_next, index, weight)
    l_all, g_all = _run_gpu(*inputs)
    l_next, g_next = _run_gpu(*inputs, needs=(False, False, True, True))
    assert l_all == l_next
    assert g_next[0] is None and g_next[1] is None
    for a, b in ((g_next[2], g_all[2]), (g_next[3], g_all[3])):
        assert util.rel_l2(a.numpy(), b.numpy()) < 1e-6


def test_forward_losses_are_bitwise_identical_across_calls():
    from manigaussian_b200 import gaussian_renderer as GR
    xyz, rot, xyz_next, rot_next = (t.cuda() for t in _cloud("uniform", 100_000, seed=10))
    index, weight = (t.cuda() for t in _knn_lists(xyz.cpu(), 20))
    a = GR.neighbour_regularisers(xyz, rot, xyz_next, rot_next, index, weight)
    b = GR.neighbour_regularisers(xyz, rot, xyz_next, rot_next, index, weight)
    for n in ("rigid", "rotation", "isometry"):
        assert a[n].item() == b[n].item()
        assert a[n].view(1).view(torch.int32).item() == b[n].view(1).view(torch.int32).item()


def test_cuda_graph_replay_on_new_values():
    from manigaussian_b200 import gaussian_renderer as GR
    P, k = 5000, 20
    xyz, rot, xyz_next, rot_next = _cloud("uniform", P, seed=11)
    index, weight = _knn_lists(xyz, k)
    static = [t.cuda().requires_grad_() for t in (xyz, rot, xyz_next, rot_next)]
    s_index, s_weight = index.cuda(), weight.cuda()

    def step():
        for t in static:
            t.grad = None
        out = GR.neighbour_regularisers(*static, s_index, s_weight)
        total = _COT[0] * out["rigid"] + _COT[1] * out["rotation"] + _COT[2] * out["isometry"]
        total.backward()
        return torch.stack([out["rigid"], out["rotation"], out["isometry"]]).detach()

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
    new = _cloud("uniform", P, seed=12)
    new_index, new_weight = _knn_lists(new[0], k)
    with torch.no_grad():
        for t, v in zip(static, new):
            t.copy_(v.cuda())
        s_index.copy_(new_index.cuda())
        s_weight.copy_(new_weight.cuda())
    graph.replay()
    torch.cuda.synchronize()
    lr, gr = _run_ref(*new, new_index, new_weight)
    np.testing.assert_allclose(cap.cpu().numpy(), lr, rtol=1e-5)
    for t, b in zip(static, gr):
        assert util.rel_l2(t.grad.cpu().numpy(), b.numpy()) < 1e-4


def test_repeated_calls_do_not_grow_device_memory():
    xyz, rot, xyz_next, rot_next = _cloud("uniform", 20_000, seed=13)
    index, weight = _knn_lists(xyz, 20)
    inputs = (xyz, rot, xyz_next, rot_next, index, weight)
    for _ in range(3):
        _run_gpu(*inputs)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for _ in range(20):
        _run_gpu(*inputs)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= before


def test_a_call_on_a_non_current_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import gaussian_renderer as GR
    xyz, rot, xyz_next, rot_next = _cloud("uniform", 3000, seed=14)
    index, weight = _knn_lists(xyz, 8)
    d1 = torch.device("cuda:1")
    ins = [t.to(d1).requires_grad_() for t in (xyz, rot, xyz_next, rot_next)]
    out = GR.neighbour_regularisers(*ins, index.to(d1), weight.to(d1))
    assert out["rigid"].device == d1
    sum(c * out[n] for c, n in zip(_COT, ("rigid", "rotation", "isometry"))).backward()
    lr, gr = _run_ref(xyz, rot, xyz_next, rot_next, index, weight)
    np.testing.assert_allclose([float(out[n]) for n in ("rigid", "rotation", "isometry")], lr, rtol=1e-5)
    for t, b in zip(ins, gr):
        assert t.grad.device == d1
        assert util.rel_l2(t.grad.cpu().numpy(), b.numpy()) < 1e-4
