"""Neighbour regularisers without a GPU: the float64 reference (tests/neighbour_reg_ref64.py) against INTEGRATION.md's
restatement, gradcheck of the reference and its conventions (zero offsets and j = i, padded and out-of-range slots, a zero
quaternion, rot == rot_next), the C ABI's declarations, exports and argument errors, and the Python surface's refusals
(gaussian_renderer.neighbour_regularisers)."""
import os
import re

import numpy as np
import pytest
import torch

import neighbour_reg_ref64 as N64
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR


def _inputs(P=60, k=5, seed=0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(P, 3, generator=g, dtype=dtype)
    rot = torch.randn(P, 4, generator=g, dtype=dtype)
    xyz_next = xyz + 0.05 * torch.randn(P, 3, generator=g, dtype=dtype)
    rot_next = rot + 0.1 * torch.randn(P, 4, generator=g, dtype=dtype)
    index = torch.stack([torch.randperm(P, generator=g)[:k] for _ in range(P)])
    weight = torch.rand(P, k, generator=g, dtype=dtype)
    return xyz, rot, xyz_next, rot_next, index, weight


def _grads(fn, xyz, rot, xyz_next, rot_next, index, weight, cot=(1.0, 0.7, 1.3)):
    ins = [t.clone().requires_grad_() for t in (xyz, rot, xyz_next, rot_next)]
    out = fn(*ins, index, weight)
    sum(c * o for c, o in zip(cot, out)).backward()
    return [o.detach() for o in out], [t.grad for t in ins]


def test_reference_equals_the_integration_restatement_without_padding():
    inp = _inputs(P=200, k=20, seed=1)
    lr, gr = _grads(N64.neighbour_reg_ref64, *inp)
    li, gi = _grads(N64.integration_restatement, *inp)
    for a, b in zip(lr, li):
        assert torch.allclose(a, b, rtol=1e-13, atol=0)
    for a, b in zip(gr, gi):
        assert torch.allclose(a, b, rtol=1e-11, atol=1e-15)


def test_gradcheck_of_the_reference():
    xyz, rot, xyz_next, rot_next, index, weight = _inputs(P=12, k=4, seed=2)
    index[0, 1] = -1
    index[3, 0] = 12

    def f(a, b, c, d):
        r, t, i = N64.neighbour_reg_ref64(a, b, c, d, index, weight)
        return r + 0.5 * t + 2.0 * i
    assert torch.autograd.gradcheck(f, tuple(t.clone().requires_grad_() for t in (xyz, rot, xyz_next, rot_next)))


def test_zero_offsets_and_self_slots_add_nothing():
    xyz, rot, xyz_next, rot_next, index, weight = _inputs(P=20, k=4, seed=3)
    base, _ = _grads(N64.neighbour_reg_ref64, xyz, rot, xyz_next, rot_next, index, weight)
    # slot 0 of every row points to the Gaussian itself: its terms are 0 and so are its gradients
    idx = torch.cat([torch.arange(20)[:, None], index], 1)
    w = torch.cat([torch.ones(20, 1, dtype=weight.dtype), weight], 1)
    out, g = _grads(N64.neighbour_reg_ref64, xyz, rot, xyz_next, rot_next, idx, w)
    for a, b in zip(out, base):
        assert torch.allclose(a * 5, b * 4, rtol=1e-13)
    gs = _grads(N64.neighbour_reg_ref64, xyz, rot, xyz_next, rot_next, idx[:, :1], w[:, :1])[1]
    assert all(torch.isfinite(t).all() and (t == 0).all() for t in gs)
    # duplicate points: o = 0 with o' = 0 gives a zero isometry term and no NaN
    xyz[1], xyz_next[1] = xyz[0], xyz_next[0]
    out, g = _grads(N64.neighbour_reg_ref64, xyz, rot, xyz_next, rot_next, torch.tensor([[1]] * 20), torch.ones(20, 1,
                                                                                                               dtype=xyz.dtype))
    assert all(torch.isfinite(t).all() for t in g)


def test_padded_and_out_of_range_slots_are_skipped():
    xyz, rot, xyz_next, rot_next, index, weight = _inputs(P=30, k=6, seed=4)
    bad = index.clone()
    bad[:, 4] = -1
    bad[:, 5] = torch.tensor([30, 10 ** 9, -7] * 10)
    out, g = _grads(N64.neighbour_reg_ref64, xyz, rot, xyz_next, rot_next, bad, weight)
    kept, gk = _grads(N64.neighbour_reg_ref64, xyz, rot, xyz_next, rot_next, index[:, :4], weight[:, :4])
    for a, b in zip(out, kept):  # the same sums over P k = 30 * 6 instead of 30 * 4
        assert torch.allclose(a * 6, b * 4, rtol=1e-13)
    for a, b in zip(g, gk):
        assert torch.allclose(a * 6, b * 4, rtol=1e-12, atol=1e-15)


def test_zero_quaternion_gives_identity_rotation_and_finite_gradients():
    xyz, rot, xyz_next, rot_next, index, weight = _inputs(P=16, k=3, seed=5)
    rot[2] = 0.0
    rot_next[5] = 0.0
    out, g = _grads(N64.neighbour_reg_ref64, xyz, rot, xyz_next, rot_next, index, weight)
    assert all(torch.isfinite(t).all() for t in list(out) + g)
    # below the clamp the gradient is that of x / 1e-12: at 0 it is the upstream gradient of q times 1e12
    rel = N64.qmul(torch.nn.functional.normalize(rot_next, dim=-1), torch.zeros(16, 4, dtype=rot.dtype))
    assert (rel[2] == 0).all()
    assert g[1][2].abs().max() > 1e6


def test_equal_rotations_give_identity_rel_and_r():
    xyz, rot, xyz_next, _, index, weight = _inputs(P=25, k=5, seed=6)
    q = torch.nn.functional.normalize(rot, dim=-1)
    rel = N64.qmul(q, q * q.new_tensor([1.0, -1.0, -1.0, -1.0]))
    assert torch.allclose(rel, rel.new_tensor([1.0, 0, 0, 0]).expand_as(rel), atol=1e-15)
    assert torch.allclose(N64.qrot(rel), torch.eye(3, dtype=rel.dtype).expand(25, 3, 3), atol=1e-15)
    # R = I: rigid is the plain offset change, rotation is 0
    rigid, rotation, _ = N64.neighbour_reg_ref64(xyz, rot, xyz_next, rot.clone(), index, weight)
    off = xyz[index] - xyz[:, None]
    off_next = xyz_next[index] - xyz_next[:, None]
    assert torch.allclose(rigid, (weight * (off_next - off).norm(dim=-1)).mean(), rtol=1e-12)
    assert rotation.abs() < 1e-14


def test_zero_gaussians_give_zeros():
    e3, e4 = torch.zeros(0, 3, dtype=torch.float64), torch.zeros(0, 4, dtype=torch.float64)
    out = N64.neighbour_reg_ref64(e3, e4, e3, e4, torch.zeros(0, 5, dtype=torch.int64), torch.zeros(0, 5, dtype=torch.float64))
    assert [float(t) for t in out] == [0.0, 0.0, 0.0]


# --------------------------------------------------------------------------- C ABI
_CALLS = ("mgs_neighbour_reg_state_bytes", "mgs_neighbour_reg", "mgs_neighbour_reg_backward")


def test_header_declares_and_the_library_exports_the_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    for sym in _CALLS:
        assert re.search(r"\b%s\s*\(" % sym, hdr)
        assert sym in _binding.EXPORTED_SYMBOLS
        assert hasattr(_binding.lib(), sym)
    L = _binding.lib()
    assert L.mgs_neighbour_reg_state_bytes(1000, 20) >= 1000 * (48 + 48 + 48)
    assert L.mgs_neighbour_reg_state_bytes(0, 20) > 0


_S = 4096  # a non-NULL address: every call below fails before it could be used


@pytest.mark.parametrize("args,code,msg", [
    ((_S, 10, 33, _S, _S, _S, _S, _S, _S, _S), -2, "at most 32"),
    ((_S, 10, 0, _S, _S, _S, _S, _S, _S, _S), -1, "k must be"),
    ((_S, -1, 3, _S, _S, _S, _S, _S, _S, _S), -1, "P must be"),
    ((None, 10, 3, _S, _S, _S, _S, _S, _S, _S), -1, "required"),
    ((_S, 10, 3, _S, _S, _S, _S, _S, _S, None), -1, "required"),
    ((_S, 10, 3, None, _S, _S, _S, _S, _S, _S), -1, "required"),
    ((_S, 10, 3, _S, None, _S, _S, _S, _S, _S), -1, "required"),
    ((_S, 10, 3, _S, _S, None, _S, _S, _S, _S), -1, "required"),
    ((_S, 10, 3, _S, _S, _S, None, _S, _S, _S), -1, "required"),
    ((_S, 10, 3, _S, _S, _S, _S, None, _S, _S), -1, "required"),
    ((_S, 10, 3, _S, _S, _S, _S, _S, None, _S), -1, "required"),
])
def test_argument_errors_return_their_code_without_touching_a_gpu(args, code, msg):
    L = _binding.lib()
    assert L.mgs_neighbour_reg(*args, 0, None) == code
    assert msg in _binding.last_error() and "mgs_neighbour_reg" in _binding.last_error()
    assert L.mgs_neighbour_reg_backward(*args, None, None, None, None, 0, None) == code
    assert msg in _binding.last_error() and "mgs_neighbour_reg_backward" in _binding.last_error()


def test_backward_with_no_gaussians_is_a_no_op():
    L = _binding.lib()
    assert L.mgs_neighbour_reg_backward(_S, 0, 3, None, None, None, None, None, None, _S, None, None, None, None, 0, None) == 0


# --------------------------------------------------------------------------- Python surface
def _t(P=8, k=3):
    return dict(xyz=torch.zeros(P, 3), rot=torch.zeros(P, 4), xyz_next=torch.zeros(P, 3), rot_next=torch.zeros(P, 4),
                index=torch.zeros(P, k, dtype=torch.int64), weight=torch.zeros(P, k))


@pytest.mark.parametrize("case,match", [
    (dict(xyz=torch.zeros(8, 4)), r"xyz: expected \[8,3\]"),
    (dict(rot=torch.zeros(8, 3)), r"rot: expected \[8,4\]"),
    (dict(xyz_next=torch.zeros(7, 3)), r"xyz_next: expected \[8,3\]"),
    (dict(rot_next=torch.zeros(8, 4, dtype=torch.float64)), "float32"),
    (dict(index=torch.zeros(8, 3, dtype=torch.int32)), "int64"),
    (dict(index=torch.zeros(8, dtype=torch.int64)), "index: expected"),
    (dict(index=torch.zeros(9, 3, dtype=torch.int64)), "index: expected"),
    (dict(weight=torch.zeros(8, 4)), r"weight: expected \[8,k\]"),
    (dict(weight=torch.zeros(8, 3, dtype=torch.float16)), "float32"),
    (dict(index=torch.zeros(8, 33, dtype=torch.int64), weight=torch.zeros(8, 33)), "1 .. 32"),
    (dict(index=torch.zeros(8, 0, dtype=torch.int64), weight=torch.zeros(8, 0)), "1 .. 32"),
    (dict(weight=torch.zeros(8, 3, requires_grad=True)), "requires grad"),
    (dict(xyz=np.zeros((8, 3), np.float32)), "expected a tensor"),
    (dict(rot=torch.zeros(8, 4, device="meta")), "expected a tensor on cpu"),
])
def test_neighbour_regularisers_rejects_bad_arguments(case, match):
    kw = _t()
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.neighbour_regularisers(**kw)


def test_neighbour_regularisers_has_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.neighbour_regularisers(**_t())
