"""Control-graph deformation without a GPU: gradcheck of the float64 reference (tests/deform_ref64.py) in all six inputs and
its conventions (rows without weight or valid slots unchanged, k = 1 as a rigid motion, q and -q alike, identity nodes), the
C ABI's declarations, exports, state size and argument errors, and the Python surface's refusals
(gaussian_renderer.deform_gaussians)."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import deform_ref64 as D64
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR
from neighbour_reg_ref64 import qmul, qrot


def _inputs(P=40, N=7, k=4, seed=0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(P, 3, generator=g, dtype=dtype)
    rot = F.normalize(torch.randn(P, 4, generator=g, dtype=dtype), dim=-1)
    node_xyz = torch.rand(N, 3, generator=g, dtype=dtype)
    node_rot = torch.randn(N, 4, generator=g, dtype=dtype)
    node_t = 0.1 * torch.randn(N, 3, generator=g, dtype=dtype)
    index = torch.stack([torch.randperm(N, generator=g)[:k] for _ in range(P)])
    weight = torch.rand(P, k, generator=g, dtype=dtype)
    return xyz, rot, node_xyz, node_rot, node_t, index, weight


def test_gradcheck_of_the_reference_in_all_six_inputs():
    xyz, rot, node_xyz, node_rot, node_t, index, weight = _inputs(P=10, N=5, k=3, seed=1)
    index[0, 1] = -1
    index[3, 0] = 5
    index[4, 2] = index[4, 0]  # one node twice in a row
    weight[2, 0] = -0.4        # a negative weight
    node_rot[1, 0] = -abs(node_rot[1, 0])  # a flipped node

    def f(a, b, c, d, e, w):
        out_xyz, out_rot = D64.deform_ref64(a, b, c, d, e, index, w)
        return out_xyz, out_rot
    assert torch.autograd.gradcheck(f, tuple(t.clone().requires_grad_() for t in (xyz, rot, node_xyz, node_rot, node_t, weight)))


def test_rows_without_weight_or_valid_slots_are_unchanged_bitwise():
    xyz, rot, node_xyz, node_rot, node_t, index, weight = _inputs(P=30, N=6, k=5, seed=2)
    rot = torch.randn(30, 4, dtype=torch.float64)  # not unit: used as given
    weight[0] = 0.0
    index[1] = -1
    index[2] = torch.tensor([6, -1, 10 ** 9, -7, 6])
    out_xyz, out_rot = D64.deform_ref64(xyz, rot, node_xyz, node_rot, node_t, index, weight)
    for i in (0, 1, 2):
        assert torch.equal(out_xyz[i], xyz[i]) and torch.equal(out_rot[i], rot[i])
    assert not torch.equal(out_xyz[3], xyz[3])


def test_one_slot_with_unit_weight_is_the_node_rigid_motion():
    xyz, rot, node_xyz, node_rot, node_t, _, _ = _inputs(P=25, N=4, k=1, seed=3)
    index = torch.randint(0, 4, (25, 1))
    out_xyz, out_rot = D64.deform_ref64(xyz, rot, node_xyz, node_rot, node_t, index, torch.ones(25, 1, dtype=torch.float64))
    q = F.normalize(node_rot, dim=-1)
    q = torch.where(q[:, :1] < 0, -q, q)
    j = index[:, 0]
    p = node_xyz[j]
    want = (qrot(q[j]) @ (xyz - p)[..., None]).squeeze(-1) + p + node_t[j]
    assert torch.allclose(out_xyz, want, rtol=0, atol=1e-14)
    assert torch.allclose(out_rot, qmul(q[j], rot), rtol=0, atol=1e-15)


def test_a_node_and_its_negation_give_the_same_output():
    xyz, rot, node_xyz, node_rot, node_t, index, weight = _inputs(P=30, N=6, k=4, seed=4)
    a = D64.deform_ref64(xyz, rot, node_xyz, node_rot, node_t, index, weight)
    flip = torch.tensor([1.0, -1.0, 1.0, -1.0, -1.0, 1.0], dtype=torch.float64)[:, None]
    b = D64.deform_ref64(xyz, rot, node_xyz, node_rot * flip, node_t, index, weight)
    for x, y in zip(a, b):
        assert torch.allclose(x, y, rtol=0, atol=1e-15)


def test_identity_nodes_change_nothing():
    xyz, rot, node_xyz, _, _, index, weight = _inputs(P=30, N=6, k=4, seed=5)
    e = torch.tensor([[1.0, 0.0, 0.0, 0.0]], dtype=torch.float64).expand(6, 4)
    out_xyz, out_rot = D64.deform_ref64(xyz, rot, node_xyz, 3.0 * e, torch.zeros(6, 3, dtype=torch.float64), index, weight)
    assert torch.allclose(out_xyz, xyz, rtol=0, atol=1e-15)
    assert torch.allclose(out_rot, rot, rtol=0, atol=1e-15)


def test_no_nodes_return_the_cloud():
    xyz, rot, _, _, _, _, _ = _inputs(P=5, seed=6)
    e3, e4 = torch.zeros(0, 3, dtype=torch.float64), torch.zeros(0, 4, dtype=torch.float64)
    out = D64.deform_ref64(xyz, rot, e3, e4, e3, torch.full((5, 2), -1), torch.ones(5, 2, dtype=torch.float64))
    assert torch.equal(out[0], xyz) and torch.equal(out[1], rot)


# --------------------------------------------------------------------------- C ABI
_CALLS = ("mgs_deform_state_bytes", "mgs_deform", "mgs_deform_backward")


def test_header_declares_and_the_library_exports_the_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    for sym in _CALLS:
        assert re.search(r"\b%s\s*\(" % sym, hdr)
        assert sym in _binding.EXPORTED_SYMBOLS
        assert hasattr(_binding.lib(), sym)


def test_state_size_grows_with_gaussians_and_nodes_and_not_with_k():
    L = _binding.lib()
    base = L.mgs_deform_state_bytes(1000, 100, 8)
    assert base >= 1000 * 16 + 100 * 128
    assert L.mgs_deform_state_bytes(2000, 100, 8) > base
    assert L.mgs_deform_state_bytes(1000, 200, 8) > base
    assert L.mgs_deform_state_bytes(1000, 100, 32) >= base
    assert L.mgs_deform_state_bytes(0, 0, 1) > 0


_S = 4096  # a non-NULL address: every call below fails before it could be used


# (state, P, N, k, xyz, rot, node_xyz, node_rot, node_t, index, weight)
@pytest.mark.parametrize("args,code,msg", [
    ((_S, 10, 4, 33, _S, _S, _S, _S, _S, _S, _S), -2, "at most 32"),
    ((_S, 10, 4, 0, _S, _S, _S, _S, _S, _S, _S), -1, "k must be"),
    ((_S, -1, 4, 3, _S, _S, _S, _S, _S, _S, _S), -1, "P and N must be"),
    ((_S, 10, -1, 3, _S, _S, _S, _S, _S, _S, _S), -1, "P and N must be"),
    ((None, 10, 4, 3, _S, _S, _S, _S, _S, _S, _S), -1, "state is required"),
    ((_S, 10, 4, 3, None, _S, _S, _S, _S, _S, _S), -1, "required with P > 0"),
    ((_S, 10, 4, 3, _S, None, _S, _S, _S, _S, _S), -1, "required with P > 0"),
    ((_S, 10, 4, 3, _S, _S, _S, _S, _S, None, _S), -1, "required with P > 0"),
    ((_S, 10, 4, 3, _S, _S, _S, _S, _S, _S, None), -1, "required with P > 0"),
    ((_S, 10, 4, 3, _S, _S, None, _S, _S, _S, _S), -1, "required with N > 0"),
    ((_S, 10, 4, 3, _S, _S, _S, None, _S, _S, _S), -1, "required with N > 0"),
    ((_S, 10, 4, 3, _S, _S, _S, _S, None, _S, _S), -1, "required with N > 0"),
])
def test_argument_errors_return_their_code_without_touching_a_gpu(args, code, msg):
    L = _binding.lib()
    assert L.mgs_deform(*args, _S, _S, 0, None) == code
    assert msg in _binding.last_error() and "mgs_deform" in _binding.last_error()
    assert L.mgs_deform_backward(*args, None, None, None, None, None, None, None, None, 0, None) == code
    assert msg in _binding.last_error() and "mgs_deform_backward" in _binding.last_error()


@pytest.mark.parametrize("outs", [(None, _S), (_S, None)])
def test_forward_needs_its_outputs(outs):
    L = _binding.lib()
    assert L.mgs_deform(_S, 10, 4, 3, _S, _S, _S, _S, _S, _S, _S, *outs, 0, None) == -1
    assert "out_xyz and out_rot are required" in _binding.last_error()


# --------------------------------------------------------------------------- Python surface
def _t(P=8, N=5, k=3):
    return dict(xyz=torch.zeros(P, 3), rot=torch.zeros(P, 4), node_xyz=torch.zeros(N, 3), node_rot=torch.zeros(N, 4),
                node_t=torch.zeros(N, 3), index=torch.zeros(P, k, dtype=torch.int64), weight=torch.zeros(P, k))


@pytest.mark.parametrize("case,match", [
    (dict(xyz=torch.zeros(8, 4)), r"xyz: expected \[8,3\]"),
    (dict(rot=torch.zeros(8, 3)), r"rot: expected \[8,4\]"),
    (dict(node_xyz=torch.zeros(5, 4)), r"node_xyz: expected \[5,3\]"),
    (dict(node_rot=torch.zeros(6, 4)), r"node_rot: expected \[5,4\]"),
    (dict(node_t=torch.zeros(5)), r"node_t: expected \[5,3\]"),
    (dict(node_t=torch.zeros(5, 3, dtype=torch.float64)), "float32"),
    (dict(index=torch.zeros(8, 3, dtype=torch.int32)), "int64"),
    (dict(index=torch.zeros(8, dtype=torch.int64)), "index: expected"),
    (dict(index=torch.zeros(9, 3, dtype=torch.int64)), "index: expected"),
    (dict(weight=torch.zeros(8, 4)), r"weight: expected \[8,k\]"),
    (dict(weight=torch.zeros(8, 3, dtype=torch.float16)), "float32"),
    (dict(index=torch.zeros(8, 33, dtype=torch.int64), weight=torch.zeros(8, 33)), "1 .. 32"),
    (dict(index=torch.zeros(8, 0, dtype=torch.int64), weight=torch.zeros(8, 0)), "1 .. 32"),
    (dict(xyz=np.zeros((8, 3), np.float32)), "expected a tensor"),
    (dict(node_rot=torch.zeros(5, 4, device="meta")), "expected a tensor on cpu"),
])
def test_deform_gaussians_rejects_bad_arguments(case, match):
    kw = _t()
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.deform_gaussians(**kw)


def test_deform_gaussians_has_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.deform_gaussians(**_t())
    kw = _t()
    kw["weight"] = kw["weight"].requires_grad_()  # a learnable weight is accepted, and still needs the GPU
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.deform_gaussians(**kw)
