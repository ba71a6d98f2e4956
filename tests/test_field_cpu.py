"""The field query without a GPU: the C ABI's declarations and argument checks, query_field / voxelize's input checks, and
the float64 reference's own checks (an isotropic Gaussian's analytic value, the support box, the voxel-centre convention)."""
import math
import os
import re

import numpy as np
import pytest
import torch

import field_ref64 as F64
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR


def test_field_calls_are_declared_and_exported():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read(), flags=re.S)
    L = _binding.lib()
    for name in ("mgs_field_query", "mgs_field_query_backward"):
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _binding.EXPORTED_SYMBOLS and hasattr(L, name)


_CB = _binding.ALLOC_FN(lambda u, n: 0)  # never called: every case fails before anything is allocated


def _fwd(Q=4, P=4, C=3, points=4096, means=4096, scales=4096, rot=4096, opac=4096, feat=4096, cf=0, dens=4096, out=4096, cb=_CB):
    return _binding.lib().mgs_field_query(cb, None, cb, None, Q, P, C, points, means, scales, rot, opac, feat, cf, dens, out, 0, None)


def _bwd(Q=4, P=4, C=3, state=4096, pairs=4096, points=4096, scales=4096, rot=4096, feat=4096, cf=0, gd=4096, gf=4096):
    return _binding.lib().mgs_field_query_backward(state, pairs, Q, P, C, points, scales, rot, feat, cf, gd, gf,
                                                   4096, 4096, 4096, 4096, 4096, 4096, 0, None)


@pytest.mark.parametrize("case,code,msg", [
    ("C_neg", -2, "channel count"), ("C_513", -2, "channel count"), ("Q0", -1, "Q and P"), ("P0", -1, "Q and P"),
    ("no_alloc", -1, "allocator"), ("no_points", -1, "points"), ("no_opac", -1, "opacities"), ("no_density", -1, "out_density"),
    ("no_features", -1, "features"), ("no_out_features", -1, "out_features"), ("cf2", -1, "channel_first"),
])
def test_forward_argument_errors_return_their_code_without_touching_a_gpu(case, code, msg):
    kw = {"C_neg": dict(C=-1), "C_513": dict(C=513), "Q0": dict(Q=0), "P0": dict(P=-3), "no_alloc": dict(cb=_binding.ALLOC_FN()),
          "no_points": dict(points=None), "no_opac": dict(opac=None), "no_density": dict(dens=None), "no_features": dict(feat=None),
          "no_out_features": dict(out=None), "cf2": dict(cf=2)}[case]
    rc = _fwd(**kw)
    assert rc == code and msg in _binding.last_error(), (rc, _binding.last_error())


@pytest.mark.parametrize("case,code,msg", [
    ("C_513", -2, "channel count"), ("Q0", -1, "Q and P"), ("no_state", -1, "state"), ("no_pairs", -1, "pair_state"),
    ("no_scales", -1, "scales"), ("no_features", -1, "features"), ("cf2", -1, "channel_first"),
])
def test_backward_argument_errors_return_their_code_without_touching_a_gpu(case, code, msg):
    kw = {"C_513": dict(C=513), "Q0": dict(Q=0), "no_state": dict(state=None), "no_pairs": dict(pairs=None),
          "no_scales": dict(scales=None), "no_features": dict(feat=None), "cf2": dict(cf=2)}[case]
    rc = _bwd(**kw)
    assert rc == code and msg in _binding.last_error(), (rc, _binding.last_error())


def test_without_features_the_feature_pointers_may_be_null():
    # C = 0 passes the feature checks; Q = 0 then fails, so nothing is enqueued
    rc = _fwd(Q=0, C=0, feat=None, out=None)
    assert rc == -1 and "Q and P" in _binding.last_error()


def _cloud(P=6, C=None):
    a = dict(pts_xyz=torch.zeros(P, 3), rotations=torch.zeros(P, 4), scales=torch.zeros(P, 3), opacity=torch.zeros(P, 1))
    if C is not None:
        a["features"] = torch.zeros(P, C)
    return a


@pytest.mark.parametrize("case,match", [
    ("rotations_shape", "rotations: expected"), ("opacity_shape", "opacity: expected"), ("scales_dtype", "scales: expected float32"),
    ("features_rows", "features: expected"), ("features_width", "at most 512"), ("features_dtype", "features: expected float32"),
    ("points_shape", "points: expected"), ("points_dtype", "points: expected float32"), ("device", "CUDA tensor"),
])
def test_query_field_rejects_mismatches(case, match):
    a = _cloud(C=3)
    pts = torch.zeros(5, 3)
    if case == "rotations_shape":
        a["rotations"] = torch.zeros(6, 3)
    elif case == "opacity_shape":
        a["opacity"] = torch.zeros(5, 1)
    elif case == "scales_dtype":
        a["scales"] = a["scales"].double()
    elif case == "features_rows":
        a["features"] = torch.zeros(5, 3)
    elif case == "features_width":
        a["features"] = torch.zeros(6, 513)
    elif case == "features_dtype":
        a["features"] = a["features"].half()
    elif case == "points_shape":
        pts = torch.zeros(5, 2)
    elif case == "points_dtype":
        pts = pts.double()
    with pytest.raises(ValueError, match=match):
        GR.query_field(pts, a["pts_xyz"], a["rotations"], a["scales"], a["opacity"], a["features"])


@pytest.mark.parametrize("bounds,res,match", [
    ((0, 0, 0, 1, 1), 4, "bounds"), ((0, 0, 0, 1, 0, 1), 4, "bounds"), ((0, 0, 0, 1, 1, 1), 0, "resolution"),
    ((0, 0, 0, 1, 1, 1), (4, 4), "resolution"),
])
def test_voxelize_rejects_bad_grids(bounds, res, match):
    a = _cloud()
    with pytest.raises(ValueError, match=match):
        GR.voxelize(bounds, res, a["pts_xyz"], a["rotations"], a["scales"], a["opacity"])


def test_voxelize_rejects_a_bad_cloud():
    a = _cloud()
    with pytest.raises(ValueError, match="voxelize: scales"):
        GR.voxelize((0, 0, 0, 1, 1, 1), 4, a["pts_xyz"], a["rotations"], torch.zeros(6, 2), a["opacity"])


def test_voxel_centres_are_lo_plus_half_cells_in_x_major_order():
    pts, n = GR.voxel_centres((-0.3, -0.5, 0.6, 0.7, 0.5, 1.6), (4, 5, 2), "cpu")
    assert n == [4, 5, 2] and pts.shape == (40, 3)
    g = pts.view(4, 5, 2, 3)
    for (i, j, k) in ((0, 0, 0), (3, 4, 1), (1, 2, 0)):
        want = [-0.3 + (i + 0.5) * 1.0 / 4, -0.5 + (j + 0.5) * 1.0 / 5, 0.6 + (k + 0.5) * 1.0 / 2]
        assert np.allclose(g[i, j, k].numpy(), want, atol=1e-6)


def test_reference_isotropic_gaussian_has_its_analytic_value():
    s, o = 0.05, 0.8
    q = torch.tensor([[0.3, -0.2, 0.9, 0.1]], dtype=torch.float64)  # any rotation of an isotropic Gaussian
    mu = torch.tensor([[0.1, 0.2, 0.3]], dtype=torch.float64)
    r = torch.tensor([0.0, 0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 4.0], dtype=torch.float64) * s
    x = mu + r[:, None] * torch.tensor([0.6, 0.0, 0.8], dtype=torch.float64)
    f = torch.tensor([[2.0, -1.0]], dtype=torch.float64)
    d, feat = F64.field(x, mu, torch.full((1, 3), s, dtype=torch.float64), q, torch.tensor([o], dtype=torch.float64), f)
    want = o * torch.exp(-0.5 * (r / s) ** 2)
    want = torch.where(want >= F64.THRESH, want, torch.zeros_like(want))
    assert torch.allclose(d, want, rtol=1e-12, atol=0) and want[-1] == 0 and want[-2] > 0
    assert torch.allclose(feat, want[:, None] * f, rtol=1e-12, atol=0)


def test_reference_support_lies_in_the_computed_box():
    rng = np.random.default_rng(5)
    P = 64
    q = torch.tensor(rng.normal(size=(P, 4)))
    s = torch.tensor(np.exp(rng.normal(np.log(0.03), 0.8, (P, 3))))
    s[::7, 2] = 1e-4  # flat Gaussians
    o = torch.tensor(rng.uniform(0.01, 1.0, P))
    mu = torch.zeros(P, 3, dtype=torch.float64)
    box = F64.support_box(mu, s, q, o)
    hits = 0
    for i in range(P):
        # samples of the ellipsoid's surface and interior, mapped from the unit ball through x = R^T S u sqrt(cut)
        u = torch.tensor(rng.normal(size=(4000, 3)))
        u = u / u.norm(dim=1, keepdim=True) * torch.tensor(rng.uniform(0, 1, (4000, 1))) ** (1 / 3)
        u[:500] /= u[:500].norm(dim=1, keepdim=True)
        cut = -2.0 * math.log(F64.THRESH / float(o[i]))
        x = (u * s[i] * math.sqrt(cut)) @ F64.rotation_rows(q[i:i + 1])[0]
        g, _ = F64.field(x, mu[i:i + 1], s[i:i + 1], q[i:i + 1], o[i:i + 1])
        inside = g > 0
        hits += int(inside.sum())
        assert (x[inside].abs() <= box[i] * (1 + 1e-9)).all(), i
        # the box is tight: the support reaches every face
        assert torch.allclose(x[:500].abs().max(0).values, box[i], rtol=0.05), i
    assert hits > 0


def test_reference_drops_gaussians_without_support():
    mu = torch.zeros(4, 3, dtype=torch.float64)
    s = torch.full((4, 3), 0.1, dtype=torch.float64)
    s[1, 0] = 0.0
    q = torch.tensor([[1.0, 0, 0, 0]] * 4, dtype=torch.float64)
    q[2] = float("nan")
    o = torch.tensor([0.5, 0.5, 0.5, 1.0 / 255.0], dtype=torch.float64)
    assert F64.valid(mu, s, q, o).tolist() == [True, False, False, False]
    d, _ = F64.field(torch.zeros(1, 3, dtype=torch.float64), mu, s, q, o)
    assert float(d) == 0.5
