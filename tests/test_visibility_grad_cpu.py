"""The point-visibility backward without a GPU: the float64 statement (tests/visibility_grad_ref64.py), the C ABI's exports and
argument checks, and point_visibility(differentiable=True)'s input checks.

* gradcheck of the reference's uv, depth and T with the decisions frozen, in the points, the cloud, the view and projection
  matrices and tan_fov, for all four camera models, with and without the anti-aliased opacity.
* Every new argument error of mgs_visibility_views_backward returns its code and sets mgs_last_error before anything is
  enqueued (the pointers are never dereferenced, so no device is touched); Q = 0 enqueues nothing.
"""
import os

import numpy as np
import pytest
import torch

import util
import visibility_grad_ref64 as VG
from manigaussian_b200 import _binding
from test_visibility_cpu import _cloud, _settings, _views

D64 = torch.float64


def _scene(model, seed=0):
    from test_planar_depth_gpu import _model_kw
    inp = util.make_inputs(P=64, W=48, H=40, F=0, seed=seed)
    view = _model_kw(inp, model)[1]
    g = inp["g"]
    rng = np.random.default_rng(seed)
    # six Gaussians well inside the pinhole clamp |t.xy / t.z| <= 1.3 tan_fov, where the backward's J is J's derivative
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).T
    t = np.asarray(g["means3D"], np.float64) @ vm[:3, :3].T + vm[:3, 3]
    inside = (np.abs(t[:, 0] / t[:, 2]) < 1.1 * view["tanfovx"]) & (np.abs(t[:, 1] / t[:, 2]) < 1.1 * view["tanfovy"]) & (t[:, 2] > 0.5)
    sel = np.nonzero(inside)[0][:6]
    assert len(sel) == 6
    means = np.asarray(g["means3D"], np.float64)[sel]
    pts = means[[0, 2, 4]] + 0.05 * rng.standard_normal((3, 3))
    # each point accepts a few Gaussians in a fixed order; small opacities keep every alpha below the 0.99 clamp
    accepted = [np.array([1, 3]), np.array([0, 5, 2]), np.array([4])]
    # scales 10 x the scene's so that every accepted footprint reaches its point
    return view, means, 10.0 * np.asarray(g["scales"], np.float64)[sel], np.asarray(g["rotations"], np.float64)[sel], pts, accepted


@pytest.mark.parametrize("model,aa", [("pinhole", False), ("ortho", False), ("fisheye", False), ("distorted", False),
                                      ("pinhole", True), ("fisheye", True)])
def test_reference_gradients_pass_gradcheck(model, aa):
    view, means, scales, rots, pts, acc = _scene(model)
    opac = np.full((6, 1), 0.3)
    leaves = [torch.tensor(x, dtype=D64, requires_grad=True) for x in (pts, means, scales, rots, opac)]
    vm = torch.tensor(np.asarray(view["viewmatrix"], np.float64), requires_grad=True)
    pm = torch.tensor(np.asarray(view["projmatrix"], np.float64), requires_grad=True)
    tf = torch.tensor([view["tanfovx"], view["tanfovy"]], dtype=D64, requires_grad=True)
    wT, wuv, wd = (torch.tensor(np.random.default_rng(3).standard_normal(s)) for s in ((3,), (3, 2), (3,)))

    def f(p, m, s, r, o, vm_, pm_, tf_):
        v = dict(view, viewmatrix=vm_, projmatrix=pm_, tanfovx=tf_[0], tanfovy=tf_[1])
        uv, d, T = VG.outputs(p, m, o, v, acc, scales=s, rotations=r, antialias=aa)
        assert (T < 0.9).all() and (T > 0.01).all()
        return (wT * T).sum() + (wuv * uv).sum() + (wd * d).sum()

    assert torch.autograd.gradcheck(f, leaves + [vm, pm, tf], eps=1e-6, atol=1e-5, rtol=1e-4)


def test_reference_T_is_the_product_over_the_accepted_candidates():
    view, means, scales, rots, pts, acc = _scene("pinhole")
    t = lambda x: torch.tensor(x, dtype=D64)  # noqa: E731
    uv, d, T = VG.outputs(t(pts), t(means), t(np.full(6, 0.3)), view, acc, scales=t(scales), rotations=t(rots))
    S = VG.P64.covariance(t(scales), t(rots))
    mu, conic, _ = VG._screen_conic(t(means), S, view, False)
    for q, ids in enumerate(acc):
        want = 1.0
        for i in ids:
            dx, dy = (mu[i] - uv[q]).tolist()
            A, B, C = conic[i].tolist()
            want *= 1.0 - 0.3 * np.exp(-0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy)
        assert abs(float(T[q]) - want) <= 1e-12
    assert torch.allclose(d, VG.F64.view_space(t(pts), view)[:, 2])


def test_visibility_backward_symbols_are_declared_and_exported():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    L = _binding.lib()
    for sym in ("mgs_visibility_views_backward", "mgs_visibility_backward_scratch_bytes"):
        assert f"{sym}(" in hdr and sym in _binding.EXPORTED_SYMBOLS and hasattr(L, sym)
    # gb, the uv cotangents and the camera rows of both paths grow with P and Q
    a, b, c = (L.mgs_visibility_backward_scratch_bytes(P, Q) for P, Q in ((1000, 1000), (2000, 1000), (1000, 2000)))
    assert b - a >= 1000 * 12 * 4 and c - a >= 1000 * 2 * 4


def _bcall(V=1, views=None, P=4, Q=3, out_T=4096, dT=4096, dcov=None, cov=None):
    L = _binding.lib()
    views = _views(max(V, 1)) if views is None else views
    for v in views:
        v.dL_dmean2D = v.dL_dmean2D or 4096
    return L.mgs_visibility_views_backward(V, views, 0, None, None, None, None, P, 0, 0, Q, 4096, 4096, None, 4096, 4096, 4096, 1.0,
                                           4096, cov, out_T, dT, None, None, 4096, 4096, 4096, None, None, dcov, None, 0, None)


@pytest.mark.parametrize("case,msg", [
    ("V0", "at least one view"),
    ("no_T", "out_T"),
    ("no_backward_scratch", "backward scratch"),
    ("cov3D_grad", "dL_dcov3D needs cov3D_precomp"),
    ("no_scratch", "blend_scratch"),
])
def test_invalid_arguments_return_error_codes_without_touching_a_gpu(case, msg):
    views = _views()
    kw = {}
    if case == "V0":
        kw["V"] = 0
    elif case == "no_T":
        kw["out_T"] = None
    elif case == "no_backward_scratch":
        views[0].dL_dmean2D = None
        L = _binding.lib()
        rc = L.mgs_visibility_views_backward(1, views, 0, None, None, None, None, 4, 0, 0, 3, 4096, 4096, None, 4096, 4096, 4096,
                                             1.0, 4096, None, 4096, 4096, None, None, 4096, None, None, None, None, None, None, 0,
                                             None)
        assert rc == -1 and msg in _binding.last_error(), (rc, _binding.last_error())
        return
    elif case == "cov3D_grad":
        kw["dcov"] = 4096
    elif case == "no_scratch":
        views[0].blend_scratch = None
    rc = _bcall(views=views, **kw)
    assert rc == -1 and msg in _binding.last_error(), (rc, _binding.last_error())


def test_zero_points_is_a_no_op():
    assert _bcall(Q=0) == 0
    # without dL_dT, out_T is not needed
    assert _bcall(Q=0, out_T=None, dT=None) == 0


@pytest.mark.parametrize("flag", ["yes", 1, torch.tensor(True), None])
def test_differentiable_must_be_a_bool(flag):
    from manigaussian_b200 import gaussian_renderer as GR
    a = _cloud()
    with pytest.raises(ValueError, match="differentiable: expected True or False"):
        GR.point_visibility(_settings(), torch.zeros(5, 3), a["pts_xyz"], a["rotations"], a["scales"], a["opacity"],
                            differentiable=flag)


@pytest.mark.parametrize("case,match", [
    ("rotations_shape", "rotations: expected"),
    ("points_dtype", "points: expected float32"),
    ("device", "CUDA tensor"),
])
def test_differentiable_point_visibility_rejects_mismatches(case, match):
    """the differentiable path runs the same input checks before it builds its node"""
    from manigaussian_b200 import gaussian_renderer as GR
    a = _cloud()
    pts = torch.zeros(5, 3, requires_grad=True)
    if case == "rotations_shape":
        a["rotations"] = torch.zeros(6, 3)
    elif case == "points_dtype":
        pts = torch.zeros(5, 3, dtype=D64, requires_grad=True)
    with pytest.raises(ValueError, match=match):
        GR.point_visibility(_settings(), pts, a["pts_xyz"], a["rotations"], a["scales"], a["opacity"], differentiable=True)
