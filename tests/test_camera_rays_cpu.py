"""Camera rays without a GPU: the float64 statement (tests/rays_ref64.py), the C ABI's exports and argument checks, and
camera_rays' input checks.

* The reference's rays project back through the forward maps to their pixel at every depth (1e-9 px), for all four camera
  models, and gradcheck passes in the pixels, viewmatrix, projmatrix and tan_fov.
* The validity rules at theta_max, at r_max and across a fold where det Dd <= 0.
* Every argument error of mgs_camera_rays and its backward returns its code and sets mgs_last_error before anything is
  enqueued (the pointers are never dereferenced, so no device is touched); Q = 0 enqueues nothing.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import rays_ref64 as R
import util
from manigaussian_b200 import _binding

D64 = torch.float64
MODELS = ("pinhole", "ortho", "fisheye", "distorted")


def _view(model):
    from test_planar_depth_gpu import _model_kw
    inp = util.make_inputs(P=8, W=48, H=40, F=0, seed=0)
    return _model_kw(inp, model)[1]


def _pixels(view, n=64, seed=0):
    rng = np.random.default_rng(seed)
    px = np.stack([rng.uniform(-0.5, view["W"] - 0.5, n), rng.uniform(-0.5, view["H"] - 0.5, n)], -1)
    return torch.tensor(px, dtype=D64)


@pytest.mark.parametrize("model", MODELS)
def test_reference_rays_project_back_to_their_pixels(model):
    view = _view(model)
    pix = _pixels(view)
    o, d, ok = R.rays(pix, view)
    assert bool(ok.all())
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).T
    # direction's view-space z component is 1
    assert np.abs(d.numpy() @ vm[2, :3] - 1).max() < 1e-12
    for z in (0.5, 2.0, 7.5):
        uv, depth = R.round_trip(o, d, z, view)
        assert (uv - pix).abs().max() < 1e-9, (uv - pix).abs().max()
        assert (depth - z).abs().max() < 1e-12


@pytest.mark.parametrize("model", MODELS)
def test_reference_gradients_pass_gradcheck(model):
    view = _view(model)
    pix = _pixels(view, n=5, seed=1).requires_grad_(True)
    vm = torch.tensor(np.asarray(view["viewmatrix"], np.float64), requires_grad=True)
    pm = torch.tensor(np.asarray(view["projmatrix"], np.float64), requires_grad=True)
    tf = torch.tensor([view["tanfovx"], view["tanfovy"]], dtype=D64, requires_grad=True)
    wo, wd = (torch.tensor(np.random.default_rng(3).standard_normal((5, 3))) for _ in range(2))

    def f(p, vm_, pm_, tf_):
        o, d, ok = R.rays(p, dict(view, viewmatrix=vm_, projmatrix=pm_, tanfovx=tf_[0], tanfovy=tf_[1]))
        assert bool(ok.all())
        return (wo * o).sum() + (wd * d).sum()

    assert torch.autograd.gradcheck(f, (pix, vm, pm, tf), eps=1e-6, atol=1e-6, rtol=1e-5)


def test_fisheye_validity_at_theta_max():
    view = _view("fisheye")
    fe = view["fisheye"]
    k, tmax = [float(x) for x in fe[2:6]], float(fe[6])
    fx, fy = (float(x) for x in R._focal(view))
    td_max = tmax * R._rho(tmax, k)
    # along +x from the principal point: theta_d just inside and just outside the limit
    u = float(fe[0]) + fx * td_max * np.array([0.999, 1.001])
    pix = torch.tensor(np.stack([u, np.full(2, float(fe[1]))], -1), dtype=D64)
    o, d, ok = R.rays(pix, view)
    assert ok.tolist() == [True, False]
    assert torch.isnan(d[1]).all() and torch.isnan(o[1]).all()
    # the valid ray's points keep theta <= theta_max: the forward cull passes
    p = o[:1] + 2.0 * d[:1]
    assert bool(R.F64.valid(p, view).all())


def test_fisheye_axis_pixel_is_the_optical_axis():
    view = _view("fisheye")
    fe = view["fisheye"]
    o, d, ok = R.rays(torch.tensor([[float(fe[0]), float(fe[1])]], dtype=D64), view)
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).T
    assert bool(ok.all()) and np.allclose(d.numpy()[0], vm[2, :3], atol=1e-12)


def test_distorted_validity_at_r_max_and_across_a_fold():
    view = _view("distorted")
    fx, _ = (float(x) for x in R._focal(view))
    cx, cy = view["distortion"][:2]
    # r_max: a pixel whose undistorted radius is just inside / outside 0.3
    dc = list(view["distortion"][:10]) + [0.3]
    v2 = dict(view, distortion=tuple(dc))
    k1, k2 = dc[2], dc[3]
    xd = lambda r: r * (1 + k1 * r * r + k2 * r ** 4)  # noqa: E731  (on the x axis the tangential terms add p2 (3 r^2))
    p2 = dc[5]
    u = [cx + fx * (xd(r) + 3 * p2 * r * r) for r in (0.299, 0.301)]
    o, d, ok = R.rays(torch.tensor([[u[0], cy], [u[1], cy]], dtype=D64), v2)
    assert ok.tolist() == [True, False]
    # a fold: strong barrel distortion (k1 = -1) turns back at r^2 = 1/3, and det Dd <= 0 from there to r = 1 (beyond r = 1
    # the far branch, culled here by r_max = 1, folds back into the image with det Dd > 0).  A pixel just past the turning
    # point's image is reached only across the fold, so it has no valid ray; one just inside it does.
    dc = (cx, cy, -1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)
    v3 = dict(view, distortion=dc)
    r_turn = np.sqrt(1 / 3)
    xd_turn = r_turn * (1 - r_turn ** 2)
    pix = torch.tensor([[cx + fx * 0.95 * xd_turn, cy], [cx + fx * 1.05 * xd_turn, cy]], dtype=D64)
    o, d, ok = R.rays(pix, v3)
    assert ok.tolist() == [True, False]
    r2, det = R.F64.distortion_r2_det((d[:1] @ torch.tensor(np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).T[:3, :3]).T), dc)
    assert float(det[0]) > 0


def test_camera_ray_symbols_are_declared_and_exported():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    L = _binding.lib()
    for sym in ("mgs_camera_rays", "mgs_camera_rays_backward", "mgs_camera_rays_scratch_bytes"):
        assert f"{sym}(" in hdr and sym in _binding.EXPORTED_SYMBOLS and hasattr(L, sym)
    # one row of 27 camera and 2 focal-length terms per 128 rays
    assert L.mgs_camera_rays_scratch_bytes(128) == 29 * 4 and L.mgs_camera_rays_scratch_bytes(129) == 2 * 29 * 4
    assert L.mgs_camera_rays_scratch_bytes(0) == 0


def _views(V=1, W=8, H=6):
    views = (_binding.View * V)()
    for v in views:
        v.width, v.height, v.tan_fovx, v.tan_fovy = W, H, 0.5, 0.5
        v.viewmatrix, v.projmatrix = 4096, 4096
    return views


def _fwd(V=1, views=None, ortho=None, fisheye=None, Q=3, pixels=4096, out=4096):
    L = _binding.lib()
    views = _views(max(V, 1)) if views is None else views
    return L.mgs_camera_rays(V, views, None, ortho, fisheye, None, Q, pixels, out, out, out, 0, None)


def _bwd(views=None, Q=3, pixels=4096, dpix=None, cam=None, intr=None):
    L = _binding.lib()
    views = _views() if views is None else views
    return L.mgs_camera_rays_backward(1, views, intr, None, None, None, Q, pixels, 4096, 4096, dpix, cam, 0, None)


@pytest.mark.parametrize("case,msg", [
    ("V0", "at least one view"),
    ("Q_neg", "Q must be"),
    ("no_matrix", "matrices"),
    ("size", "bad size"),
    ("grid_size", "Q must equal width * height"),
    ("grid_mixed", "Q must equal width * height"),
    ("no_output", "out_origin"),
    ("ortho", "ortho"),
    ("fisheye", "theta_max"),
])
def test_forward_argument_errors_return_before_anything_is_enqueued(case, msg):
    views, kw = _views(), {}
    if case == "V0":
        kw["V"] = 0
    elif case == "Q_neg":
        kw["Q"] = -1
    elif case == "no_matrix":
        views[0].projmatrix = None
    elif case == "size":
        views[0].height = 0
    elif case == "grid_size":
        kw.update(pixels=None, Q=47)
    elif case == "grid_mixed":
        views = _views(2)
        views[1].width = 9
        kw.update(V=2, pixels=None, Q=48)
    elif case == "no_output":
        kw["out"] = None
    elif case == "ortho":
        kw["ortho"] = (ctypes.c_int * 1)(2)
    elif case == "fisheye":
        fe = (_binding.ViewFisheye * 1)()
        fe[0].fisheye, fe[0].theta_max = 1, 2.0
        kw["fisheye"] = fe
    rc = _fwd(views=views, **kw)
    assert rc == -1 and msg in _binding.last_error(), (rc, _binding.last_error())


@pytest.mark.parametrize("case,msg", [
    ("dpix_grid", "dL_dpixels needs pixels"),
    ("no_scratch", "needs scratch"),
    ("tan_fov_no_scratch", "needs scratch"),
    ("grid_size", "Q must equal width * height"),
])
def test_backward_argument_errors_return_before_anything_is_enqueued(case, msg):
    kw = {}
    if case == "dpix_grid":
        kw.update(pixels=None, Q=48, dpix=4096)
    elif case == "no_scratch":
        cam = (_binding.ViewCameraGrad * 1)()
        cam[0].dL_dviewmatrix = 4096
        kw["cam"] = cam
    elif case == "tan_fov_no_scratch":
        intr = (_binding.ViewIntrinsics * 1)()
        intr[0].tan_fov, intr[0].dL_dtan_fov = 4096, 4096
        kw["intr"] = intr
    elif case == "grid_size":
        kw.update(pixels=None, Q=5)
    rc = _bwd(**kw)
    assert rc == -1 and msg in _binding.last_error(), (rc, _binding.last_error())


def test_zero_rays_is_a_no_op():
    assert _fwd(Q=0, pixels=None, out=None) == 0
    assert _bwd(Q=0, pixels=None) == 0
    assert _bwd(Q=0, dpix=4096) == 0


def _settings(V=2, W=8, H=6, device="cpu"):
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    return [GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4, device=device), torch.eye(4, device=device), 0,
                                          torch.zeros(3), False, False, False) for _ in range(V)]


@pytest.mark.parametrize("case,match", [
    ("no_views", "at least one view"),
    ("device", "CUDA viewmatrix"),
])
def test_camera_rays_rejects_mismatches(case, match):
    from manigaussian_b200 import gaussian_renderer as GR
    views = [] if case == "no_views" else _settings()
    with pytest.raises(ValueError, match=match):
        GR.camera_rays(views)
