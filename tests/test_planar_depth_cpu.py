"""Planar depth without a GPU: the float64 reference (tests/planar_ref64.py) against finite differences and geometry, and the
C ABI's argument checks (include/mgs_rasterizer.h, mgs_render_options.planar_depth)."""
import ctypes as C

import numpy as np
import pytest
import torch

import planar_ref64 as R64

D64 = torch.float64


def _view(model="pinhole", W=64, H=48):
    vm = np.eye(4)
    vm[3, :3] = [0.1, -0.2, 0.0]  # column-major storage: translation in the last row
    tx, ty = 0.6, 0.45
    fx = W / (2 * tx)
    znear, zfar = 0.1, 100.0
    P = np.zeros((4, 4))
    P[0, 0], P[1, 1] = 1 / tx, 1 / ty
    P[2, 2], P[2, 3], P[3, 2] = zfar / (zfar - znear), -zfar * znear / (zfar - znear), 1.0
    full = vm @ P.T
    view = dict(viewmatrix=vm.reshape(-1), projmatrix=full.reshape(-1), W=W, H=H, tanfovx=tx, tanfovy=ty)
    cx, cy = (W - 1) / 2, (H - 1) / 2
    if model == "ortho":
        Po = np.diag([1 / 2.0, 1 / 1.5, 1 / (zfar - znear), 1.0])
        view.update(ortho=True, tanfovx=2.0, tanfovy=1.5, projmatrix=(vm @ Po.T).reshape(-1))
    elif model == "fisheye":
        view.update(fisheye=(cx, cy, 0.03, -0.01, 0.002, -0.001))
    elif model == "distorted":
        view.update(distortion=(cx, cy, -0.08, 0.02, 0.003, -0.002, 0.001, 0.01, 0.0, 0.0))
    return view, fx


def _cloud(P=12, seed=0):
    rng = np.random.default_rng(seed)
    m = np.c_[rng.uniform(-0.8, 0.8, (P, 2)), rng.uniform(2.0, 4.0, P)]
    s = rng.uniform(0.02, 0.3, (P, 3))
    q = rng.standard_normal((P, 4))
    return (torch.tensor(x, dtype=D64, requires_grad=True) for x in (m, s, q))


@pytest.mark.parametrize("model", ["pinhole", "ortho", "fisheye", "distorted"])
def test_reference_gradients_match_finite_differences(model):
    view, _ = _view(model)
    m, s, q = _cloud()
    w = torch.tensor(np.random.default_rng(3).standard_normal((12, 3)), dtype=D64)
    f = lambda m, s, q: (R64.quads(m, s, q, view)[0] * w).sum()  # noqa: E731
    assert torch.autograd.gradcheck(f, (m, s, q), eps=1e-6, atol=1e-6, rtol=1e-5)


@pytest.mark.parametrize("model", ["pinhole", "ortho", "fisheye", "distorted"])
def test_gaussian_facing_the_camera_on_the_axis_has_a_flat_depth(model):
    view, _ = _view(model)
    vm = np.asarray(view["viewmatrix"]).reshape(4, 4)
    off = 1e-7 if model == "fisheye" else 0.0  # the fisheye map's closed form is 0 / 0 on the axis itself
    m = torch.tensor([[off - vm[3, 0], -vm[3, 1], 3.0]], dtype=D64)  # view-space (0, 0, 3)
    s = torch.tensor([[0.2, 0.1, 0.01]], dtype=D64)
    q = torch.tensor([[0.9, 0.0, 0.0, 0.3]], dtype=D64)  # a rotation about the view axis only
    quad, _ = R64.quads(m, s, q, view)
    quad = quad.detach()
    assert float(quad[0, :2].abs().max()) < 1e-9
    assert abs(float(R64.planar_depth_at(3.0, quad[0], 10.0, 7.0)) - 3.0) < 1e-6


def test_thin_tilted_gaussian_follows_its_plane():
    """a very thin Gaussian in the plane z = 3 + 0.6 x (view space): near its centre the planar depth matches the ray-plane
    intersection to second order in the pixel offset; its centre depth is off by the slope"""
    view, fx = _view("pinhole", 200, 150)
    W, H = view["W"], view["H"]
    vm = np.asarray(view["viewmatrix"]).reshape(4, 4)
    slope = 0.6
    n = np.array([-slope, 0.0, 1.0]) / np.hypot(1, slope)
    u = np.array([1.0, 0.0, slope]) / np.hypot(1, slope)
    Rw = np.stack([u, [0.0, 1.0, 0.0], n], 1)
    qw = np.sqrt(1 + np.trace(Rw)) / 2
    q = torch.tensor([[qw, (Rw[2, 1] - Rw[1, 2]) / (4 * qw), (Rw[0, 2] - Rw[2, 0]) / (4 * qw), (Rw[1, 0] - Rw[0, 1]) / (4 * qw)]],
                     dtype=D64)
    t0 = np.array([0.0, 0.0, 3.0])
    m = torch.tensor([t0 - vm[3, :3]], dtype=D64)
    s = torch.tensor([[0.4, 0.4, 1e-5]], dtype=D64)
    quad, _ = R64.quads(m, s, q, view)
    mu = R64.screen_mean(m, view)[0].numpy()
    errs = {}
    for d in (4.0, 2.0):
        px, py = mu[0] + d, mu[1] + 0.5 * d
        rx, ry = (px - (W - 1) / 2) / fx, (py - (H - 1) / 2) / fx
        depth = t0[2] * n[2] / (n[0] * rx + n[1] * ry + n[2])  # the ray (rx, ry, 1) s meets the plane n . (t - t0) = 0
        planar = float(R64.planar_depth_at(t0[2], quad[0], px, py))
        errs[d] = abs(planar - depth)
        assert abs(t0[2] - depth) > 20 * errs[d]
    assert errs[2.0] < errs[4.0] / 3  # second order: halving the offset quarters the error (up to the dilation's share)


def test_planar_depth_option_argument_checks():
    from manigaussian_b200 import _binding as B
    from manigaussian_b200 import rasterizer as R
    L = B.lib()
    views = (B.View * 1)()
    normal = (B.ViewNormal * 1)()
    buf = (C.c_float * 4)()
    normal[0].out_normal = C.addressof(buf)
    rest = (1, 0, 0, 0) + (None,) * 4 + (None, None, 1.0, None, None, 0, 0, None)
    for flag, nrm in ((2, None), (1, normal)):
        rc = L.mgs_forward_views(1, views, B.RenderOptions(normal=nrm, planar_depth=flag), *rest)
        assert rc == B.MGS_ERR_INVALID_ARG if hasattr(B, "MGS_ERR_INVALID_ARG") else rc != 0
        assert b"planar_depth" in L.mgs_last_error()
    s = R.GaussianRasterizationSettings(4, 4, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False,
                                        False, False, planar_depth=True)
    assert s.planar_depth and "planar_depth=True" in repr(s) and s._replace(image_height=8).planar_depth
    assert not s._replace(planar_depth=False).planar_depth
    with pytest.raises(ValueError):
        R._planar_flag([s], None, True)
    with pytest.raises(ValueError):
        R._planar_flag([s, s._replace(planar_depth=False)])
