"""The flow plane without a GPU: the float64 reference (tests/flow_ref64.py) against finite differences and geometry, and the
argument checks of the C ABI (include/mgs_rasterizer.h, flow plane) and of the Python entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

import flow_ref64 as F64

D64 = torch.float64


def _view(model="pinhole", W=64, H=48):
    vm = np.eye(4)
    vm[3, :3] = [0.1, -0.2, 0.0]  # column-major storage: translation in the last row
    tx, ty = 0.6, 0.45
    znear, zfar = 0.1, 100.0
    P = np.zeros((4, 4))
    P[0, 0], P[1, 1] = 1 / tx, 1 / ty
    P[2, 2], P[2, 3], P[3, 2] = zfar / (zfar - znear), -zfar * znear / (zfar - znear), 1.0
    view = dict(viewmatrix=vm.reshape(-1), projmatrix=(vm @ P.T).reshape(-1), W=W, H=H, tanfovx=tx, tanfovy=ty)
    cx, cy = (W - 1) / 2, (H - 1) / 2
    if model == "ortho":
        Po = np.diag([1 / 2.0, 1 / 1.5, 1 / (zfar - znear), 1.0])
        view.update(ortho=True, tanfovx=2.0, tanfovy=1.5, projmatrix=(vm @ Po.T).reshape(-1))
    elif model == "fisheye":
        view.update(fisheye=(cx, cy, 0.03, -0.01, 0.002, -0.001, 1.4))
    elif model == "distorted":
        view.update(distortion=(cx, cy, -0.05, 0.01, 0.001, -0.002, 0.0, 0.0, 0.0, 0.0, float("inf")))
    return view


def _cloud(P=6, seed=0):
    g = torch.Generator().manual_seed(seed)
    mu = torch.rand((P, 3), generator=g, dtype=D64) * torch.tensor([1.0, 0.8, 1.0], dtype=D64) - \
        torch.tensor([0.5, 0.4, -2.0], dtype=D64)
    nxt = mu + 0.05 * torch.randn((P, 3), generator=g, dtype=D64)
    return mu, nxt


@pytest.mark.parametrize("model", ["pinhole", "ortho", "fisheye", "distorted"])
def test_reference_against_finite_differences(model):
    view = _view(model)
    mu, nxt = _cloud()
    vm = torch.tensor(view["viewmatrix"], dtype=D64, requires_grad=True)
    pm = torch.tensor(view["projmatrix"], dtype=D64, requires_grad=True)
    tf = torch.tensor([view["tanfovx"], view["tanfovy"]], dtype=D64, requires_grad=True)
    mu.requires_grad_(True)
    nxt.requires_grad_(True)

    def f(mu, nxt, vm, pm, tf):
        v = dict(view, viewmatrix=vm, projmatrix=pm, tanfovx=tf[0], tanfovy=tf[1])
        d, ok = F64.delta(mu, nxt, v)
        assert bool(ok.all())
        return d

    assert torch.autograd.gradcheck(f, (mu, nxt, vm, pm, tf), eps=1e-6, atol=1e-5, rtol=1e-4)


def test_ortho_translation_parallel_to_the_image_plane():
    view = _view("ortho")
    mu, _ = _cloud()
    dt = torch.tensor([0.03, -0.02, 0.0], dtype=D64)
    d, ok = F64.delta(mu, mu + dt, view)
    fx, fy = view["W"] / (2 * view["tanfovx"]), view["H"] / (2 * view["tanfovy"])
    assert bool(ok.all())
    assert torch.allclose(d, torch.tensor([fx * 0.03, fy * -0.02], dtype=D64).expand_as(d), atol=1e-9)


def test_pinhole_motion_along_the_camera_ray_has_no_flow():
    view = _view("pinhole")
    mu, _ = _cloud()
    vm = torch.tensor(view["viewmatrix"], dtype=D64).reshape(4, 4).T
    centre = -vm[:3, :3].T @ vm[:3, 3]  # the camera centre in world space
    d, ok = F64.delta(mu, centre + 1.7 * (mu - centre), view)
    assert bool(ok.all())
    # zero up to the projection's own 1e-7 in 1 / (w + 1e-7): it moves m by |ndc| 1e-7 / w (W / 2) < 1e-5 px here
    assert float(d.abs().max()) < 1e-5


def test_next_mean_behind_the_near_plane_is_zero_with_zero_gradient():
    view = _view("pinhole")
    mu, nxt = _cloud(P=3)
    nxt = nxt.clone()
    nxt[1, 2] = 0.05  # view-space z = 0.05 < NEAR_Z
    mu.requires_grad_(True)
    nxt.requires_grad_(True)
    d, ok = F64.delta(mu, nxt, view)
    assert ok.tolist() == [True, False, True]
    assert float(d[1].abs().max()) == 0.0
    d.sum().backward()
    assert float(nxt.grad[1].abs().max()) == 0.0 and float(mu.grad[1].abs().max()) == 0.0


def test_same_mean_gives_exactly_zero():
    for model in ("pinhole", "ortho", "fisheye", "distorted"):
        mu, _ = _cloud()
        d, _ = F64.delta(mu, mu.clone(), _view(model))
        assert float(d.abs().max()) == 0.0


def test_flow_option_argument_checks():
    from manigaussian_b200 import _binding as B
    L = B.lib()
    views = (B.View * 1)()
    buf = (C.c_float * 16)()
    means = C.addressof(buf)

    def flow(out=True, dpix=False, vm=False):
        fl = (B.ViewFlow * 1)()
        fl[0].out_flow = C.addressof(buf) if out else None
        fl[0].dL_dpix_flow = C.addressof(buf) if dpix else None
        fl[0].next_viewmatrix = C.addressof(buf) if vm else None
        return fl

    normal = (B.ViewNormal * 1)()
    normal[0].out_normal = C.addressof(buf)
    dm = (B.ViewDepthMask * 1)()
    dm[0].target_depth = C.addressof(buf)
    rest = (1, 0, 0, 0) + (None,) * 4 + (None, None, 1.0, None, None, 0, 0, None)
    cases = [  # (normal, depth / mask, planar_depth, flow, next means, what the error names)
        (normal, None, 0, flow(), means, b"normal plane"),
        (None, None, 1, flow(), means, b"planar_depth"),
        (None, dm, 0, flow(), means, b"depth / mask"),
        (None, None, 0, flow(), None, b"next-frame means"),
        (None, None, 0, flow(out=False, dpix=True), means, b"out_flow"),
        (None, None, 0, flow(vm=True), means, b"next_projmatrix"),
    ]
    for nrm, d, pln, fl, nxt, what in cases:
        opts = B.RenderOptions(depth_mask=d, normal=nrm, planar_depth=pln, flow=fl, flow_next=(B.CloudFlow * 1)((nxt, None)))
        rc = L.mgs_forward_views(1, views, opts, *rest)
        assert rc == -1, what
        assert what in L.mgs_last_error(), (what, L.mgs_last_error())


def test_python_argument_errors():
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200 import gaussian_renderer as G
    with pytest.raises(ValueError):
        R._check_flow(torch.zeros(4, 3), True, False, None)
    with pytest.raises(ValueError):
        R._check_flow(torch.zeros(4, 3), False, True, None)
    with pytest.raises(ValueError):
        R._check_flow(torch.zeros(4, 3), False, False, (None,) * 6)
    R._check_flow(None, True, True, None)
    with pytest.raises(ValueError):
        R._flow_array([None], torch.zeros(4, 2), None, 4, torch.device("cpu"), [])
    with pytest.raises(ValueError):
        R._flow_array([None], torch.zeros(4, 3, dtype=torch.float64), None, 4, torch.device("cpu"), [])
    s = R.GaussianRasterizationSettings(4, 4, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False,
                                        False, False)
    pts = torch.zeros(4, 3)
    assert G._flow_inputs([s], pts, torch.zeros(4, 3), None, None, None, 0, False) is None
    with pytest.raises(ValueError):  # wrong shape
        G._flow_inputs([s], pts, torch.zeros(5, 3), None, None, None, 0, False)
    with pytest.raises(ValueError):  # other intrinsics
        G._flow_inputs([s], pts, torch.zeros(4, 3), [s._replace(tanfovx=0.6)], None, None, 0, False)
    with pytest.raises(ValueError):  # other image size
        G._flow_inputs([s], pts, torch.zeros(4, 3), [s._replace(image_width=8)], None, None, 0, False)
    with pytest.raises(ValueError):  # other model
        G._flow_inputs([s], pts, torch.zeros(4, 3), [s._replace(orthographic=True)], None, None, 0, False)
    with pytest.raises(ValueError):  # a pose that requires grad
        G._flow_inputs([s], pts, torch.zeros(4, 3), [s._replace(viewmatrix=torch.eye(4, requires_grad=True))], None, None, 0, False)
    poses = G._flow_inputs([s], pts, torch.zeros(4, 3), [s._replace(viewmatrix=2 * torch.eye(4))], None, None, 0, False)
    assert torch.equal(poses[0][0], 2 * torch.eye(4))
    for kw in (dict(return_normal=True), dict(planar_depth=True), dict(sync_gradients=True),
               dict(targets={"rgb": torch.zeros(1, 3, 4, 4)})):
        with pytest.raises(ValueError):
            G.render_views([s], pts, torch.zeros(4, 4), torch.ones(4, 3), torch.ones(4, 1), pts_rgb=torch.zeros(4, 3),
                           flow_xyz=torch.zeros(4, 3), **kw)
