"""Distorted-pinhole views without a GPU: the float64 reference against OpenCV and torch autograd, the camera builders,
distortion_r_max and the C ABI's checks.

* tests/distorted_ref64.py's screen means and J match cv2.projectPoints (and its Jacobian's d/dtvec columns, which are
  d(u, v)/dt at a zero pose) to 1e-9 relative, when OpenCV is installed.
* The reference matches torch float64 autograd of an independent restatement to 1e-9 relative: the records (means2D, conic,
  o_eff, depth), dL/dmeans3D, dL/dcov3D (or the scales and rotations), dL/dsh, dL/dopacity, the 27 camera terms and
  dL/dtan_fov.  The restatement takes J from autograd of the mean map, with vm and tan_fov as leaves.
* With all coefficients 0 the records and per-Gaussian gradients are the pinhole reference's inside the clamp region.
* distortion_r_max: the fold of k1 < 0 alone, a zero of the rational denominator, monotone coefficients, 4- and 5-entry D.
* Each broken convention of distorted_ref64.MUTATIONS moves a checked element past twice its bound.
* Bad distortion parameters in the render options and the lift return MGS_ERR_INVALID_ARG before anything is enqueued.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import distorted_ref64 as D64
import project_ref64 as P64
import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding, cameras, scenes
from manigaussian_b200.rasterizer import GaussianRasterizationSettings

# an Azure-Kinect-like rational 8-coefficient calibration (strong distortion) and a RealSense-like 5-coefficient one
KINECT_D = (0.45, -0.08, 0.0006, -0.0004, -0.01, 0.78, 0.02, -0.06)
REALSENSE_D = (0.12, -0.25, 0.001, -0.0015, 0.1)


def _look(eye, target):
    fwd = np.asarray(target, np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    if np.linalg.norm(right) < 1e-6:
        right = np.array([1.0, 0.0, 0.0])
    right /= np.linalg.norm(right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, np.cross(fwd, right), fwd, eye
    return c2w


def dcam(W=40, H=32, D=KINECT_D, eye=(0.6, -0.4, 0.9), f=None, r_max=None):
    """a distorted camera looking at the scene centre from close by, so the cloud spans a wide field"""
    f = f if f is not None else W / 2.5
    return D64.distorted_cam(W, H, f, f * 1.02, (W - 1) / 2 + 0.3, (H - 1) / 2 - 0.2, D, _look(np.array(eye), scenes.SCENE_CENTER),
                             r_max)


def _scene(name, P=48, seed=0):
    deg = {"sh0": 0, "sh1": 1, "sh2": 2, "sh3": 3}.get(name, 1)
    g = scenes.make_gaussians(P, sh_degree=deg, seed=seed + deg)
    g["cov3D_precomp"] = None
    rng = np.random.default_rng(seed)
    g["rotations"] = (g["rotations"] * rng.uniform(0.3, 3.0, (P, 1))).astype(np.float32)
    g["scales"] = (g["scales"] * 4.0).astype(np.float32)
    if name == "precomp_cov":
        S = P64.cov3d(g)[0]
        g["cov3D_precomp"] = np.stack([S[0][0].v, S[0][1].v, S[0][2].v, S[1][1].v, S[1][2].v, S[2][2].v], 1).astype(np.float32)
        g["scales"] = g["rotations"] = None
    if g.get("shs") is not None:
        g["shs"][:, 0, :] -= 1.2
    D = REALSENSE_D if name == "rs5" else KINECT_D
    return g, dcam(D=D), name.startswith("aa")


def _mean_map_torch(t, cam, fx, fy):
    cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, _ = (float(np.float32(v)) for v in cam["distortion"])
    x, y = t[:, 0] / t[:, 2], t[:, 1] / t[:, 2]
    r2 = x * x + y * y
    R = (1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3) / (1 + k4 * r2 + k5 * r2 ** 2 + k6 * r2 ** 3)
    xd = x * R + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
    yd = y * R + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
    return torch.stack([fx * xd + cx, fy * yd + cy], 1)


def _torch_loss_distorted(g, cam, cot, mod, aa):
    """An independent torch restatement of one distorted view with every input a leaf, in the conventions of
    test_fisheye_cpu's restatement: the screen mean is OpenCV's map of t, J its autograd Jacobian w.r.t. t"""
    d = torch.float64
    T = lambda a: torch.tensor(np.asarray(a, np.float32).astype(np.float64), dtype=d)  # noqa: E731
    p = T(g["means3D"]).requires_grad_()
    leaves = dict(dL_dmeans3D=p)
    if g.get("scales") is not None:
        se = (T(g["scales"]) * float(np.float32(mod))).detach().requires_grad_()
        q = T(g["rotations"]).requires_grad_()
        leaves.update(dL_dscales=se, dL_drotations=q)
        r, x, y, z = q.unbind(1)
        Rq = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                          2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                          2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
        Sig = Rq @ torch.diag_embed(se * se) @ Rq.transpose(1, 2)
    else:
        c6 = T(g["cov3D_precomp"]).requires_grad_()
        leaves["dL_dcov3D"] = c6
        Sig = torch.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], 1)
    o = T(g["opacities"]).reshape(-1).requires_grad_()
    leaves["dL_dopacity"] = o
    vm16 = T(np.asarray(cam["viewmatrix"]).reshape(-1)).requires_grad_()
    pm16 = torch.zeros(16, dtype=d, requires_grad=True)   # not read: its gradient must be zero
    cp = T(np.asarray(cam["campos"]).reshape(-1)).requires_grad_()
    tan0 = np.array([np.float32(cam["tanfovx"]), np.float32(cam["tanfovy"])], np.float64)
    tan = torch.tensor(tan0, dtype=d, requires_grad=True)
    leaves.update(dL_dviewmatrix=vm16, dL_dprojmatrix=pm16, dL_dcampos=cp, dL_dtan_fov=tan)
    vw = P64.view_of(cam)
    fx, fy = vw["fx"] * (tan0[0] / tan[0]), vw["fy"] * (tan0[1] / tan[1])
    vm = vm16.reshape(4, 4).T
    t = p @ vm[:3, :3].T + vm[:3, 3]
    uv = _mean_map_torch(t, cam, fx, fy)
    J = torch.stack([torch.autograd.grad(uv[:, i].sum(), t, create_graph=True)[0] for i in range(2)], 1)   # [P,2,3]
    Mx = J @ vm[:3, :3]
    cov = Mx @ Sig @ Mx.transpose(1, 2)
    h = float(np.float32(0.3))
    a, b, c = cov[:, 0, 0] + h, cov[:, 0, 1], cov[:, 1, 1] + h
    det = a * c - b * b
    kk = (det * det / (det * det + float(np.float32(1e-7)))).detach()
    sc = lambda x: x.detach() + (x - x.detach()) * kk  # noqa: E731
    C_ = lambda k: torch.tensor(np.asarray(cot[k], np.float64), dtype=d)  # noqa: E731
    gco = C_("dL_dconic")
    conic = torch.stack([c / det, -b / det, a / det], 1)
    tz = t[:, 2]
    ndc = (2.0 * uv + 1.0) / torch.tensor([cam["W"], cam["H"]], dtype=d) - 1.0
    loss = (ndc * C_("dL_dmean2D")).sum() + (sc(c / det) * gco[:, 0] + 2 * sc(-b / det) * gco[:, 1] + sc(a / det) * gco[:, 2]).sum()
    oe = o
    if aa:
        rr = (cov[:, 0, 0] * cov[:, 1, 1] - b * b) / det
        oe = o * torch.sqrt(rr.clamp_min(P64.AA_CLAMP))
    loss = loss + (oe * C_("dL_dopacity")).sum() + (tz * C_("dL_ddepth")).sum()
    if g.get("shs") is not None:
        sh = T(g["shs"]).requires_grad_()
        leaves["dL_dsh"] = sh
        v = p - cp
        dr = v / v.norm(dim=1, keepdim=True)
        x, y, z = dr.unbind(1)
        xx, yy, zz = x * x, y * y, z * z
        basis = [torch.full_like(x, P64.SH_C0), -P64.SH_C1 * y, P64.SH_C1 * z, -P64.SH_C1 * x]
        c2, c3 = P64.SH_C2, P64.SH_C3
        basis += [c2[0] * x * y, c2[1] * y * z, c2[2] * (2 * zz - xx - yy), c2[3] * x * z, c2[4] * (xx - yy)]
        basis += [c3[0] * y * (3 * xx - yy), c3[1] * x * y * z, c3[2] * y * (4 * zz - xx - yy), c3[3] * z * (2 * zz - 3 * xx - 3 * yy),
                  c3[4] * x * (4 * zz - xx - yy), c3[5] * z * (xx - yy), c3[6] * x * (xx - 3 * yy)]
        n = (int(g["sh_degree"]) + 1) ** 2
        rgb = sum(basis[k][:, None] * sh[:, k, :] for k in range(n)) + 0.5
        loss = loss + (torch.relu(rgb) * C_("dL_dcolor")).sum()
    recs = dict(means2D=uv.detach().numpy(), conic=conic.detach().numpy(), opacity=oe.detach().numpy(), depth=tz.detach().numpy(),
                J=J.detach().numpy())
    return loss, leaves, recs


def _close(got, want, e=None, what=""):
    tol = 1e-9 * max(np.abs(want).max(), 1e-300) + (16 * 2.0 ** -53 * np.asarray(e) if e is not None else 0.0)
    assert np.all(np.abs(np.asarray(got) - want) <= tol), (what, np.abs(np.asarray(got) - want).max(), np.abs(want).max())


def _live(g, cam, mod, aa):
    fw = D64.forward(g, cam, mod, antialias=aa)
    live = ~fw["culled"]
    sel = {k: (v[live] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(live) else v) for k, v in g.items()}
    return sel, int(live.sum()), fw


def _ref_J(g, cam):
    vw = D64.view_of(cam)
    J, _, _ = D64._jacobian(D64._t(P64._cols(g["means3D"]), vw), vw, second=False)
    return np.stack([np.stack([J[i][j].v for j in range(3)], -1) for i in range(2)], 1)


AUTOGRAD = ["sh0", "sh1", "sh2", "sh3", "precomp_cov", "aa1", "rs5"]


@pytest.mark.parametrize("scene", AUTOGRAD)
def test_reference_matches_torch_float64_autograd(scene):
    import test_project_ref64_cpu as CPU
    g, cam, aa = _scene(scene)
    mod = 0.9
    sel, n, fw0 = _live(g, cam, mod, aa)
    assert n >= 24 and fw0["r2"][~fw0["culled"]].max() > 0.25   # a wide view: far from the axis, where the terms matter
    fw = D64.forward(sel, cam, mod, antialias=aa)
    cot = CPU.seeded_cotangents(n, 5, depth=True)
    rb = D64.backward(sel, [cam], [cot], mod, antialias=aa)
    loss, leaves, recs = _torch_loss_distorted(sel, cam, cot, mod, aa)
    for q in ("means2D", "conic", "opacity", "depth"):
        _close(fw[q], recs[q], what=q)
    _close(_ref_J(sel, cam), recs["J"], what="J")
    loss.backward()
    for name, leaf in leaves.items():
        want = leaf.grad.numpy() if leaf.grad is not None else np.zeros(tuple(leaf.shape))
        if name in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos"):
            got, e, _ = rb["camera"][0][name]
        elif name == "dL_dtan_fov":
            got, e, _ = rb["tan_fov"][0]
        elif name == "dL_dsh":
            got, e, _ = rb["dL_dsh"]
            n_ = (int(sel["sh_degree"]) + 1) ** 2
            got, e, want = got[:, :n_], e[:, :n_], want[:, :n_]
        else:
            got, e, _ = rb[name]
            if name == "dL_dopacity":
                want = want.reshape(-1)
        _close(got, want, e, name)
    assert np.abs(rb["camera"][0]["dL_dprojmatrix"][0]).max() == 0


@pytest.mark.parametrize("D", [KINECT_D, REALSENSE_D, (-0.3, 0.1, 0.01, -0.02)], ids=["kinect8", "realsense5", "brown4"])
def test_means_and_J_match_opencv(D):
    """cv2.projectPoints of t with a zero pose: its screen points are the means, and its Jacobian's d/dtvec columns (3:6)
    are d(u, v)/dt = J"""
    cv2 = pytest.importorskip("cv2")
    g, cam, _ = _scene("sh1")
    cam = dcam(D=D)
    sel, n, _ = _live(g, cam, 1.0, False)
    fw = D64.forward(sel, cam)
    vw = D64.view_of(cam)
    t = np.stack([x.v for x in D64._t(P64._cols(sel["means3D"]), vw)], 1)
    K = np.array([[vw["fx"], 0, float(np.float32(cam["distortion"][0]))], [0, vw["fy"], float(np.float32(cam["distortion"][1]))],
                  [0, 0, 1.0]])
    Dc = np.array([float(np.float32(x)) for x in cam["distortion"][2:10]])
    uv, jac = cv2.projectPoints(t.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, Dc)
    uv = uv.reshape(-1, 2)
    _close(fw["means2D"], uv, what="means2D vs cv2")
    Jcv = jac[:, 3:6].reshape(n, 2, 3)
    _close(_ref_J(sel, cam), Jcv, what="J vs cv2")


def test_zero_coefficients_give_the_pinhole_records_and_gradients():
    """All coefficients 0: the records and per-Gaussian gradients are the pinhole reference's for Gaussians inside the
    clamp region (the pinhole Jacobian is unclamped there).  The pinhole matrix of cameras.projection_from_intrinsics places
    the optical axis at (cx - 0.5, cy - 0.5) of the blend's pixel grid, the distorted model at (cx, cy): the means differ by
    that half pixel."""
    import test_project_ref64_cpu as CPU
    g, _, _ = _scene("sh1")
    cam = dcam(D=(0.0,) * 8, f=40 / 1.5)
    pin = {k: v for k, v in cam.items() if k != "distortion"}
    fp = P64.forward(g, pin)
    inside = ~fp["culled"] & ~fp["border"]
    vw = P64.view_of(pin)
    t = np.stack([x.v for x in D64._t(P64._cols(g["means3D"]), vw)], 1)
    inside &= (np.abs(t[:, 0] / t[:, 2]) < vw["limx"]) & (np.abs(t[:, 1] / t[:, 2]) < vw["limy"])
    sel = {k: (v[inside] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(inside) else v) for k, v in g.items()}
    n = int(inside.sum())
    assert n >= 16
    fd, fp = D64.forward(sel, cam), P64.forward(sel, pin)
    assert not fd["culled"].any()
    np.testing.assert_allclose(fd["means2D"] - 0.5, fp["means2D"], rtol=0, atol=2e-4)
    np.testing.assert_allclose(fd["conic"], fp["conic"], rtol=1e-9, atol=1e-12)
    cot = CPU.seeded_cotangents(n, 5, depth=True)
    gd, gp = D64.backward(sel, [cam], [cot]), P64.backward(sel, [pin], [cot])
    for q in ("dL_dmeans3D", "dL_dscales", "dL_drotations", "dL_dopacity", "dL_dsh"):
        # the pinhole mean's path runs through the float32 projmatrix, whose entries round apart from fx: 3e-7 of dL/dmeans3D
        # (a mean cotangent taken in the wrong units would be off by W / 2)
        tol = 1e-5 if q == "dL_dmeans3D" else 1e-9
        np.testing.assert_allclose(gd[q][0], gp[q][0], rtol=0, atol=tol * np.abs(gp[q][0]).max(), err_msg=q)


# --------------------------------------------------------------------------- r_max
def test_distortion_r_max():
    k1 = -0.3
    assert cameras.distortion_r_max([k1, 0, 0, 0])[0] == pytest.approx(1 / math.sqrt(-3 * k1), rel=1e-12)
    # a zero of the rational denominator 1 + k4 r^2 before any fold of the numerator: r = 1 / sqrt(-k4)
    assert cameras.distortion_r_max([0.0, 0, 0, 0, 0, -0.25, 0, 0])[0] == pytest.approx(2.0, rel=1e-9)
    # monotone coefficients: no fold
    assert cameras.distortion_r_max([0.1, 0.01, 0, 0, 0.001])[0] == math.inf
    assert cameras.distortion_r_max([0.0] * 8)[0] == math.inf
    # 4- and 5-entry D are padded with zeros
    for D in ([-0.2, 0.01, 0.001, 0.002], [-0.2, 0.01, 0.001, 0.002, -0.003]):
        r = cameras.distortion_r_max(D)[0]
        r8 = cameras.distortion_r_max(list(D) + [0.0] * (8 - len(D)))[0]
        assert r == r8 and np.isfinite(r)
        d = (D + [0.0])[:5]
        rr = lambda x: x * (1 + d[0] * x * x + d[1] * x ** 4 + d[4] * x ** 6)  # noqa: E731
        assert rr(r * 0.999) < rr(r) and rr(r * 1.001) < rr(r) + 1e-9   # a maximum of r R
    with pytest.raises(ValueError, match="thin-prism"):
        cameras.distortion_r_max([0.0] * 12)
    with pytest.raises(ValueError, match="thin-prism"):
        cameras.distortion_r_max([0.0] * 14)
    with pytest.raises(ValueError):
        cameras.distortion_r_max([0.0] * 6)


def test_cull_past_the_fold():
    g, _, _ = _scene("sh1")
    cam = dcam(D=(-0.3, 0, 0, 0))
    fw = D64.forward(g, cam)
    r2max = cam["distortion"][10] ** 2
    front = np.stack([x.v for x in D64._t(P64._cols(g["means3D"]), D64.view_of(cam))], 1)[:, 2] > P64.NEAR_Z
    assert ((fw["r2"] > r2max) & front).any() and ((fw["r2"] < r2max) & front).any()
    assert np.all(fw["radius"][(fw["r2"] > r2max) & ~fw["border"]] == 0)


# --------------------------------------------------------------------------- sensitivity
@pytest.mark.parametrize("mutation", D64.MUTATIONS)
def test_each_broken_convention_moves_a_checked_element_past_twice_its_bound(mutation):
    import test_project_ref64_cpu as CPU
    g, cam, _ = _scene("sh1")
    sel, n, _ = _live(g, cam, 1.0, False)
    cot = CPU.seeded_cotangents(n, 5, depth=True)
    fw, rb = D64.forward(sel, cam), D64.backward(sel, [cam], [cot])
    D64.MUTATE.add(mutation)
    try:
        fm, bm = D64.forward(sel, cam), D64.backward(sel, [cam], [cot])
    finally:
        D64.MUTATE.clear()
    worst = 0.0
    for q in ("means2D", "conic"):
        worst = max(worst, float((np.abs(fm[q] - fw[q]) / (P64.U * fw[q + "_B"] + 1e-30)).max()))
    for q in ("dL_dmeans3D", "dL_dscales", "dL_drotations"):
        v, e, d = rb[q]
        worst = max(worst, float((np.maximum(np.abs(bm[q][0] - v) - d, 0) / (P64.U * e + 1e-30)).max()))
    assert worst > 2.0, (mutation, worst)


# --------------------------------------------------------------------------- builders
def test_builders_tan_fov_r_max_and_errors():
    W, H = 64, 48
    c2w = _look(np.array([1.0, -2.0, 2.0]), scenes.SCENE_CENTER)
    K = np.array([[30.0, 0, 31.5], [0, 28.0, 23.5], [0, 0, 1]])
    cb = cameras.build_distorted_cameras(K[None], np.array([KINECT_D]), c2w[None], W, H)
    assert cb.tanfovx == [pytest.approx(W / 60.0)] and cb.tanfovy == [pytest.approx(H / 56.0)] and cb.FovX is None
    cx, cy, *d, rm = cb.distortion[0]
    assert (cx, cy) == (31.5, 23.5) and tuple(d) == KINECT_D and rm == cameras.distortion_r_max(KINECT_D)[0]
    s = cb.settings(0, torch.zeros(3), 0, False)
    assert s.distortion == cb.distortion[0] and not s.orthographic and s.fisheye is None
    with pytest.raises(ValueError):
        cb.as_novel_view()
    rs = cameras.build_distorted_cameras(K[None], np.array([REALSENSE_D]), c2w[None], W, H, r_max=0.9)
    assert rs.distortion[0][2:10] == (*REALSENSE_D[:4], REALSENSE_D[4], 0.0, 0.0, 0.0) and rs.distortion[0][10] == 0.9
    w2c = torch.from_numpy(np.linalg.inv(c2w)).requires_grad_()
    f = torch.tensor([[30.0, 28.0]], dtype=torch.float64, requires_grad=True)
    lb = cameras.distorted_camera_batch(w2c, f, [[31.5, 23.5]], [KINECT_D], W, H)
    assert lb.tanfovx is None and lb.fisheye is None and lb.distortion == cb.distortion
    assert torch.allclose(lb.tan_fov, torch.tensor([[W / 60.0, H / 56.0]], dtype=torch.float64))
    lb.tan_fov.sum().backward()
    assert torch.allclose(f.grad, torch.tensor([[-W / (2 * 30.0 ** 2), -H / (2 * 28.0 ** 2)]], dtype=torch.float64))
    hb = cameras.distorted_camera_batch(w2c, [[30.0, 28.0]], [[31.5, 23.5]], [KINECT_D], W, H)
    assert hb.tanfovx == [pytest.approx(W / 60.0)] and hb.distortion == cb.distortion
    torch.testing.assert_close(hb.world_view_transform.float(), cb.world_view_transform, atol=1e-6, rtol=1e-6)
    with pytest.raises(ValueError, match="thin-prism"):
        cameras.build_distorted_cameras(K[None], np.zeros((1, 12)), c2w[None], W, H)
    with pytest.raises(ValueError):
        cameras.build_distorted_cameras(K[None], np.array([[np.inf, 0, 0, 0]]), c2w[None], W, H)
    with pytest.raises(ValueError):
        cameras.distorted_camera_batch(w2c, [[30.0, 28.0]], [[31.5, 23.5]], [KINECT_D], W, H, r_max=0.0)


def test_settings_attribute():
    args = (8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False, False)
    s = GaussianRasterizationSettings(*args)
    assert s.distortion is None and len(tuple(s)) == 13 and GaussianRasterizationSettings._fields == s._fields
    dc = dict(cx=3.5, cy=3.5, k1=0.1, k2=0.0, p1=0.0, p2=0.0, k3=0.0, k4=0.0, k5=0.0, k6=0.0, r_max=math.inf)
    d = GaussianRasterizationSettings(*args, distortion=dc)
    assert d.distortion == (3.5, 3.5, 0.1, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, math.inf)
    assert d._replace(image_width=16).distortion == d.distortion and d._replace(distortion=None).distortion is None
    assert "distortion=(3.5" in repr(d)
    with pytest.raises(ValueError):
        GaussianRasterizationSettings(*args, orthographic=True, distortion=dc)
    with pytest.raises(ValueError):
        GaussianRasterizationSettings(*args, fisheye=(3.5, 3.5, 0, 0, 0, 0, 1.0), distortion=dc)
    with pytest.raises(ValueError):
        GaussianRasterizationSettings(*args, distortion=(1.0, 2.0))


BAD = [("flag", dict(distorted=2)), ("ortho", dict()), ("fisheye", dict()), ("nan", dict(p2=float("nan"))),
       ("inf", dict(k6=float("inf"))), ("cx", dict(cx=float("inf"))), ("zero", dict(r_max=0.0)), ("neg", dict(r_max=-1.0)),
       ("rnan", dict(r_max=float("nan")))]


@pytest.mark.parametrize("what,bad", BAD, ids=[b[0] for b in BAD])
def test_distortion_option_checks_its_parameters(what, bad):
    L = _binding.lib()
    views = (_binding.View * 2)()
    for v in views:
        v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
        for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                     "radii", "out_color", "dL_dpix", "blend_scratch"):
            setattr(v, name, 4096)
        v.binning_capacity = 1
    dc = (_binding.ViewDistortion * 2)()
    dc[1].distorted, dc[1].cx, dc[1].cy, dc[1].r_max = 1, 3.5, 3.5, math.inf
    for k, x in bad.items():
        setattr(dc[1], k, x)
    ortho = (ctypes.c_int * 2)(0, 1) if what == "ortho" else None
    fe = None
    if what == "fisheye":
        fe = (_binding.ViewFisheye * 2)()
        fe[1].fisheye, fe[1].cx, fe[1].cy, fe[1].theta_max = 1, 3.5, 3.5, 1.5
    opts = _binding.RenderOptions(ortho=ortho, fisheye=fe, distortion=dc)
    # pointers are never dereferenced: the parameters are checked before anything is enqueued
    rcs = [
        L.mgs_forward_views(2, views, opts, 4, 0, 0, 0, 4096, None, 4096, None, 4096, 4096, 1.0, 4096, None, 0, 0, None),
        L.mgs_backward_views(2, views, opts, 4, 0, 0, 0, 4096, None, 4096, None, 4096, 1.0, 4096, None, 4096, 4096, None, None, None,
                             None, None, None, 0, 0, 3, 0, None),
        L.mgs_lift_views(2, views, None, 0, None, ortho, fe, dc, 4, 0, 0, 0, 4096, None, 4096, 4096, 4096, 1.0, 4096, None,
                                   None, 4096, 0, None)]
    clouds = (_binding.Cloud * 1)()
    c = clouds[0]
    c.P, c.means3D, c.colors_precomp, c.opacities, c.scales, c.rotations = 4, 4096, 4096, 4096, 4096, 4096
    c.dL_dmean3D, c.dL_dopacity = 4096, 4096
    offs = (ctypes.c_int * 2)(0, 2)
    rcs.append(L.mgs_forward_clouds(1, clouds, offs, views, opts, 0, 0, 0, 1.0, 0, 0, None))
    rcs.append(L.mgs_backward_clouds(1, clouds, offs, views, opts, 0, 0, 0, 1.0, 0, 0, None))
    for rc in rcs:
        assert rc == -1 and "distortion" in _binding.last_error(), (what, rc, _binding.last_error())
