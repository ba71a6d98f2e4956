"""Fisheye views without a GPU: the float64 reference, the series branch, the camera builders and the C ABI's checks.

* tests/fisheye_ref64.py matches torch float64 autograd of an independent restatement to 1e-9 relative: the records
  (means2D, conic, o_eff, depth), dL/dmeans3D, dL/dcov3D (or the scales and rotations), dL/dsh, dL/dopacity, the 27 camera
  terms and dL/dtan_fov.  The restatement takes J from autograd of the mean map, with vm and tan_fov as leaves.
* The radial terms are continuous through r / z in {0, 1e-7, 1e-4, 1e-2, 1/8 +- ulp}: an fp32 restatement of
  csrc/fisheye.cuh stays within the reference's bound on both sides of the series threshold.
* With k = 0 and a small-angle scene, the fisheye records converge to the pinhole records as the angles shrink.
* Builders: tan_fov = W / (2 fx), theta_max against the root of rho', learnable focal lengths; the errors.
* Each broken convention of fisheye_ref64.MUTATIONS moves a checked element past twice its bound.
* Bad fisheye parameters in the render options and the lift return MGS_ERR_INVALID_ARG before anything is enqueued.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import fisheye_ref64 as F64
import project_ref64 as P64
import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding, cameras, scenes
from manigaussian_b200.rasterizer import GaussianRasterizationSettings

UMI_K = (-0.0318, 0.0019, -0.0015, 0.0002)   # a GoPro-like Kannala-Brandt calibration (about 155 degrees)


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


def fcam(W=40, H=32, k=(0.0, 0.0, 0.0, 0.0), eye=(0.6, -0.4, 0.9), f=None):
    """a fisheye camera looking at the scene centre from close by, so the cloud spans a wide angle"""
    f = f if f is not None else W / 3.0
    return F64.fisheye_cam(W, H, f, f * 1.02, (W - 1) / 2 + 0.3, (H - 1) / 2 - 0.2, k, _look(np.array(eye), scenes.SCENE_CENTER))


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
    k = UMI_K if name == "kb4" else (0.05, -0.01, 0.0, 0.0) if name == "aa1" else (0.0, 0.0, 0.0, 0.0)
    return g, fcam(k=k), name.startswith("aa")


def _torch_loss_fisheye(g, cam, cot, mod, aa):
    """An independent torch restatement of one fisheye view with every input a leaf: means, scale_modifier * scales and
    rotations (or cov3D), opacities, SHs, vm [16], campos [3] and {tan_fovx, tan_fovy}.  The screen mean is
    fx theta_d t.x / r + cx (fx = W / (2 tan_fovx)), J its autograd Jacobian w.r.t. t (kept in the graph); the reference's
    conventions as in test_ortho_cpu."""
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
    cx, cy, k1, k2, k3, k4, _ = (float(np.float32(v)) for v in cam["fisheye"])
    vm = vm16.reshape(4, 4).T
    t = p @ vm[:3, :3].T + vm[:3, 3]

    def mean_map(t):
        x, y, z = t.unbind(1)
        r = torch.sqrt(x * x + y * y)
        th = torch.atan2(r, z)
        t2 = th * th
        thd = th * (1 + k1 * t2 + k2 * t2 ** 2 + k3 * t2 ** 3 + k4 * t2 ** 4)
        return torch.stack([fx * thd * x / r + cx, fy * thd * y / r + cy], 1)

    uv = mean_map(t)
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
    # dL_dmean2D is the cotangent of ndc = (2 u + 1) / W - 1, as in every restatement of the project (test_ortho_cpu, ...)
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
    recs = dict(means2D=uv.detach().numpy(), conic=conic.detach().numpy(), opacity=oe.detach().numpy(), depth=tz.detach().numpy())
    return loss, leaves, recs


def _close(got, want, e=None, what=""):
    tol = 1e-9 * max(np.abs(want).max(), 1e-300) + (16 * 2.0 ** -53 * np.asarray(e) if e is not None else 0.0)
    assert np.all(np.abs(np.asarray(got) - want) <= tol), (what, np.abs(np.asarray(got) - want).max(), np.abs(want).max())


def _live(g, cam, mod, aa):
    fw = F64.forward(g, cam, mod, antialias=aa)
    live = ~fw["culled"]
    sel = {k: (v[live] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(live) else v) for k, v in g.items()}
    return sel, int(live.sum()), fw


AUTOGRAD = ["sh0", "sh1", "sh2", "sh3", "precomp_cov", "aa1", "kb4"]


@pytest.mark.parametrize("scene", AUTOGRAD)
def test_reference_matches_torch_float64_autograd(scene):
    import test_project_ref64_cpu as CPU
    g, cam, aa = _scene(scene)
    mod = 0.9
    sel, n, fw0 = _live(g, cam, mod, aa)
    assert n >= 24 and fw0["theta"][~fw0["culled"]].max() > 0.8   # a wide view: angles beyond 45 degrees
    fw = F64.forward(sel, cam, mod, antialias=aa)
    cot = CPU.seeded_cotangents(n, 5, depth=True)
    rb = F64.backward(sel, [cam], [cot], mod, antialias=aa)
    loss, leaves, recs = _torch_loss_fisheye(sel, cam, cot, mod, aa)
    for q in ("means2D", "conic", "opacity", "depth"):
        _close(fw[q], recs[q], what=q)
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


# --------------------------------------------------------------------------- the series branch
def _radial_f32(x, y, z, k):
    """csrc/fisheye.cuh's fisheye_radial<true> in numpy float32, in the kernel's operation order"""
    f = np.float32
    x, y, z = f(x), f(y), f(z)
    k1, k2, k3, k4 = (f(v) for v in k)
    r2 = x * x + y * y
    r = np.sqrt(r2)
    s = r2 + z * z
    is_ = f(1) / s
    iz = f(1) / z
    th = f(np.arctan2(np.float64(r), np.float64(z)))
    t2 = th * th
    rho = f(1) + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)))
    D1 = f(1) + t2 * (f(3) * k1 + t2 * (f(5) * k2 + t2 * (f(7) * k3 + t2 * (f(9) * k4))))
    e2 = r2 * iz * iz
    ser = e2 < f(F64.SERIES_E2)
    q = iz * (f(1) + e2 * (f(-1 / 3) + e2 * (f(0.2) + e2 * f(-1 / 7)))) if ser else th / r
    a = q * rho
    g = D1 * is_
    c0 = f(2) * k1 - f(2 / 3)
    c1 = f(4) * (k2 - k1) + f(0.8)
    c2 = f(5.6) * k1 - f(10) * k2 + f(6) * k3 - f(6 / 7)
    iz3 = iz * iz * iz
    c = iz3 * (c0 + e2 * (c1 + e2 * c2)) if ser else (D1 * z * is_ - a) / r2
    D2r = q * (f(6) * k1 + t2 * (f(20) * k2 + t2 * (f(42) * k3 + t2 * (f(72) * k4))))
    is2 = is_ * is_
    C1 = iz3 * iz * iz * (f(2) * c1 + f(4) * c2 * e2) if ser else ((D2r * z * z - f(2) * z * D1) * is2 - f(3) * c) / r2
    cz = (f(2) * D1 - D2r * z) * is2
    gz = -(D2r * r2 + f(2) * z * D1) * is2
    return dict(a=a, c=c, g=g, C1=C1, cz=cz, gz=gz, series=ser)


@pytest.mark.parametrize("k", [(0.0, 0.0, 0.0, 0.0), UMI_K, (0.3, -0.2, 0.05, -0.01)])
def test_radial_terms_are_continuous_through_the_series_threshold(k):
    z = 1.7
    thr = math.sqrt(F64.SERIES_E2)
    es = [0.0, 1e-7, 1e-4, 1e-2, thr * (1 - 2 ** -22), thr * (1 + 2 ** -22), 0.3]
    branches = set()
    for e in es:
        x, y = np.float32(0.6 * e * z), np.float32(0.8 * e * z)
        E = P64.E
        ref = F64.radial(E(np.array([float(x)])), E(np.array([float(y)])), E(np.array([float(np.float32(z))])), k)
        got = _radial_f32(x, y, z, k)
        branches.add(bool(got["series"]))
        for q in ("a", "c", "g", "C1", "cz", "gz"):
            v, b = float(ref[q].v[0]), float(np.asarray(ref[q].e + 0 * ref[q].v)[0])
            assert abs(float(got[q]) - v) <= 2.0 * P64.U * b + 1e-30, (e, q, float(got[q]), v, b)
    assert branches == {True, False}
    # the limits the definition states
    ref0 = F64.radial(P64.E(np.zeros(1)), P64.E(np.zeros(1)), P64.E(np.array([z])), k)
    k1 = float(np.float32(k[0]))
    assert ref0["a"].v[0] == pytest.approx(1 / z) and ref0["c"].v[0] == pytest.approx((2 * k1 - 2 / 3) / z ** 3)


def test_small_angles_converge_to_the_pinhole_records_and_gradients():
    """k = 0 fisheye and the pinhole camera of the same K agree more closely as the cloud's angles shrink (error ~ theta^2),
    in the records and in the per-Gaussian gradients of the same blend-stage cotangents (the mean's cotangent is w.r.t. ndc
    for both models, so a wrong scale of the fisheye mean's cotangent shows as a gap that does not shrink).
    The pinhole matrix of cameras.projection_from_intrinsics places the optical axis at (cx - 0.5, cy - 0.5) of the blend's
    pixel grid (the reference's convention), the fisheye model at (cx, cy) (OpenCV's): the means differ by that half pixel."""
    g = scenes.make_gaussians(24, sh_degree=1, seed=4)
    g["cov3D_precomp"] = None
    target = scenes.SCENE_CENTER.astype(np.float64)
    direction = np.array([1.5, -1.0, 1.3]) / np.linalg.norm([1.5, -1.0, 1.3])
    W, H = 64, 48
    errs, gerrs = [], []
    import test_project_ref64_cpu as CPU
    cot = CPU.seeded_cotangents(len(g["means3D"]), 5, depth=True)
    for D in (3.0, 30.0, 300.0):
        f = 40.0 * D
        cam = F64.fisheye_cam(W, H, f, f, (W - 1) / 2, (H - 1) / 2, (0, 0, 0, 0), _look(target + D * direction, target))
        fw = F64.forward(g, cam)
        pin = P64.forward(g, {k: v for k, v in cam.items() if k != "fisheye"})
        errs.append(np.abs(fw["conic"] - pin["conic"]).max() / np.abs(pin["conic"]).max())
        errs.append(np.abs(fw["means2D"] - pin["means2D"] - 0.5).max())
        assert not fw["culled"].any() and not pin["culled"].any()
        gb = F64.backward(g, [cam], [cot])
        pb = P64.backward(g, [{k: v for k, v in cam.items() if k != "fisheye"}], [cot])
        gerrs.append(max(np.abs(gb[q][0] - pb[q][0]).max() / np.abs(pb[q][0]).max()
                         for q in ("dL_dmeans3D", "dL_dscales", "dL_drotations")))
    conic, mean = errs[0::2], errs[1::2]
    assert conic[1] < conic[0] / 30 and conic[2] < conic[1] / 30, conic
    assert mean[1] < mean[0] / 30 and mean[2] < 1e-4, mean
    assert gerrs[1] < gerrs[0] / 30 and gerrs[2] < gerrs[1] / 30 and gerrs[2] < 1e-4, gerrs


# --------------------------------------------------------------------------- sensitivity
@pytest.mark.parametrize("mutation", F64.MUTATIONS)
def test_each_broken_convention_moves_a_checked_element_past_twice_its_bound(mutation):
    import test_project_ref64_cpu as CPU
    g, cam, _ = _scene("kb4")
    sel, n, _ = _live(g, cam, 1.0, False)
    cot = CPU.seeded_cotangents(n, 5, depth=True)
    fw, rb = F64.forward(sel, cam), F64.backward(sel, [cam], [cot])
    F64.MUTATE.add(mutation)
    try:
        fm, bm = F64.forward(sel, cam), F64.backward(sel, [cam], [cot])
    finally:
        F64.MUTATE.clear()
    worst = 0.0
    for q in ("means2D", "conic"):
        worst = max(worst, float((np.abs(fm[q] - fw[q]) / (P64.U * fw[q + "_B"] + 1e-30)).max()))
    for q in ("dL_dmeans3D", "dL_dscales", "dL_drotations"):
        v, e, d = rb[q]
        worst = max(worst, float((np.maximum(np.abs(bm[q][0] - v) - d, 0) / (P64.U * e + 1e-30)).max()))
    assert worst > 2.0, (mutation, worst)


# --------------------------------------------------------------------------- builders
def test_theta_max_is_the_first_zero_of_rho_prime():
    assert cameras.fisheye_theta_max([0, 0, 0, 0])[0] == pytest.approx(math.pi / 2, abs=1e-6)
    assert cameras.fisheye_theta_max([0, 0, 0, 0])[0] <= math.pi / 2
    t = cameras.fisheye_theta_max([-0.2, 0, 0, 0])[0]     # 1 - 0.6 theta^2 = 0
    assert t == pytest.approx(math.sqrt(1 / 0.6), rel=1e-6) and t <= math.sqrt(1 / 0.6)
    rp = lambda x, k: 1 + 3 * k[0] * x ** 2 + 5 * k[1] * x ** 4 + 7 * k[2] * x ** 6 + 9 * k[3] * x ** 8  # noqa: E731
    k = (-0.1, -0.05, 0.0, 0.0)                            # 1 - 0.3 x - 0.25 x^2, x = theta^2: a root at theta = 1.22
    t = cameras.fisheye_theta_max(k)[0]
    assert t < 1.3 and 0 <= rp(t, k) < 1e-6 and rp(t + 1e-5, k) < 0 and min(rp(x, k) for x in np.linspace(0, t, 100)) >= 0
    k = (-0.1, -0.05, 0.01, 0.001)                         # rho' stays positive up to pi/2
    assert cameras.fisheye_theta_max(k)[0] == pytest.approx(math.pi / 2, abs=1e-6)
    assert min(rp(x, k) for x in np.linspace(0, math.pi / 2, 100)) > 0
    with pytest.raises(ValueError):
        cameras.fisheye_theta_max([np.nan, 0, 0, 0])


def test_builders_tan_fov_theta_max_and_errors():
    W, H = 64, 48
    c2w = _look(np.array([1.0, -2.0, 2.0]), scenes.SCENE_CENTER)
    K = np.array([[30.0, 0, 31.5], [0, 28.0, 23.5], [0, 0, 1]])
    cb = cameras.build_fisheye_cameras(K[None], np.array([UMI_K]), c2w[None], W, H)
    assert cb.tanfovx == [pytest.approx(W / 60.0)] and cb.tanfovy == [pytest.approx(H / 56.0)] and cb.FovX is None
    cx, cy, k1, k2, k3, k4, tm = cb.fisheye[0]
    assert (cx, cy) == (31.5, 23.5) and (k1, k2, k3, k4) == UMI_K and tm == cameras.fisheye_theta_max(UMI_K)[0]
    s = cb.settings(0, torch.zeros(3), 0, False)
    assert s.fisheye == cb.fisheye[0] and not s.orthographic
    with pytest.raises(ValueError):
        cb.as_novel_view()
    w2c = torch.from_numpy(np.linalg.inv(c2w)).requires_grad_()
    f = torch.tensor([[30.0, 28.0]], dtype=torch.float64, requires_grad=True)
    lb = cameras.fisheye_camera_batch(w2c, f, [[31.5, 23.5]], [UMI_K], W, H)
    assert lb.tanfovx is None and torch.allclose(lb.tan_fov, torch.tensor([[W / 60.0, H / 56.0]], dtype=torch.float64))
    lb.tan_fov.sum().backward()
    assert torch.allclose(f.grad, torch.tensor([[-W / (2 * 30.0 ** 2), -H / (2 * 28.0 ** 2)]], dtype=torch.float64))
    hb = cameras.fisheye_camera_batch(w2c, [[30.0, 28.0]], [[31.5, 23.5]], [UMI_K], W, H)
    assert hb.tanfovx == [pytest.approx(W / 60.0)] and hb.fisheye == cb.fisheye
    torch.testing.assert_close(hb.world_view_transform.float(), cb.world_view_transform, atol=1e-6, rtol=1e-6)
    torch.testing.assert_close(lb.full_proj_transform.detach(), hb.full_proj_transform)   # the pinhole matrix of the same K
    with pytest.raises(ValueError):
        cameras.build_fisheye_cameras(K[None], np.array([[np.inf, 0, 0, 0]]), c2w[None], W, H)
    with pytest.raises(ValueError):
        cameras.fisheye_camera_batch(w2c, [[0.0, 28.0]], [[31.5, 23.5]], [UMI_K], W, H)


def test_settings_attribute():
    args = (8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False, False)
    s = GaussianRasterizationSettings(*args)
    assert s.fisheye is None and len(tuple(s)) == 13 and GaussianRasterizationSettings._fields == s._fields
    fe = dict(cx=3.5, cy=3.5, k1=0.1, k2=0.0, k3=0.0, k4=0.0, theta_max=1.2)
    f = GaussianRasterizationSettings(*args, fisheye=fe)
    assert f.fisheye == (3.5, 3.5, 0.1, 0.0, 0.0, 0.0, 1.2)
    assert f._replace(image_width=16).fisheye == f.fisheye and f._replace(fisheye=None).fisheye is None
    assert "fisheye=(3.5" in repr(f)
    with pytest.raises(ValueError):
        GaussianRasterizationSettings(*args, orthographic=True, fisheye=fe)
    with pytest.raises(ValueError):
        GaussianRasterizationSettings(*args, fisheye=(1.0, 2.0))


BAD = [("flag", dict(fisheye=2)), ("ortho", dict()), ("nan", dict(k2=float("nan"))), ("inf", dict(cx=float("inf"))),
       ("zero", dict(theta_max=0.0)), ("wide", dict(theta_max=1.6))]


@pytest.mark.parametrize("what,bad", BAD, ids=[b[0] for b in BAD])
def test_fisheye_option_checks_its_parameters(what, bad):
    L = _binding.lib()
    views = (_binding.View * 2)()
    for v in views:
        v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
        for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                     "radii", "out_color", "dL_dpix", "blend_scratch"):
            setattr(v, name, 4096)
        v.binning_capacity = 1
    fe = (_binding.ViewFisheye * 2)()
    fe[1].fisheye, fe[1].cx, fe[1].cy, fe[1].theta_max = 1, 3.5, 3.5, 1.5
    for k, x in bad.items():
        setattr(fe[1], k, x)
    ortho = (ctypes.c_int * 2)(0, 1) if what == "ortho" else None
    opts = _binding.RenderOptions(ortho=ortho, fisheye=fe)
    # pointers are never dereferenced: the parameters are checked before anything is enqueued
    rcs = [
        L.mgs_forward_views(2, views, opts, 4, 0, 0, 0, 4096, None, 4096, None, 4096, 4096, 1.0, 4096, None, 0, 0, None),
        L.mgs_backward_views(2, views, opts, 4, 0, 0, 0, 4096, None, 4096, None, 4096, 1.0, 4096, None, 4096, 4096, None, None, None,
                             None, None, None, 0, 0, 3, 0, None),
        L.mgs_lift_views(2, views, None, 0, None, ortho, fe, None, 4, 0, 0, 0, 4096, None, 4096, 4096, 4096, 1.0, 4096, None, None,
                                 4096, 0, None)]
    clouds = (_binding.Cloud * 1)()
    c = clouds[0]
    c.P, c.means3D, c.colors_precomp, c.opacities, c.scales, c.rotations = 4, 4096, 4096, 4096, 4096, 4096
    c.dL_dmean3D, c.dL_dopacity = 4096, 4096
    offs = (ctypes.c_int * 2)(0, 2)
    rcs.append(L.mgs_forward_clouds(1, clouds, offs, views, opts, 0, 0, 0, 1.0, 0, 0, None))
    rcs.append(L.mgs_backward_clouds(1, clouds, offs, views, opts, 0, 0, 0, 1.0, 0, 0, None))
    for rc in rcs:
        assert rc == -1 and "fisheye" in _binding.last_error(), (what, rc, _binding.last_error())
