"""The projection kernels (project.cu, project_bwd.cu), Gaussian by Gaussian, against the float64 reference
(tests/project_ref64.py).

* Single view, inputs known exactly: the forward's records (radius, tiles, means2D, depth, cov3D, conic, o, rgb, clamp bits,
  extent) are compared with `project_ref64.forward`; `mgs_backward` is called through the C ABI with a dL_dconic buffer and
  every output prefilled with NaN.  With AA off and no depth cotangent its dL_dmean2D, dL_dconic, dL_dcolor and dL_dopacity
  are bit for bit the blend-stage record project_bwd consumed, so they feed the float64 chain and the bound is the chain's
  rounding alone; every per-Gaussian output is compared.
* AA on (needles on both sides of the 2.5e-5 clamp, degrees 1-3), depth on, several views and several clouds: the per-view cotangents come from blend_ref64 on our own records and
  pixel masks (as test_blend_pairs_gpu.run_kernels does), their bounds carried through the chain; the kernels' sums over
  V in {1, 4, 16, 17, 33} views (17 and 33 cross MAX_BWD_VIEWS = 16), shared or per-view dL_dmeans2D, accumulate onto a
  seeded buffer, 20 clouds x 2 views, a cloud of 17 views, degrees 2 and 3 through the clouds kernel.
* Every instantiation of project_bwd (views / clouds x AA x NSH in {12, 27, 48}) is run by a listed case (INSTANTIATIONS).
* The output contract of mgs_backward and mgs_backward_views: with each nullable output NULL in turn and the others
  prefilled with NaN, every output given is fully written, and within the float64 bounds (mgs_backward) or equal to the
  all-outputs call up to the blend's atomic reordering (mgs_backward_views).

Gaussians with a borderline decision (project_ref64.BAND) in any view are left out of the comparison of their rows.

Measured on an H100 80GB HBM3 (400 W power limit): worst raw ratio |x - ref64| / (u e) per scene, single view (KAPPA in
project_ref64 = 4x the worst of these and of the C oracle's):

| scene | depth | means2D | conic | rgb | cov3D | extent | dmeans3D | dcov3D | dsh | dscales | drotations |
|---|---|---|---|---|---|---|---|---|---|---|---|
| clamp_x / clamp_y | 0.58 | 0.39 | 0.084 | 0.43 | 0.32 | 0.021 | 0.10 | 0.054 | 0.46 | 0.028 | 0.026 |
| near | 0.40 | 0.25 | 0.082 | 0.56 | 0.28 | 0.026 | 0.25 | 0.062 | 0.45 | 0.016 | 0.010 |
| quat_scale (0.7 / 1.0 / 1.9) | 0.50 | 0.37 | 0.14 | 0.51 | 0.43 | 0.058 | 0.20 | 0.10 | 0.49 | 0.074 | 0.048 |
| sh0 - sh3 (M = (deg+1)^2 / 16) | 0.71 | 0.58 | 0.088 | 0.50 | 0.33 | 0.040 | 0.31 | 0.085 | 0.48 | 0.051 | 0.026 |
| precomp_cov / precomp_sr | 0.55 | 0.44 | 0.094 | - | 0.28 | 0.035 | 0.24 | 0.056 | - | 0.030 | 0.029 |
| ragged_f32 | 0.80 | 0.62 | 0.14 | 0.79 | 0.36 | 0.028 | 0.29 | 0.15 | 0.50 | 0.050 | 0.038 |
| sh3_big | 0.81 | 0.89 | 0.17 | 0.28 | 0.34 | 0.032 | 0.22 | 0.12 | 0.48 | 0.040 | 0.028 |
| mg_real_f3 | 0.85 | 0.93 | 0.16 | 0.86 | 0.46 | 0.033 | 0.33 | 0.15 | 0.50 | 0.076 | 0.047 |

AA on (aa1 / aa2 / aa3, one view, blend_ref64 cotangents): records depth 0.59, means2D 0.54, conic 0.15, rgb 0.53,
cov3D 0.29, extent 0.15, o_eff 0.37; the chain's sums dL_dscales 0.041, dL_dopacity 0.058, every other output within its
inherited bound d.  These needles found the AA backward recovering the undilated covariance as (S' - 0.3 I), which cancels
to a relative error of u 0.3 / c0 on them (raw ratios up to 137); project_bwd.cu now keeps a0, c0 from before the low-pass.
Several views and clouds (AA and depth cotangents on): every kernel output lies within the inherited blend_ref64 bound d
(raw ratio 0 for every quantity).  All 45 cases take about 28 s.
"""
import numpy as np
import pytest

import blend_ref64 as B64
import project_ref64 as P64
import util
from manigaussian_b200 import scenes

pytestmark = pytest.mark.gpu


# --------------------------------------------------------------------------- scene construction (numpy only)
def _place(cam, px, py, z):
    """World-space means projecting to pixel (px, py) at view depth z (test_blend_pairs_gpu.place, shapes dropped)."""
    import test_blend_pairs_gpu as BP
    px = np.asarray(px, np.float64).ravel()
    return BP.place(cam, px, py, z, BP.iso(len(px), 1.0), np.full(len(px), 0.5), F=0)["means3D"]


def _view_quat(cam, n):
    """Quaternions whose R(q) has the camera's axes as columns: scales then act along view x, y, z."""
    from scipy.spatial.transform import Rotation
    Rw = cam["viewmatrix"].astype(np.float64).T[:3, :3]        # world -> view
    x, y, z, w = Rotation.from_matrix(Rw.T).as_quat()
    return np.tile(np.array([w, x, y, z]), (n, 1))


def _gauss(cam, means, scales, rotations=None, opac=None, deg=1, M=None, seed=0, dc=None, colors=False, cov=False,
           modifier=1.0):
    rng = np.random.default_rng(seed)
    n = len(means)
    if rotations is None:
        q = rng.normal(0, 1, (n, 4))
        rotations = q / np.linalg.norm(q, axis=1, keepdims=True)
    g = dict(means3D=np.asarray(means, np.float32), opacities=(rng.uniform(0.2, 0.9, (n, 1)) if opac is None else
                                                               np.asarray(opac).reshape(n, 1)).astype(np.float32),
             scales=np.asarray(scales, np.float32), rotations=np.asarray(rotations, np.float32), cov3D_precomp=None,
             shs=None, sh_degree=deg, colors_precomp=None, feature=None)
    if colors:
        g["colors_precomp"] = rng.random((n, 3)).astype(np.float32)
        g["sh_degree"] = 0
    else:
        M = (deg + 1) ** 2 if M is None else M
        sh = rng.normal(0, 0.3, (n, M, 3))
        sh[:, 0, :] = rng.normal(0, 1.0, (n, 3)) if dc is None else dc
        g["shs"] = sh.astype(np.float32)
    if cov:
        s = g["scales"].astype(np.float64) * np.float32(modifier)
        q = g["rotations"].astype(np.float64)
        Rm = np.stack([_rot(qq) for qq in q])
        Sig = Rm @ (s[:, :, None] ** 2 * np.transpose(Rm, (0, 2, 1)))
        g["cov3D_precomp"] = Sig[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32)
        g["scales"] = g["rotations"] = None
    return g


def _rot(q):
    r, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                     [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                     [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])


RATIOS_CLAMP = (1.2, 1.31, 1.5, 3.0)


def scene_clamp(axis):
    """Means at |t.x / t.z| (axis 0) or |t.y / t.z| (axis 1) = {1.2, 1.31, 1.5, 3} tan_fov on both sides, big splats that
    still reach the image.  Edge asserted: at least 8 on-screen Gaussians past the 1.3 tan_fov clamp on the axis."""
    W, H = 64, 48
    cam = scenes.make_camera(W, H, 1, 4)
    rng = np.random.default_rng(31 + axis)
    r = np.repeat(np.array(RATIOS_CLAMP), 6) * np.tile([1, -1], 12)
    z = rng.uniform(1.0, 2.5, len(r))
    other = rng.uniform(-0.6, 0.6, len(r))
    if axis == 0:
        px, py = r * W / 2 + W / 2 - 0.5, other * H / 2 + H / 2 - 0.5
    else:
        px, py = other * W / 2 + W / 2 - 0.5, r * H / 2 + H / 2 - 0.5
    means = _place(cam, px, py, z)
    scales = (z[:, None] * rng.uniform(0.25, 0.6, (len(r), 3)))
    return dict(cam=cam, g=_gauss(cam, means, scales, deg=1, seed=3 + axis), edge=("clamp", axis, 8))


def scene_near():
    """View depths just below and above the 0.2 near plane, at 0.25 and 0.5, and behind the camera.  Edge asserted: 8
    culled by the near plane, 8 kept with t.z < 0.26."""
    W, H = 48, 48
    cam = scenes.make_camera(W, H, 2, 4)
    z = np.repeat(np.array([0.2 - 1e-3, 0.2 - 1e-5, 0.2 + 1e-5, 0.2 + 1e-3, 0.25, 0.5, -0.5, -2.0]), 2)
    rng = np.random.default_rng(41)
    px, py = rng.uniform(10, 38, len(z)), rng.uniform(10, 38, len(z))
    means = _place(cam, px, py, z)
    scales = np.abs(z)[:, None] * rng.uniform(0.002, 0.02, (len(z), 3))
    return dict(cam=cam, g=_gauss(cam, means, scales, deg=1, seed=5), edge=("near",))


QNORMS = (0.05, 0.5, 1.0, 3.0, 20.0)


def scene_quat_scale(modifier=0.7):
    """Quaternion norms {0.05, 0.5, 1, 3, 20}, the identity and r = 0; scales from 1e-5 to 0.5 with anisotropy up to 1e4
    (needles, where the 0.3 px^2 dilation dominates det).  Edge asserted: every norm present on screen, and at least 8
    on-screen needles whose minor screen-space variance is below 0.03 px^2 (the dilation at least 10x larger)."""
    W, H = 64, 64
    cam = scenes.make_camera(W, H, 3, 4)
    rng = np.random.default_rng(51)
    n = 70
    q = rng.normal(0, 1, (n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    nq = np.array(QNORMS)[np.arange(n) % len(QNORMS)]
    q *= nq[:, None]
    q[0] = (1, 0, 0, 0)
    q[1, 0] = 0.0
    s = np.exp(rng.uniform(np.log(1e-4), np.log(0.05), (n, 3)))
    s[::3, 0] = rng.uniform(0.02, 0.5, len(s[::3]))                       # needles: anisotropy up to 1e4
    s[::3, 1:] = s[::3, :1] * rng.uniform(1e-4, 1e-3, (len(s[::3]), 2))
    s[5] = 1e-5
    s /= (nq ** 2)[:, None]                                                 # R(q) scales the covariance by |q|^4
    means = _place(cam, rng.uniform(4, 60, n), rng.uniform(4, 60, n), rng.uniform(1.0, 2.0, n))
    g = _gauss(cam, means, s, rotations=q, deg=1, seed=7)
    return dict(cam=cam, g=g, scale_modifier=modifier, edge=("quat",))


def scene_sh(deg, M=None):
    """SH degree `deg` with M = (deg + 1)^2 or 16; DC terms near -0.5 / C0 so that about half the channels clamp; views along
    the camera axis (means on the image centre) among random ones.  Edge asserted: 25-75 % of live channels clamped."""
    W, H = 48, 40
    cam = scenes.make_camera(W, H, 0, 4)
    rng = np.random.default_rng(61 + deg)
    n = 80
    px, py = rng.uniform(2, 46, n), rng.uniform(2, 38, n)
    px[:6], py[:6] = W / 2 - 0.5, H / 2 - 0.5
    means = _place(cam, px, py, rng.uniform(0.8, 2.5, n))
    dc = (-0.5 + rng.normal(0, 0.05, (n, 3))) / P64.SH_C0
    g = _gauss(cam, means, rng.uniform(0.003, 0.03, (n, 3)), deg=deg, M=M, seed=11 + deg, dc=dc)
    g["shs"][:, 1:] *= 0.15
    return dict(cam=cam, g=g, edge=("sh",))


def scene_precomp(cov):
    """colors_precomp with cov3D_precomp (cov) or with scales / rotations."""
    W, H = 40, 40
    cam = scenes.make_camera(W, H, 1, 4)
    rng = np.random.default_rng(71)
    n = 60
    means = _place(cam, rng.uniform(0, 40, n), rng.uniform(0, 40, n), rng.uniform(0.8, 2.0, n))
    g = _gauss(cam, means, rng.uniform(0.003, 0.05, (n, 3)), seed=13, colors=True, cov=cov)
    return dict(cam=cam, g=g, edge=())


def scene_aa(deg):
    """AA on, degree `deg`: needles whose r = det0 / det straddles the 2.5e-5 clamp, plus ordinary splats.  Edge asserted:
    at least 4 live Gaussians on each side of the clamp."""
    W, H = 48, 48
    cam = scenes.make_camera(W, H, 2, 4)
    rng = np.random.default_rng(81 + deg)
    n, m = 24, 40
    z = rng.uniform(1.0, 1.6, n)
    fx = W / (2 * cam["tanfovx"])
    lam = np.geomspace(2e-6, 3e-5, n)                     # minor-axis variance in px^2: r ~ lam / 0.3
    s = np.stack([np.full(n, 0.05), np.sqrt(lam) * z / fx, np.full(n, 1e-4)], 1)
    means = _place(cam, rng.uniform(8, 40, n), rng.uniform(8, 40, n), z)
    g1 = _gauss(cam, means, s, rotations=_view_quat(cam, n), deg=deg, seed=17)
    means2 = _place(cam, rng.uniform(0, 48, m), rng.uniform(0, 48, m), rng.uniform(1.0, 2.0, m))
    g2 = _gauss(cam, means2, rng.uniform(0.003, 0.03, (m, 3)), deg=deg, seed=19)
    g = {k: (None if g1[k] is None else (np.concatenate([g1[k], g2[k]]) if isinstance(g1[k], np.ndarray) else g1[k]))
         for k in g1}
    return dict(cam=cam, g=g, antialias=True, edge=("aa",))


def scene_random(kw):
    inp = util.make_inputs(**kw)
    return dict(cam=inp["cam"], g=inp["g"], edge=())


SCENES = {
    "clamp_x": lambda: scene_clamp(0),
    "clamp_y": lambda: scene_clamp(1),
    "near": scene_near,
    "quat_scale": lambda: scene_quat_scale(0.7),
    "quat_scale_1": lambda: scene_quat_scale(1.0),
    "quat_scale_19": lambda: scene_quat_scale(1.9),
    "sh0": lambda: scene_sh(0), "sh0_m16": lambda: scene_sh(0, 16),
    "sh1": lambda: scene_sh(1), "sh1_m16": lambda: scene_sh(1, 16),
    "sh2": lambda: scene_sh(2), "sh2_m16": lambda: scene_sh(2, 16),
    "sh3": lambda: scene_sh(3), "sh3_m16": lambda: scene_sh(3, 16),
    "precomp_cov": lambda: scene_precomp(True),
    "precomp_sr": lambda: scene_precomp(False),
    "aa1": lambda: scene_aa(1), "aa2": lambda: scene_aa(2), "aa3": lambda: scene_aa(3),
    "ragged_f32": lambda: scene_random(dict(P=5000, W=200, H=120, F=0, seed=3)),
    "sh3_big": lambda: scene_random(dict(P=1500, W=128, H=96, F=0, seed=5, sh_degree=3, scale0=0.04)),
    "mg_real_f3": lambda: scene_random(dict(P=16384, W=128, H=128, F=0, seed=2)),   # ManiGaussian's regime
}


# --------------------------------------------------------------------------- running the kernels
def _t(x):
    return util._t(x)


def _arr(R, which, name, state, a0, a1, dtype, count):
    import torch
    off = R.state_array(which, name, state, a0, a1) - state.data_ptr()
    nbytes = count * torch.empty((), dtype=dtype).element_size()
    return state[off:off + nbytes].view(dtype).cpu().numpy()


def records(R, geomB, P):
    """The projection's per-Gaussian records of one view, read from its geometry state."""
    import torch
    k = dict(means2D=_arr(R, "geometry", "means2D", geomB, P, 0, torch.float32, 2 * P).reshape(P, 2),
             conic_opacity=_arr(R, "geometry", "conic_opacity", geomB, P, 0, torch.float32, 4 * P).reshape(P, 4),
             rgbd=_arr(R, "geometry", "rgbd", geomB, P, 0, torch.float32, 4 * P).reshape(P, 4),
             cov3D=_arr(R, "geometry", "cov3D", geomB, P, 0, torch.float32, 6 * P).reshape(P, 6),
             depths=_arr(R, "geometry", "depths", geomB, P, 0, torch.float32, P),
             tiles_touched=_arr(R, "geometry", "tiles_touched", geomB, P, 0, torch.int32, P),
             clamped=_arr(R, "geometry", "clamped", geomB, P, 0, torch.uint8, P),
             extent=_arr(R, "geometry", "extent", geomB, P, 0, torch.float32, 2 * P).reshape(P, 2))
    k["rgb"] = k["rgbd"][:, :3]
    return k


def settings(cam, deg, aa=False):
    from manigaussian_b200 import rasterizer as R
    return R.GaussianRasterizationSettings(cam["H"], cam["W"], cam["tanfovx"], cam["tanfovy"], _t(np.zeros(3, np.float32)), 1.0,
                                           _t(cam["viewmatrix"]), _t(cam["projmatrix"]), deg, _t(cam["campos"]), False, False,
                                           False, antialiasing=aa)


def g_args(g):
    return dict(means3D=_t(g["means3D"]), colors=_t(g["colors_precomp"]), opacity=_t(g["opacities"]), scales=_t(g["scales"]),
                rotations=_t(g["rotations"]), cov3D_precomp=_t(g["cov3D_precomp"]), sh=_t(g["shs"]))


def mgs_backward_call(sc, fw, omit=(), prefill=np.nan, accumulate=0, seed=0):
    """mgs_backward through the C ABI on the single-view forward `fw`; every output prefilled with `prefill`, the outputs
    named in `omit` passed as NULL.  Returns numpy outputs (None where omitted)."""
    import torch
    from manigaussian_b200 import _binding
    g, cam = sc["g"], sc["cam"]
    P, W, H = len(g["means3D"]), cam["W"], cam["H"]
    M = 0 if g["shs"] is None else g["shs"].shape[1]
    shapes = dict(dL_dmean2D=(P, 3), dL_dconic=(P, 4), dL_dopacity=(P, 1), dL_dcolor=(P, 3), dL_dmean3D=(P, 3),
                  dL_dcov3D=(P, 6), dL_dsh=(P, max(M, 1), 3), dL_dscale=(P, 3), dL_drot=(P, 4))
    out = {k: (None if k in omit else torch.full(s, prefill, dtype=torch.float32, device="cuda")) for k, s in shapes.items()}
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    a = g_args(g)
    dpix = _t(np.random.default_rng(seed + 101).normal(0, 1, (3, H, W)).astype(np.float32))
    scratch = torch.empty((_binding.lib().mgs_backward_scratch_bytes(P),), dtype=torch.uint8, device="cuda")
    vm, pm, cp, bg = _t(cam["viewmatrix"]), _t(cam["projmatrix"]), _t(cam["campos"]), _t(np.zeros(3, np.float32))
    rc = _binding.lib().mgs_backward(
        P, int(g["sh_degree"]), M, 0, int(fw["R"]), bg.data_ptr(), W, H, a["means3D"].data_ptr(), ptr(a["sh"]) if M else None,
        ptr(a["colors"]) if g["colors_precomp"] is not None else None, None,
        ptr(a["scales"]) if g["scales"] is not None else None, float(sc.get("scale_modifier", 1.0)),
        ptr(a["rotations"]) if g["rotations"] is not None else None,
        ptr(a["cov3D_precomp"]) if g["cov3D_precomp"] is not None else None, vm.data_ptr(), pm.data_ptr(), cp.data_ptr(),
        float(cam["tanfovx"]), float(cam["tanfovy"]), fw["radii_t"].data_ptr(), fw["geomB"].data_ptr(), fw["binB"].data_ptr(),
        fw["imgB"].data_ptr(), dpix.data_ptr(), None, None, ptr(out["dL_dmean2D"]), ptr(out["dL_dconic"]),
        ptr(out["dL_dopacity"]), ptr(out["dL_dcolor"]), None, ptr(out["dL_dmean3D"]), ptr(out["dL_dcov3D"]),
        ptr(out["dL_dsh"]) if M else None, ptr(out["dL_dscale"]), ptr(out["dL_drot"]), scratch.data_ptr(), accumulate, 0,
        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0, _binding.last_error()
    res = {k: (None if v is None else v.cpu().numpy()) for k, v in out.items()}
    if not M:
        res["dL_dsh"] = None
    return res


def single_forward(sc):
    import torch
    from manigaussian_b200 import rasterizer as R
    g, cam = sc["g"], sc["cam"]
    a = g_args(g)
    P = len(g["means3D"])
    out = R.rasterize_gaussians_raw(_t(np.zeros(3, np.float32)), a["means3D"], a["colors"], torch.zeros((P, 3), device="cuda"),
                                    a["opacity"], a["scales"], a["rotations"], float(sc.get("scale_modifier", 1.0)),
                                    a["cov3D_precomp"], _t(cam["viewmatrix"]), _t(cam["projmatrix"]), cam["tanfovx"],
                                    cam["tanfovy"], cam["H"], cam["W"], a["sh"], g["sh_degree"], _t(cam["campos"]), False,
                                    False, False)
    torch.cuda.synchronize()
    Rn, _, _, radii, geomB, binB, imgB = out[:7]
    k = records(R, geomB, P)
    k.update(R=Rn, radii=radii.cpu().numpy(), radii_t=radii, geomB=geomB, binB=binB, imgB=imgB)
    return k


def _exact_cot(b):
    return dict(dL_dmean2D=b["dL_dmean2D"][:, :2], dL_dconic=b["dL_dconic"][:, [0, 1, 3]], dL_dopacity=b["dL_dopacity"][:, 0],
                dL_dcolor=b["dL_dcolor"], dL_ddepth=None)


def _bits(c):
    return c.astype(np.int64)


MEASURED = {}


def _record(name, rows):
    for k, v in rows.items():
        MEASURED[k] = max(MEASURED.get(k, 0.0), v)
    print(f"[{name}] " + " ".join(f"{k}={v:.3g}" for k, v in rows.items()))


def _bwd_names(b):
    return dict(dL_dmeans3D=b["dL_dmean3D"], dL_dcov3D=b["dL_dcov3D"], dL_dsh=b["dL_dsh"], dL_dscales=b["dL_dscale"],
                dL_drotations=b["dL_drot"], dL_dopacity=b["dL_dopacity"][:, 0], dL_dcolors=b["dL_dcolor"],
                dL_dmeans2D=b["dL_dmean2D"][None, :, :2])


SINGLE = ["clamp_x", "clamp_y", "near", "quat_scale", "quat_scale_1", "quat_scale_19", "sh0", "sh0_m16", "sh1", "sh1_m16",
          "sh2", "sh2_m16", "sh3", "sh3_m16", "precomp_cov", "precomp_sr", "ragged_f32", "sh3_big",
          "mg_real_f3"]


@pytest.mark.parametrize("scene", SINGLE)
def test_single_view_per_gaussian(scene):
    import test_project_ref64_cpu as CPU
    sc = SCENES[scene]()
    g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
    fw = single_forward(sc)
    b = mgs_backward_call(sc, fw)
    for k, v in b.items():
        assert v is None or not np.isnan(v).any(), f"{k}: {int(np.isnan(v).sum())} elements never written"
    ref = P64.forward(g, cam, mod)
    keep = ~ref["border"]
    rows = {}
    got = dict(fw, cov3D=fw["cov3D"] if g["scales"] is not None else None)
    problems = CPU.compare_forward(ref, got, keep, rows, "fwd")
    rb = P64.backward(g, [cam], [_exact_cot(b)], mod, live=[fw["radii"] > 0], clamped=[_bits(fw["clamped"])])
    problems += CPU.compare_backward(rb, _bwd_names(b), keep & ~rb["border"], rows, "bwd",
                                     names=CPU.BWD + ("dL_dopacity", "dL_dcolors"))
    # culled Gaussians: radius 0 and exactly zero gradient rows
    dead = fw["radii"] == 0
    for k in ("dL_dmean3D", "dL_dmean2D", "dL_dconic", "dL_dopacity", "dL_dcolor", "dL_dcov3D", "dL_dscale", "dL_drot", "dL_dsh"):
        if b[k] is not None and dead.any():
            assert not np.any(b[k][dead]), (k, "a culled Gaussian has a non-zero gradient row")
    _record(scene, rows)
    _assert_edge(sc, ref, fw)
    assert not problems, "\n".join(problems)


def _assert_edge(sc, ref, fw):
    e = sc.get("edge", ())
    live = fw["radii"] > 0
    if not e:
        return
    if e[0] == "clamp":
        out = ~(ref["inx"] if e[1] == 0 else ref["iny"])
        n = int((live & out & ~ref["border"]).sum())
        assert n >= e[2], f"only {n} on-screen Gaussians past the clamp on axis {e[1]}"
    elif e[0] == "near":
        z = ref["depth"]
        assert int((~live & (z <= P64.NEAR_Z)).sum()) == 8 and int((live & (z < 0.26)).sum()) >= 4, (z, fw["radii"])
    elif e[0] == "quat":
        n = np.linalg.norm(sc["g"]["rotations"].astype(np.float64), axis=1)
        for qn in P64_QNORMS:
            assert np.any(live & np.isclose(n, qn, rtol=1e-3)), qn
        a0, b, c0, _ = P64.screen_covariance(sc["g"], sc["cam"], sc.get("scale_modifier", 1.0))
        lmin = 0.5 * (a0 + c0) - np.sqrt(0.25 * (a0 - c0) ** 2 + b * b)
        n = int((live & ~ref["border"] & (lmin < 0.03)).sum())
        assert n >= 8, f"only {n} needles where the dilation dominates"
    elif e[0] == "aa":
        a0, b, c0, det = P64.screen_covariance(sc["g"], sc["cam"], sc.get("scale_modifier", 1.0))
        r = (a0 * c0 - b * b) / det
        ok = live & ~ref["border"]
        lo, hi = int((ok & (r < P64.AA_CLAMP)).sum()), int((ok & (r > P64.AA_CLAMP)).sum())
        assert lo >= 4 and hi >= 4, f"{lo} live Gaussians below the 2.5e-5 clamp, {hi} above"
    elif e[0] == "sh":
        bits = fw["clamped"][live]
        share = np.unpackbits(bits[:, None], axis=1)[:, -3:].mean()
        assert 0.25 <= share <= 0.75, share


P64_QNORMS = QNORMS


@pytest.mark.parametrize("scene", ["aa1", "aa2", "aa3"])
def test_antialiased_view_per_gaussian(scene):
    """The anti-aliased projection (one view through mgs_forward_views / mgs_backward_views with antialiasing = 1, depth cotangents on):
    every record, o_eff included, against project_ref64.forward(antialias=True), and every per-Gaussian output against the
    AA chain fed blend_ref64's cotangents, on needles both sides of the 2.5e-5 clamp."""
    import test_project_ref64_cpu as CPU
    sc = SCENES[scene]()
    g, cam = sc["g"], sc["cam"]
    recs, cots, got, _ = run_views(g, [cam], aa=True, seed=7)
    ref = P64.forward(g, cam, antialias=True)
    rows = {}
    problems = CPU.compare_forward(ref, recs[0], ~ref["border"], rows, "fwd")
    problems += check_sums(scene, g, [cam], recs, cots, got, True, True)
    _record(scene, rows)
    _assert_edge(sc, ref, recs[0])
    assert not problems, "\n".join(problems)


# --------------------------------------------------------------------------- several views / clouds, blend_ref64 cotangents
def view_cotangents(R, o, P, cam, ct_color, ct_depth):
    """One view of a multi-view forward: its records, and the blend-stage cotangents blend_ref64 computes from our records
    and pixel masks, with their bounds (KAPPA u B of blend_ref64)."""
    import torch
    W, H = cam["W"], cam["H"]
    geomB, binB, imgB = o[4], o[5], o[6]
    Rn, cap = o.num_rendered(), int(o[0])
    assert not o.overflowed()
    T = ((W + 15) // 16) * ((H + 15) // 16)
    S = (cap + 11) & ~3
    k = records(R, geomB, P)
    k["radii"] = o[3].cpu().numpy()
    st = dict(W=W, H=H, ranges=_arr(R, "image", "ranges", imgB, W, H, torch.int32, 2 * T).view(np.uint32).reshape(T, 2),
              point_list=_arr(R, "binning", "point_list", binB, cap, 0, torch.int32, Rn).view(np.uint32),
              means2D=k["means2D"], conic_opacity=k["conic_opacity"], colors=k["rgbd"][:, :3], depth=k["rgbd"][:, 3],
              feature=None, bg=np.zeros(3, np.float32), g_color=ct_color, g_feature=None, g_depth=ct_depth, g_alpha=None)
    bl = _arr(R, "binning", "block_lists", binB, cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    pmk = _arr(R, "binning", "pixel_masks", binB, cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    nw = _arr(R, "image", "block_nwalk", imgB, W, H, torch.int32, 8 * T).view(np.uint32).reshape(T, 8)
    ref = B64.blend(st, B64.masks_from_blocks(st, bl, pmk, nw))
    kb = lambda q: B64.KAPPA[q] * B64.U * ref[q + "_B"]  # noqa: E731
    cot = dict(dL_dmean2D=ref["dL_dmeans2D"], dL_dmean2D_B=kb("dL_dmeans2D"), dL_dconic=ref["dL_dconic"],
               dL_dconic_B=kb("dL_dconic"), dL_dopacity=ref["dL_dopacity"], dL_dopacity_B=kb("dL_dopacity"),
               dL_dcolor=ref["dL_dcolors"], dL_dcolor_B=kb("dL_dcolors"), dL_ddepth=ref["dL_ddepth"],
               dL_ddepth_B=kb("dL_ddepth"))
    return k, cot


def run_views(g, cams, aa=False, shared=True, accumulate=False, mod=1.0, seed=0):
    import torch
    from manigaussian_b200 import rasterizer as R
    deg = int(g["sh_degree"])
    views = [settings(c, deg, aa) for c in cams]
    a = g_args(g)
    outs, streams = R.rasterize_views_raw(views, a["means3D"], a["colors"], None, a["opacity"], a["scales"], a["rotations"], mod,
                                          a["cov3D_precomp"], a["sh"], deg, False, return_depth=True, antialiasing=aa)
    torch.cuda.synchronize()
    P = len(g["means3D"])
    rng = np.random.default_rng(seed + 5)
    gc = [rng.normal(0, 1, (3, c["H"], c["W"])).astype(np.float32) for c in cams]
    gd = [rng.normal(0, 1, (c["H"], c["W"])).astype(np.float32) for c in cams]
    recs, cots = [], []
    for v, c in enumerate(cams):
        k, cot = view_cotangents(R, outs[v], P, c, gc[v], gd[v])
        recs.append(k)
        cots.append(cot)
    seedbuf = None
    acc = None
    M = 0 if g["shs"] is None else g["shs"].shape[1]
    if accumulate:
        seedbuf = dict(dL_dmeans3D=rng.normal(0, 1, (P, 3)), dL_dmeans2D=rng.normal(0, 1, (P, 3)), dL_dopacity=rng.normal(0, 1, (P, 1)),
                       dL_dscales=rng.normal(0, 1, (P, 3)), dL_drotations=rng.normal(0, 1, (P, 4)),
                       dL_dsh=rng.normal(0, 1, (P, M, 3)) if M else None)
        seedbuf = {k: (None if v is None else v.astype(np.float32)) for k, v in seedbuf.items()}
        acc = {k: (None if v is None else _t(v)) for k, v in seedbuf.items()}
    m2 = None if shared else torch.full((len(cams), P, 3), np.nan, device="cuda")
    if accumulate and not shared:
        # per-view rows belong to their view: written, not added to, whatever `accumulate` says
        seedbuf.pop("dL_dmeans2D")
    grads = R.rasterize_views_backward_raw(views, outs, streams, [_t(x) for x in gc], None, a["means3D"], a["colors"], None,
                                           a["scales"], a["rotations"], mod, a["cov3D_precomp"], a["sh"], deg, False,
                                           grads_depth=[_t(x) for x in gd], accumulate_into=acc, means2D_per_view=m2,
                                           accumulate=accumulate, antialiasing=aa)
    torch.cuda.synchronize()
    names = ("dL_dmeans2D", "dL_dcolors", "dL_dfeature", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
             "dL_drotations")
    got = {n: (None if t is None else t.cpu().numpy()) for n, t in zip(names, grads)}
    return recs, cots, got, seedbuf


def check_sums(name, g, cams, recs, cots, got, aa, shared, mod=1.0, seedbuf=None):
    import test_project_ref64_cpu as CPU
    rb = P64.backward(g, cams, cots, mod, antialias=aa, live=[k["radii"] > 0 for k in recs],
                      clamped=[_bits(k["clamped"]) for k in recs], shared_mean2D=shared)
    keep = ~rb["border"]
    cmp = dict(got)
    m2 = np.asarray(cmp.pop("dL_dmeans2D"))
    cmp["dL_dmeans2D"] = (m2[None] if shared else m2)[..., :2]
    cmp["dL_dopacity"] = cmp["dL_dopacity"][:, 0]
    if seedbuf is not None:   # accumulate: the kernels added onto the seeded buffers
        for k, v in seedbuf.items():
            if v is None:
                continue
            x = (v[None, :, :2] if k == "dL_dmeans2D" else v).reshape(cmp[k].shape).astype(np.float64)
            cmp[k] = cmp[k] - x
            # each launch (16 views at most) adds its partial sum onto the buffer in fp32: u |seed + sum| per launch
            val, e, d = rb[k]
            rb[k] = (val, e, d + -(-len(cams) // 16) * P64.U * (np.abs(x) + np.abs(val)))
    rows = {}
    names = ("dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations", "dL_dopacity", "dL_dcolors", "dL_dmeans2D")
    # dL_dmeans2D is [V,P,2]: keep applies along P
    problems = CPU.compare_backward(rb, {k: v for k, v in cmp.items() if k != "dL_dmeans2D"}, keep, rows, "sum", names=names[:-1])
    v, e, d = rb["dL_dmeans2D"]
    x = cmp["dL_dmeans2D"]
    r = np.maximum(np.abs(x - v) - d, 0.0)[:, keep] / (P64.U * e[:, keep] + 1e-30)
    rows["sum dL_dmeans2D"] = float(r.max()) if r.size else 0.0
    if r.size and r.max() > P64.KAPPA["dL_dmeans2D"]:
        problems.append(f"dL_dmeans2D: {int((r > P64.KAPPA['dL_dmeans2D']).sum())} out of bound, worst {r.max():.3g}")
    for kk, vv in got.items():
        if vv is not None:
            assert not np.isnan(vv).any(), (kk, "elements never written")
    _record(name, rows)
    return problems


def _cloud_g(P, deg, seed, precomp=False):
    g = scenes.make_gaussians(P, sh_degree=deg, seed=seed, precomp_colors=precomp)
    g["cov3D_precomp"] = None
    g["shs"] = g["shs"] if not precomp else None
    # un-normalised quaternions and clamped channels in every cloud
    g["rotations"] = (g["rotations"] * np.random.default_rng(seed).uniform(0.3, 3.0, (P, 1))).astype(np.float32)
    if g["shs"] is not None:
        g["shs"][:, 0, :] -= 1.2
    return g


VIEW_CASES = [(1, True, False, False, 1), (4, True, False, True, 1), (16, False, False, False, 2), (17, True, True, False, 3),
              (17, False, False, True, 3), (33, True, False, False, 1), (33, False, True, True, 2), (4, True, False, False, 0)]


@pytest.mark.parametrize("V,shared,accumulate,aa,deg", VIEW_CASES,
                         ids=[f"V{v}-{'shared' if s else 'per_view'}-{'acc' if a else 'write'}-{'aa' if x else 'noaa'}-deg{d}"
                              for v, s, a, x, d in VIEW_CASES])
def test_views_sum_over_views(V, shared, accumulate, aa, deg):
    """rasterize_views_backward_raw (mgs_backward_views) over V views of one cloud, depth cotangents on, against the float64
    sum over views of the chain fed blend_ref64's cotangents."""
    W, H = 32, 24
    g = _cloud_g(160, deg, 90 + V + deg)
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    recs, cots, got, sb = run_views(g, cams, aa, shared, accumulate, seed=V)
    problems = check_sums(f"views V={V}", g, cams, recs, cots, got, aa, shared, seedbuf=sb)
    assert not problems, "\n".join(problems)


CLOUD_CASES = [("20x2", [2] * 20, 1, False), ("1x17", [17], 1, True), ("deg2", [3, 2], 2, False), ("deg3", [2, 3], 3, True),
               ("deg2_aa", [2, 2], 2, True), ("deg3_noaa", [3], 3, False), ("deg1_aa", [2], 1, True), ("precomp", [2, 2], 0, False)]


@pytest.mark.parametrize("name,nv,deg,aa", CLOUD_CASES, ids=[c[0] for c in CLOUD_CASES])
def test_clouds_sum_over_views(name, nv, deg, aa):
    """rasterize_clouds_backward_raw (mgs_backward_clouds): every cloud's sums over its own views."""
    import torch
    from manigaussian_b200 import rasterizer as R
    W, H = 32, 24
    clouds, gs, camss = [], [], []
    for b, n in enumerate(nv):
        g = _cloud_g(120 + 7 * b, deg, 200 + b, precomp=(name == "precomp"))
        cams = [scenes.make_camera(W, H, v + b, n + b) for v in range(n)]
        a = g_args(g)
        clouds.append(dict(views=[settings(c, deg, aa) for c in cams], means3D=a["means3D"], sh=a["sh"], colors=a["colors"],
                           opacity=a["opacity"], scales=a["scales"], rotations=a["rotations"], cov3D_precomp=a["cov3D_precomp"]))
        gs.append(g)
        camss.append(cams)
    outs, streams = R.rasterize_clouds_raw(clouds, deg, False, return_depth=True, antialiasing=aa)
    torch.cuda.synchronize()
    rng = np.random.default_rng(len(nv))
    problems = []
    per = []
    for b, c in enumerate(clouds):
        P = len(gs[b]["means3D"])
        gc = [rng.normal(0, 1, (3, H, W)).astype(np.float32) for _ in camss[b]]
        gd = [rng.normal(0, 1, (H, W)).astype(np.float32) for _ in camss[b]]
        rc = [view_cotangents(R, outs[b][v], P, cam, gc[v], gd[v]) for v, cam in enumerate(camss[b])]
        per.append(rc)
        c["grad_color"] = _t(np.stack(gc))
        c["grad_depth"] = _t(np.stack(gd))
    grads = R.rasterize_clouds_backward_raw(clouds, outs, streams, deg, False, antialiasing=aa)
    torch.cuda.synchronize()
    for b, gr in enumerate(grads):
        got = {k: (None if v is None else v.cpu().numpy()) for k, v in gr.items()}
        got.pop("dL_dfeature", None)
        problems += check_sums(f"clouds {name} #{b}", gs[b], camss[b], [r[0] for r in per[b]], [r[1] for r in per[b]], got, aa,
                               False)
    assert not problems, "\n".join(problems)


# --------------------------------------------------------------------------- coverage of the 12 instantiations
# (kernel, NSH, AA) -> the case above whose configuration runs it.  The launchers dispatch on the SH degree (<= 1 -> 12,
# 2 -> 27, 3 -> 48) and AA only; the coverage test launches each case's configuration (entry point, degree, AA, view and
# cloud counts) at a smaller P under the profiler and checks the kernel it names.
INSTANTIATIONS = {
    ("views", 12, False): "test_single_view_per_gaussian[sh1]",
    ("views", 27, False): "test_single_view_per_gaussian[sh2]",
    ("views", 48, False): "test_single_view_per_gaussian[sh3]",
    ("views", 12, True): "test_views_sum_over_views[V4-shared-write-aa-deg1]",
    ("views", 27, True): "test_views_sum_over_views[V33-per_view-acc-aa-deg2]",
    ("views", 48, True): "test_views_sum_over_views[V17-per_view-write-aa-deg3]",
    ("clouds", 12, False): "test_clouds_sum_over_views[20x2]",
    ("clouds", 27, False): "test_clouds_sum_over_views[deg2]",
    ("clouds", 48, False): "test_clouds_sum_over_views[deg3_noaa]",
    ("clouds", 12, True): "test_clouds_sum_over_views[1x17]",
    ("clouds", 27, True): "test_clouds_sum_over_views[deg2_aa]",
    ("clouds", 48, True): "test_clouds_sum_over_views[deg3]",
}


def _launched(fn, attempts=3):
    """Demangled names of the project_bwd kernels `fn` launches (torch.profiler, CUDA activities).

    CUPTI hands kernel records to the profiler asynchronously, and a trace can come back without its last records -- here
    the project_bwd kernel, which ends the backward.  So once `fn`'s work has completed, a marker kernel (a one-pixel
    mgs_loss_heads) runs inside the same window: a trace that holds the marker holds everything that completed before it.
    A trace without the marker is incomplete and the capture is repeated; one with it is taken as it is."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from manigaussian_b200 import _binding as B
    buf = torch.zeros(16, device="cuda")
    p = [buf[i:].data_ptr() for i in range(0, 16, 4)]
    for _ in range(attempts):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
            B.check(B.lib().mgs_loss_heads(1, 0, 1, p[0], None, p[1], None, p[2], None, p[3],
                                           torch.cuda.current_stream().cuda_stream), "mgs_loss_heads")
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        if any("loss_heads_kernel" in n for n in names):
            break
    return {n for n in names if "project_bwd" in n}


def _case_runner(case):
    name, arg = case.split("[")
    arg = arg[:-1]
    if name == "test_single_view_per_gaussian":
        sc = SCENES[arg]()
        fw = single_forward(sc)
        return lambda: mgs_backward_call(sc, fw)
    if name == "test_views_sum_over_views":
        V, shared, accumulate, aa, deg = next(c for c in VIEW_CASES if f"V{c[0]}-{'shared' if c[1] else 'per_view'}-"
                                              f"{'acc' if c[2] else 'write'}-{'aa' if c[3] else 'noaa'}-deg{c[4]}" == arg)
        g = _cloud_g(64, deg, 7)
        cams = [scenes.make_camera(32, 24, v, V) for v in range(V)]
        return lambda: run_views(g, cams, aa, shared, accumulate)
    nm, nv, deg, aa = next(c for c in CLOUD_CASES if c[0] == arg)

    def run():
        import torch
        from manigaussian_b200 import rasterizer as R
        clouds = []
        for b, n in enumerate(nv):
            a = g_args(_cloud_g(64, deg, 300 + b))
            cams = [scenes.make_camera(32, 24, v, n) for v in range(n)]
            clouds.append(dict(views=[settings(c, deg, aa) for c in cams], means3D=a["means3D"], sh=a["sh"], colors=a["colors"],
                               opacity=a["opacity"], scales=a["scales"], rotations=a["rotations"], cov3D_precomp=None,
                               grad_color=torch.ones((n, 3, 24, 32), device="cuda")))
        outs, streams = R.rasterize_clouds_raw(clouds, deg, False, antialiasing=aa)
        R.rasterize_clouds_backward_raw(clouds, outs, streams, deg, False, antialiasing=aa)
    return run


def test_every_project_bwd_instantiation_is_run():
    """Each of the 12 instantiations is launched by the configuration of the case the table names (checked on the launch)."""
    assert len(INSTANTIATIONS) == 12
    missing = []
    for (kind, nsh, aa), case in INSTANTIATIONS.items():
        names = _launched(_case_runner(case))
        want = [n for n in names if f"project_bwd_{kind}_kernel<{nsh}," in n and (", true>" in n) == aa]
        if not want:
            missing.append(((kind, nsh, aa), case, sorted(names)))
    assert not missing, missing


# --------------------------------------------------------------------------- output contract of mgs_backward
NULLABLE = ("dL_dconic", "dL_dcolor", "dL_dcov3D", "dL_dsh", "dL_dscale", "dL_drot")


@pytest.mark.parametrize("scene", ["near", "precomp_cov", "sh2"])
def test_mgs_backward_writes_every_output_it_is_given(scene):
    """With each nullable output NULL in turn (the rest prefilled with NaN), every output given is fully written and
    within the float64 bounds of the all-outputs call: dL_dconic rows of culled Gaussians are zeros, dL_dmean3D keeps its SH
    view-direction term without dL_dsh, dL_dscale / dL_drot are written on their own and are zeros with cov3D_precomp."""
    import test_project_ref64_cpu as CPU
    sc = SCENES[scene]()
    g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
    fw = single_forward(sc)
    full = mgs_backward_call(sc, fw)
    problems = []
    for omit in NULLABLE:
        b = mgs_backward_call(sc, fw, omit={omit})
        for k, v in b.items():
            if v is not None and np.isnan(v).any():
                problems.append(f"{omit} NULL: {k} has {int(np.isnan(v).sum())} elements never written")
        if omit in ("dL_dconic", "dL_dcolor"):
            # the chain's input is not returned: compare with the all-outputs call (the blend's atomics reorder sums)
            for k in ("dL_dmean3D", "dL_dcov3D", "dL_dsh", "dL_dscale", "dL_drot"):
                if b[k] is not None and not np.allclose(b[k], full[k], rtol=1e-4, atol=1e-5 * np.abs(full[k]).max()):
                    problems.append(f"{omit} NULL: {k} differs from the all-outputs call")
            continue
        # every other call returns its own blend-stage cotangents: its outputs against the float64 chain on them
        rb = P64.backward(g, [cam], [_exact_cot(b)], mod, live=[fw["radii"] > 0], clamped=[_bits(fw["clamped"])])
        problems += CPU.compare_backward(rb, _bwd_names(b), ~rb["border"], {}, f"{omit} NULL:",
                                         names=CPU.BWD + ("dL_dopacity", "dL_dcolors"))
    dead = fw["radii"] == 0
    if dead.any():
        assert np.all(full["dL_dconic"][dead] == 0)
    if g["scales"] is None:
        assert np.all(full["dL_dscale"] == 0) and np.all(full["dL_drot"] == 0)
    assert not problems, "\n".join(problems)


VIEWS_NULLABLE = ("dL_dcolor", "dL_dcov3D", "dL_dsh", "dL_dscale", "dL_drot")


@pytest.mark.parametrize("scene", ["near", "precomp_cov", "sh2"])
def test_backward_views_call_writes_every_output_it_is_given(scene):
    """mgs_backward_views over two views (shared dL_dmean2D), each nullable output NULL in turn and every other output
    prefilled with NaN: every output given is fully written and equals the all-outputs call up to the reordering of the
    blend's atomic sums.  dL_dmean3D keeps its SH view-direction term without dL_dsh, dL_dscale / dL_drot are written on
    their own, and are zeros with cov3D_precomp."""
    import torch
    from manigaussian_b200 import _binding, rasterizer as R
    sc = SCENES[scene]()
    g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
    cams = [cam, scenes.make_camera(cam["W"], cam["H"], 0, 4)]
    deg = int(g["sh_degree"])
    views = [settings(c, deg) for c in cams]
    a = g_args(g)
    outs, streams = R.rasterize_views_raw(views, a["means3D"], a["colors"], None, a["opacity"], a["scales"], a["rotations"], mod,
                                          a["cov3D_precomp"], a["sh"], deg, False)
    torch.cuda.synchronize()
    L = _binding.lib()
    P = len(g["means3D"])
    M = 0 if g["shs"] is None else g["shs"].shape[1]
    rng = np.random.default_rng(13)
    gc = [_t(rng.normal(0, 1, (3, c["H"], c["W"])).astype(np.float32)) for c in cams]
    shapes = dict(dL_dmean2D=(P, 3), dL_dmean3D=(P, 3), dL_dopacity=(P, 1), dL_dcolor=(P, 3), dL_dcov3D=(P, 6),
                  dL_dsh=(P, max(M, 1), 3), dL_dscale=(P, 3), dL_drot=(P, 4))
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731

    def call(omit=()):
        out = {k: (None if k in omit else torch.full(s, np.nan, dtype=torch.float32, device="cuda")) for k, s in shapes.items()}
        arr = (_binding.View * len(views))()
        keep = []
        for v, s in enumerate(views):
            keep.append(R._backward_view(L, arr[v], s, outs[v], torch.device("cuda"), P, gc[v], None, None))
            arr[v].dL_dmean2D = ptr(out["dL_dmean2D"])
            arr[v].stream = streams[v].cuda_stream
        rc = L.mgs_backward_views(len(views), arr, None, P, deg, M, 0, ptr(a["means3D"]), ptr(a["sh"]) if M else None,
                                  ptr(a["colors"]) if g["colors_precomp"] is not None else None, None,
                                  ptr(a["scales"]) if g["scales"] is not None else None, float(mod),
                                  ptr(a["rotations"]) if g["rotations"] is not None else None,
                                  ptr(a["cov3D_precomp"]) if g["cov3D_precomp"] is not None else None,
                                  ptr(out["dL_dmean3D"]), ptr(out["dL_dopacity"]), ptr(out["dL_dcolor"]), None,
                                  ptr(out["dL_dcov3D"]), ptr(out["dL_dsh"]) if M else None, ptr(out["dL_dscale"]),
                                  ptr(out["dL_drot"]), 1, 0, 3, 0, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert rc == 0, _binding.last_error()
        res = {k: (None if v is None else v.cpu().numpy()) for k, v in out.items()}
        if not M:
            res["dL_dsh"] = None
        return res

    full = call()
    problems = []
    for omit in VIEWS_NULLABLE:
        b = call({omit})
        for k, v in b.items():
            if v is None:
                continue
            if np.isnan(v).any():
                problems.append(f"{omit} NULL: {k} has {int(np.isnan(v).sum())} elements never written")
            elif not np.allclose(v, full[k], rtol=1e-4, atol=1e-5 * np.abs(full[k]).max()):
                problems.append(f"{omit} NULL: {k} differs from the all-outputs call")
    if g["scales"] is None:
        assert np.all(full["dL_dscale"] == 0) and np.all(full["dL_drot"] == 0)
    assert not np.isnan(np.concatenate([v.ravel() for v in full.values() if v is not None])).any()
    assert not problems, "\n".join(problems)
