"""Camera gradients without a GPU: the differentiable camera builder and the C ABI's argument checks.

* cameras.camera_batch(w2c, intr, ...) builds the same matrices as build_cameras on the golden calibrations (2e-6
  relative, as build_cameras is held to the reference), and its matrices are differentiable in w2c (float64 gradcheck).
* The camera-gradient symbols are exported, and their argument errors return MGS_ERR_INVALID_ARG before anything is
  enqueued.
* tests/camera_ref64.py, the float64 camera chain, matches torch float64 autograd of an independent restatement of the
  projection with the camera as leaves to 1e-9 relative (clamp x / y, near, quat_scale, SH degrees 0-3 with M = 16,
  precomp_cov, AA at degrees 1 and 3), and each of its mutations (the J term dropped, the t p outer product transposed,
  the depth cotangent left out, the campos sign flipped, the pm[4c + 3] term dropped, the true d/dt.z at the clamp)
  moves a checked element past twice its bound.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding, cameras

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "cameras.npz"))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.parametrize("name", ["square128", "wide"])
def test_camera_batch_matches_build_cameras(name):
    W, H = (int(x) for x in GOLD[f"{name}_WH"])
    intr, extr = GOLD[f"{name}_intr"], GOLD[f"{name}_extr"]
    ref = cameras.build_cameras(torch.from_numpy(intr), torch.from_numpy(extr), W, H)
    w2c = torch.from_numpy(np.linalg.inv(extr.astype(np.float64))).float()
    cb = cameras.camera_batch(w2c, intr, W, H)
    assert cb.FovX == ref.FovX and cb.FovY == ref.FovY and cb.tanfovx == ref.tanfovx
    for f in ("world_view_transform", "full_proj_transform", "camera_center"):
        assert rel(getattr(cb, f).numpy(), getattr(ref, f).numpy()) < 2e-6, f


def test_camera_batch_is_differentiable_in_w2c():
    intr = GOLD["wide_intr"][:2]
    w2c = torch.from_numpy(np.linalg.inv(GOLD["wide_extr"][:2].astype(np.float64))).requires_grad_()

    def f(m):
        cb = cameras.camera_batch(m, intr, 160, 120)
        return cb.world_view_transform, cb.full_proj_transform, cb.camera_center

    assert torch.autograd.gradcheck(f, (w2c,))
    cb = cameras.camera_batch(w2c, intr, 160, 120)
    assert cb.world_view_transform.requires_grad and cb.camera_center.requires_grad


def test_camera_option_checks_its_arguments():
    L = _binding.lib()
    assert hasattr(L, "mgs_camera_grad_scratch_bytes") and "mgs_camera_grad_scratch_bytes" in _binding.EXPORTED_SYMBOLS
    assert L.mgs_camera_grad_scratch_bytes(1) == 27 * 4
    assert L.mgs_camera_grad_scratch_bytes(16384) == 128 * 27 * 4
    assert L.mgs_camera_grad_scratch_bytes(16385) == 129 * 27 * 4
    views = (_binding.View * 1)()
    v = views[0]
    v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
    for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                 "radii", "dL_dpix", "blend_scratch"):
        setattr(v, name, 4096)
    v.binning_capacity = 1
    cam = (_binding.ViewCameraGrad * 1)()
    cam[0].dL_dviewmatrix = 4096   # an output without scratch
    cam = _binding.RenderOptions(camera_grad=cam)
    rc = L.mgs_backward_views(1, views, cam, 4, 0, 0, 0, 4096, None, 4096, None, None, 1.0, None, 4096,
                              4096, 4096, None, None, None, None, None, None, 0, 0, 3, 0, None)
    assert rc == -1 and "scratch" in _binding.last_error()
    clouds = (_binding.Cloud * 1)()
    c = clouds[0]
    c.P, c.means3D, c.colors_precomp, c.dL_dmean3D, c.dL_dopacity = 4, 4096, 4096, 4096, 4096
    offs = (ctypes.c_int * 2)(0, 1)
    rc = L.mgs_backward_clouds(1, clouds, offs, views, cam, 0, 0, 0, 1.0, 0, 0, None)
    assert rc == -1 and "scratch" in _binding.last_error()


# --------------------------------------------------------------------------- the float64 camera chain (camera_ref64)
def _torch_loss_cam(g, cam, cot, mod, aa):
    """test_project_ref64_cpu._torch_loss restated with the camera as leaves: vm [16], pm [16] and campos [3] in the ABI's
    layout.  The reference's quirks as `detach`, as there: outside the frustum clamp t.x_c = (+-lim t.z).detach(), the
    quaternion un-normalised, 2 gB on the conic's b, w = 1 / (det^2 + 1e-7), the SH clamp a relu.  tan_fov and the focal
    lengths are constants."""
    import project_ref64 as P64
    d = torch.float64
    T = lambda a: torch.tensor(np.asarray(a, np.float32).astype(np.float64), dtype=d)  # noqa: E731
    p = T(g["means3D"])
    vm16 = T(np.asarray(cam["viewmatrix"]).reshape(-1)).requires_grad_()
    pm16 = T(np.asarray(cam["projmatrix"]).reshape(-1)).requires_grad_()
    cp = T(np.asarray(cam["campos"]).reshape(-1)).requires_grad_()
    leaves = dict(dL_dviewmatrix=vm16, dL_dprojmatrix=pm16, dL_dcampos=cp)
    if g.get("scales") is not None:
        se = T(g["scales"]) * float(np.float32(mod))
        q = T(g["rotations"])
        r, x, y, z = q.unbind(1)
        Rq = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                          2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                          2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
        Sig = Rq @ torch.diag_embed(se * se) @ Rq.transpose(1, 2)
    else:
        c6 = T(g["cov3D_precomp"])
        Sig = torch.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], 1)
    o = T(g["opacities"]).reshape(-1)
    vm = vm16.reshape(4, 4).T
    pm = pm16.reshape(4, 4).T
    t = p @ vm[:3, :3].T + vm[:3, 3]
    vw = P64.view_of(cam)
    fx, fy, lx, ly = vw["fx"], vw["fy"], vw["limx"], vw["limy"]
    tz = t[:, 2]
    ux, uy = t[:, 0] / tz, t[:, 1] / tz
    cx = torch.where((ux >= -lx) & (ux <= lx), t[:, 0], (ux.clamp(-lx, lx) * tz).detach())
    cy = torch.where((uy >= -ly) & (uy <= ly), t[:, 1], (uy.clamp(-ly, ly) * tz).detach())
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * cx / tz ** 2], 1), torch.stack([zero, fy / tz, -fy * cy / tz ** 2], 1)], 1)
    Mx = J @ vm[:3, :3]
    cov = Mx @ Sig @ Mx.transpose(1, 2)
    h = float(np.float32(0.3))
    a, b, c = cov[:, 0, 0] + h, cov[:, 0, 1], cov[:, 1, 1] + h
    det = a * c - b * b
    k = (det * det / (det * det + float(np.float32(1e-7)))).detach()
    sc = lambda x: x.detach() + (x - x.detach()) * k  # noqa: E731
    hom = torch.cat([p, torch.ones_like(tz)[:, None]], 1) @ pm.T
    ndc = hom[:, :2] / (hom[:, 3:4] + float(np.float32(1e-7)))
    C_ = lambda k: torch.tensor(np.asarray(cot[k], np.float64), dtype=d)  # noqa: E731
    gco = C_("dL_dconic")
    loss = (ndc * C_("dL_dmean2D")).sum() + (sc(c / det) * gco[:, 0] + 2 * sc(-b / det) * gco[:, 1] + sc(a / det) * gco[:, 2]).sum()
    oe = o
    if aa:
        rr = (cov[:, 0, 0] * cov[:, 1, 1] - b * b) / det
        oe = o * torch.sqrt(rr.clamp_min(P64.AA_CLAMP))
    loss = loss + (oe * C_("dL_dopacity")).sum()
    if cot.get("dL_ddepth") is not None:
        loss = loss + (tz * C_("dL_ddepth")).sum()
    if g.get("shs") is not None:
        sh = T(g["shs"])
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
    return loss, leaves


def _scene(name):
    import test_project_ref64_gpu as S
    return S.SCENES[name]()


CAM_AUTOGRAD = [("clamp_x", False), ("clamp_y", False), ("near", False), ("quat_scale", False), ("sh0_m16", False),
                ("sh1_m16", False), ("sh2_m16", False), ("sh3_m16", False), ("precomp_cov", False), ("aa1", True), ("aa3", True)]


@pytest.mark.parametrize("scene,aa", CAM_AUTOGRAD, ids=[s for s, _ in CAM_AUTOGRAD])
def test_camera_chain_matches_torch_float64_autograd(scene, aa):
    import camera_ref64 as C64
    import project_ref64 as P64
    import test_project_ref64_cpu as CPU
    sc = _scene(scene)
    g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
    ref = P64.forward(g, cam, mod, antialias=aa)
    live = ~ref["culled"]
    sel = {k: (v[live] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(live) else v) for k, v in g.items()}
    cot = CPU.seeded_cotangents(int(live.sum()), 3, depth=True)
    rc = C64.camera_grads(sel, [cam], [cot], mod, antialias=aa)[0]
    loss, leaves = _torch_loss_cam(sel, cam, cot, mod, aa)
    loss.backward()
    for name, leaf in leaves.items():
        want = leaf.grad.numpy() if leaf.grad is not None else np.zeros(leaf.shape)   # degree 0: no view direction
        got, e, _ = rc[name]
        tol = 1e-9 * np.abs(want).max() + 16 * 2.0 ** -53 * e
        assert np.all(np.abs(got - want) <= tol), (name, np.abs(got - want).max(), np.abs(want).max())
    if g.get("shs") is not None and int(g["sh_degree"]) > 0:
        assert np.abs(rc["dL_dcampos"][0]).max() > 0
    else:
        assert not rc["dL_dcampos"][0].any()


def test_every_camera_mutation_moves_a_checked_element_past_twice_its_bound():
    import camera_ref64 as C64
    import project_ref64 as P64
    import test_project_ref64_cpu as CPU
    scenes = ("clamp_x", "clamp_y", "near", "sh1", "quat_scale")
    base, moved = {}, {m: 0.0 for m in C64.CAM_MUTATIONS}
    for name in scenes:
        sc = _scene(name)
        g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
        fw = P64.forward(g, cam, mod)
        cot = CPU.seeded_cotangents(len(g["means3D"]), 4, depth=True)
        ref = C64.camera_grads(g, [cam], [cot], mod)[0]
        base[name] = ref
        for m in C64.CAM_MUTATIONS:
            mut = C64.camera_grads(g, [cam], [cot], mod, mutate={m})[0]
            for q in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos"):
                v, e, d = ref[q]
                r = np.abs(mut[q][0] - v) / (C64.KAPPA_CAM * (P64.U * e + d) + 1e-30)
                moved[m] = max(moved[m], float(r.max()))
        del fw
    assert all(r > 2.0 for r in moved.values()), moved
