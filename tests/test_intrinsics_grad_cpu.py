"""Learnable intrinsics without a GPU: the float64 focal-length chain, the differentiable camera builder and the C ABI.

* tests/intrinsics_ref64.py, the float64 chain of dL/dtan_fov, matches torch float64 autograd of an independent restatement
  of the projection with {tan_fovx, tan_fovy} as leaves to 1e-9 relative, on the projection edge scenes: Gaussians clamped
  on each side of both axes, SH degrees 0-3, and anti-aliased needles on both sides of the 2.5e-5 clamp.  Each of its
  mutations (the clamp term dropped, the unclamped t in J, H without the AA compensation, dL/dfx in place of dL/dtan_fov)
  moves an entry past twice its bound.
* cameras.camera_batch with an intr that requires grad builds the matrices of build_cameras (float32 rounding), a [B,2]
  device-side tan_fov, and passes a float64 gradcheck from intr and w2c to all four camera tensors.
* The argument errors of the intrinsics option return MGS_ERR_INVALID_ARG before anything is enqueued.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding, cameras

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "cameras.npz"))


def _scene(name):
    import test_project_ref64_gpu as S
    return S.SCENES[name]()


def _torch_loss_intr(g, cam, cot, mod, aa):
    """The conic and (AA) opacity terms of the blend-stage loss, with tan_fovx / tan_fovy as float64 leaves: fx = W / (2 tan)
    and the clamp limit 1.3 tan, with their fp32 values as the kernels use them and their exact derivatives; the clamped
    cx = +-1.3 tan tz outside the frustum clamp.  Everything else as test_camera_grad_cpu._torch_loss_cam."""
    import project_ref64 as P64
    d = torch.float64
    T = lambda a: torch.tensor(np.asarray(a, np.float32).astype(np.float64), dtype=d)  # noqa: E731
    p = T(g["means3D"])
    tans = [T(cam["tanfovx"]).reshape(()).requires_grad_(), T(cam["tanfovy"]).reshape(()).requires_grad_()]
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
    vm = T(np.asarray(cam["viewmatrix"]).reshape(-1)).reshape(4, 4).T
    vw = P64.view_of(cam)
    t = p @ vm[:3, :3].T + vm[:3, 3]
    tz = t[:, 2]
    f, cl = [], []
    for ax, (size, f32v, lim32) in enumerate(((vw["W"], vw["fx"], vw["limx"]), (vw["H"], vw["fy"], vw["limy"]))):
        tan = tans[ax]
        dtan = tan - tan.detach()
        fa = f32v + (-f32v / tan.detach()) * dtan      # fp32 fx, d fx / d tan = -fx / tan
        lim = lim32 + 1.3 * dtan
        u = t[:, ax] / tz
        inside = (u >= -lim32) & (u <= lim32)
        sgn = torch.where(u > 0, 1.0, -1.0).to(d)
        f.append(fa)
        cl.append(torch.where(inside, t[:, ax], sgn * lim * tz))
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([f[0] / tz, zero, -f[0] * cl[0] / tz ** 2], 1),
                     torch.stack([zero, f[1] / tz, -f[1] * cl[1] / tz ** 2], 1)], 1)
    Mx = J @ vm[:3, :3]
    cov = Mx @ Sig @ Mx.transpose(1, 2)
    h = float(np.float32(0.3))
    a, b, c = cov[:, 0, 0] + h, cov[:, 0, 1], cov[:, 1, 1] + h
    det = a * c - b * b
    k = (det * det / (det * det + float(np.float32(1e-7)))).detach()
    sc = lambda x: x.detach() + (x - x.detach()) * k  # noqa: E731
    C_ = lambda name: torch.tensor(np.asarray(cot[name], np.float64), dtype=d)  # noqa: E731
    gco = C_("dL_dconic")
    loss = (sc(c / det) * gco[:, 0] + 2 * sc(-b / det) * gco[:, 1] + sc(a / det) * gco[:, 2]).sum()
    if aa:
        rr = (cov[:, 0, 0] * cov[:, 1, 1] - b * b) / det
        loss = loss + (o * torch.sqrt(rr.clamp_min(P64.AA_CLAMP)) * C_("dL_dopacity")).sum()
    return loss, tans


INTR_AUTOGRAD = [("clamp_x", False), ("clamp_y", False), ("near", False), ("quat_scale", False), ("sh0_m16", False),
                 ("sh1_m16", False), ("sh2_m16", False), ("sh3_m16", False), ("precomp_cov", False), ("aa1", True), ("aa3", True)]


@pytest.mark.parametrize("scene,aa", INTR_AUTOGRAD, ids=[s for s, _ in INTR_AUTOGRAD])
def test_intrinsics_chain_matches_torch_float64_autograd(scene, aa):
    import intrinsics_ref64 as I64
    import project_ref64 as P64
    import test_project_ref64_cpu as CPU
    sc = _scene(scene)
    g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
    ref = P64.forward(g, cam, mod, antialias=aa)
    live = ~ref["culled"]
    sel = {k: (v[live] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(live) else v) for k, v in g.items()}
    cot = CPU.seeded_cotangents(int(live.sum()), 3, depth=True)
    got, e, _ = I64.tan_fov_grads(sel, [cam], [cot], mod, antialias=aa)[0]
    loss, tans = _torch_loss_intr(sel, cam, cot, mod, aa)
    loss.backward()
    want = np.array([float(t.grad) for t in tans])
    tol = 1e-9 * np.abs(want).max() + 16 * 2.0 ** -53 * e
    assert np.all(np.abs(got - want) <= tol), (np.abs(got - want).max(), want)
    assert np.abs(want).max() > 0
    if scene in ("clamp_x", "clamp_y"):
        # the scene has Gaussians past the clamp on both sides of its axis
        import project_ref64 as P64b
        G = P64b._geometry(P64b._cols(sel["means3D"]), P64b.cov3d(sel, mod)[0], P64b.view_of(cam))
        ax = 0 if scene == "clamp_x" else 1
        u = (G["t"][ax] / G["tz"]).v
        outside = ~(G["inx"] if ax == 0 else G["iny"])
        assert (outside & (u > 0)).any() and (outside & (u < 0)).any()


def test_every_intrinsics_mutation_moves_an_entry_past_twice_its_bound():
    import intrinsics_ref64 as I64
    import project_ref64 as P64
    import test_project_ref64_cpu as CPU
    moved = {m: 0.0 for m in I64.INTR_MUTATIONS}
    for name, aa in (("clamp_x", False), ("clamp_y", False), ("sh1", False), ("aa1", True), ("aa3", True)):
        sc = _scene(name)
        g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
        cot = CPU.seeded_cotangents(len(g["means3D"]), 4, depth=True)
        v, e, d = I64.tan_fov_grads(g, [cam], [cot], mod, antialias=aa)[0]
        for m in I64.INTR_MUTATIONS:
            mut = I64.tan_fov_grads(g, [cam], [cot], mod, antialias=aa, mutate={m})[0][0]
            r = np.abs(mut - v) / (I64.KAPPA_INTR * (P64.U * e + d) + 1e-30)
            moved[m] = max(moved[m], float(r.max()))
    assert all(r > 2.0 for r in moved.values()), moved


# --------------------------------------------------------------------------- camera_batch with a learnable intr
@pytest.mark.parametrize("name", ["square128", "wide"])
def test_learnable_camera_batch_matches_build_cameras(name):
    W, H = (int(x) for x in GOLD[f"{name}_WH"])
    intr, extr = GOLD[f"{name}_intr"], GOLD[f"{name}_extr"]
    ref = cameras.build_cameras(torch.from_numpy(intr), torch.from_numpy(extr), W, H)
    w2c = torch.from_numpy(np.linalg.inv(extr.astype(np.float64))).float()
    K = torch.from_numpy(intr).float().requires_grad_()
    cb = cameras.camera_batch(w2c, K, W, H)
    assert cb.FovX is None and cb.tanfovx is None and len(cb) == len(ref)
    for f in ("world_view_transform", "full_proj_transform", "camera_center"):
        a, b = getattr(cb, f).detach().double().numpy(), getattr(ref, f).double().numpy()
        assert np.linalg.norm(a - b) / np.linalg.norm(b) < 2e-6, f
    want = np.stack([np.array(ref.tanfovx), np.array(ref.tanfovy)], 1)
    assert np.abs(cb.tan_fov.detach().double().numpy() - want).max() <= 2e-6 * np.abs(want).max()
    assert cb.tan_fov.requires_grad and cb.full_proj_transform.requires_grad
    st = cb.settings(0, torch.zeros(3), 1, False)
    assert torch.is_tensor(st.tanfovx) and st.tanfovx.dim() == 0
    with pytest.raises(ValueError):
        cb.as_novel_view()


def test_learnable_camera_batch_gradcheck():
    intr = torch.from_numpy(GOLD["wide_intr"][:2].astype(np.float64)).requires_grad_()
    w2c = torch.from_numpy(np.linalg.inv(GOLD["wide_extr"][:2].astype(np.float64))).requires_grad_()

    def f(m, k):
        cb = cameras.camera_batch(m, k, 160, 120)
        return cb.world_view_transform, cb.full_proj_transform, cb.camera_center, cb.tan_fov

    assert torch.autograd.gradcheck(f, (w2c, intr))


def test_other_intr_forms_are_unchanged():
    intr = GOLD["wide_intr"][:2]
    w2c = torch.from_numpy(np.linalg.inv(GOLD["wide_extr"][:2].astype(np.float64))).float()
    for form in (intr, torch.from_numpy(intr), torch.from_numpy(intr).float()):
        cb = cameras.camera_batch(w2c, form, 160, 120)
        assert cb.tan_fov is None and cb.FovX is not None and len(cb.tanfovx) == 2
        w, h, fx = 160, 120, float(intr[0, 0, 0])
        assert abs(cb.tanfovx[0] - w / (2 * fx)) < 1e-12 and isinstance(cb.tanfovy[0], float) and h


# --------------------------------------------------------------------------- the C ABI
def test_intrinsics_option_checks_its_arguments():
    L = _binding.lib()
    views = (_binding.View * 1)()
    v = views[0]
    v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
    for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                 "radii", "dL_dpix", "blend_scratch"):
        setattr(v, name, 4096)
    v.binning_capacity = 1
    intr = (_binding.ViewIntrinsics * 1)()
    intr[0].tan_fov, intr[0].dL_dtan_fov = 4096, 4096
    # dL_dtan_fov with no camera entry, then with a camera entry that has no scratch
    for cam in (None, (_binding.ViewCameraGrad * 1)()):
        opts = _binding.RenderOptions(camera_grad=cam, intrinsics=intr)
        rc = L.mgs_backward_views(1, views, opts, 4, 0, 0, 0, 4096, None, 4096, None, None, 1.0, None,
                                  4096, 4096, 4096, None, None, None, None, None, None, 0, 0, 3, 0, None)
        assert rc == -1 and "scratch" in _binding.last_error()
        clouds = (_binding.Cloud * 1)()
        c = clouds[0]
        c.P, c.means3D, c.colors_precomp, c.dL_dmean3D, c.dL_dopacity = 4, 4096, 4096, 4096, 4096
        offs = (ctypes.c_int * 2)(0, 1)
        rc = L.mgs_backward_clouds(1, clouds, offs, views, opts, 0, 0, 0, 1.0, 0, 0, None)
        assert rc == -1 and "scratch" in _binding.last_error()
    # the forward checks its other arguments before reading intr
    rc = L.mgs_forward_views(0, views, _binding.RenderOptions(intrinsics=intr), 4, 0, 0, 0, 4096, None, 4096, None, 4096, None, 1.0,
                             None, None, 0, 0, None)
    assert rc == -1
    rc = L.mgs_forward_views(1, views, _binding.RenderOptions(intrinsics=intr, antialiasing=2), 4, 0, 0, 0, 4096, None, 4096, None,
                             4096, None, 1.0, None, None, 0, 0, None)
    assert rc == -1 and "antialiasing" in _binding.last_error()
    # the camera-grad scratch keeps its size: the focal-length rows live in the geometry state
    assert L.mgs_camera_grad_scratch_bytes(16385) == 129 * 27 * 4
