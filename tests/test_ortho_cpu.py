"""Orthographic views without a GPU: the float64 reference, the camera builders and the C ABI's argument checks.

* tests/ortho_ref64.py, the float64 orthographic projection and its backward, matches torch float64 autograd of an
  independent restatement to 1e-9 relative: the records (means2D, conic, o_eff, depth), dL/dmeans3D, dL/dcov3D (or the
  scales and rotations), dL/dsh, dL/dopacity, the 27 camera terms and dL/dtan_fov, with AA on and off.
* A pinhole camera pulled back to distance D with tan_fov = h / D converges to the orthographic conic as D grows.
* The builders' matrices give d px / d t.x = fx and d py / d t.y = fy, the Jacobian's entries, and top_down_camera maps
  the workspace box onto the image.
* An ortho flag other than 0 or 1 returns MGS_ERR_INVALID_ARG before anything is enqueued.
* GaussianRasterizationSettings.orthographic: default, _replace and repr; CameraBatch.as_novel_view refuses orthographic
  cameras.
"""
import ctypes

import numpy as np
import pytest
import torch

import ortho_ref64 as O64
import project_ref64 as P64
import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding, cameras, scenes
from manigaussian_b200.rasterizer import GaussianRasterizationSettings


def _look(eye, target):
    """camera-to-world pose at `eye` looking at `target` (x right, y down, z forward)"""
    fwd = np.asarray(target, np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    if np.linalg.norm(right) < 1e-6:
        right = np.array([1.0, 0.0, 0.0])
    right /= np.linalg.norm(right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, np.cross(fwd, right), fwd, eye
    return c2w


def _scene(name, P=48, seed=0):
    """(g, cam, aa) of a small orthographic scene"""
    deg = {"sh0": 0, "sh1": 1, "sh2": 2, "sh3": 3}.get(name, 1)
    g = scenes.make_gaussians(P, sh_degree=deg, seed=seed + deg, precomp_colors=(name == "precomp_cov"))
    g["cov3D_precomp"] = None
    rng = np.random.default_rng(seed)
    g["rotations"] = (g["rotations"] * rng.uniform(0.3, 3.0, (P, 1))).astype(np.float32)
    g["scales"] = (g["scales"] * 4.0).astype(np.float32)
    if name == "precomp_cov":
        S = P64.cov3d(g)[0]
        g["cov3D_precomp"] = np.stack([S[0][0].v, S[0][1].v, S[0][2].v, S[1][1].v, S[1][2].v, S[2][2].v], 1).astype(np.float32)
        g["scales"] = g["rotations"] = None
    if g.get("shs") is not None:
        g["shs"][:, 0, :] -= 1.2   # some clamped channels
    eye = np.array([0.2 + 1.5, -1.0, 2.4])
    cam = O64.ortho_cam(40, 32, 0.7, 0.56, _look(eye, scenes.SCENE_CENTER))
    return g, cam, name.startswith("aa")


def _torch_loss_ortho(g, cam, cot, mod, aa):
    """An independent torch restatement of one orthographic view with every input a leaf: means, scale_modifier * scales
    and rotations (or cov3D), opacities, SHs, vm [16], pm [16], campos [3] in the ABI's layout and {tan_fovx, tan_fovy}.
    J = [[W / (2 tan_fovx), 0, 0], [0, H / (2 tan_fovy), 0]] (valued with the host's fp32 focal lengths).  The reference's
    conventions as in test_project_ref64_cpu: 2 gB on the conic's b, w = 1 / (det^2 + 1e-7), the SH clamp a relu."""
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
    pm16 = T(np.asarray(cam["projmatrix"]).reshape(-1)).requires_grad_()
    cp = T(np.asarray(cam["campos"]).reshape(-1)).requires_grad_()
    tan0 = np.array([np.float32(cam["tanfovx"]), np.float32(cam["tanfovy"])], np.float64)
    tan = torch.tensor(tan0, dtype=d, requires_grad=True)
    leaves.update(dL_dviewmatrix=vm16, dL_dprojmatrix=pm16, dL_dcampos=cp, dL_dtan_fov=tan)
    vw = P64.view_of(cam)
    fx, fy = vw["fx"] * (tan0[0] / tan[0]), vw["fy"] * (tan0[1] / tan[1])
    vm, pm = vm16.reshape(4, 4).T, pm16.reshape(4, 4).T
    t = p @ vm[:3, :3].T + vm[:3, 3]
    tz = t[:, 2]
    zero = torch.zeros(())
    J = torch.stack([torch.stack([fx, zero, zero]), torch.stack([zero, fy, zero])])
    Mx = J @ vm[:3, :3]
    cov = Mx @ Sig @ Mx.T
    h = float(np.float32(0.3))
    a, b, c = cov[:, 0, 0] + h, cov[:, 0, 1], cov[:, 1, 1] + h
    det = a * c - b * b
    k = (det * det / (det * det + float(np.float32(1e-7)))).detach()
    sc = lambda x: x.detach() + (x - x.detach()) * k  # noqa: E731
    hom = torch.cat([p, torch.ones_like(tz)[:, None]], 1) @ pm.T
    ndc = hom[:, :2] / (hom[:, 3:4] + float(np.float32(1e-7)))
    C_ = lambda k: torch.tensor(np.asarray(cot[k], np.float64), dtype=d)  # noqa: E731
    gco = C_("dL_dconic")
    conic = torch.stack([c / det, -b / det, a / det], 1)
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
    W, H = cam["W"], cam["H"]
    pix = ((ndc + 1.0) * torch.tensor([W, H], dtype=d) - 1.0) * 0.5
    recs = dict(means2D=pix.detach().numpy(), conic=conic.detach().numpy(), opacity=oe.detach().numpy(), depth=tz.detach().numpy())
    return loss, leaves, recs


def _close(got, want, e=None, what=""):
    tol = 1e-9 * max(np.abs(want).max(), 1e-300) + (16 * 2.0 ** -53 * np.asarray(e) if e is not None else 0.0)
    assert np.all(np.abs(np.asarray(got) - want) <= tol), (what, np.abs(np.asarray(got) - want).max(), np.abs(want).max())


AUTOGRAD = ["sh0", "sh1", "sh2", "sh3", "precomp_cov", "aa1", "aa3"]


@pytest.mark.parametrize("scene", AUTOGRAD)
def test_reference_matches_torch_float64_autograd(scene):
    import test_project_ref64_cpu as CPU
    g, cam, aa = _scene(scene)
    if scene == "aa3":
        g = scenes.make_gaussians(48, sh_degree=3, seed=9)
        g["cov3D_precomp"] = None
        g["scales"][:16, 2] = 1e-4   # needles on both sides of the compensation's clamp
    mod = 0.9
    fw = O64.forward(g, cam, mod, antialias=aa)
    live = ~fw["culled"]
    assert live.sum() >= 24
    sel = {k: (v[live] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(live) else v) for k, v in g.items()}
    fw = O64.forward(sel, cam, mod, antialias=aa)
    cot = CPU.seeded_cotangents(int(live.sum()), 5, depth=True)
    rb = O64.backward(sel, [cam], [cot], mod, antialias=aa)
    loss, leaves, recs = _torch_loss_ortho(sel, cam, cot, mod, aa)
    # the records
    _close(fw["means2D"], recs["means2D"], what="means2D")
    _close(fw["conic"], recs["conic"], what="conic")
    _close(fw["opacity"], recs["opacity"], what="opacity")
    _close(fw["depth"], recs["depth"], what="depth")
    loss.backward()
    for name, leaf in leaves.items():
        want = leaf.grad.numpy() if leaf.grad is not None else np.zeros(tuple(leaf.shape))
        if name in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos"):
            got, e, _ = rb["camera"][0][name]
        elif name == "dL_dtan_fov":
            got, e, _ = rb["tan_fov"][0]
        elif name == "dL_dsh":
            got, e, _ = rb["dL_dsh"]
            n = (int(sel["sh_degree"]) + 1) ** 2
            got, e, want = got[:, :n], e[:, :n], want[:, :n]
        else:
            got, e, _ = rb[name]
            if name == "dL_dopacity":
                want = want.reshape(-1)
        _close(got, want, e, name)
    # the camera centre only through the view direction; tan_fov always moves the conic
    assert np.abs(rb["tan_fov"][0][0]).min() > 0


def test_pinhole_pulled_back_converges_to_the_orthographic_conic():
    """A pinhole camera at distance D along the same axis, with tan_fov = h / D, sees the orthographic conic as D grows:
    the relative difference falls like 1 / D."""
    g, cam, _ = _scene("sh1", P=24, seed=3)
    target = scenes.SCENE_CENTER.astype(np.float64)
    direction = np.array([1.5, -1.0, 1.3]) / np.linalg.norm([1.5, -1.0, 1.3])
    W, H, hw, hh = 40, 32, 0.7, 0.56
    ref = O64.forward(g, O64.ortho_cam(W, H, hw, hh, _look(target + 2.0 * direction, target)), 1.0)
    errs = []
    for D in (10.0, 100.0, 1000.0):
        c2w = _look(target + D * direction, target)
        w2c = np.linalg.inv(c2w)
        tx, ty = hw / D, hh / D
        K = np.array([[W / (2 * tx), 0, W / 2], [0, H / (2 * ty), H / 2], [0, 0, 1]])
        proj = cameras.projection_from_intrinsics(0.1, 2 * D, K, H, W)
        cam = dict(W=W, H=H, tanfovx=tx, tanfovy=ty, viewmatrix=w2c.T, projmatrix=w2c.T @ proj.T,
                   campos=c2w[:3, 3])
        # float64 matrices: the comparison is of the model, not of fp32 rounding
        vw = P64.view_of(cam)
        vw.update(fx=W / (2 * tx), fy=H / (2 * ty), limx=1.3 * tx, limy=1.3 * ty,
                  Rv=w2c[:3, :3], tv=w2c[:3, 3])
        S = P64.cov3d(g)[0]
        G = P64._geometry(P64._cols(g["means3D"]), S, vw)
        conic = np.stack([(G["c"] / G["det"]).v, (-(G["b"] / G["det"])).v, (G["a"] / G["det"]).v], 1)
        errs.append(np.abs(conic - ref["conic"]).max() / np.abs(ref["conic"]).max())
    assert errs[0] < 0.2 and errs[1] < errs[0] / 5 and errs[2] < errs[1] / 5, errs


@pytest.mark.parametrize("half", [(0.5, 0.5), (0.8, 0.3)])
def test_builder_matrices_match_the_jacobian(half):
    """The screen mean of build_ortho_cameras / ortho_camera_batch moves by fx per unit of t.x and fy per unit of t.y, and
    not with t.z: the Jacobian J = [[fx, 0, 0], [0, fy, 0]] the kernels use."""
    W, H = 64, 48
    c2w = _look(np.array([1.0, -2.0, 2.0]), scenes.SCENE_CENTER)
    cb = cameras.build_ortho_cameras(c2w[None], np.array([half]), W, H)
    cb2 = cameras.ortho_camera_batch(torch.from_numpy(np.linalg.inv(c2w)).float(), half, W, H)
    for full, wvt in ((cb.host["full_proj_transform"][0], cb.host["world_view_transform"][0]),
                      (cb2.full_proj_transform[0].numpy(), cb2.world_view_transform[0].numpy())):
        full, wvt = full.astype(np.float64), wvt.astype(np.float64)
        c2w_ = np.linalg.inv(wvt.T)

        def px(t):
            hom = np.append(c2w_[:3, :3] @ t + c2w_[:3, 3], 1.0) @ full
            assert abs(hom[3] - 1.0) < 1e-6
            return ((hom[:2] / hom[3] + 1.0) * np.array([W, H]) - 1.0) * 0.5

        t0 = np.array([0.1, -0.05, 1.0])
        fx, fy = W / (2 * half[0]), H / (2 * half[1])
        for axis, want in ((0, (fx, 0.0)), (1, (0.0, fy)), (2, (0.0, 0.0))):
            dt = np.zeros(3)
            dt[axis] = 1e-3
            np.testing.assert_allclose((px(t0 + dt) - px(t0)) / 1e-3, want, atol=1e-3 * max(fx, fy))
    assert cb.ortho and cb2.ortho and cb.FovX is None and cb.tanfovx == [half[0]] and cb.tanfovy == [half[1]]


def test_learnable_half_extent_lives_on_the_device_and_is_differentiable():
    w2c = torch.from_numpy(np.linalg.inv(_look(np.array([1.0, -2.0, 2.0]), scenes.SCENE_CENTER))).requires_grad_()
    h = torch.tensor([[0.6, 0.4]], dtype=torch.float64, requires_grad=True)
    cb = cameras.ortho_camera_batch(w2c, h, 32, 24)
    assert cb.tan_fov is h or torch.equal(cb.tan_fov, h)
    assert cb.tanfovx is None and cb.ortho
    s = cb.settings(0, torch.zeros(3), 0, False)
    assert s.orthographic and torch.is_tensor(s.tanfovx)
    assert torch.autograd.gradcheck(lambda m, k: cameras.ortho_camera_batch(m, k, 32, 24).full_proj_transform, (w2c, h))


def test_top_down_camera_maps_the_box_onto_the_image():
    bounds = scenes.SCENE_BOUNDS.astype(np.float64)
    W, H = 100, 100
    cb = cameras.top_down_camera(bounds, W, H)
    full = cb.host["full_proj_transform"][0].astype(np.float64)
    wvt = cb.host["world_view_transform"][0].astype(np.float64)
    x0, y0, z0, x1, y1, z1 = bounds

    def pix(p):
        hom = np.append(p, 1.0) @ full
        return ((hom[:2] / hom[3] + 1.0) * np.array([W, H]) - 1.0) * 0.5

    for z in (z0, z1):
        np.testing.assert_allclose(pix([x0, y1, z]), [-0.5, -0.5], atol=1e-4)        # x_min, y_max: top-left corner
        np.testing.assert_allclose(pix([x1, y0, z]), [W - 0.5, H - 0.5], atol=1e-4)  # x_max, y_min: bottom-right corner
    depth = lambda p: (np.append(p, 1.0) @ wvt)[2]  # noqa: E731
    assert depth([0.2, 0.0, z1]) > P64.NEAR_Z and depth([0.2, 0.0, z0]) - depth([0.2, 0.0, z1]) == pytest.approx(z1 - z0)
    s = cb.settings(0, torch.zeros(3), 0, False)
    assert s.orthographic and s.tanfovx == pytest.approx(0.5) and s.tanfovy == pytest.approx(0.5)
    with pytest.raises(ValueError):
        cameras.top_down_camera(bounds, W, H, margin=0.1)
    with pytest.raises(ValueError):
        cameras.top_down_camera([0, 0, 0, -1, 1, 1], W, H)


def test_settings_attribute_default_replace_and_repr():
    args = (8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False, False)
    s = GaussianRasterizationSettings(*args)
    assert s.orthographic is False and len(tuple(s)) == 13
    o = GaussianRasterizationSettings(*args, orthographic=True)
    assert o.orthographic and not o.antialiasing and tuple(o)[:2] == (8, 8)
    r = o._replace(image_width=16)
    assert r.orthographic and r.image_width == 16
    assert not o._replace(orthographic=False).orthographic
    assert o._replace(antialiasing=True).orthographic
    assert "orthographic=True" in repr(o) and "orthographic=False" in repr(s)
    assert GaussianRasterizationSettings._make(tuple(o)).orthographic is False   # the 13 fields carry no camera model


def test_as_novel_view_refuses_orthographic_cameras():
    cb = cameras.build_ortho_cameras(np.eye(4)[None], 0.5, 16, 16)
    with pytest.raises(ValueError):
        cb.as_novel_view()


def test_ortho_option_checks_its_flags():
    L = _binding.lib()
    views = (_binding.View * 2)()
    for v in views:
        v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
        for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                     "radii", "out_color", "dL_dpix", "blend_scratch"):
            setattr(v, name, 4096)
        v.binning_capacity = 1
    bad = (ctypes.c_int * 2)(0, 2)
    # pointers are never dereferenced: the flags are checked before anything is enqueued
    rc = L.mgs_forward_views(2, views, _binding.RenderOptions(ortho=bad), 4, 0, 0, 0, 4096, None, 4096, None, 4096,
                             4096, 1.0, 4096, None, 0, 0, None)
    assert rc == -1 and "ortho" in _binding.last_error()
    rc = L.mgs_backward_views(2, views, _binding.RenderOptions(ortho=bad), 4, 0, 0, 0, 4096, None, 4096, None,
                              4096, 1.0, 4096, None, 4096, 4096, None, None, None, None, None, None, 0, 0, 3, 0, None)
    assert rc == -1 and "ortho" in _binding.last_error()
    rc = L.mgs_lift_views(2, views, None, 0, None, bad, None, None, 4, 0, 0, 0, 4096, None, 4096, 4096, 4096, 1.0, 4096, None, None,
                                4096, 0, None)
    assert rc == -1 and "ortho" in _binding.last_error()
    clouds = (_binding.Cloud * 1)()
    c = clouds[0]
    c.P, c.means3D, c.colors_precomp, c.opacities, c.scales, c.rotations = 4, 4096, 4096, 4096, 4096, 4096
    c.dL_dmean3D, c.dL_dopacity = 4096, 4096
    offs = (ctypes.c_int * 2)(0, 2)
    neg = (ctypes.c_int * 2)(-1, 0)
    rc = L.mgs_forward_clouds(1, clouds, offs, views, _binding.RenderOptions(ortho=neg), 0, 0, 0, 1.0, 0, 0, None)
    assert rc == -1 and "ortho" in _binding.last_error()
    rc = L.mgs_backward_clouds(1, clouds, offs, views, _binding.RenderOptions(ortho=neg), 0, 0, 0, 1.0, 0, 0, None)
    assert rc == -1 and "ortho" in _binding.last_error()
