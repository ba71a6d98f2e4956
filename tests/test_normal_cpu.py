"""The float64 reference of the per-Gaussian surface normal (tests/normal_ref64.py) against torch float64 autograd of an
independent restatement (the rotation matrix assembled by torch ops, the axis picked by a gather), on unit and non-unit
quaternions, tied scales, edge-on Gaussians and Gaussians behind the camera; the axis as an eigenvector of the covariance the
projection builds; four broken conventions each move a checked element; and the C ABI's argument errors."""
import ctypes

import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
import normal_ref64 as N
from manigaussian_b200 import _binding


def _cloud(P=64, seed=0):
    rng = np.random.default_rng(seed)
    means = rng.uniform(-1, 1, (P, 3))
    scales = rng.uniform(0.01, 0.3, (P, 3))
    q = rng.standard_normal((P, 4))
    q *= (np.geomspace(0.05, 20, P) / np.linalg.norm(q, axis=1))[:, None]  # |q| from 0.05 to 20
    q[:4] /= np.linalg.norm(q[:4], axis=1)[:, None]                         # and some unit ones
    scales[4, 1] = scales[4, 0] = 0.02                                      # two equal shortest: index 0
    scales[5, 2] = scales[5, 1] = 0.01                                      # two equal shortest: index 1
    scales[6] = 0.05                                                        # all equal: index 0
    campos = np.array([0.3, -0.2, 3.0])
    # Gaussians 7, 8 exactly edge-on: the camera in the plane through the mean, orthogonal to the axis
    a, _, _, _ = N.axis(scales, q)
    for i in (7, 8):
        t = np.cross(a[i], [0.0, 0.0, 1.0])
        means[i] = campos - 2.0 * t / np.linalg.norm(t)
    means[9] = campos + np.array([0.0, 0.0, 5.0])  # behind a camera that looks down -z
    return means, scales, q, campos


def _torch_normals(means, scales, q, campos, cot):
    """independent restatement: R from torch ops on the normalised quaternion, column by gather, sign detached"""
    q = q.clone().requires_grad_(True)
    qh = q / q.norm(dim=1, keepdim=True)
    r, x, y, z = qh.unbind(1)
    R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], 1),
                     torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], 1),
                     torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1)], 1)
    k = torch.argmin(scales, dim=1)
    # torch.argmin does not promise the first minimum: resolve ties to the lowest index
    k = torch.where(scales[:, 0] <= scales.min(dim=1).values, torch.zeros_like(k), k)
    k = torch.where((scales[:, 1] <= scales.min(dim=1).values) & (k != 0), torch.ones_like(k), k)
    a = torch.gather(R, 2, k[:, None, None].expand(-1, 3, 1))[:, :, 0]
    s = torch.where(((campos[None] - means) * a).sum(1) >= 0, 1.0, -1.0).detach()
    n = a * s[:, None]
    (n * cot).sum().backward()
    return n.detach().numpy(), q.grad.numpy()


def test_reference_matches_float64_autograd():
    means, scales, q, campos = _cloud()
    rng = np.random.default_rng(1)
    cot = rng.standard_normal(means.shape)
    n, d = N.normals(means, scales, q, campos)
    g = N.rotation_grad(means, scales, q, [campos], [cot])
    tn, tg = _torch_normals(*(torch.from_numpy(x) for x in (means, scales, q, campos, cot)))
    assert abs(d[7]) < 1e-12 and abs(d[8]) < 1e-12  # edge-on by construction
    sure = np.abs(d) > 1e-9                         # the sign of an exact zero depends on rounding: compare up to sign there
    assert np.abs(n[sure] - tn[sure]).max() < 1e-9
    assert np.abs(np.abs(n[~sure]) - np.abs(tn[~sure])).max() < 1e-9
    scale = np.abs(tg).max(axis=1, keepdims=True) + 1e-30
    assert (np.abs(g[sure] - tg[sure]) / scale[sure]).max() < 1e-9
    assert np.abs(np.linalg.norm(n, axis=1) - 1).max() < 1e-12
    assert list(N.shortest_axis(scales)[4:7]) == [0, 1, 0]
    assert d[9] < 0 or d[9] >= 0  # behind the camera: defined either way, no NaN
    assert np.isfinite(n).all() and np.isfinite(g).all()


def test_two_views_sum_with_their_signs():
    means, scales, q, campos = _cloud(seed=2)
    rng = np.random.default_rng(3)
    cams = [campos, -campos]
    cots = [rng.standard_normal(means.shape) for _ in cams]
    g = N.rotation_grad(means, scales, q, cams, cots)
    one = sum(N.rotation_grad(means, scales, q, [c], [t]) for c, t in zip(cams, cots))
    assert np.abs(g - one).max() < 1e-12
    s0, s1 = N.facing(N.axis(scales, q)[0], means, cams[0])[0], N.facing(N.axis(scales, q)[0], means, cams[1])[0]
    assert (s0 != s1).any() and (s0 == s1).any()


def test_axis_is_the_eigenvector_of_the_projections_covariance():
    """Sigma = (S R)^T (S R) assembled as the projection kernel does (csrc/project.cu, cov3d_from_scale_rot: R given column
    by column), from the normalised quaternion: the chosen axis is its eigenvector of the smallest eigenvalue s_k^2"""
    means, scales, q, campos = _cloud(seed=4)
    qh = q / np.linalg.norm(q, axis=1)[:, None]
    a, k, _, _ = N.axis(scales, q)
    for i in range(len(k)):
        r, x, y, z = qh[i]
        cols = [[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]]
        R = np.array(cols).T          # column-major, as the kernel's m3()
        M = np.diag(scales[i]) @ R
        Sigma = M.T @ M
        assert np.abs(Sigma @ a[i] - scales[i, k[i]] ** 2 * a[i]).max() < 1e-12
        assert scales[i, k[i]] == scales[i].min()


@pytest.mark.parametrize("broken", ["argmax", "no_flip", "no_normalization_jacobian", "row"])
def test_broken_conventions_move_a_checked_element(broken):
    means, scales, q, campos = _cloud(seed=5)
    rng = np.random.default_rng(6)
    cot = rng.standard_normal(means.shape)
    n, d = N.normals(means, scales, q, campos)
    g = N.rotation_grad(means, scales, q, [campos], [cot])
    if broken == "argmax":
        bn, _ = N.normals(means, scales, q, campos, argmax=True)
        moved = np.abs(bn - n).max()
    elif broken == "no_flip":
        bn, _ = N.normals(means, scales, q, campos, flip=False)
        assert (d < 0).any()
        moved = np.abs(bn - n).max()
    elif broken == "row":
        bn, _ = N.normals(means, scales, q, campos, row=True)
        moved = np.abs(bn - n).max()
    else:
        bg = N.rotation_grad(means, scales, q, [campos], [cot], normalization_jacobian=False)
        moved = np.abs(bg - g).max()
    assert moved > 1e-3


def test_state_queries_grow_only_with_normals():
    L = _binding.lib()
    for P in (1, 1000, 500000):
        assert L.mgs_geometry_state_bytes_normal(P) >= L.mgs_geometry_state_bytes(P) + 16 * P
        assert L.mgs_backward_scratch_bytes_normal(P) >= L.mgs_backward_scratch_bytes(P) + 16 * P
    out, out2 = ctypes.c_void_p(), ctypes.c_void_p()
    base = 1 << 20
    assert L.mgs_state_array(b"geometry", b"nrm", ctypes.c_void_p(base), 1000, 0, ctypes.byref(out)) == 0
    assert L.mgs_state_array(b"geometry", b"rgbd", ctypes.c_void_p(base), 1000, 0, ctypes.byref(out2)) == 0
    assert out.value % 16 == 0 and out.value + 16 * 1000 <= base + L.mgs_geometry_state_bytes_normal(1000)
    assert out.value >= base + L.mgs_geometry_state_bytes(1000) - 128 - 127  # behind every other array


def _views_call(L, forward, normal, cov3D=False, cam_pos=True, depth_mask=None):
    """mgs_forward_views / mgs_backward_views with a normal plane and fake non-NULL pointers: every refusal happens before
    anything is enqueued"""
    p = ctypes.c_void_p(4096)
    w = (_binding.View * 1)()
    v = w[0]
    v.viewmatrix = v.projmatrix = v.background = v.geometry_state = v.binning_state = v.image_state = 4096
    v.out_color = v.radii = v.dL_dpix = v.blend_scratch = 4096
    v.cam_pos = 4096 if cam_pos else None
    v.width = v.height = 16
    v.tan_fovx = v.tan_fovy = 0.5
    geo = (p, p, None, None, p, None if cov3D else p, 1.0, None if cov3D else p, p if cov3D else None)
    opts = _binding.RenderOptions(depth_mask=depth_mask, normal=normal)
    if forward:
        return L.mgs_forward_views(1, w, opts, 10, 1, 4, 0, *geo, 0, 0, None)
    geo = (p, p, None, None, None if cov3D else p, 1.0, None if cov3D else p, p if cov3D else None)
    return L.mgs_backward_views(1, w, opts, 10, 1, 4, 0, *geo,
                                p, p, None, None, None, p, p, p, 1, 0, 3, 0, None)


def test_normal_option_errors_before_anything_is_enqueued():
    L = _binding.lib()
    n = (_binding.ViewNormal * 1)()
    n[0].out_normal = 4096
    assert _views_call(L, True, n, cov3D=True) == -1 and "scales and rotations" in _binding.last_error()
    assert _views_call(L, True, n, cam_pos=False) == -1 and "cam_pos" in _binding.last_error()
    n[0].dL_dpix_normal = 4096
    assert _views_call(L, False, n, cov3D=True) == -1 and "scales and rotations" in _binding.last_error()
    n[0].out_normal = None
    assert _views_call(L, False, n) == -1 and "out_normal" in _binding.last_error()
    n[0].out_normal = 4096
    dm = (_binding.ViewDepthMask * 1)()
    dm[0].target_mask, dm[0].cot_alpha_mask, dm[0].loss_acc = 4096, 4096, 4096
    assert _views_call(L, False, n, depth_mask=dm) == -1 and "depth / mask" in _binding.last_error()
