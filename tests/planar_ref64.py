"""Float64 restatement of planar depth (include/mgs_rasterizer.h, mgs_render_options.planar_depth), in torch so that its gradients
come from autograd rather than from the hand chain of project_bwd.cu.

For Gaussian i in a view with t = Rv p + tv: Sigma_c = Rv S Rv^T, J the view model's 2x3 screen Jacobian in pixels, Q the
blend's conic inv(J Sigma_c J^T + 0.3 I), k = e3^T Sigma_c J^T, (a, b) = k Q, and the depth at pixel (px, py) is
z + a (px - mu_x) + b (py - mu_y), mu the screen mean in pixels.  quads() returns {a, b, e = -(a mu_x + b mu_y)} per Gaussian.

A view is a dict: viewmatrix (16, column-major as the kernels read it: Rv[r][c] = vm[4 c + r]), projmatrix (16, likewise),
W, H, tanfovx, tanfovy, and optionally "ortho" (bool), "fisheye" (cx, cy, k1..k4) or "distortion" (cx, cy, k1, k2, p1, p2, k3,
k4, k5, k6).
"""
import numpy as np
import torch

D64 = torch.float64


def _t(x):
    return x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, np.float64), dtype=D64)


def rotation(q):
    """R(q) of the un-normalised quaternion (r, x, y, z), as project.cu forms it"""
    r, x, y, z = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
        torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
        torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def covariance(scales, rotations, scale_modifier=1.0):
    """S = R diag(s^2) R^T, [P,3,3]"""
    R = rotation(rotations)
    s = scale_modifier * scales
    return R @ torch.diag_embed(s * s) @ R.transpose(-1, -2)


def _map(t, view):
    """the view's screen position (u, v) in pixels of view-space points t [P,3], and whether J takes the pinhole clamp"""
    W, H = view["W"], view["H"]
    fx, fy = W / (2.0 * view["tanfovx"]), H / (2.0 * view["tanfovy"])
    x, y, z = t.unbind(-1)
    if view.get("fisheye") is not None:
        cx, cy, k1, k2, k3, k4 = view["fisheye"][:6]
        r = torch.sqrt(x * x + y * y)
        th = torch.atan2(r, z)
        th2 = th * th
        thd = th * (1 + th2 * (k1 + th2 * (k2 + th2 * (k3 + th2 * k4))))
        s = thd / r
        return torch.stack([fx * s * x + cx, fy * s * y + cy], -1)
    if view.get("distortion") is not None:
        cx, cy, k1, k2, p1, p2, k3, k4, k5, k6 = view["distortion"][:10]
        xn, yn = x / z, y / z
        r2 = xn * xn + yn * yn
        R = (1 + r2 * (k1 + r2 * (k2 + r2 * k3))) / (1 + r2 * (k4 + r2 * (k5 + r2 * k6)))
        xd = xn * R + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
        yd = yn * R + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
        return torch.stack([fx * xd + cx, fy * yd + cy], -1)
    raise ValueError("pinhole and orthographic means go through projmatrix")


def _jacobian(t, view):
    """J [P,2,3] in pixels, differentiable in t"""
    W, H = view["W"], view["H"]
    fx, fy = W / (2.0 * view["tanfovx"]), H / (2.0 * view["tanfovy"])
    P = t.shape[0]
    zero = torch.zeros(P, dtype=D64)
    if view.get("ortho"):
        return torch.stack([torch.stack([zero + fx, zero, zero], -1), torch.stack([zero, zero + fy, zero], -1)], -2)
    if view.get("fisheye") is not None or view.get("distortion") is not None:
        tt = t if t.requires_grad else t.detach().requires_grad_(True)
        with torch.enable_grad():
            uv = _map(tt, view)
            rows = [torch.autograd.grad(uv[:, j].sum(), tt, create_graph=True)[0] for j in range(2)]
        return torch.stack(rows, -2)
    # pinhole: the Jacobian at t.xy clamped to 1.3 tan_fov t.z
    x, y, z = t.unbind(-1)
    limx, limy = 1.3 * view["tanfovx"], 1.3 * view["tanfovy"]
    cx = torch.clamp(x / z, -limx, limx) * z
    cy = torch.clamp(y / z, -limy, limy) * z
    return torch.stack([torch.stack([fx / z, zero, -fx * cx / (z * z)], -1),
                        torch.stack([zero, fy / z, -fy * cy / (z * z)], -1)], -2)


def screen_mean(means3D, view):
    """mu [P,2] in pixels: through projmatrix (pinhole, orthographic) or the view's lens map"""
    vm = _t(view["viewmatrix"]).reshape(4, 4).T  # row-major: t = vm[:3,:3] p + vm[:3,3]
    t = means3D @ vm[:3, :3].T + vm[:3, 3]
    if view.get("fisheye") is not None or view.get("distortion") is not None:
        return _map(t, view)
    pm = _t(view["projmatrix"]).reshape(4, 4).T
    h = means3D @ pm[:, :3].T + pm[:, 3]
    ndc = h[:, :2] / (h[:, 3:4] + 1e-7)
    return torch.stack([((ndc[:, 0] + 1.0) * view["W"] - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * view["H"] - 1.0) * 0.5], -1)


def quads(means3D, scales, rotations, view, scale_modifier=1.0, cov3D=None):
    """{a, b, e} [P,3] and the conic (A, B, C) [P,3], differentiable in means3D, scales, rotations (or cov3D [P,3,3])"""
    vm = _t(view["viewmatrix"]).reshape(4, 4).T
    Rv = vm[:3, :3]
    t = means3D @ Rv.T + vm[:3, 3]
    S = covariance(scales, rotations, scale_modifier) if cov3D is None else cov3D
    J = _jacobian(t, view)
    M = J @ Rv                                                     # [P,2,3]
    cov2 = M @ S @ M.transpose(-1, -2) + 0.3 * torch.eye(2, dtype=D64)
    Q = torch.linalg.inv(cov2)
    k = ((Rv[2] @ S).unsqueeze(-2) @ M.transpose(-1, -2)).squeeze(-2)  # [P,2]: e3^T Rv S Rv^T J^T
    ab = (k.unsqueeze(-2) @ Q).squeeze(-2)
    mu = screen_mean(means3D, view)
    e = -(ab[:, 0] * mu[:, 0] + ab[:, 1] * mu[:, 1])
    return torch.stack([ab[:, 0], ab[:, 1], e], -1), torch.stack([Q[:, 0, 0], Q[:, 0, 1], Q[:, 1, 1]], -1)


def planar_depth_at(z, quad, px, py):
    """d_i(p) = z + a px + b py + e"""
    return z + quad[..., 0] * px + quad[..., 1] * py + quad[..., 2]


def packed_cov(c6):
    """the symmetric [P,3,3] of the 6 packed entries 00 01 02 11 12 22 (off-diagonals appear twice: their gradient is the sum)"""
    return torch.stack([torch.stack([c6[:, 0], c6[:, 1], c6[:, 2]], -1), torch.stack([c6[:, 1], c6[:, 3], c6[:, 4]], -1),
                        torch.stack([c6[:, 2], c6[:, 4], c6[:, 5]], -1)], -2)


def full_chain(means3D, scales, rotations, view, dquad, mask=None, cov3D=None, tan_fov=None):
    """dL/d of sum dquad * quads w.r.t. means3D [P,3], scales [P,3] and rotations [P,4] (or packed cov3D [P,6]), the stored
    viewmatrix [16] and projmatrix [16], and {tan_fovx, tan_fovy} (float64 numpy; None where an input is not given)"""
    m = _t(means3D).clone().requires_grad_(True)
    leaves = [m]
    if cov3D is None:
        s, r = (_t(x).clone().requires_grad_(True) for x in (scales, rotations))
        leaves += [s, r]
        S = covariance(s, r)
    else:
        c = _t(cov3D).clone().requires_grad_(True)
        leaves.append(c)
        S = packed_cov(c)
    vm = _t(view["viewmatrix"]).clone().requires_grad_(True)
    pm = _t(view["projmatrix"]).clone().requires_grad_(True)
    tf = _t([view["tanfovx"], view["tanfovy"]] if tan_fov is None else tan_fov).clone().requires_grad_(True)
    v = dict(view, viewmatrix=vm, projmatrix=pm, tanfovx=tf[0], tanfovy=tf[1])
    q, _ = quads(m, None, None, v, cov3D=S)
    w = _t(dquad)
    if mask is not None:
        w = w * _t(mask.astype(np.float64))[:, None]
    gr = torch.autograd.grad((q * w).sum(), leaves + [vm, pm, tf], allow_unused=True)
    return [None if g is None else g.numpy() for g in gr]


def quad_chain(means3D, scales, rotations, view, dquad, mask=None, scale_modifier=1.0):
    """dL/d(means3D, scales, rotations) of sum dquad * quads (float64 numpy [P,3], [P,3], [P,4]); rows outside mask carry none"""
    m, s, r = (_t(x).clone().requires_grad_(True) for x in (means3D, scales, rotations))
    q, _ = quads(m, s, r, view, scale_modifier)
    w = _t(dquad)
    if mask is not None:
        w = w * _t(mask.astype(np.float64))[:, None]
    gm, gs, gr = torch.autograd.grad((q * w).sum(), (m, s, r))
    return gm.numpy(), gs.numpy(), gr.numpy()
