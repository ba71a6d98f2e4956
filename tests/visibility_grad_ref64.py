"""Float64 restatement of the point-visibility backward (include/mgs_rasterizer.h, mgs_visibility_views_backward), in torch so
that its gradients come from autograd rather than from the hand chains of visibility.cu and project_bwd.cu.

* `decisions`: per in-view point the accepted candidates of visibility_ref64's walk (the tile, the depth cut, the 1/255 cut
  and the stop), from a view's projected and sorted state, and its `border` flag.  They are constants of the outputs.
* `outputs`: uv, depth and T of the points with those decisions frozen, differentiable end to end in the points, the cloud
  (means, scales, rotations or a packed cov3D, opacities), the view and projection matrices and tan_fov.  uv and depth come
  from flow_ref64 / planar_ref64's screen_mean (every camera model), each Gaussian's screen mean and conic from
  planar_ref64's projection (J of the model, the 0.3 px^2 low-pass) with the per-Gaussian backward's convention at the
  pinhole clamp (project_ref64's: a clamped t.x / t.z holds t.z), the anti-aliased opacity from
  aa_oracle's definition, and T = prod (1 - alpha_i) over the accepted candidates with alpha = min(0.99, o G) whose clamp
  is transparent to the gradient, as in blend_ref64 and the blend backward.
"""
import numpy as np
import torch

import blend_ref64 as R64
import flow_ref64 as F64
import planar_ref64 as P64
import visibility_ref64 as V64

D64 = torch.float64


def decisions(st, uv, d, inside):
    """(accepted: per point an int64 array of Gaussian ids in list order (empty where not inside), border [Q])"""
    _, border = V64.transmittance(st, uv, d, inside)
    W, H = st["W"], st["H"]
    tiles = V64.tile_of(np.where(inside[:, None], uv, 0.0), W, H)
    acc = [np.zeros(0, np.int64) for _ in range(len(d))]
    for q in np.nonzero(inside)[0]:
        u, v = float(uv[q, 0]), float(uv[q, 1])
        r0, r1 = (int(x) for x in st["ranges"][tiles[q]])
        ids = st["point_list"][r0:r1].astype(np.int64)
        ids = ids[st["depths"][ids].astype(np.float64) < d[q]]
        m = st["means2D"][ids].astype(np.float64)
        co = st["conic_opacity"][ids].astype(np.float64)
        dx, dy = m[:, 0] - u, m[:, 1] - v
        power = -0.5 * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy
        alpha = np.minimum(R64.ALPHA_MAX, co[:, 3] * np.exp(power))
        ok = (power <= 0) & (alpha >= R64.ALPHA_MIN)
        cp = np.cumprod(np.where(ok, 1.0 - alpha, 1.0))
        stop = ok & (cp < R64.T_STOP)
        end = int(np.argmax(stop)) if stop.any() else len(ids)
        acc[q] = ids[:end][ok[:end]]
    return acc, border


def _jacobian(t, view):
    """J [P,2,3] in pixels, with the per-Gaussian backward's convention at the pinhole clamp (include/mgs_rasterizer.h, camera
    gradients): a clamped cx = +-1.3 tan_fovx t.z holds t.z constant, so only tan_fov reaches it, and d/dt.x is masked; an
    unclamped cx is t.x.  Other models as planar_ref64."""
    if view.get("ortho") or view.get("fisheye") is not None or view.get("distortion") is not None:
        return P64._jacobian(t, view)
    W, H = view["W"], view["H"]
    tx, ty = view["tanfovx"], view["tanfovy"]
    fx, fy = W / (2.0 * tx), H / (2.0 * ty)
    x, y, z = t.unbind(-1)
    zero = torch.zeros_like(z)

    def held(a, tan):
        lim = 1.3 * tan
        r = a / z
        out = (r > lim) | (r < -lim)
        return torch.where(out, torch.sign(r).detach() * lim * z.detach(), a)

    cx, cy = held(x, tx), held(y, ty)
    return torch.stack([torch.stack([fx / z + zero, zero, -fx * cx / (z * z)], -1),
                        torch.stack([zero, fy / z + zero, -fy * cy / (z * z)], -1)], -2)


def _screen_conic(means3D, S, view, antialias):
    """screen means [P,2], conics (A, B, C) [P,3] and the anti-aliased opacity factor [P] (1 without antialias)"""
    vm = P64._t(view["viewmatrix"]).reshape(4, 4).T
    Rv = vm[:3, :3]
    t = means3D @ Rv.T + vm[:3, 3]
    M = _jacobian(t, view) @ Rv
    cov0 = M @ S @ M.transpose(-1, -2)
    cov = cov0 + 0.3 * torch.eye(2, dtype=D64)
    det0 = cov0[:, 0, 0] * cov0[:, 1, 1] - cov0[:, 0, 1] * cov0[:, 1, 0]
    det = cov[:, 0, 0] * cov[:, 1, 1] - cov[:, 0, 1] * cov[:, 1, 0]
    conic = torch.stack([cov[:, 1, 1] / det, -cov[:, 0, 1] / det, cov[:, 0, 0] / det], -1)
    s = torch.sqrt(torch.clamp(det0 / det, min=2.5e-5)) if antialias else torch.ones_like(det)
    return P64.screen_mean(means3D, view), conic, s


def outputs(points, means3D, opacities, view, accepted, scales=None, rotations=None, cov3D=None, antialias=False):
    """(uv [Q,2], depth [Q], T [Q]) in float64 torch with the decisions `accepted` frozen; T = 1 where nothing is accepted.
    The view dict may hold tensors (viewmatrix, projmatrix, tanfovx, tanfovy) to differentiate in."""
    uv = F64.screen_mean(points, view)
    depth = F64.view_space(points, view)[:, 2]
    S = P64.covariance(scales, rotations) if cov3D is None else P64.packed_cov(cov3D)
    mu, conic, s = _screen_conic(means3D, S, view, antialias)
    return uv, depth, screen_transmittance(uv, mu, conic, opacities.reshape(-1) * s, accepted)


def screen_transmittance(uv, mu, conic, opacity, accepted):
    """T [Q] = prod (1 - alpha_i) over each point's accepted Gaussians, from the points' uv [Q,2] and the Gaussians' screen
    means [P,2], conics (A, B, C) [P,3] and (effective) opacities [P]: the screen-space half of `outputs`"""
    qi = np.concatenate([np.full(len(a), q, np.int64) for q, a in enumerate(accepted)] + [np.zeros(0, np.int64)])
    gi = np.concatenate(list(accepted) + [np.zeros(0, np.int64)])
    qi, gi = torch.as_tensor(qi), torch.as_tensor(gi)
    d = mu[gi] - uv[qi]
    A, B, C = conic[gi].unbind(-1)
    power = -0.5 * (A * d[:, 0] ** 2 + C * d[:, 1] ** 2) - B * d[:, 0] * d[:, 1]
    a = opacity[gi] * torch.exp(power)
    alpha = a - (a - torch.clamp(a, max=R64.ALPHA_MAX)).detach()  # the 0.99 clamp passes the gradient through
    logT = torch.zeros(uv.shape[0], dtype=D64).index_add(0, qi, torch.log1p(-alpha))
    return torch.exp(logT)
