"""Float64 restatement of the flow plane's per-Gaussian displacement (include/mgs_rasterizer.h, flow plane), in torch so that
its gradients come from autograd rather than from the hand chain of flow.cu.

delta_i = valid_i ? m'_i - m_i : 0, m = screen_mean(mu, view) and m' = screen_mean(mu', next view), both built with
planar_ref64.screen_mean (every camera model).  valid_i: the next mean passes the projection's cull of a mean (view-space
z > NEAR_Z; fisheye theta <= theta_max; distorted r2 <= r_max^2 and det Dd > 0).  Views are planar_ref64's dicts; a
fisheye view's parameters may carry theta_max as a 7th entry and a distorted view's r_max as an 11th.  Differentiable in
both means, the view and projection matrices and tan_fov (pass tensors in the view dict).
"""
import torch

import planar_ref64 as P64

NEAR_Z = 0.2
D64 = torch.float64


def view_space(means3D, view):
    vm = P64._t(view["viewmatrix"]).reshape(4, 4).T
    return means3D @ vm[:3, :3].T + vm[:3, 3]


def valid(means3D, view):
    """[P] bool: the projection's cull of a mean for the view's model"""
    t = view_space(means3D, view).detach()
    x, y, z = t.unbind(-1)
    ok = z > NEAR_Z
    fe, dc = view.get("fisheye"), view.get("distortion")
    if fe is not None and len(fe) > 6:
        ok = ok & (torch.atan2(torch.sqrt(x * x + y * y), z) <= float(fe[6]))
    if dc is not None:
        r_max = float(dc[10]) if len(dc) > 10 else float("inf")
        r2, det = distortion_r2_det(t, dc)
        ok = ok & (r2 <= r_max * r_max) & (det > 0)
    return ok


def distortion_r2_det(t, dc):
    """r2 and det Dd of view-space points t [P,3] under distortion parameters dc (cx, cy, k1, k2, p1, p2, k3, k4, k5, k6[, r_max])"""
    x, y, z = t.unbind(-1)
    cx, cy, k1, k2, p1, p2, k3, k4, k5, k6 = (float(v) for v in dc[:10])
    xn, yn = x / z, y / z
    r2 = xn * xn + yn * yn
    N = 1 + r2 * (k1 + r2 * (k2 + r2 * k3))
    Q = 1 + r2 * (k4 + r2 * (k5 + r2 * k6))
    N1 = k1 + r2 * (2 * k2 + r2 * 3 * k3)
    Q1 = k4 + r2 * (2 * k5 + r2 * 3 * k6)
    R = N / Q
    R1 = (N1 - R * Q1) / Q
    d00 = R + 2 * xn * xn * R1 + 2 * p1 * yn + 6 * p2 * xn
    d01 = 2 * xn * yn * R1 + 2 * p1 * xn + 2 * p2 * yn
    d11 = R + 2 * yn * yn * R1 + 6 * p1 * yn + 2 * p2 * xn
    return r2, d00 * d11 - d01 * d01


def screen_mean(means3D, view):
    return P64.screen_mean(means3D, view)


def delta(means3D, next_means3D, view, next_view=None):
    """(delta [P,2] in pixels, valid [P] bool); next_view: the view with its next-frame pose, or None for the view itself"""
    nv = view if next_view is None else next_view
    ok = valid(next_means3D, nv)
    d = screen_mean(next_means3D, nv) - screen_mean(means3D, view)
    return torch.where(ok.unsqueeze(-1), d, torch.zeros_like(d)), ok
