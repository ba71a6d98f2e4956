"""Float64 restatement of camera rays (include/mgs_rasterizer.h, mgs_camera_rays), in torch, built on the forward maps the
other references share (planar_ref64.screen_mean / _map, flow_ref64's culls), so that a ray is checked against the map it
inverts rather than against a second statement of the inverse.

* Pinhole and orthographic: the 3x3 system of the header, solved with torch.linalg.solve.
* Fisheye: theta from theta rho(theta) = theta_d by bisection to float64 precision, then (X, Y) = tan(theta) (xd, yd) / theta_d.
* Both lens models: p = Rv^-1 (z (X, Y, 1) - tv), Rv^T (...) for a rigid pose.
* Distorted: Newton's method on the lens map at t.z = 1 to float64 precision.
* Gradients: the lens solutions are found without autograd, then one Newton step of the forward map is taken with autograd on;
  at the root that step's derivative is the implicit-function derivative -J^-1 dF, so the pixels, the view and projection
  matrices and tan_fov reach the rays exactly to first order.  The fisheye axis pixel (theta_d = 0) is (0, 0) with no
  correction step: the forward reference has no value there.

A view is planar_ref64's dict; a fisheye view's parameters carry theta_max as a 7th entry and a distorted view's r_max as an
11th (flow_ref64's convention).
"""
import numpy as np
import torch

import flow_ref64 as F64
import planar_ref64 as P64

D64 = torch.float64


def _focal(view):
    return view["W"] / (2.0 * P64._t(view["tanfovx"])), view["H"] / (2.0 * P64._t(view["tanfovy"]))


def _rho(th, k):
    t2 = th * th
    return 1 + t2 * (k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3])))


def fisheye_theta(theta_d, fe):
    """theta in [0, theta_max] with theta rho(theta) = theta_d (float64 numpy), and whether theta_d <= theta_max rho(theta_max)"""
    k, tmax = [float(x) for x in fe[2:6]], float(fe[6])
    ok = theta_d <= tmax * _rho(tmax, k)
    lo, hi = np.zeros_like(theta_d), np.full_like(theta_d, tmax)
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        big = mid * _rho(mid, k) > theta_d
        hi, lo = np.where(big, mid, hi), np.where(big, lo, mid)
    return 0.5 * (lo + hi), ok


def _lens_jacobian(XY, view):
    """(xd, yd)-space residual map's value [Q,2] and Jacobian [Q,2,2] in pixels at t = (X, Y, 1)"""
    t = torch.cat([XY, torch.ones_like(XY[:, :1])], -1).detach().requires_grad_(True)
    vw = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in view.items()}
    with torch.enable_grad():
        uv = P64._map(t, vw)
        rows = [torch.autograd.grad(uv[:, j].sum(), t, retain_graph=True)[0][:, :2] for j in range(2)]
    return uv.detach(), torch.stack(rows, -2)


def _unmap(pixels, view):
    """(X, Y) [Q,2] with the view's lens map at t = (X, Y, 1) equal to pixels, and valid [Q]"""
    fx, fy = _focal(view)
    fe, dc = view.get("fisheye"), view.get("distortion")
    c = fe if fe is not None else dc
    with torch.no_grad():
        xd = ((pixels[:, 0] - float(c[0])) / fx).numpy()
        yd = ((pixels[:, 1] - float(c[1])) / fy).numpy()
        if fe is not None:
            td = np.hypot(xd, yd)
            th, ok = fisheye_theta(td, fe)
            s = np.where(td > 0, np.tan(th) / np.where(td > 0, td, 1.0), 1.0)
            XY = torch.tensor(np.stack([s * xd, s * yd], -1), dtype=D64)
            ok = ok & np.isfinite(s) & (s >= 0)
            axis = torch.as_tensor(td == 0)
        else:
            XY = torch.tensor(np.stack([xd, yd], -1), dtype=D64)
            for _ in range(60):
                uv, J = _lens_jacobian(XY, view)
                step = torch.linalg.solve(J, (pixels.detach() - uv).unsqueeze(-1)).squeeze(-1)
                XY = XY + torch.nan_to_num(step)
            uv, _ = _lens_jacobian(XY, view)
            r_max = float(dc[10]) if len(dc) > 10 else float("inf")
            r2, det = F64.distortion_r2_det(torch.cat([XY, torch.ones_like(XY[:, :1])], -1), dc)
            ok = ((r2 <= r_max * r_max) & (det > 0) & ((uv - pixels.detach()).norm(dim=-1) <= 1e-9 * (1 + fx.detach()))).numpy()
            axis = torch.zeros(len(XY), dtype=torch.bool)
    # one Newton step with autograd on: the implicit derivative at the root
    safe = torch.where(axis[:, None], torch.full_like(XY, 1e-3), XY)
    _, J = _lens_jacobian(safe, view)
    uv = P64._map(torch.cat([safe, torch.ones_like(safe[:, :1])], -1), view)
    stepped = safe - torch.linalg.solve(J, (uv - pixels).unsqueeze(-1)).squeeze(-1)
    return torch.where(axis[:, None], XY, stepped), torch.as_tensor(ok)


def rays(pixels, view):
    """(origin [Q,3], direction [Q,3], valid [Q] bool) of pixel positions [Q,2] (float64) in the view; origin and direction
    are NaN where invalid.  Differentiable in pixels and the view's tensors (viewmatrix, projmatrix, tanfovx, tanfovy)."""
    vm = P64._t(view["viewmatrix"]).reshape(4, 4).T  # row-major: t = vm[:3, :3] p + vm[:3, 3]
    Q = pixels.shape[0]
    if view.get("fisheye") is not None or view.get("distortion") is not None:
        XY, ok = _unmap(pixels, view)
        Rv, tv = vm[:3, :3], vm[:3, 3]
        Ri = torch.linalg.inv(Rv)
        origin = (-(Ri @ tv)).expand(Q, 3)
        direction = torch.cat([XY, torch.ones_like(XY[:, :1])], -1) @ Ri.T
        ok = ok & torch.isfinite(torch.linalg.det(Rv.detach())) & (torch.linalg.det(Rv.detach()) != 0)
    else:
        pm = P64._t(view["projmatrix"]).reshape(4, 4).T  # h = pm[:, :3] p + pm[:, 3]
        nx = (2 * pixels[:, 0] + 1) / view["W"] - 1
        ny = (2 * pixels[:, 1] + 1) / view["H"] - 1
        A = torch.stack([pm[0, :3] - nx[:, None] * pm[3, :3], pm[1, :3] - ny[:, None] * pm[3, :3], vm[2, :3].expand(Q, 3)], -2)
        w = pm[3, 3] + 1e-7
        b = torch.stack([nx * w - pm[0, 3], ny * w - pm[1, 3], (-vm[2, 3]).expand(Q)], -1)
        det = torch.linalg.det(A.detach())
        ok = torch.isfinite(det) & (det != 0)
        e3 = torch.zeros_like(b)
        e3[:, 2] = 1
        sol = torch.linalg.solve(A, torch.stack([b, e3], -1))
        origin, direction = sol[..., 0], sol[..., 1]
    nan = torch.full_like(direction, float("nan"))
    return torch.where(ok[:, None], origin, nan), torch.where(ok[:, None], direction, nan), ok


def round_trip(origin, direction, z, view):
    """screen_mean of origin + z direction (z [Q] or a scalar), and its view-space depth"""
    p = origin + (z[:, None] if torch.is_tensor(z) and z.dim() else z) * direction
    return F64.screen_mean(p, view), F64.view_space(p, view)[:, 2]
