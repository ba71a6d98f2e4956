"""Float64 restatement of TSDF fusion (include/mgs_rasterizer.h, mgs_tsdf_fuse).

For each voxel centre x (voxel_centres' float32 point, taken exactly into float64) and the views in order: the map and
cull of every camera model come from visibility_ref64.project (planar_ref64's screen_mean and flow_ref64's cull), the
pixel is (floor(px + 0.5), floor(py + 0.5)) inside [-0.5, W - 0.5) x [-0.5, H - 0.5), d = depth[v, j, i] is skipped where
it is not finite or <= 0, s = d - z is skipped below -trunc, and f = min(1, s / trunc) enters the running averages of the
tsdf and the colour with unit weights.

`border` flags the voxels where the kernel's float32 may decide a view differently: px or py within BAND_PX of a
half-integer (the pixel and the image bounds; BAND_PX is relative to W + H, the scale of the fp32 pixel map's rounding),
s within a relative BAND of -trunc, z within BAND of NEAR_Z, a fisheye's
theta within BAND of theta_max, or a distorted view's r2 within BAND of r_max^2 or det Dd within BAND of 0.
"""
import numpy as np
import torch

import flow_ref64 as F64
import visibility_ref64 as V64

BAND = 1e-5     # relative width of the depth, truncation and cull decision bands
# pixels per pixel of W + H: the fp32 map forms (ndc + 1) W / 2 from an ndc carrying a few ulps of error, ~1e-4 px at W = 640
BAND_PX = 1e-6


def _cull_border(p, view):
    t = F64.view_space(torch.as_tensor(p), view).numpy()
    x, y, z = t[:, 0], t[:, 1], t[:, 2]
    b = np.abs(z - F64.NEAR_Z) <= BAND * np.maximum(1.0, np.abs(z))
    fe, dc = view.get("fisheye"), view.get("distortion")
    if fe is not None and len(fe) > 6:
        th = np.arctan2(np.sqrt(x * x + y * y), z)
        b |= np.abs(th - float(fe[6])) <= BAND
    if dc is not None:
        with np.errstate(divide="ignore", invalid="ignore"):
            r2, det = (a.numpy() for a in F64.distortion_r2_det(torch.as_tensor(t), dc))
        r_max = float(dc[10]) if len(dc) > 10 else float("inf")
        if np.isfinite(r_max):
            b |= np.abs(r2 - r_max * r_max) <= BAND * r_max * r_max
        b |= np.abs(det) <= BAND
    return b


def fuse(points, views, depth, trunc, color=None, state=None):
    """(tsdf [Q], weight [Q], color [Q,C] or None, border [Q]) of float32 points [Q,3] (as float64) under views (planar_ref64
    dicts, each with W and H), depth [V,H,W] and color [V,C,H,W] (numpy float32); state: an earlier (tsdf, weight, color)
    to continue from"""
    p = np.asarray(points, np.float64)
    Q = len(p)
    C = 0 if color is None else color.shape[1]
    if state is None:
        ts, w, col = np.ones(Q), np.zeros(Q), np.zeros((Q, C))
    else:
        ts, w = (np.array(a, np.float64) for a in state[:2])
        col = np.array(state[2], np.float64) if C else np.zeros((Q, 0))
    border = np.zeros(Q, bool)
    for v, view in enumerate(views):
        W, H = view["W"], view["H"]
        uv, z, ok = V64.project(p, view)
        border |= _cull_border(p, view)
        inside = V64.in_view(uv, ok, W, H)
        with np.errstate(invalid="ignore"):
            for c in (uv[:, 0] + 0.5, uv[:, 1] + 0.5):
                border |= ok & (np.abs(c - np.round(c)) <= BAND_PX * (W + H))
        ii = np.where(inside, np.minimum(np.floor(np.where(inside, uv[:, 0], 0) + 0.5), W - 1), 0).astype(np.int64)
        jj = np.where(inside, np.minimum(np.floor(np.where(inside, uv[:, 1], 0) + 0.5), H - 1), 0).astype(np.int64)
        d = depth[v][jj, ii].astype(np.float64)
        live = inside & np.isfinite(d) & (d > 0)
        s = np.where(live, d - np.where(live, z, 0), 0.0)
        border |= live & (np.abs(s + trunc) <= BAND * np.maximum(1.0, np.abs(d)))
        upd = live & (s >= -trunc)
        f = np.minimum(1.0, s / trunc)
        w1 = w + 1
        ts = np.where(upd, (ts * w + f) / w1, ts)
        if C:
            cv = color[v][:, jj, ii].T.astype(np.float64)
            col = np.where(upd[:, None], (col * w[:, None] + cv) / w1[:, None], col)
        w = np.where(upd, w1, w)
    return ts, w, (col if C else None), border


def plane_closed_form(points, view, D, trunc):
    """(tsdf, weight) of one pinhole view of the fronto-parallel plane at view-space depth D (depth image D everywhere),
    for points that project inside the image: min(1, (D - z) / trunc) with weight 1 where D - z >= -trunc, else 1, 0"""
    z = F64.view_space(torch.as_tensor(np.asarray(points, np.float64)), view)[:, 2].numpy()
    s = D - z
    upd = (s >= -trunc) & (z > F64.NEAR_Z)
    return np.where(upd, np.minimum(1.0, s / trunc), 1.0), upd.astype(np.float64)
