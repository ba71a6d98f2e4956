"""Float64 restatement of point visibility (include/mgs_rasterizer.h, mgs_visibility_views).

* `project`: (u, v), depth t.z and the cull of each point under a view, with flow_ref64's map of a mean (planar_ref64's
  screen_mean, every camera model) and its cull; `in_view` adds the image bounds [-0.5, W - 0.5) x [-0.5, H - 0.5).
* `transmittance`: T = prod (1 - alpha_i) over the instances of the point's 16x16 tile with depth z_i < d, in the view's
  tile-list order, with blend_ref64's constants (0.99 clamp, 1/255 cut, 1e-4 stop) and its alpha expression evaluated at the
  continuous (u, v).  The view's projected and sorted state (ranges, point_list, means2D, conic_opacity, depths) is an input,
  as in blend_ref64.  Each point also gets a `border` flag where fp32 may decide differently: alpha within a band of 1/255,
  power within a band of 0, z_i within a band of d, T within a band of 1e-4, or u + 0.5 / v + 0.5 within a band of a tile
  edge.
"""
import numpy as np
import torch

import blend_ref64 as R64
import flow_ref64 as F64

BAND = 1e-5    # relative width of the alpha, power and depth decision bands (fp32 rounding of a few operations and expf)
T_BAND = 1e-4  # relative width of the stop's band (the running product drifts by about one rounding per factor)


def project(points, view):
    """(uv [Q,2], depth [Q], ok [Q]) of float64 points [Q,3] under a planar_ref64 view dict; uv and depth NaN where the cull
    fails"""
    p = torch.as_tensor(np.asarray(points, np.float64))
    ok = F64.valid(p, view).numpy()
    uv = F64.screen_mean(p, view).detach().numpy()
    z = F64.view_space(p, view)[:, 2].detach().numpy()
    uv[~ok] = np.nan
    z = np.where(ok, z, np.nan)
    return uv, z, ok


def in_view(uv, ok, W, H):
    u, v = uv[:, 0], uv[:, 1]
    with np.errstate(invalid="ignore"):
        return ok & (u >= -0.5) & (u < W - 0.5) & (v >= -0.5) & (v < H - 0.5)


def tile_of(uv, W, H):
    """the tile of pixel (floor(u + 0.5), floor(v + 0.5)), the pixel clamped into the image"""
    gx = (W + 15) // 16
    ix = np.minimum(np.floor(uv[:, 0] + 0.5), W - 1).astype(np.int64)
    iy = np.minimum(np.floor(uv[:, 1] + 0.5), H - 1).astype(np.int64)
    return (iy // 16) * gx + ix // 16


def transmittance(st, uv, d, inside):
    """(T [Q], border [Q]) of points at uv [Q,2] with depth d [Q]; T = 1 where `inside` is False"""
    Q = len(d)
    T = np.ones(Q)
    border = np.zeros(Q, bool)
    W, H = st["W"], st["H"]
    tiles = tile_of(np.where(inside[:, None], uv, 0.0), W, H)
    for q in np.nonzero(inside)[0]:
        u, v = float(uv[q, 0]), float(uv[q, 1])
        for c in (u + 0.5, v + 0.5):
            r = c % 16.0
            border[q] |= min(r, 16.0 - r) <= 1e-3
        r0, r1 = (int(x) for x in st["ranges"][tiles[q]])
        ids = st["point_list"][r0:r1].astype(np.int64)
        z = st["depths"][ids].astype(np.float64)
        border[q] |= bool(np.isfinite(d[q]) and np.any(np.abs(z - d[q]) <= BAND * abs(d[q])))
        ids = ids[z < d[q]]
        m = st["means2D"][ids].astype(np.float64)
        co = st["conic_opacity"][ids].astype(np.float64)
        dx, dy = m[:, 0] - u, m[:, 1] - v
        a, b, c, o = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
        power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
        mag = 0.5 * (np.abs(a) * dx * dx + np.abs(c) * dy * dy) + np.abs(b * dx * dy)
        alpha = np.minimum(R64.ALPHA_MAX, o * np.exp(power))
        ok = (power <= 0) & (alpha >= R64.ALPHA_MIN)
        near = (np.abs(power) <= BAND * mag) | (np.abs(alpha - R64.ALPHA_MIN) <= BAND * R64.ALPHA_MIN)
        # the running product over the accepted pairs; the walk ends at the first one that would take it below 1e-4
        cp = np.cumprod(np.where(ok, 1.0 - alpha, 1.0))
        stop = ok & (cp < R64.T_STOP)
        end = int(np.argmax(stop)) if stop.any() else len(ids)
        T[q] = cp[end - 1] if end > 0 else 1.0
        walked = np.arange(len(ids)) <= end
        border[q] |= bool(np.any(walked & (near | (ok & (np.abs(cp - R64.T_STOP) <= T_BAND * R64.T_STOP)))))
    return T, border

