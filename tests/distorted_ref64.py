"""Float64 reference of the OpenCV distorted-pinhole projection (include/mgs_rasterizer.h, "Distorted-pinhole views"), with
bounds.

A distorted view maps t = Rv p + tv to (u, v) = (fx xd + cx, fy yd + cy), (xd, yd) OpenCV's radially, tangentially and
rationally distorted (x, y) = t.xy / t.z, and has the Jacobian J = diag(fx, fy) Dd [[1/z, 0, -x/z], [0, 1/z, -y/z]]
(Dd = d(xd, yd) / d(x, y); csrc/distortion.cuh), with no frustum clamp; the depth, dilation, compensation, conic, radius and
extent are the pinhole view's.  The records therefore come from project_ref64.forward with its geometry and screen mean
replaced (the only places the camera model enters the forward), plus the cull r2 > r_max^2 or det Dd <= 0.  The backward
restates project_bwd.cu's chain for distorted views: dL/dt = J^T (du, dv) + dL/dJ : dJ/dt + the depth cotangent, with
(du, dv) = (dm0 / (W / 2), dm1 / (H / 2)), the camera terms with the full J^T Q and no projection matrix, and
dL/dtan_fovx = -(du (u - cx) + sum_j dJ0j J0j) / tan_fovx (y likewise).

Values carry project_ref64's bounds (E: rounding bound e in units of u, inherited bound d).  The map is a rational
polynomial: every term is the kernel's own expression, evaluated in float64 with its first-order rounding bound.

`backward` returns what ortho_ref64.backward returns.  A camera dict carries its parameters under "distortion" =
(cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, r_max).
"""
import contextlib

import numpy as np

import ortho_ref64 as O64
import project_ref64 as P64
from project_ref64 import E, _b, _cot, dot, f32, sqrt, where

# Broken conventions for the sensitivity test (tests/test_distorted_cpu.py): names in MUTATE are applied while set.
MUTATIONS = ("p1_p2_swapped", "k3_from_slot_3", "no_Dd_in_J", "dm_as_pixel_cotangent", "cx_half_pixel")
MUTATE = set()
F = lambda x: float(f32(x))  # noqa: E731


def coefficients(dc):
    """(k1, k2, p1, p2, k3, k4, k5, k6) as the kernels read them from a camera's "distortion" entry (OpenCV's order)"""
    d = [F(v) for v in dc[2:10]]
    if "p1_p2_swapped" in MUTATE:
        d[2], d[3] = d[3], d[2]
    if "k3_from_slot_3" in MUTATE:
        d[4] = d[3]
    return d


def terms(x, y, k, second=True):
    """distortion.cuh's distortion_terms over E arrays: r2, xd, yd, Dd (d00, d01, d11) and (second) hxxx, hxxy, hxyy, hyyy"""
    k1, k2, p1, p2, k3, k4, k5, k6 = k
    xx, yy, xy = x * x, y * y, x * y
    r2 = xx + yy
    N = 1.0 + r2 * (k1 + r2 * (k2 + r2 * k3))
    Q = 1.0 + r2 * (k4 + r2 * (k5 + r2 * k6))
    N1 = k1 + r2 * (E(2.0) * k2 + r2 * (E(3.0) * k3))
    Q1 = k4 + r2 * (E(2.0) * k5 + r2 * (E(3.0) * k6))
    iQ = 1.0 / Q
    R = N * iQ
    R1 = (N1 - R * Q1) * iQ
    o = dict(r2=r2, R=R)
    o["xd"] = x * R + E(2.0 * p1) * xy + p2 * (r2 + 2.0 * xx)
    o["yd"] = y * R + p1 * (r2 + 2.0 * yy) + E(2.0 * p2) * xy
    o["d00"] = R + 2.0 * xx * R1 + E(2.0 * p1) * y + E(6.0 * p2) * x
    o["d01"] = 2.0 * xy * R1 + E(2.0 * p1) * x + E(2.0 * p2) * y
    o["d11"] = R + 2.0 * yy * R1 + E(6.0 * p1) * y + E(2.0 * p2) * x
    if second:
        N2 = E(2.0 * k2) + E(6.0 * k3) * r2
        Q2 = E(2.0 * k5) + E(6.0 * k6) * r2
        R2 = (N2 - 2.0 * R1 * Q1 - R * Q2) * iQ
        o["hxxx"] = x * (6.0 * R1 + 4.0 * xx * R2) + 6.0 * p2
        o["hxxy"] = y * (2.0 * R1 + 4.0 * xx * R2) + 2.0 * p1
        o["hxyy"] = x * (2.0 * R1 + 4.0 * yy * R2) + 2.0 * p2
        o["hyyy"] = y * (6.0 * R1 + 4.0 * yy * R2) + 6.0 * p1
    return o


def _dc(vw):
    return vw["distortion"]


def _t(p, vw):
    Rv, tv = vw["Rv"], vw["tv"]
    return [dot([float(Rv[r][c]) for c in range(3)], p) + float(tv[r]) for r in range(3)]


def _jacobian(t, vw, second=True):
    x_, y_, z = t
    iz = 1.0 / z
    x, y = x_ * iz, y_ * iz
    ds = terms(x, y, coefficients(_dc(vw)), second)
    fx, fy = vw["fx"], vw["fy"]
    if "no_Dd_in_J" in MUTATE:
        d00, d01, d11 = E(np.ones_like(x.v)), E(np.zeros_like(x.v)), E(np.ones_like(x.v))
    else:
        d00, d01, d11 = ds["d00"], ds["d01"], ds["d11"]
    J = [[fx * d00 * iz, fx * d01 * iz, -1.0 * fx * (d00 * x + d01 * y) * iz],
         [fy * d01 * iz, fy * d11 * iz, -1.0 * fy * (d01 * x + d11 * y) * iz]]
    return J, ds, (x, y, iz)


def _geometry(p, S, vw, mutate=()):
    """project_ref64._geometry for a distorted view: same keys (no clamp), plus J, the distortion terms ds and (x, y, iz)"""
    t = _t(p, vw)
    tz = t[2]
    P = tz.v.shape[0]
    J, ds, xyz = _jacobian(t, vw)
    Rv = vw["Rv"]
    m0 = [dot(J[0], [float(Rv[j][c]) for j in range(3)]) for c in range(3)]
    m1 = [dot(J[1], [float(Rv[j][c]) for j in range(3)]) for c in range(3)]
    u0 = [dot(S[c], m0) for c in range(3)]
    u1 = [dot(S[c], m1) for c in range(3)]
    a0, b, c0 = dot(m0, u0), dot(m0, u1), dot(m1, u1)
    a, c = a0 + F(0.3), c0 + F(0.3)
    det = a * c - b * b
    ones = np.ones(P, bool)
    return dict(t=t, tz=tz, inx=ones, iny=ones, cx=E(np.zeros(P)), cy=E(np.zeros(P)), m0=m0, m1=m1, u0=u0, u1=u1, a0=a0,
                c0=c0, a=a, b=b, c=c, det=det, border=np.zeros(P, bool), J=J, ds=ds, xyz=xyz)


def _means2D(p, vw):
    """The distorted screen mean (fx xd + cx, fy yd + cy); h and iw are not used for a distorted view"""
    t = _t(p, vw)
    iz = 1.0 / t[2]
    ds = terms(t[0] * iz, t[1] * iz, coefficients(_dc(vw)), second=False)
    dc = _dc(vw)
    half = 0.5 if "cx_half_pixel" in MUTATE else 0.0
    return [vw["fx"] * ds["xd"] + (F(dc[0]) + half), vw["fy"] * ds["yd"] + (F(dc[1]) + half)], None, None


def view_of(cam, W=None, H=None):
    vw = _VIEW_OF(cam, W, H)
    vw["distortion"] = tuple(cam["distortion"])
    return vw


_VIEW_OF = P64.view_of


@contextlib.contextmanager
def _distorted_model():
    saved = P64._geometry, P64._means2D, P64.view_of
    P64._geometry, P64._means2D, P64.view_of = _geometry, _means2D, view_of
    try:
        yield
    finally:
        P64._geometry, P64._means2D, P64.view_of = saved


def forward(g, cam, scale_modifier=1.0, antialias=False):
    """project.cu's records of one distorted view (project_ref64.forward's dict and bounds), with the fold cull: a mean
    with r2 > r_max^2 or det Dd <= 0 is culled (radius 0, no tiles); either test within 4 u e of its threshold is border."""
    with _distorted_model():
        out = P64.forward(g, cam, scale_modifier, antialias)
        vw = view_of(cam)
        t = _t(P64._cols(g["means3D"]), vw)
        iz = 1.0 / t[2]
        ds = terms(t[0] * iz, t[1] * iz, coefficients(cam["distortion"]), second=False)
    r2max = F(cam["distortion"][10]) ** 2
    r2max = float(f32(r2max)) if np.isfinite(r2max) else np.inf
    detd = ds["d00"] * ds["d11"] - ds["d01"] * ds["d01"]
    front = t[2].v > P64.NEAR_Z
    cut = ((ds["r2"].v > r2max) | (detd.v <= 0)) & front
    out["culled"] = out["culled"] | cut
    out["radius"] = np.where(out["culled"], 0, out["radius"])
    out["tiles_touched"] = np.where(out["culled"], 0, out["tiles_touched"])
    border = P64.within(detd, 0.0) & front
    if np.isfinite(r2max):
        border |= P64.within(ds["r2"], r2max) & front
    out["border"] = out["border"] | border
    out["r2"], out["det_Dd"] = ds["r2"].v, detd.v
    return out


def _view(g, cam, c, S, lv, cl, antialias):
    """One distorted view's contributions, in ortho_ref64._view's layout"""
    with _distorted_model():
        return _view_distorted(g, cam, c, S, lv, cl, antialias)


def _view_distorted(g, cam, c, S, lv, cl, antialias):
    p = P64._cols(g["means3D"])
    P = p[0].v.shape[0]
    vw = view_of(cam)
    zero = E(np.zeros(P))
    gate = lambda x: where(lv, x, 0.0)  # noqa: E731
    dm = [gate(_cot(c["dL_dmean2D"][:, i], _b(c, "dL_dmean2D", i))) for i in range(2)]
    # dm is w.r.t. ndc = (2 u + 1) / W - 1 (the blend's convention); the distorted mean (u, v) is in pixels
    du = dm if "dm_as_pixel_cotangent" in MUTATE else [dm[0] / (0.5 * cam["W"]), dm[1] / (0.5 * cam["H"])]
    gA, gB, gC = (gate(_cot(c["dL_dconic"][:, i], _b(c, "dL_dconic", i))) for i in range(3))
    gop_v = gate(_cot(c["dL_dopacity"], _b(c, "dL_dopacity")))
    dcol = [gate(_cot(c["dL_dcolor"][:, i], _b(c, "dL_dcolor", i))) for i in range(3)]
    dd = c.get("dL_ddepth")
    ddepth = gate(_cot(dd, c.get("dL_ddepth_B"))) if dd is not None else zero
    G = _geometry(p, S, vw)
    a, b, cc, det = G["a"], G["b"], G["c"], G["det"]
    m0, m1, u0, u1 = G["m0"], G["m1"], G["u0"], G["u1"]
    wgt = 1.0 / (det * det + F(1e-7))
    e00, e01 = cc * gA - b * gB, cc * gB - b * gC
    e10, e11 = a * gB - b * gA, a * gC - b * gB
    H00 = -wgt * (e00 * cc - e01 * b)
    H01 = -wgt * (e01 * a - e00 * b)
    H11 = -wgt * (e11 * a - e10 * b)
    if antialias:
        o_raw = E(np.asarray(g["opacities"], f32).reshape(-1).astype(np.float64))
        a0, c0 = G["a0"], G["c0"]
        d0 = a0 * c0 - b * b
        r = d0 / det
        on = r.v > P64.AA_CLAMP
        s_ = sqrt(where(on, r, P64.AA_CLAMP))
        gop = where(lv, s_ * gop_v, 0.0)
        k = 0.5 * gop_v * (o_raw * s_)
        i0 = 1.0 / where(on, d0, 1.0)
        i1 = 1.0 / det
        H00 = H00 + where(on, k * (c0 * i0 - cc * i1), 0.0)
        H11 = H11 + where(on, k * (a0 * i0 - a * i1), 0.0)
        H01 = H01 + where(on, k * b * (i1 - i0), 0.0)
    else:
        gop = gop_v
    h0 = [H00 * m0[i] + H01 * m1[i] for i in range(3)]
    h1 = [H01 * m0[i] + H11 * m1[i] for i in range(3)]
    D = [[where(lv, m0[i] * h0[j] + m1[i] * h1[j], 0.0) if j >= i else None for j in range(3)] for i in range(3)]
    Rv = vw["Rv"]
    q0 = [2.0 * (H00 * u0[i] + H01 * u1[i]) for i in range(3)]
    q1 = [2.0 * (H01 * u0[i] + H11 * u1[i]) for i in range(3)]
    dJ = [[dot(q, [float(x) for x in Rv[j]]) for j in range(3)] for q in (q0, q1)]
    J, ds = G["J"], G["ds"]
    nx, ny, iz = G["xyz"]
    fx, fy = vw["fx"], vw["fy"]
    # G = F dL/dJ; K = G P^T against dDd/d(x, y); N = Dd G against dP/dt; (gx, gy) = dL/d(x, y), with J^T (du, dv)
    G0 = [fx * dJ[0][j] for j in range(3)]
    G1 = [fy * dJ[1][j] for j in range(3)]
    K00 = (G0[0] - nx * G0[2]) * iz
    Kx = (G0[1] - ny * G0[2] + G1[0] - nx * G1[2]) * iz
    K11 = (G1[1] - ny * G1[2]) * iz
    eu, ev = fx * du[0], fy * du[1]
    gx = K00 * ds["hxxx"] + Kx * ds["hxxy"] + K11 * ds["hxyy"] + ds["d00"] * eu + ds["d01"] * ev
    gy = K00 * ds["hxxy"] + Kx * ds["hxyy"] + K11 * ds["hyyy"] + ds["d01"] * eu + ds["d11"] * ev
    N00 = ds["d00"] * G0[0] + ds["d01"] * G1[0]
    N02 = ds["d00"] * G0[2] + ds["d01"] * G1[2]
    N11 = ds["d01"] * G0[1] + ds["d11"] * G1[1]
    N12 = ds["d01"] * G0[2] + ds["d11"] * G1[2]
    dt = [(gx - N02 * iz) * iz, (gy - N12 * iz) * iz,
          (2.0 * (N02 * nx + N12 * ny) - N00 - N11) * (iz * iz) - (gx * nx + gy * ny) * iz + ddepth]
    gp = [where(lv, dot([float(Rv[0][i]), float(Rv[1][i]), float(Rv[2][i])], dt), 0.0) for i in range(3)]
    terms_ = []
    for cidx in range(4):
        for r in range(3):
            if cidx < 3:
                terms_.append(dt[r] * p[cidx] + J[0][r] * q0[cidx] + J[1][r] * q1[cidx])
            else:
                terms_.append(dt[r])
    terms_ += [zero] * 12          # projmatrix is not read
    has_sh = g.get("shs") is not None
    dsh, cp = None, [zero, zero, zero]
    if has_sh:
        deg = int(g["sh_degree"])
        sh = np.asarray(g["shs"], f32).astype(np.float64)
        M = sh.shape[1]
        dRGB = [where(((cl >> ch) & 1).astype(bool), 0.0, dcol[ch]) for ch in range(3)]
        vv, ln = P64._direction(p, vw)
        il = 1.0 / ln
        xd, yd, zd = (vi * il for vi in vv)
        basis = P64._sh_basis(xd, yd, zd, deg)
        ddir = [zero, zero, zero]
        dsh = [[zero] * 3 for _ in range(M)]
        for kk in range((deg + 1) ** 2):
            B_, grad = basis[kk]
            for ch in range(3):
                if kk < M:
                    dsh[kk][ch] = B_ * dRGB[ch]
            s_ = dot([E(sh[:, kk, ch]) for ch in range(3)], dRGB)
            ddir = [ddir[i] + P64._e(grad[i]) * s_ for i in range(3)]
        along = dot([xd, yd, zd], ddir)
        for i, di in enumerate((xd, yd, zd)):
            t_ = (ddir[i] - di * along) * il
            gp[i] = gp[i] + where(lv, t_, 0.0)
            cp[i] = -1.0 * t_
    terms_ += cp
    ax = fx * ds["xd"]     # u - cx
    ay = fy * ds["yd"]
    tanx, tany = F(cam["tanfovx"]), F(cam["tanfovy"])
    intr = [-1.0 * (du[0] * ax + dot(dJ[0], J[0])) / tanx, -1.0 * (du[1] * ay + dot(dJ[1], J[1])) / tany]
    return dict(gp=gp, D=D, gop=where(lv, gop, 0.0), dm=dm, dcol=dcol, dsh=dsh, cam=[where(lv, t_, 0.0) for t_ in terms_],
                intr=[where(lv, t_, 0.0) for t_ in intr])


def backward(g, cams, cot, scale_modifier=1.0, antialias=False, live=None, clamped=None, shared_mean2D=False):
    """project_bwd.cu's per-Gaussian chain over the distorted views `cams` (ortho_ref64.backward's arguments and results)"""
    saved = O64.forward, O64._view
    O64.forward, O64._view = forward, _view
    try:
        return O64.backward(g, cams, cot, scale_modifier, antialias, live, clamped, shared_mean2D)
    finally:
        O64.forward, O64._view = saved


def distorted_cam(W, H, fx, fy, cx, cy, D, c2w, r_max=None):
    """A camera dict in project_ref64's layout of a distorted view: tanfovx = W / (2 fx), the pinhole projmatrix of the
    same K (not read by the kernels), and "distortion" = (cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, r_max) from OpenCV's D
    (4, 5 or 8 entries)."""
    from manigaussian_b200 import cameras
    w2c = np.linalg.inv(np.asarray(c2w, np.float64))
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    proj = cameras.projection_from_intrinsics(0.1, 10.0, K, H, W)
    wvt = w2c.T
    d8 = list(np.asarray(D, np.float64)) + [0.0] * (8 - len(D))
    rm = float(cameras.distortion_r_max(np.asarray(D, np.float64))[0]) if r_max is None else float(r_max)
    return dict(W=W, H=H, tanfovx=W / (2.0 * fx), tanfovy=H / (2.0 * fy), viewmatrix=wvt.astype(np.float32),
                projmatrix=(wvt @ proj.T).astype(np.float32), campos=np.linalg.inv(wvt)[3, :3].astype(np.float32),
                distortion=(float(cx), float(cy), *(float(x) for x in d8), rm))
