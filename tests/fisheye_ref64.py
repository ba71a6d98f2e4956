"""Float64 reference of the Kannala-Brandt fisheye projection (include/mgs_rasterizer.h, "Fisheye views"), with bounds.

A fisheye view maps t = Rv p + tv to (u, v) = (fx a t.x + cx, fy a t.y + cy), a = theta_d / r, and has the Jacobian
J = [[fx (a + c x^2), fx c x y, -fx x g], [fy c x y, fy (a + c y^2), -fy y g]] (c = (b - a) / r^2, b = D1 z / s, g = D1 / s;
csrc/fisheye.cuh), with no frustum clamp; the depth, dilation, compensation, conic, radius and extent are the pinhole
view's.  The records therefore come from project_ref64.forward with its geometry and screen mean replaced (the only places
the camera model enters the forward), plus the theta_max cull.  The backward restates project_bwd.cu's chain for fisheye
views: dL/dt = J^T (du, dv) + dL/dJ : dJ/dt + the depth cotangent, with (du, dv) = (dm0 / (W / 2), dm1 / (H / 2)) the
pixel-space cotangent of the mean (the blend's dL/dmean2D, dm, is w.r.t. ndc), the camera terms take the full J^T Q and
no projection matrix, and dL/dtan_fovx = -(du (u - cx) + sum_j dJ0j J0j) / tan_fovx (y likewise).

Values carry project_ref64's bounds (E: rounding bound e in units of u, inherited bound d).  Each radial term's value is
the model's (the closed form in float64, or below r / z = 1e-3 its series to (r/z)^6, exact to float64 there); its bound is
the rounding bound of the kernel's own expression -- the closed form, or below r / z = 1/8 (SERIES_E2) the truncated series
-- plus, on the series branch, the truncation bound of that series (its first omitted term, times 2).

`backward` returns what ortho_ref64.backward returns: per-Gaussian sums over the views, per view the 35 camera outputs and
the 2 tan_fov outputs.  A camera dict carries its fisheye parameters under "fisheye" = (cx, cy, k1, k2, k3, k4, theta_max).
"""
import contextlib

import numpy as np

import ortho_ref64 as O64
import project_ref64 as P64
from blend_ref64 import U
from project_ref64 import E, _b, _cot, dot, f32, sqrt, where

SERIES_E2 = 1.0 / 64.0   # fisheye.cuh FISHEYE_SERIES_E2
# Broken conventions for the sensitivity test (tests/test_fisheye_cpu.py): names in MUTATE are applied while set.
MUTATIONS = ("theta_r_over_z", "no_rho_prime_in_J", "no_JT_dm", "dm_as_pixel_cotangent", "cx_half_pixel")
MUTATE = set()
F = lambda x: float(f32(x))  # noqa: E731


def _atan2(y, x):
    """atan2 with a bound: the first-order propagation of the operands' bounds plus 4 |result| (CUDA's atan2f is within a
    few ulp)"""
    v = np.arctan2(y.v, x.v)
    s = y.v * y.v + x.v * x.v
    k = 1.0 / np.where(s > 0, s, 1.0)
    return E(v, (np.abs(x.v) * y.e + np.abs(y.v) * x.e) * k + 4.0 * np.abs(v), (np.abs(x.v) * y.d + np.abs(y.v) * x.d) * k)


def _model(v, kern, trunc=0.0):
    """E with the model's value v, the kernel expression kern's bounds, plus an absolute truncation bound"""
    return E(v, kern.e + np.asarray(trunc) / U + 0 * v, kern.d + 0 * v)


def _series_coefs(k):
    k1, k2, k3, k4 = k
    return (2 * k1 - 2 / 3, 4 * (k2 - k1) + 0.8, 5.6 * k1 - 10 * k2 + 6 * k3 - 6 / 7,
            -6544 * k1 / 945 + 152 * k2 / 9 - 56 * k3 / 3 + 8 * k4 + 8 / 9)


def radial(x, y, z, k, second=True):
    """fisheye.cuh's fisheye_radial over E arrays: theta, a, c, g and (second) C1, cz, gz"""
    k1, k2, k3, k4 = (F(v) for v in k)
    r2 = x * x + y * y
    r = sqrt(r2)
    s = r2 + z * z
    is_ = 1.0 / s
    iz = 1.0 / z
    th = _atan2(r, z) if "theta_r_over_z" not in MUTATE else r / z
    t2 = th * th
    rho = 1.0 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)))
    D1 = 1.0 + t2 * (E(3.0) * k1 + t2 * (E(5.0) * k2 + t2 * (E(7.0) * k3 + t2 * (E(9.0) * k4))))
    e2 = r2 * iz * iz
    ser = e2.v < SERIES_E2
    tiny = e2.v < 1e-6
    rs = np.where(r.v > 0, r.v, 1.0)
    r2s = np.where(r2.v > 0, r2.v, 1.0)
    # kernel expressions on both branches (the value of the untaken one is replaced below)
    q_ser = iz * (1.0 + e2 * (F(-1 / 3) + e2 * (F(0.2) + e2 * F(-1 / 7))))
    q_dir = th / E(rs, r.e, r.d)
    c0, c1, c2, c3 = _series_coefs((k1, k2, k3, k4))
    c0k, c1k = E(2.0) * k1 - F(2 / 3), E(4.0) * (E(k2) - k1) + F(0.8)
    c2k = E(F(5.6)) * k1 - E(10.0) * k2 + E(6.0) * k3 - F(6 / 7)
    iz3 = iz * iz * iz
    a_k = where(ser, q_ser, q_dir) * rho
    c_ser = iz3 * (c0k + e2 * (c1k + e2 * c2k))
    c_dir = (D1 * z * is_ - a_k) / E(r2s, r2.e, r2.d)
    # model values: closed form, or (r / z < 1e-3) the series to e^6
    zz, ee = z.v, e2.v
    qv = np.where(tiny, (1 - ee / 3 + ee ** 2 / 5 - ee ** 3 / 7) / zz, th.v / rs)
    av = qv * rho.v
    cv = np.where(tiny, (c0 + ee * (c1 + ee * (c2 + ee * c3))) / zz ** 3, (D1.v * zz / s.v - av) / r2s)
    tq = ee ** 4 / 9 / zz * 2
    tc = np.abs(c3) * ee ** 3 / zz ** 3 * 2
    out = dict(theta=th, rho=rho, D1=D1, series=ser)
    out["a"] = _model(av, a_k, np.where(ser, tq * np.abs(rho.v), 0.0))
    out["g"] = D1 * is_
    out["c"] = _model(cv, where(ser, c_ser, c_dir), np.where(ser, tc, 0.0))
    if second:
        D2r_k = where(ser, q_ser, q_dir) * (E(6.0) * k1 + t2 * (E(20.0) * k2 + t2 * (E(42.0) * k3 + t2 * (E(72.0) * k4))))
        D2r = qv * (6 * k1 + t2.v * (20 * k2 + t2.v * (42 * k3 + t2.v * 72 * k4)))
        is2 = is_ * is_
        C1_ser = iz3 * iz * iz * (2.0 * c1k + E(4.0) * c2k * e2)
        C1_dir = ((D2r_k * z * z - 2.0 * z * D1) * is2 - 3.0 * where(ser, c_ser, c_dir)) / E(r2s, r2.e, r2.d)
        C1v = np.where(tiny, (2 * c1 + ee * (4 * c2 + ee * 6 * c3)) / zz ** 5,
                       ((D2r * zz * zz - 2 * zz * D1.v) / s.v ** 2 - 3 * cv) / r2s)
        out["C1"] = _model(C1v, where(ser, C1_ser, C1_dir), np.where(ser, 6 * np.abs(c3) * ee ** 2 / zz ** 5 * 2, 0.0))
        cz_k = (2.0 * D1 - D2r_k * z) * is2
        gz_k = -1.0 * (D2r_k * r2 + 2.0 * z * D1) * is2
        out["cz"] = _model((2 * D1.v - D2r * zz) / s.v ** 2, cz_k, np.where(ser, tq * np.abs(D2r * zz) / s.v ** 2, 0.0))
        out["gz"] = _model(-(D2r * r2.v + 2 * zz * D1.v) / s.v ** 2, gz_k, 0.0)
    return out


def _fe(vw):
    return vw["fisheye"]


def _jacobian(t, vw):
    x, y, z = t
    fr = radial(x, y, z, _fe(vw)[2:6])
    fx, fy = vw["fx"], vw["fy"]
    cxy = fr["c"] * x * y
    g = fr["g"] if "no_rho_prime_in_J" not in MUTATE else fr["g"] / fr["D1"]
    J = [[fx * (fr["a"] + fr["c"] * x * x), fx * cxy, -fx * x * g],
         [fy * cxy, fy * (fr["a"] + fr["c"] * y * y), -fy * y * g]]
    return J, fr


def _geometry(p, S, vw, mutate=()):
    """project_ref64._geometry for a fisheye view: same keys (no clamp), plus J and the radial terms fr"""
    Rv, tv = vw["Rv"], vw["tv"]
    t = [dot([float(Rv[r][c]) for c in range(3)], p) + float(tv[r]) for r in range(3)]
    tz = t[2]
    P = tz.v.shape[0]
    J, fr = _jacobian(t, vw)
    m0 = [dot(J[0], [float(Rv[j][c]) for j in range(3)]) for c in range(3)]
    m1 = [dot(J[1], [float(Rv[j][c]) for j in range(3)]) for c in range(3)]
    u0 = [dot(S[c], m0) for c in range(3)]
    u1 = [dot(S[c], m1) for c in range(3)]
    a0, b, c0 = dot(m0, u0), dot(m0, u1), dot(m1, u1)
    a, c = a0 + F(0.3), c0 + F(0.3)
    det = a * c - b * b
    ones = np.ones(P, bool)
    return dict(t=t, tz=tz, inx=ones, iny=ones, cx=E(np.zeros(P)), cy=E(np.zeros(P)), m0=m0, m1=m1, u0=u0, u1=u1, a0=a0,
                c0=c0, a=a, b=b, c=c, det=det, border=np.zeros(P, bool), J=J, fr=fr)


def _means2D(p, vw):
    """The fisheye screen mean (fx a t.x + cx, fy a t.y + cy); h and iw are not used for a fisheye view"""
    Rv, tv = vw["Rv"], vw["tv"]
    t = [dot([float(Rv[r][c]) for c in range(3)], p) + float(tv[r]) for r in range(3)]
    fr = radial(t[0], t[1], t[2], _fe(vw)[2:6], second=False)
    fe = _fe(vw)
    half = 0.5 if "cx_half_pixel" in MUTATE else 0.0
    return [vw["fx"] * fr["a"] * t[0] + (F(fe[0]) + half), vw["fy"] * fr["a"] * t[1] + (F(fe[1]) + half)], None, None


def view_of(cam, W=None, H=None):
    vw = _VIEW_OF(cam, W, H)
    vw["fisheye"] = tuple(cam["fisheye"])
    return vw


_VIEW_OF = P64.view_of


@contextlib.contextmanager
def _fisheye_model():
    saved = P64._geometry, P64._means2D, P64.view_of
    P64._geometry, P64._means2D, P64.view_of = _geometry, _means2D, view_of
    try:
        yield
    finally:
        P64._geometry, P64._means2D, P64.view_of = saved


def forward(g, cam, scale_modifier=1.0, antialias=False):
    """project.cu's records of one fisheye view (project_ref64.forward's dict and bounds), with the theta_max cull: a mean
    with theta > theta_max is culled (radius 0, no tiles); a theta within 4 u e of theta_max is border."""
    with _fisheye_model():
        out = P64.forward(g, cam, scale_modifier, antialias)
        vw = view_of(cam)
        p = P64._cols(g["means3D"])
        t = [dot([float(vw["Rv"][r][c]) for c in range(3)], p) + float(vw["tv"][r]) for r in range(3)]
        th = radial(t[0], t[1], t[2], vw["fisheye"][2:6], second=False)["theta"]
    tmax = F(cam["fisheye"][6])
    cut = (th.v > tmax) & (t[2].v > P64.NEAR_Z)
    out["culled"] = out["culled"] | cut
    out["radius"] = np.where(out["culled"], 0, out["radius"])
    out["tiles_touched"] = np.where(out["culled"], 0, out["tiles_touched"])
    out["border"] = out["border"] | P64.within(th, tmax)
    out["theta"] = th.v
    return out


def _view(g, cam, c, S, lv, cl, antialias):
    """One fisheye view's contributions, in ortho_ref64._view's layout"""
    with _fisheye_model():
        return _view_fisheye(g, cam, c, S, lv, cl, antialias)


def _view_fisheye(g, cam, c, S, lv, cl, antialias):
    p = P64._cols(g["means3D"])
    P = p[0].v.shape[0]
    vw = view_of(cam)
    zero = E(np.zeros(P))
    gate = lambda x: where(lv, x, 0.0)  # noqa: E731
    dm = [gate(_cot(c["dL_dmean2D"][:, i], _b(c, "dL_dmean2D", i))) for i in range(2)]
    # dm is w.r.t. ndc = (2 u + 1) / W - 1 (the blend's convention); the fisheye mean (u, v) is in pixels
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
    J, fr = G["J"], G["fr"]
    x, y, _ = G["t"]
    fx, fy = vw["fx"], vw["fy"]
    A, Bs, Cc = fx * dJ[0][0], fx * dJ[0][1] + fy * dJ[1][0], fx * dJ[0][2]
    Ee, Ff = fy * dJ[1][1], fy * dJ[1][2]
    c_, C1, cz, g_, gz = fr["c"], fr["C1"], fr["cz"], fr["g"], fr["gz"]
    cx2, cy2 = c_ + C1 * x * x, c_ + C1 * y * y
    dt = [A * x * (2.0 * c_ + cx2) + Bs * y * cx2 + Ee * x * cy2 - Cc * (g_ - cz * x * x) + Ff * cz * x * y,
          A * y * cx2 + Bs * x * cy2 + Ee * y * (2.0 * c_ + cy2) + Cc * cz * x * y - Ff * (g_ - cz * y * y),
          A * (cz * x * x - g_) + Bs * cz * x * y + Ee * (cz * y * y - g_) - (Cc * x + Ff * y) * gz + ddepth]
    if "no_JT_dm" not in MUTATE:
        dt = [dt[i] + J[0][i] * du[0] + J[1][i] * du[1] for i in range(3)]
    gp = [where(lv, dot([float(Rv[0][i]), float(Rv[1][i]), float(Rv[2][i])], dt), 0.0) for i in range(3)]
    terms = []
    for cidx in range(4):
        for r in range(3):
            if cidx < 3:
                terms.append(dt[r] * p[cidx] + J[0][r] * q0[cidx] + J[1][r] * q1[cidx])
            else:
                terms.append(dt[r])
    terms += [zero] * 12          # projmatrix is not read
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
    terms += cp
    ax = fx * fr["a"] * x     # u - cx
    ay = fy * fr["a"] * y
    tanx, tany = F(cam["tanfovx"]), F(cam["tanfovy"])
    intr = [-1.0 * (du[0] * ax + dot(dJ[0], J[0])) / tanx, -1.0 * (du[1] * ay + dot(dJ[1], J[1])) / tany]
    return dict(gp=gp, D=D, gop=where(lv, gop, 0.0), dm=dm, dcol=dcol, dsh=dsh, cam=[where(lv, t_, 0.0) for t_ in terms],
                intr=[where(lv, t_, 0.0) for t_ in intr])


def backward(g, cams, cot, scale_modifier=1.0, antialias=False, live=None, clamped=None, shared_mean2D=False):
    """project_bwd.cu's per-Gaussian chain over the fisheye views `cams` (ortho_ref64.backward's arguments and results)"""
    saved = O64.forward, O64._view
    O64.forward, O64._view = forward, _view
    try:
        return O64.backward(g, cams, cot, scale_modifier, antialias, live, clamped, shared_mean2D)
    finally:
        O64.forward, O64._view = saved


def fisheye_cam(W, H, fx, fy, cx, cy, k, c2w, theta_max=None):
    """A camera dict in project_ref64's layout of a fisheye view: tanfovx = W / (2 fx), the pinhole projmatrix of the same K
    (not read by the kernels), and "fisheye" = (cx, cy, k1..k4, theta_max)."""
    from manigaussian_b200 import cameras
    w2c = np.linalg.inv(np.asarray(c2w, np.float64))
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    proj = cameras.projection_from_intrinsics(0.1, 10.0, K, H, W)
    wvt = w2c.T
    tm = float(cameras.fisheye_theta_max(np.asarray(k, np.float64))[0]) if theta_max is None else float(theta_max)
    return dict(W=W, H=H, tanfovx=W / (2.0 * fx), tanfovy=H / (2.0 * fy), viewmatrix=wvt.astype(np.float32),
                projmatrix=(wvt @ proj.T).astype(np.float32), campos=np.linalg.inv(wvt)[3, :3].astype(np.float32),
                fisheye=(float(cx), float(cy), *(float(x) for x in k), tm))
