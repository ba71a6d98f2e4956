"""Float64 reference of the orthographic projection (include/mgs_rasterizer.h, "Orthographic views"), with bounds.

An orthographic view has J = [[fx, 0, 0], [0, fy, 0]] (fx = W / (2 tan_fovx), tan_fov* its half extents) and no frustum
clamp; the screen mean, depth, dilation, compensation, conic, radius and extent are the pinhole view's.  The records
therefore come from project_ref64.forward with its per-view geometry replaced by `_geometry` below (the only place the
Jacobian enters the forward).  The backward restates project_bwd.cu's chain for orthographic views: M = J Rv has rows
fx Rv0 and fy Rv1, dL/dt = (0, 0, dL/ddepth), the camera terms take J^T Q = (fx q0, fy q1, 0), and
dL/dtan_fovx = -(fx / tan_fovx) dJ00 (y likewise).  Values carry project_ref64's bounds (E: rounding bound e in units of u,
inherited bound d).

`backward` returns what project_ref64.backward returns (per-Gaussian sums over the views) plus, per view, the 35 camera
outputs and the 2 tan_fov outputs with camera_ref64's summation bound.
"""
import contextlib

import numpy as np

import camera_ref64 as C64
import project_ref64 as P64
from project_ref64 import E, _b, _cot, dot, f32, where


def _geometry(p, S, vw, mutate=()):
    """project_ref64._geometry for an orthographic view: same keys, J without t, no clamp (inx = iny = True)."""
    Rv, tv = vw["Rv"], vw["tv"]
    t = [dot([float(Rv[r][c]) for c in range(3)], p) + float(tv[r]) for r in range(3)]
    tz = t[2]
    P = tz.v.shape[0]
    fx, fy = E(np.full(P, vw["fx"])), E(np.full(P, vw["fy"]))
    m0 = [fx * float(Rv[0][c]) for c in range(3)]
    m1 = [fy * float(Rv[1][c]) for c in range(3)]
    u0 = [dot(S[c], m0) for c in range(3)]
    u1 = [dot(S[c], m1) for c in range(3)]
    a0, b, c0 = dot(m0, u0), dot(m0, u1), dot(m1, u1)
    a, c = a0 + float(f32(0.3)), c0 + float(f32(0.3))
    det = a * c - b * b
    ones = np.ones(P, bool)
    return dict(t=t, tz=tz, inx=ones, iny=ones, cx=E(np.zeros(P)), cy=E(np.zeros(P)), m0=m0, m1=m1, u0=u0, u1=u1, a0=a0,
                c0=c0, a=a, b=b, c=c, det=det, border=np.zeros(P, bool))


@contextlib.contextmanager
def _ortho_geometry():
    saved = P64._geometry
    P64._geometry = _geometry
    try:
        yield
    finally:
        P64._geometry = saved


def forward(g, cam, scale_modifier=1.0, antialias=False):
    """project.cu's records of one orthographic view (project_ref64.forward's dict and bounds)."""
    with _ortho_geometry():
        return P64.forward(g, cam, scale_modifier, antialias)


def _view(g, cam, c, S, lv, cl, antialias):
    """One orthographic view's contributions: per-Gaussian (gp [3], D [6 as 3x3 upper], gop, dm [2], dsh, dcol) and the
    camera / tan_fov terms (lists of E over the Gaussians, gated by lv)."""
    p = P64._cols(g["means3D"])
    P = p[0].v.shape[0]
    vw = P64.view_of(cam)
    zero = E(np.zeros(P))
    gate = lambda x: where(lv, x, 0.0)  # noqa: E731
    dm = [gate(_cot(c["dL_dmean2D"][:, i], _b(c, "dL_dmean2D", i))) for i in range(2)]
    gA, gB, gC = (gate(_cot(c["dL_dconic"][:, i], _b(c, "dL_dconic", i))) for i in range(3))
    gop_v = gate(_cot(c["dL_dopacity"], _b(c, "dL_dopacity")))
    dcol = [gate(_cot(c["dL_dcolor"][:, i], _b(c, "dL_dcolor", i))) for i in range(3)]
    dd = c.get("dL_ddepth")
    ddepth = gate(_cot(dd, c.get("dL_ddepth_B"))) if dd is not None else zero
    G = _geometry(p, S, vw)
    a, b, cc, det = G["a"], G["b"], G["c"], G["det"]
    m0, m1, u0, u1 = G["m0"], G["m1"], G["u0"], G["u1"]
    wgt = 1.0 / (det * det + float(f32(1e-7)))
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
        s = P64.sqrt(where(on, r, P64.AA_CLAMP))
        gop = where(lv, s * gop_v, 0.0)
        k = 0.5 * gop_v * (o_raw * s)
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
    dJ00 = dot(q0, [float(x) for x in Rv[0]])
    dJ11 = dot(q1, [float(x) for x in Rv[1]])
    fx, fy = vw["fx"], vw["fy"]
    dt = [zero, zero, ddepth]   # J does not move with t: depth = t.z is the only path
    _, h, iw = P64._means2D(p, vw)
    pm = vw["pm"]
    kx, ky = h[0] * iw * iw, h[1] * iw * iw
    gp = []
    for i in range(3):
        gi = dot([float(Rv[0][i]), float(Rv[1][i]), float(Rv[2][i])], dt)
        gi = gi + (float(pm[4 * i]) * iw - float(pm[4 * i + 3]) * kx) * dm[0] + \
            (float(pm[4 * i + 1]) * iw - float(pm[4 * i + 3]) * ky) * dm[1]
        gp.append(where(lv, gi, 0.0))
    # camera terms (camera_ref64's layout): dL/dRv = dt p^T + J^T dL/dM, dL/dtv = dt, the projection matrix, campos
    terms = []
    for cidx in range(4):
        for r in range(3):
            if cidx < 3:
                x = dt[r] * p[cidx]
                x = x + (fx * q0[cidx] if r == 0 else fy * q1[cidx] if r == 1 else zero)
                terms.append(x)
            else:
                terms.append(dt[r])
    ax, ay, aw = dm[0] * iw, dm[1] * iw, -(dm[0] * kx + dm[1] * ky)
    for cidx in range(4):
        ph = p[cidx] if cidx < 3 else E(np.ones(P))
        terms += [ax * ph, ay * ph, aw * ph]
    has_sh = g.get("shs") is not None
    dsh, cp = None, [zero, zero, zero]
    if has_sh:
        deg = int(g["sh_degree"])
        sh = np.asarray(g["shs"], f32).astype(np.float64)
        M = sh.shape[1]
        dRGB = [where(((cl >> ch) & 1).astype(bool), 0.0, dcol[ch]) for ch in range(3)]
        vv, ln = P64._direction(p, vw)
        il = 1.0 / ln
        x, y, z = (vi * il for vi in vv)
        basis = P64._sh_basis(x, y, z, deg)
        ddir = [zero, zero, zero]
        dsh = [[zero] * 3 for _ in range(M)]
        for kk in range((deg + 1) ** 2):
            B, grad = basis[kk]
            for ch in range(3):
                if kk < M:
                    dsh[kk][ch] = B * dRGB[ch]
            s_ = dot([E(sh[:, kk, ch]) for ch in range(3)], dRGB)
            ddir = [ddir[i] + P64._e(grad[i]) * s_ for i in range(3)]
        along = dot([x, y, z], ddir)
        for i, di in enumerate((x, y, z)):
            t_ = (ddir[i] - di * along) * il
            gp[i] = gp[i] + where(lv, t_, 0.0)
            cp[i] = -1.0 * t_
    terms += cp
    intr = [-(fx / float(f32(cam["tanfovx"]))) * dJ00, -(fy / float(f32(cam["tanfovy"]))) * dJ11]
    return dict(gp=gp, D=D, gop=where(lv, gop, 0.0), dm=dm, dcol=dcol, dsh=dsh, cam=[where(lv, t_, 0.0) for t_ in terms],
                intr=[where(lv, t_, 0.0) for t_ in intr])


def backward(g, cams, cot, scale_modifier=1.0, antialias=False, live=None, clamped=None, shared_mean2D=False):
    """project_bwd.cu's per-Gaussian chain over the orthographic views `cams` (arguments and per-Gaussian results as
    project_ref64.backward), plus "camera" [V] of dicts dL_dviewmatrix / dL_dprojmatrix / dL_dcampos (camera_ref64 layout)
    and "tan_fov" [V] of (val [2], e [2], d [2])."""
    p = P64._cols(g["means3D"])
    P = p[0].v.shape[0]
    S, R, se, q = P64.cov3d(g, scale_modifier)
    has_sh = g.get("shs") is not None
    M = np.asarray(g["shs"]).shape[1] if has_sh else 0
    deg = int(g["sh_degree"]) if has_sh else 0
    zero = E(np.zeros(P))
    gp = [zero, zero, zero]
    D = [[zero] * 3 for _ in range(3)]
    gop, gcol = zero, [zero, zero, zero]
    gsh = [[zero] * 3 for _ in range(M)]
    m2d, border, cams_out, intr_out = [], np.zeros(P, bool), [], []
    depth = C64.sum_depth(P)
    cols = [4 * (k // 3) + k % 3 for k in range(12)] + [16 + 4 * (k // 3) + (0, 1, 3)[k % 3] for k in range(12)] + [32, 33, 34]
    for v, cam in enumerate(cams):
        fw = forward(g, cam, scale_modifier, antialias)
        border |= fw["border"]
        lv = ~fw["culled"] if live is None else np.asarray(live[v], bool)
        cl = fw["clamped"] if clamped is None else np.asarray(clamped[v]).astype(np.int64)
        r = _view(g, cam, cot[v], S, lv, cl, antialias)
        gp = [gp[i] + r["gp"][i] for i in range(3)]
        for i in range(3):
            for j in range(i, 3):
                D[i][j] = D[i][j] + r["D"][i][j]
        gop = gop + r["gop"]
        gcol = [gcol[i] + r["dcol"][i] for i in range(3)]
        if has_sh:
            for k in range(M):
                for ch in range(3):
                    if k < (deg + 1) ** 2:
                        gsh[k][ch] = gsh[k][ch] + r["dsh"][k][ch]
        if shared_mean2D:
            m2d = [r["dm"][0] + m2d[0], r["dm"][1] + m2d[1]] if m2d else r["dm"]
        else:
            m2d.append(r["dm"])
        sums = []
        for ts in (r["cam"], r["intr"]):
            val = np.array([t_.v.sum() for t_ in ts])
            e = np.array([(t_.e + 0 * t_.v).sum() + depth * np.abs(t_.v).sum() for t_ in ts])
            d = np.array([(t_.d + 0 * t_.v).sum() for t_ in ts])
            sums.append((val, e, d))
        full = [np.zeros(35) for _ in range(3)]
        for arr, src in zip(full, sums[0]):
            arr[cols] = src
        cams_out.append(dict(dL_dviewmatrix=tuple(a[:16] for a in full), dL_dprojmatrix=tuple(a[16:32] for a in full),
                             dL_dcampos=tuple(a[32:] for a in full)))
        intr_out.append(sums[1])
    out = {}
    pack = lambda xs: (np.stack([x.v for x in xs], -1), np.stack([x.e + 0 * x.v for x in xs], -1),  # noqa: E731
                       np.stack([x.d + 0 * x.v for x in xs], -1))
    out["dL_dmeans3D"] = pack(gp)
    out["dL_dopacity"] = tuple(x[:, 0] for x in pack([gop]))
    out["dL_dcolors"] = pack(gcol)
    out["dL_dcov3D"] = pack([D[0][0], 2.0 * D[0][1], 2.0 * D[0][2], D[1][1], 2.0 * D[1][2], D[2][2]])
    out["dL_dmeans2D"] = tuple(np.stack(z, 0) for z in zip(*[pack(m) for m in ([m2d] if shared_mean2D else m2d)]))
    if has_sh:
        rows = [pack(gsh[k]) for k in range(M)]
        out["dL_dsh"] = tuple(np.stack([r_[i] for r_ in rows], 1) for i in range(3))
    if R is not None:
        Dm = [[D[min(i, j)][max(i, j)] for j in range(3)] for i in range(3)]
        dscale, A = [], [[None] * 3 for _ in range(3)]
        for j in range(3):
            gl = [2.0 * se[j] * dot([Dm[i][k] for k in range(3)], [R[k][j] for k in range(3)]) for i in range(3)]
            dscale.append(dot([R[i][j] for i in range(3)], gl))
            for i in range(3):
                A[i][j] = gl[i] * se[j]
        r_, x, y, z = q
        drot = [2.0 * (z * (A[1][0] - A[0][1]) + y * (A[0][2] - A[2][0]) + x * (A[2][1] - A[1][2])),
                2.0 * (y * (A[0][1] + A[1][0]) + z * (A[0][2] + A[2][0]) + r_ * (A[2][1] - A[1][2])) - 4.0 * x * (A[1][1] + A[2][2]),
                2.0 * (x * (A[0][1] + A[1][0]) + r_ * (A[0][2] - A[2][0]) + z * (A[1][2] + A[2][1])) - 4.0 * y * (A[0][0] + A[2][2]),
                2.0 * (r_ * (A[1][0] - A[0][1]) + x * (A[0][2] + A[2][0]) + y * (A[1][2] + A[2][1])) - 4.0 * z * (A[0][0] + A[1][1])]
        out["dL_dscales"] = pack(dscale)
        out["dL_drotations"] = pack(drot)
    else:
        out["dL_dscales"] = (np.zeros((P, 3)),) * 3
        out["dL_drotations"] = (np.zeros((P, 4)),) * 3
    out["border"] = border
    out["camera"], out["tan_fov"] = cams_out, intr_out
    return out


def ortho_cam(W, H, half_w, half_h, c2w, znear=0.01, zfar=10.0):
    """A camera dict in project_ref64's layout (viewmatrix / projmatrix in the ABI's transposed float32 layout) of an
    orthographic view with half extents (half_w, half_h) and camera-to-world pose c2w [4,4]."""
    from manigaussian_b200 import cameras
    w2c = np.linalg.inv(np.asarray(c2w, np.float64))
    proj = cameras.projection_orthographic(znear, zfar, half_w, half_h)
    wvt = w2c.T
    full = wvt @ proj.T
    return dict(W=W, H=H, tanfovx=float(half_w), tanfovy=float(half_h), viewmatrix=wvt.astype(np.float32),
                projmatrix=full.astype(np.float32), campos=np.linalg.inv(wvt)[3, :3].astype(np.float32))
