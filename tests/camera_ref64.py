"""Float64 reference of the camera gradients (include/mgs_rasterizer.h, "Camera gradients"), beside project_ref64.

Per view, the same per-Gaussian chain as project_ref64.backward (the same records, masks and error-carrying values `E`):
dt with the x / y clamp masks and the depth cotangent, Q = [q0; q1] = 2 H M S with the AA compensation in H, the
screen-mean cotangent dm with iw, kx, ky, and the SH branch's direction gradient.  From them each live Gaussian gives the
27 non-constant terms of the view's 35 outputs:
  dL/dvm[4c + r] = dt[r] p[c] + (J^T Q)[r][c] (r, c < 3),  dL/dvm[12 + r] = dt[r],
  dL/dpm[4c + {0, 1, 3}] = (dm0 iw, dm1 iw, -(dm0 kx + dm1 ky)) ph[c],  dL/dcampos = -(dd - dir along) / |v|,
and the view's gradient is their sum over its live Gaussians.  `camera_grads` returns (val, e, d) per view for the 16 + 16 + 3
floats.  The bound of the sum: each term's own (e, d), plus `depth` u |term| in e for the fp32 additions of the kernels' fixed
summation tree (a first-order bound for any order whose longest chain of additions is `depth`).

Borderline clamp decisions (t.x / t.z or t.y / t.z within 4 u e of the limit) are not dropped: the kernel's decision may
differ from float64's, which switches d/dt.x (d/dt.y) between 0 and its unmasked value; |unmasked d/dt| times |p[c]| (and 1
for the translation) joins the bound d of the entries it reaches.  Decisions on the cull and the radius come from the
caller (`live`, the kernel's radii), the clamp bits from `clamped`.

`mutate` breaks one convention on purpose (CAM_MUTATIONS, and project_ref64's "true_dtz"): the sensitivity test shows each
moves a checked element past twice its bound.
"""
import numpy as np

import project_ref64 as P64
from project_ref64 import E, U, _cot, _b, dot, f32, sqrt, where

CAM_MUTATIONS = ("cam_no_J", "cam_tp_transposed", "cam_no_depth", "cam_campos_sign", "cam_no_pm3", "true_dtz")
# an entry is within bound when |x - val| <= KAPPA_CAM (u e + d); KAPPA_CAM is 4x the largest |x - val| / (u e + d) measured against the kernels over the 12 CAM cases of
# tests/test_camera_grad_gpu.py (0.0016, H100 80GB HBM3): the summation term depth u sum |term| is a worst case the fixed
# trees stay far below
KAPPA_CAM = 0.0064


def sum_depth(P):
    """longest chain of fp32 additions from a term to its output: 5 (warp halving) + 4 (the CTA's warps) + the reduce's
    rows per thread + 8 (its tree over 256 partials)"""
    rows = -(-int(P) // 128)
    return 5 + 4 + -(-rows // 256) + 8


def _view_terms(g, cam, c, S, lv, cl, antialias, mutate):
    """The 27 per-Gaussian terms of one view (a list of E over the Gaussians) and the extra inherited bound per term from
    borderline clamp decisions."""
    p = P64._cols(g["means3D"])
    P = p[0].v.shape[0]
    vw = P64.view_of(cam)
    zero = E(np.zeros(P))
    gate = lambda x: where(lv, x, 0.0)  # noqa: E731
    dm = [gate(_cot(c["dL_dmean2D"][:, i], _b(c, "dL_dmean2D", i))) for i in range(2)]
    gA, gB, gC = (gate(_cot(c["dL_dconic"][:, i], _b(c, "dL_dconic", i))) for i in range(3))
    gop_v = gate(_cot(c["dL_dopacity"], _b(c, "dL_dopacity")))
    dcol = [gate(_cot(c["dL_dcolor"][:, i], _b(c, "dL_dcolor", i))) for i in range(3)]
    dd_ = c.get("dL_ddepth")
    ddepth = gate(_cot(dd_, c.get("dL_ddepth_B"))) if (dd_ is not None and "cam_no_depth" not in mutate) else zero
    G = P64._geometry(p, S, vw)
    tz, a, b, cc, det = G["tz"], G["a"], G["b"], G["c"], G["det"]
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
        s = sqrt(where(on, r, P64.AA_CLAMP))
        k = 0.5 * gop_v * (o_raw * s)
        i0 = 1.0 / where(on, d0, 1.0)
        i1 = 1.0 / det
        H00 = H00 + where(on, k * (c0 * i0 - cc * i1), 0.0)
        H11 = H11 + where(on, k * (a0 * i0 - a * i1), 0.0)
        H01 = H01 + where(on, k * b * (i1 - i0), 0.0)
    Rv = vw["Rv"]
    q0 = [2.0 * (H00 * u0[i] + H01 * u1[i]) for i in range(3)]
    q1 = [2.0 * (H01 * u0[i] + H11 * u1[i]) for i in range(3)]
    dJ00 = dot(q0, [float(x) for x in Rv[0]])
    dJ02 = dot(q0, [float(x) for x in Rv[2]])
    dJ11 = dot(q1, [float(x) for x in Rv[1]])
    dJ12 = dot(q1, [float(x) for x in Rv[2]])
    fx, fy = vw["fx"], vw["fy"]
    iz = 1.0 / tz
    iz2 = iz * iz
    iz3 = iz2 * iz
    dtx_u, dty_u = -fx * iz2 * dJ02, -fy * iz2 * dJ12
    dtx, dty = where(G["inx"], dtx_u, 0.0), where(G["iny"], dty_u, 0.0)
    dtz = (-fx * iz2 * dJ00 - fy * iz2 * dJ11 + 2.0 * fx * G["cx"] * iz3 * dJ02 + 2.0 * fy * G["cy"] * iz3 * dJ12 + ddepth)
    if "true_dtz" in mutate:
        lx = np.where(G["inx"], 0.0, np.sign(G["cx"].v) * vw["limx"])
        ly = np.where(G["iny"], 0.0, np.sign(G["cy"].v) * vw["limy"])
        dtz = dtz + E(-fx * lx) * iz2 * dJ02 + E(-fy * ly) * iz2 * dJ12
    dt = [dtx, dty, dtz]
    ux, uy = G["t"][0] / tz, G["t"][1] / tz
    bx = P64.within(ux, vw["limx"]) | P64.within(ux, -vw["limx"])
    by = P64.within(uy, vw["limy"]) | P64.within(uy, -vw["limy"])
    flip = [np.where(bx & lv, np.abs(dtx_u.v) + U * dtx_u.e, 0.0), np.where(by & lv, np.abs(dty_u.v) + U * dty_u.e, 0.0),
            np.zeros(P)]
    J00, J11 = fx * iz, fy * iz
    J02, J12 = -fx * G["cx"] * iz2, -fy * G["cy"] * iz2
    terms, extra = [], []
    for cidx in range(4):
        for r in range(3):
            if cidx < 3:
                pr = p[r] if "cam_tp_transposed" in mutate else p[cidx]
                dtr = dt[cidx] if "cam_tp_transposed" in mutate else dt[r]
                x = dtr * pr
                if "cam_no_J" not in mutate:
                    x = x + (J00 * q0[cidx] if r == 0 else J11 * q1[cidx] if r == 1 else J02 * q0[cidx] + J12 * q1[cidx])
                terms.append(x)
                extra.append(flip[r] * np.abs(p[cidx].v))
            else:
                terms.append(dt[r])
                extra.append(flip[r])
    _, h, iw = P64._means2D(p, vw)
    kx, ky = h[0] * iw * iw, h[1] * iw * iw
    ax, ay, aw = dm[0] * iw, dm[1] * iw, -(dm[0] * kx + dm[1] * ky)
    for cidx in range(4):
        ph = p[cidx] if cidx < 3 else E(np.ones(P))
        terms += [ax * ph, ay * ph, (zero if "cam_no_pm3" in mutate else aw * ph)]
        extra += [np.zeros(P)] * 3
    cp = [zero, zero, zero]
    if g.get("shs") is not None:
        deg = int(g["sh_degree"])
        sh = np.asarray(g["shs"], f32).astype(np.float64)
        dRGB = [where(((cl >> ch) & 1).astype(bool), 0.0, dcol[ch]) for ch in range(3)]
        vv, ln = P64._direction(p, vw)
        il = 1.0 / ln
        x, y, z = (vi * il for vi in vv)
        basis = P64._sh_basis(x, y, z, deg)
        ddir = [zero, zero, zero]
        for kk in range((deg + 1) ** 2):
            _, grad = basis[kk]
            s_ = dot([E(sh[:, kk, ch]) for ch in range(3)], dRGB)
            ddir = [ddir[i] + P64._e(grad[i]) * s_ for i in range(3)]
        along = dot([x, y, z], ddir)
        sign = 1.0 if "cam_campos_sign" in mutate else -1.0
        cp = [sign * ((ddir[i] - di * along) * il) for i, di in enumerate((x, y, z))]
    terms += cp
    extra += [np.zeros(P)] * 3
    return [where(lv, t, 0.0) for t in terms], extra


def camera_grads(g, cams, cot, scale_modifier=1.0, antialias=False, live=None, clamped=None, depth=None, mutate=()):
    """Per view v: dict dL_dviewmatrix [16], dL_dprojmatrix [16], dL_dcampos [3], each (val, e, d).  cot[v], live[v] and
    clamped[v] as project_ref64.backward takes them; depth: the summation depth (default sum_depth(P))."""
    S = P64.cov3d(g, scale_modifier)[0]
    P = len(g["means3D"])
    depth = sum_depth(P) if depth is None else depth
    out = []
    for v, cam in enumerate(cams):
        fw = P64.forward(g, cam, scale_modifier, antialias)
        lv = ~fw["culled"] if live is None else np.asarray(live[v], bool)
        cl = fw["clamped"] if clamped is None else np.asarray(clamped[v]).astype(np.int64)
        terms, extra = _view_terms(g, cam, cot[v], S, lv, cl, antialias, mutate)
        val = np.array([t.v.sum() for t in terms])
        e = np.array([(t.e + 0 * t.v).sum() + depth * np.abs(t.v).sum() for t in terms])
        d = np.array([(t.d + 0 * t.v).sum() + x.sum() for t, x in zip(terms, extra)])
        full = [np.zeros(35) for _ in range(3)]
        cols = [4 * (k // 3) + k % 3 for k in range(12)] + [16 + 4 * (k // 3) + (0, 1, 3)[k % 3] for k in range(12)] + [32, 33, 34]
        for arr, src in zip(full, (val, e, d)):
            arr[cols] = src
        out.append(dict(dL_dviewmatrix=tuple(a[:16] for a in full), dL_dprojmatrix=tuple(a[16:32] for a in full),
                        dL_dcampos=tuple(a[32:] for a in full)))
    return out


def ratio(got, ref):
    """|got - val| / (u e + d) per entry, to compare with KAPPA_CAM"""
    v, e, d = ref
    return np.abs(np.asarray(got, np.float64) - v) / (U * e + d + 1e-30)
