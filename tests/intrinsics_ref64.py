"""Float64 reference of the focal-length gradients (include/mgs_rasterizer.h, "Learnable intrinsics"), beside camera_ref64.

Per view, the chain of camera_ref64 up to Q = [q0; q1] = 2 H M S (the AA compensation inside H) and
dJ00 = q0 . Rv0, dJ02 = q0 . Rv2, dJ11 = q1 . Rv1, dJ12 = q1 . Rv2; with fx = W / (2 tan_fovx), each live Gaussian gives
  dL/dtan_fovx = -(fx / tan_fovx) (dJ00 / tz - dJ02 cx / tz^2)  -  [x clamp active] fx dJ02 (+-1.3) / tz
and likewise for y.  `tan_fov_grads` returns (val, e, d) per view for the two floats; the bound is camera_ref64's: each
term's own (e, d), plus `depth` u |term| in e for the fixed summation tree.  A borderline clamp decision (t.x / t.z within
4 u e of the limit) switches the clamp term on or off, so its magnitude joins d.

`mutate` breaks one convention on purpose (INTR_MUTATIONS): the sensitivity test shows each moves an entry past twice its
bound.
"""
import numpy as np

import camera_ref64 as C64
import project_ref64 as P64
from project_ref64 import E, U, _b, _cot, dot, f32, where

# no_clamp: drop the clamp term; unclamped_t: t.x / t.y in place of the clamped cx / cy in the J term; no_aa: H without the
# anti-aliased compensation; fx_derivative: dL/dfx in place of dL/dtan_fovx
INTR_MUTATIONS = ("no_clamp", "unclamped_t", "no_aa", "fx_derivative")
# an entry is within bound when |x - val| <= KAPPA_INTR (u e + d): 4x the largest ratio measured against the kernels over
# the 12 CAM cases and the 4 projection edge scenes of tests/test_intrinsics_grad_gpu.py (H100 80GB HBM3): 0.0012 on the
# CAM cases, 0.0023 on clamp_y, 0.0108 on aa1 (anti-aliased needles, where the compensation's 1 / det0 amplifies the fp32
# rounding of H; still well inside the unscaled first-order bound, ratio 1)
KAPPA_INTR = 0.043


def _view_terms(g, cam, c, S, lv, antialias, mutate):
    p = P64._cols(g["means3D"])
    P = p[0].v.shape[0]
    vw = P64.view_of(cam)
    gate = lambda x: where(lv, x, 0.0)  # noqa: E731
    gA, gB, gC = (gate(_cot(c["dL_dconic"][:, i], _b(c, "dL_dconic", i))) for i in range(3))
    gop_v = gate(_cot(c["dL_dopacity"], _b(c, "dL_dopacity")))
    G = P64._geometry(p, S, vw)
    tz, a, b, cc, det = G["tz"], G["a"], G["b"], G["c"], G["det"]
    u0, u1 = G["u0"], G["u1"]
    wgt = 1.0 / (det * det + float(f32(1e-7)))
    e00, e01 = cc * gA - b * gB, cc * gB - b * gC
    e10, e11 = a * gB - b * gA, a * gC - b * gB
    H00 = -wgt * (e00 * cc - e01 * b)
    H01 = -wgt * (e01 * a - e00 * b)
    H11 = -wgt * (e11 * a - e10 * b)
    if antialias and "no_aa" not in mutate:
        o_raw = E(np.asarray(g["opacities"], f32).reshape(-1).astype(np.float64))
        a0, c0 = G["a0"], G["c0"]
        d0 = a0 * c0 - b * b
        r = d0 / det
        on = r.v > P64.AA_CLAMP
        s = P64.sqrt(where(on, r, P64.AA_CLAMP))
        k = 0.5 * gop_v * (o_raw * s)
        i0 = 1.0 / where(on, d0, 1.0)
        i1 = 1.0 / det
        H00 = H00 + where(on, k * (c0 * i0 - cc * i1), 0.0)
        H11 = H11 + where(on, k * (a0 * i0 - a * i1), 0.0)
        H01 = H01 + where(on, k * b * (i1 - i0), 0.0)
    Rv = vw["Rv"]
    q0 = [2.0 * (H00 * u0[i] + H01 * u1[i]) for i in range(3)]
    q1 = [2.0 * (H01 * u0[i] + H11 * u1[i]) for i in range(3)]
    dJ = [dot(q0, [float(x) for x in Rv[0]]), dot(q0, [float(x) for x in Rv[2]]),
          dot(q1, [float(x) for x in Rv[1]]), dot(q1, [float(x) for x in Rv[2]])]
    iz = 1.0 / tz
    terms, extra = [], []
    for ax, (f, lim, dJd, dJ2, ccl, inside) in enumerate(((vw["fx"], vw["limx"], dJ[0], dJ[1], G["cx"], G["inx"]),
                                                           (vw["fy"], vw["limy"], dJ[2], dJ[3], G["cy"], G["iny"]))):
        tan = float(f32(cam["tanfovx" if ax == 0 else "tanfovy"]))
        u = G["t"][ax] / tz
        cpos = G["t"][ax] if "unclamped_t" in mutate else ccl
        jpath = dJd * iz - dJ2 * cpos * iz * iz
        sgn = np.where(u.v > 0, 1.3, -1.3)
        clamp_u = -f * dJ2 * E(sgn) * iz
        clamp = where(inside, 0.0, clamp_u) if "no_clamp" not in mutate else E(np.zeros(P))
        x = jpath if "fx_derivative" in mutate else (-(f / tan)) * jpath + clamp
        terms.append(where(lv, x, 0.0))
        border = P64.within(u, lim) | P64.within(u, -lim)
        extra.append(np.where(border & lv, np.abs(clamp_u.v) + U * clamp_u.e, 0.0))
    return terms, extra


def tan_fov_grads(g, cams, cot, scale_modifier=1.0, antialias=False, live=None, depth=None, mutate=()):
    """Per view v: (val [2], e [2], d [2]) of {dL/dtan_fovx, dL/dtan_fovy}.  cot[v] and live[v] as camera_ref64 takes them."""
    S = P64.cov3d(g, scale_modifier)[0]
    P = len(g["means3D"])
    depth = C64.sum_depth(P) if depth is None else depth
    out = []
    for v, cam in enumerate(cams):
        if live is None:
            lv = ~P64.forward(g, cam, scale_modifier, antialias)["culled"]
        else:
            lv = np.asarray(live[v], bool)
        terms, extra = _view_terms(g, cam, cot[v], S, lv, antialias, mutate)
        val = np.array([t.v.sum() for t in terms])
        e = np.array([(t.e + 0 * t.v).sum() + depth * np.abs(t.v).sum() for t in terms])
        d = np.array([(t.d + 0 * t.v).sum() + x.sum() for t, x in zip(terms, extra)])
        out.append((val, e, d))
    return out


def ratio(got, ref):
    """|got - val| / (u e + d) per entry, to compare with KAPPA_INTR"""
    v, e, d = ref
    return np.abs(np.asarray(got, np.float64) - v) / (U * e + d + 1e-30)
