"""Float64 reference of the per-Gaussian projection (forward and backward), with a first-order bound of fp32 evaluation.

Every quantity is an `E`: its float64 value `v`, `e`, a first-order bound (in units of u = 2^-24) of the error that fp32
evaluation of the same expression accumulates from exact fp32 inputs (each operation adds |result| to the operands'
propagated bounds), and `d`, an absolute bound inherited from inputs that are themselves uncertain (the blend-stage
cotangents of blend_ref64, carried through the same linear map).  A checked value is within bound when
|value - ref| <= KAPPA[q] u e + d + tiny.

`forward` restates project.cu per Gaussian and view: cov3D from scales x scale_modifier and the un-normalised quaternion
(or cov3D_precomp), t and the depth, means2D through projmatrix, 1 / (w + 1e-7) and ndc2pix, the clamped J, the 2D
covariance + 0.3, det and conic, the radius ceil(3 sqrt(lambda_max)) and the tile rect, SH -> RGB with the +0.5 offset and
the per-channel clamp bits, the anti-aliased o_eff = o sqrt(max(2.5e-5, det0 / det)), and the blend's footprint extent.
Integer and decision outputs (culled, radius, rect, clamp bits, inside / outside the frustum clamp, the AA threshold) are
exact except where the float64 argument lies within 4 u e of the threshold: such a Gaussian is `border` for that view.

`backward` chains the blend-stage cotangents of each view (dL_dmean2D, dL_dconic (a, half-b, c), dL/do_eff, dL_dcolor,
dL_ddepth) to the per-Gaussian outputs of project_bwd.cu and sums over the views the way the kernel does.  It keeps the
reference's conventions (DGR/cuda_rasterizer/backward.cu), each marked where it is applied:
  * the x / y frustum clamp masks d/dt.x and d/dt.y, and the clamped values are constants in d/dt.z;
  * the quaternion is used un-normalised;
  * dL_dscale carries no scale_modifier factor (it is dL/d(scale_modifier * scale));
  * the conic's b cotangent arrives halved (H01 = the gradient w.r.t. ONE off-diagonal entry of S');
  * w = 1 / (det^2 + 1e-7);
  * the per-channel clamp bits mask dRGB;
  * dL_dsh is exactly zero above the active degree; dL_dcov3D carries each off-diagonal entry twice.
`mutate` (a set of names, MUTATIONS) breaks one of these on purpose: the sensitivity test shows each moves a checked
element past twice its bound on the edge scenes.
"""
import numpy as np

import blend_ref64 as B64
from blend_ref64 import U

f32 = np.float32
# Bound scale per checked quantity: 4x the largest |x - ref| / (u e) measured for that quantity over the C oracle on the
# golden and edge scenes (tests/test_project_ref64_cpu.py) and the kernels on every case of tests/test_project_ref64_gpu.py
# (H100 80GB HBM3).  The measured ratios are in those tests' docstrings.  dL_dcolors and dL_dmeans2D measured 0 everywhere
# (copies of exact inputs with AA off; with AA their inherited bound d covers the whole difference): they keep 1.
KAPPA = dict(cov3D=1.86, depth=3.5, means2D=3.7, conic=0.75, rgb=3.5, opacity=1.5, extent=0.61,
             dL_dmeans3D=1.5, dL_dcov3D=3.0, dL_dscales=0.47, dL_drotations=0.4, dL_dsh=2.0, dL_dopacity=0.23,
             dL_dcolors=1.0, dL_dmeans2D=1.0)
BAND = 4.0          # a decision is borderline when its argument is within BAND u e of the threshold
NEAR_Z = float(f32(0.2))
AA_CLAMP = float(f32(2.5e-5))
SH_C0 = float(f32(0.28209479177387814))
SH_C1 = float(f32(0.4886025119029199))
SH_C2 = [float(f32(c)) for c in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                                 0.5462742152960396)]
SH_C3 = [float(f32(c)) for c in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                                 -0.4570457994644658, 1.445305721320277, -0.5900435899266435)]
MUTATIONS = ("no_x_mask", "no_y_mask", "true_dtz", "normalise_q", "scale_mod_in_dscale", "unhalve_b", "sh_grad1",
             "sh_grad2", "sh_grad3", "ignore_clamp_bits", "sh_above_degree")


class E:
    """A float64 value with its fp32 rounding bound e (units of u) and inherited absolute bound d."""
    __slots__ = ("v", "e", "d")

    def __init__(self, v, e=0.0, d=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = e
        self.d = d

    def __add__(self, o):
        o = _e(o)
        v = self.v + o.v
        return E(v, self.e + o.e + np.abs(v), self.d + o.d)

    __radd__ = __add__

    def __sub__(self, o):
        return self + (-_e(o))

    def __rsub__(self, o):
        return _e(o) + (-self)

    def __neg__(self):
        return E(-self.v, self.e, self.d)

    def __mul__(self, o):
        o = _e(o)
        v = self.v * o.v
        a, b = np.abs(self.v), np.abs(o.v)
        return E(v, a * o.e + b * self.e + np.abs(v), a * o.d + b * self.d)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _e(o)
        v = self.v / o.v
        ib = 1.0 / np.abs(o.v)
        return E(v, (self.e + np.abs(v) * o.e) * ib + np.abs(v), (self.d + np.abs(v) * o.d) * ib)

    def __rtruediv__(self, o):
        return _e(o) / self


def _e(x):
    return x if isinstance(x, E) else E(x)


def sqrt(a):
    s = np.sqrt(np.maximum(a.v, 0.0))
    k = np.where(s > 0, 0.5 / np.where(s > 0, s, 1.0), 0.0)
    return E(s, a.e * k + s, a.d * k)


def where(c, a, b):
    a, b = _e(a), _e(b)
    bc = lambda x, y: np.where(c, x, y)  # noqa: E731
    return E(bc(a.v, b.v), bc(a.e, b.e) + 0 * a.v, bc(a.d, b.d) + 0 * a.v)


def dot(us, ws):
    s = us[0] * ws[0]
    for x, y in zip(us[1:], ws[1:]):
        s = s + x * y
    return s


def within(x, threshold, band=BAND):
    """x (an E) lies within band u e (+ d) of threshold."""
    return np.abs(x.v - threshold) <= band * U * x.e + x.d


def near_integer(x, lo, hi, band=BAND):
    """x (an E) lies within band u e of an integer k in [lo, hi] (where truncation / ceil jumps)."""
    k = np.clip(np.rint(x.v), lo, hi)
    return (np.abs(x.v - k) <= band * U * x.e + 1e-12) & (np.rint(x.v) >= lo) & (np.rint(x.v) <= hi)


# --------------------------------------------------------------------------- camera
def view_of(cam, W=None, H=None):
    """The view's constants as the kernels see them (fp32 focal lengths and clamp limits, as the host computes them)."""
    W = cam["W"] if W is None else W
    H = cam["H"] if H is None else H
    vm = np.asarray(cam["viewmatrix"], f32).reshape(-1).astype(np.float64)
    pm = np.asarray(cam["projmatrix"], f32).reshape(-1).astype(np.float64)
    tx, ty = f32(cam["tanfovx"]), f32(cam["tanfovy"])
    return dict(W=W, H=H, Rv=np.array([[vm[4 * c + r] for c in range(3)] for r in range(3)]), tv=vm[12:15], pm=pm,
                campos=np.asarray(cam["campos"], f32).reshape(-1).astype(np.float64),
                fx=float(f32(W) / (f32(2.0) * tx)), fy=float(f32(H) / (f32(2.0) * ty)),
                limx=float(f32(1.3) * tx), limy=float(f32(1.3) * ty))


def _cols(a):
    a = np.asarray(a, f32).astype(np.float64)
    return [E(a[:, i]) for i in range(a.shape[1])]


# --------------------------------------------------------------------------- forward
def rotation(q):
    """R(q) of the reference (forward.cu:134-140), q = (r, x, y, z) un-normalised: rows of E."""
    r, x, y, z = q
    one = 1.0
    return [[one - 2.0 * (y * y + z * z), 2.0 * (x * y - r * z), 2.0 * (x * z + r * y)],
            [2.0 * (x * y + r * z), one - 2.0 * (x * x + z * z), 2.0 * (y * z - r * x)],
            [2.0 * (x * z - r * y), 2.0 * (y * z + r * x), one - 2.0 * (x * x + y * y)]]


def cov3d(g, scale_modifier=1.0, mutate=()):
    """S (3x3 nested list of E), R, se (the modified scales) and q from the Gaussian inputs g."""
    if g.get("scales") is not None:
        q = _cols(g["rotations"])
        if "normalise_q" in mutate:
            n = np.sqrt(sum(x.v ** 2 for x in q))
            q = [E(x.v / n) for x in q]
        s = _cols(g["scales"])
        se = [float(f32(scale_modifier)) * x for x in s]
        R = rotation(q)
        S = [[dot([R[i][k] * se[k] * se[k] for k in range(3)], [R[j][k] for k in range(3)]) for j in range(3)] for i in range(3)]
        return S, R, se, q
    c = _cols(g["cov3D_precomp"])
    S = [[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]]
    return S, None, None, None


def _sh_basis(x, y, z, deg):
    """[(B_k, (dB/dx, dB/dy, dB/dz))] for k < (deg + 1)^2, as E."""
    out = [(E(np.full(x.v.shape, SH_C0)), (0.0, 0.0, 0.0))]
    if deg > 0:
        out += [(-SH_C1 * y, (0.0, -SH_C1, 0.0)), (SH_C1 * z, (0.0, 0.0, SH_C1)), (-SH_C1 * x, (-SH_C1, 0.0, 0.0))]
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        c = SH_C2
        out += [(c[0] * (x * y), (c[0] * y, c[0] * x, 0.0)), (c[1] * (y * z), (0.0, c[1] * z, c[1] * y)),
                (c[2] * (2.0 * zz - xx - yy), (-2.0 * c[2] * x, -2.0 * c[2] * y, 4.0 * c[2] * z)),
                (c[3] * (x * z), (c[3] * z, 0.0, c[3] * x)), (c[4] * (xx - yy), (2.0 * c[4] * x, -2.0 * c[4] * y, 0.0))]
    if deg > 2:
        c = SH_C3
        out += [(c[0] * y * (3.0 * xx - yy), (c[0] * 6.0 * x * y, c[0] * 3.0 * (xx - yy), 0.0)),
                (c[1] * (x * y) * z, (c[1] * y * z, c[1] * x * z, c[1] * x * y)),
                (c[2] * y * (4.0 * zz - xx - yy), (c[2] * -2.0 * x * y, c[2] * (4.0 * zz - xx - 3.0 * yy), c[2] * 8.0 * y * z)),
                (c[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy), (c[3] * -6.0 * x * z, c[3] * -6.0 * y * z,
                                                               c[3] * (6.0 * zz - 3.0 * xx - 3.0 * yy))),
                (c[4] * x * (4.0 * zz - xx - yy), (c[4] * (4.0 * zz - 3.0 * xx - yy), c[4] * -2.0 * x * y, c[4] * 8.0 * x * z)),
                (c[5] * z * (xx - yy), (c[5] * 2.0 * x * z, c[5] * -2.0 * y * z, c[5] * (xx - yy))),
                (c[6] * x * (xx - 3.0 * yy), (c[6] * 3.0 * (xx - yy), c[6] * -6.0 * x * y, 0.0))]
    return out


def _direction(p, vw):
    v = [p[i] - float(vw["campos"][i]) for i in range(3)]
    ln = sqrt(dot(v, v))
    return v, ln


def _geometry(p, S, vw, mutate=()):
    """Per view: t, the clamp decisions, M = J Rv rows, the dilated 2D covariance (a, b, c) and det."""
    Rv, tv = vw["Rv"], vw["tv"]
    t = [dot([float(Rv[r][c]) for c in range(3)], p) + float(tv[r]) for r in range(3)]
    tz = t[2]
    ux, uy = t[0] / tz, t[1] / tz
    inx = (ux.v >= -vw["limx"]) & (ux.v <= vw["limx"])
    iny = (uy.v >= -vw["limy"]) & (uy.v <= vw["limy"])
    cx = where(inx, ux, np.where(ux.v < 0, -vw["limx"], vw["limx"])) * tz
    cy = where(iny, uy, np.where(uy.v < 0, -vw["limy"], vw["limy"])) * tz
    fx, fy = vw["fx"], vw["fy"]
    J00, J11 = fx / tz, fy / tz
    J02, J12 = -(fx * cx) / (tz * tz), -(fy * cy) / (tz * tz)
    m0 = [J00 * float(Rv[0][c]) + J02 * float(Rv[2][c]) for c in range(3)]
    m1 = [J11 * float(Rv[1][c]) + J12 * float(Rv[2][c]) for c in range(3)]
    u0 = [dot(S[c], m0) for c in range(3)]
    u1 = [dot(S[c], m1) for c in range(3)]
    a0, b, c0 = dot(m0, u0), dot(m0, u1), dot(m1, u1)
    a, c = a0 + float(f32(0.3)), c0 + float(f32(0.3))
    det = a * c - b * b
    border = (within(ux, vw["limx"]) | within(ux, -vw["limx"]) | within(uy, vw["limy"]) | within(uy, -vw["limy"]))
    return dict(t=t, tz=tz, inx=inx, iny=iny, cx=cx, cy=cy, m0=m0, m1=m1, u0=u0, u1=u1, a0=a0, c0=c0, a=a, b=b, c=c,
                det=det, border=border)


def screen_covariance(g, cam, scale_modifier=1.0):
    """float64 (a0, b, c0) of the screen-space covariance before the 0.3 px^2 dilation, and det of the dilated one."""
    S = cov3d(g, scale_modifier)[0]
    G = _geometry(_cols(g["means3D"]), S, view_of(cam))
    return G["a0"].v, G["b"].v, G["c0"].v, G["det"].v


def _means2D(p, vw):
    pm = vw["pm"]
    h = [dot([float(pm[4 * c + r]) for c in range(3)], p) + float(pm[12 + r]) for r in (0, 1, 3)]
    iw = 1.0 / (h[2] + float(f32(1e-7)))
    out = []
    for ndc, S in ((h[0] * iw, vw["W"]), (h[1] * iw, vw["H"])):
        v = ((ndc.v + 1.0) * S - 1.0) * 0.5    # ndc2pix in double from the float ndc, rounded once to float
        out.append(E(v, ndc.e * 0.5 * S + np.abs(v), ndc.d * 0.5 * S))
    return out, h, iw


def forward(g, cam, scale_modifier=1.0, antialias=False, mutate=()):
    """project.cu's per-Gaussian records of one view, in float64 with bounds.  `g`: means3D, opacities, scales +
    rotations or cov3D_precomp, shs + sh_degree or colors_precomp.  Returns a dict of float64 arrays; `X_B` is the
    rounding bound of X (units of u), `border` [P] marks Gaussians with a borderline decision."""
    vw = view_of(cam)
    W, H = vw["W"], vw["H"]
    p = _cols(g["means3D"])
    P = p[0].v.shape[0]
    S, R, se, q = cov3d(g, scale_modifier, mutate)
    G = _geometry(p, S, vw)
    tz, a, b, c, det = G["tz"], G["a"], G["b"], G["c"], G["det"]
    out = {}
    out["cov3D"] = np.stack([S[0][0].v, S[0][1].v, S[0][2].v, S[1][1].v, S[1][2].v, S[2][2].v], 1)
    out["cov3D_B"] = np.stack([x.e + 0 * x.v for x in (S[0][0], S[0][1], S[0][2], S[1][1], S[1][2], S[2][2])], 1)
    out["depth"], out["depth_B"] = tz.v, tz.e + 0 * tz.v
    m2, _, _ = _means2D(p, vw)
    out["means2D"] = np.stack([m2[0].v, m2[1].v], 1)
    out["means2D_B"] = np.stack([m2[0].e, m2[1].e], 1) + 0 * out["means2D"]
    conic = [c / det, -b / det, a / det]
    out["conic"] = np.stack([x.v for x in conic], 1)
    out["conic_B"] = np.stack([x.e + 0 * x.v for x in conic], 1)
    mid = 0.5 * (a + c)
    disc = mid * mid - det
    big = disc.v > float(f32(0.1))
    l1 = mid + sqrt(where(big, disc, float(f32(0.1))))
    rf = 3.0 * sqrt(l1)
    radius = np.ceil(rf.v).astype(np.int64)
    border = G["border"] | within(disc, float(f32(0.1))) | near_integer(rf, -10, 1 << 30) | within(tz, NEAR_Z)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rect = []
    for m, gmax in ((m2[0], gx), (m2[1], gy)):
        lo = (m - radius.astype(np.float64)) / 16.0
        hi = (m + radius.astype(np.float64) + 15.0) / 16.0
        rect.append((np.minimum(gmax, np.maximum(0, np.trunc(lo.v))).astype(np.int64),
                     np.minimum(gmax, np.maximum(0, np.trunc(hi.v))).astype(np.int64)))
        border |= near_integer(lo, 1, gmax) | near_integer(hi, 1, gmax)
    tiles = (rect[0][1] - rect[0][0]) * (rect[1][1] - rect[1][0])
    culled = (tz.v <= NEAR_Z) | (det.v == 0) | (tiles == 0)
    out["radius"] = np.where(culled, 0, radius)
    out["rect"] = np.stack([rect[0][0], rect[1][0], rect[0][1], rect[1][1]], 1)
    out["tiles_touched"] = np.where(culled, 0, tiles)
    out["culled"] = culled
    out["inx"], out["iny"] = G["inx"], G["iny"]
    # colour
    if g.get("shs") is not None:
        v, ln = _direction(p, vw)
        x, y, z = (vi / ln for vi in v)
        deg = int(g["sh_degree"])
        sh = np.asarray(g["shs"], f32).astype(np.float64)
        basis = _sh_basis(x, y, z, deg)
        rgb, rgbB, bits = np.zeros((P, 3)), np.zeros((P, 3)), np.zeros(P, np.int64)
        for ch in range(3):
            res = basis[0][0] * E(sh[:, 0, ch])
            for k in range(1, len(basis)):
                res = res + basis[k][0] * E(sh[:, k, ch])
            res = res + 0.5
            bits |= (res.v < 0).astype(np.int64) << ch
            border |= within(res, 0.0)
            rgb[:, ch], rgbB[:, ch] = np.maximum(res.v, 0.0), res.e
        out["rgb"], out["rgb_B"], out["clamped"] = rgb, rgbB, bits
    else:
        out["rgb"] = np.asarray(g["colors_precomp"], f32).astype(np.float64)
        out["rgb_B"], out["clamped"] = np.zeros((P, 3)), np.zeros(P, np.int64)
    # opacity (AA: o_eff = o s) and the footprint extent
    o = E(np.asarray(g["opacities"], f32).reshape(-1).astype(np.float64))
    if antialias:
        d0 = G["a0"] * G["c0"] - b * b
        r = d0 / det
        border |= within(r, AA_CLAMP)
        o = o * sqrt(where(r.v > AA_CLAMP, r, AA_CLAMP))
    out["opacity"], out["opacity_B"] = o.v, o.e + 0 * o.v
    o255 = 255.0 * o
    ext = np.full((P, 2), 1e30)
    extB = np.zeros((P, 2))
    border |= within(o255, float(f32(0.999)))
    tau = E(np.log(np.maximum(o255.v, 1e-30)), o255.e / np.maximum(o255.v, 1e-30) + 1.0) * float(f32(1.0005)) + float(f32(1e-3))
    ac = conic[0] * conic[2]
    dq = ac - conic[1] * conic[1]
    cut = float(f32(1e-3)) * ac
    ok = (conic[0].v > 0) & (conic[2].v > 0) & (dq.v > cut.v)
    border |= np.abs(dq.v - cut.v) <= BAND * U * (dq.e + cut.e)
    for i, cz in enumerate((conic[2], conic[0])):
        h = sqrt(2.0 * tau * cz / dq) * float(f32(1.001)) + float(f32(0.01))
        ext[:, i] = np.where(ok, h.v, 1e30)
        extB[:, i] = np.where(ok, h.e, 0.0)
    low = ~(o255.v >= float(f32(0.999)))
    ext[low], extB[low] = -1.0, 0.0
    out["extent"], out["extent_B"] = ext, extB
    out["border"] = border
    out["has_sh"] = g.get("shs") is not None
    return out


# --------------------------------------------------------------------------- backward
def _cot(x, B=None):
    x = np.asarray(x, np.float64)
    return E(x, 0.0, 0.0 if B is None else np.asarray(B, np.float64))


def backward(g, cams, cot, scale_modifier=1.0, antialias=False, live=None, clamped=None, shared_mean2D=False, mutate=()):
    """The per-Gaussian chain of project_bwd.cu over the views `cams`, in float64 with bounds.

    cot[v]: dict of the blend-stage cotangents of view v -- dL_dmean2D [P,2], dL_dconic [P,3] (a, half-b, c),
    dL_dopacity [P] (dL/do_eff under AA), dL_dcolor [P,3], dL_ddepth [P] or None -- each with an optional `<name>_B`
    absolute bound.  live[v] [P] bool (default: not culled by `forward`) and clamped[v] [P] bits (default: `forward`'s)
    are the decisions the chain follows.  Returns dict name -> (value, e, d) for dL_dmeans3D [P,3], dL_dcov3D [P,6],
    dL_dscales [P,3], dL_drotations [P,4], dL_dsh [P,M,3], dL_dopacity [P], dL_dcolors [P,3] and dL_dmeans2D [V,P,2]
    ([1,P,2] with shared_mean2D), plus `border` [P] (a borderline decision in some view)."""
    p = _cols(g["means3D"])
    P = p[0].v.shape[0]
    S, R, se, q = cov3d(g, scale_modifier, mutate)
    o_raw = E(np.asarray(g["opacities"], f32).reshape(-1).astype(np.float64))
    has_sh = g.get("shs") is not None
    deg = int(g["sh_degree"]) if has_sh else 0
    M = np.asarray(g["shs"]).shape[1] if has_sh else 0
    sh = np.asarray(g["shs"], f32).astype(np.float64) if has_sh else None
    nb = (deg + 1) ** 2
    if "sh_above_degree" in mutate:
        nb = min(M, 16)
    zero = E(np.zeros(P))
    gp = [zero, zero, zero]
    D = [[zero] * 3 for _ in range(3)]
    gop, gcol = zero, [zero, zero, zero]
    gsh = [[zero] * 3 for _ in range(M)]
    m2d = []
    border = np.zeros(P, bool)
    for v, cam in enumerate(cams):
        vw = view_of(cam)
        fw = forward(g, cam, scale_modifier, antialias, mutate)
        border |= fw["border"]
        lv = ~fw["culled"] if live is None else np.asarray(live[v], bool)
        cl = fw["clamped"] if clamped is None else np.asarray(clamped[v]).astype(np.int64)
        c = cot[v]
        gate = lambda x: where(lv, x, 0.0)  # noqa: E731
        dm = [gate(_cot(c["dL_dmean2D"][:, i], _b(c, "dL_dmean2D", i))) for i in range(2)]
        gA, gB, gC = (gate(_cot(c["dL_dconic"][:, i], _b(c, "dL_dconic", i))) for i in range(3))
        if "unhalve_b" in mutate:
            gB = 2.0 * gB
        gop_v = gate(_cot(c["dL_dopacity"], _b(c, "dL_dopacity")))
        dcol = [gate(_cot(c["dL_dcolor"][:, i], _b(c, "dL_dcolor", i))) for i in range(3)]
        dd = c.get("dL_ddepth")
        ddepth = gate(_cot(dd, c.get("dL_ddepth_B"))) if dd is not None else zero
        G = _geometry(p, S, vw)
        tz, a, b, cc, det = G["tz"], G["a"], G["b"], G["c"], G["det"]
        m0, m1, u0, u1 = G["m0"], G["m1"], G["u0"], G["u1"]
        gcol = [gcol[i] + dcol[i] for i in range(3)]
        # dL/dS' = H = -w adj(S') G adj(S'), w = 1 / (det^2 + 1e-7); gB is the half-weight off-diagonal cotangent
        wgt = 1.0 / (det * det + float(f32(1e-7)))
        e00, e01 = cc * gA - b * gB, cc * gB - b * gC
        e10, e11 = a * gB - b * gA, a * gC - b * gB
        H00 = -wgt * (e00 * cc - e01 * b)
        H01 = -wgt * (e01 * a - e00 * b)
        H11 = -wgt * (e11 * a - e10 * b)
        # the reference (and the C oracle) write -b^2 as (det - a c), which cancels for elongated splats: its rounding
        # |a c| u enters the bound of the diagonal terms
        H00.e = H00.e + wgt.v * np.abs(a.v * cc.v) * np.abs(gC.v)
        H11.e = H11.e + wgt.v * np.abs(a.v * cc.v) * np.abs(gA.v)
        if antialias:
            a0, c0 = G["a0"], G["c0"]
            d0 = a0 * c0 - b * b
            r = d0 / det
            on = r.v > AA_CLAMP
            s = sqrt(where(on, r, AA_CLAMP))
            gop = gop + where(lv, s * gop_v, 0.0)
            o_eff = o_raw * s
            k = 0.5 * gop_v * o_eff
            i0 = 1.0 / where(on, d0, 1.0)
            i1 = 1.0 / det
            H00 = H00 + where(on, k * (c0 * i0 - cc * i1), 0.0)
            H11 = H11 + where(on, k * (a0 * i0 - a * i1), 0.0)
            H01 = H01 + where(on, k * b * (i1 - i0), 0.0)
        else:
            gop = gop + gop_v
        h0 = [H00 * m0[i] + H01 * m1[i] for i in range(3)]
        h1 = [H01 * m0[i] + H11 * m1[i] for i in range(3)]
        for i in range(3):
            for j in range(i, 3):
                D[i][j] = D[i][j] + where(lv, m0[i] * h0[j] + m1[i] * h1[j], 0.0)
        # dL/dM = 2 H (M S), dL/dJ = dL/dM Rv^T: only J00, J02, J11, J12 move with t
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
        # the frustum clamp masks d/dt.x and d/dt.y ...
        mx = G["inx"] | ("no_x_mask" in mutate)
        my = G["iny"] | ("no_y_mask" in mutate)
        dtx = where(mx, -fx * iz2 * dJ02, 0.0)
        dty = where(my, -fy * iz2 * dJ12, 0.0)
        # ... and the clamped values cx, cy are constants in d/dt.z (depth = t.z takes dL_ddepth)
        dtz = (-fx * iz2 * dJ00 - fy * iz2 * dJ11 + 2.0 * fx * G["cx"] * iz3 * dJ02 + 2.0 * fy * G["cy"] * iz3 * dJ12
               + ddepth)
        if "true_dtz" in mutate:
            # the derivative of cx = lim t.z through the clamp: d J02 / d t.z gains -fx lim / t.z^2
            lx = np.where(G["inx"], 0.0, np.sign(G["cx"].v) * vw["limx"])
            ly = np.where(G["iny"], 0.0, np.sign(G["cy"].v) * vw["limy"])
            dtz = dtz + E(-fx * lx) * iz2 * dJ02 + E(-fy * ly) * iz2 * dJ12
        dt = [dtx, dty, dtz]
        _, h, iw = _means2D(p, vw)
        pm = vw["pm"]
        kx, ky = h[0] * iw * iw, h[1] * iw * iw
        for i in range(3):
            gi = dot([float(Rv[0][i]), float(Rv[1][i]), float(Rv[2][i])], dt)
            gi = gi + (float(pm[4 * i]) * iw - float(pm[4 * i + 3]) * kx) * dm[0] + \
                (float(pm[4 * i + 1]) * iw - float(pm[4 * i + 3]) * ky) * dm[1]
            gp[i] = gp[i] + where(lv, gi, 0.0)
        if has_sh:
            ign = "ignore_clamp_bits" in mutate
            # the per-channel clamp bits mask dRGB
            dRGB = [where(((cl >> ch) & 1).astype(bool) & (not ign), 0.0, dcol[ch]) for ch in range(3)]
            vv, ln = _direction(p, vw)
            il = 1.0 / ln
            x, y, z = (vi * il for vi in vv)
            basis = _sh_basis(x, y, z, 3 if "sh_above_degree" in mutate else deg)
            ddir = [zero, zero, zero]
            flip = {1: "sh_grad1", 5: "sh_grad2", 11: "sh_grad3"}
            for kk in range(min(nb, len(basis))):
                B, grad = basis[kk]
                for ch in range(3):
                    if kk < M:
                        gsh[kk][ch] = gsh[kk][ch] + B * dRGB[ch]
                if kk >= (deg + 1) ** 2:
                    continue
                s_ = dot([E(sh[:, kk, ch]) for ch in range(3)], dRGB)
                sg = -1.0 if flip.get(kk) in mutate else 1.0
                ddir = [ddir[i] + sg * (_e(grad[i]) * s_) for i in range(3)]
            # through the normalisation: d dir / d v = (I - dir dir^T) / |v|
            along = dot([x, y, z], ddir)
            for i, di in enumerate((x, y, z)):
                gp[i] = gp[i] + where(lv, (ddir[i] - di * along) * il, 0.0)
        if shared_mean2D:
            m2d = [dm[0] + m2d[0], dm[1] + m2d[1]] if m2d else dm
        else:
            m2d.append(dm)
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
        used = nb if "sh_above_degree" in mutate else (deg + 1) ** 2
        out["dL_dsh"] = tuple(np.stack([r[i] if k < used else 0 * r[i] for k, r in enumerate(rows)], 1) for i in range(3))
    # covariance -> scale and quaternion, once, on the sum over views
    if R is not None:
        Dm = [[D[min(i, j)][max(i, j)] for j in range(3)] for i in range(3)]
        dscale, A = [], [[None] * 3 for _ in range(3)]
        for j in range(3):
            gl = [2.0 * se[j] * dot([Dm[i][k] for k in range(3)], [R[k][j] for k in range(3)]) for i in range(3)]
            # dL/d(scale_modifier * scale): the reference's dL_dscale has no scale_modifier factor
            ds = dot([R[i][j] for i in range(3)], gl)
            if "scale_mod_in_dscale" in mutate:
                ds = float(f32(scale_modifier)) * ds
            dscale.append(ds)
            for i in range(3):
                A[i][j] = gl[i] * se[j]
        r_, x, y, z = q   # the quaternion un-normalised (R(q) of the forward)
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
    return out


def _b(c, name, i=None):
    B = c.get(name + "_B")
    if B is None:
        return None
    B = np.asarray(B, np.float64)
    return B if i is None else B[:, i]


def cov3d_grad(blend, g, cam, live=None):
    """dL_dcov3D [P,6] as (value, e, d) of one view's blend-stage conic gradients -- `blend` a blend_ref64.blend() result,
    whose dL_dconic bound (KAPPA u B of blend_ref64) is inherited -- through the chain of `backward` with every other
    cotangent zero: what the kernels return for cov3D_precomp.  Also returns the view's `border` mask."""
    P = len(g["means3D"])
    cot = dict(dL_dmean2D=np.zeros((P, 2)), dL_dconic=blend["dL_dconic"],
               dL_dconic_B=B64.KAPPA["dL_dconic"] * U * blend["dL_dconic_B"], dL_dopacity=np.zeros(P),
               dL_dcolor=np.zeros((P, 3)))
    out = backward(dict(g, shs=None), [cam], [cot], live=None if live is None else [live])
    return out["dL_dcov3D"], out["border"]


def raw_ratio(got, ref):
    """max(|got - value| - d, 0) / (u e) elementwise for ref = (value, e, d): the rounding part of the difference in units of
    the chain's own bound (the inherited bound d is not scaled); within bound when <= KAPPA[q]."""
    v, e, d = ref
    return np.maximum(np.abs(np.asarray(got, np.float64) - v) - d, 0.0) / (U * e + 1e-30)


def ratio(got, ref, quantity, kappa=None):
    """|got - ref| / (kappa u e + d + tiny) for ref = (value, e, d) or (value, e); kappa defaults to KAPPA[quantity]."""
    k = KAPPA[quantity] if kappa is None else kappa
    v, e = ref[0], ref[1]
    d = ref[2] if len(ref) > 2 else 0.0
    return np.abs(np.asarray(got, np.float64) - v) / (k * U * e + d + 1e-30)
