"""Expected values of the anti-aliased projection (opacity compensation) from the unmodified C oracle (oracle/gs_oracle.c)
plus a float64 restatement of the compensation.

Definition, per Gaussian and view: Sigma2 = the screen-space covariance before the 0.3 px^2 low-pass, S' = Sigma2 + 0.3 I =
[[a, b], [b, c]], d0 = det Sigma2, d1 = det S', r = d0 / d1, s = sqrt(max(2.5e-5, r)), o_eff = o s.  o_eff replaces o in
conic_opacity.w; everything else the projection writes is unchanged.

Forward: the oracle's projection and binning (which the mode does not touch), s in float64 from the oracle's float32 world-space
covariance (`compensation`), conic_opacity.w = float32(o s), then the oracle's own blend on that state.
Backward: the oracle's blend backward gives g = dL/do_eff.  dL/do = s g.  Where r > 2.5e-5 the covariance gains
g o ds/d(a, b, c) with, b one variable,
    ds/da = (c0 - r c) / (2 s d1),   ds/dc = (a0 - r a) / (2 s d1),   ds/db = -b (1 - r) / (s d1),   a0 = a - 0.3, c0 = c - 0.3.
The oracle's preprocess backward takes its input as dL/dconic, so this (a, b, c) gradient is mapped to the conic gradient that
the preprocess backward turns into exactly it (the 3x3 linear map of backward.cu:199-210, inverted per Gaussian), added to the
blend's, and the unmodified preprocess backward chains everything to means, scales, rotations or cov3D.  With
antialiasing=False both functions are gs_oracle.forward / backward, bit for bit (tests/test_antialias_cpu.py).
tests/test_antialias_cpu.py checks the backward against central differences of this forward.
"""
import ctypes as C

import numpy as np

from oracle import gs_oracle as O

CLAMP = 2.5e-5


def screen_cov64(means3D, viewmatrix, W, H, tanfovx, tanfovy, cov3D):
    """[P,2,2] screen-space covariance before the low-pass in float64 from float32 inputs: Sigma2 = J Rv Sigma Rv^T J^T with the
    reference's clamped J (forward.cu:75-107)."""
    vm = np.asarray(viewmatrix, np.float64).reshape(-1)
    Rv = np.array([[vm[4 * c + r] for c in range(3)] for r in range(3)])
    p = np.asarray(means3D, np.float64)
    t = p @ Rv.T + vm[12:15]
    tx_, ty_ = np.float32(tanfovx), np.float32(tanfovy)
    fx, fy = np.float64(np.float32(W / (2.0 * tx_))), np.float64(np.float32(H / (2.0 * ty_)))
    limx, limy = 1.3 * np.float64(tx_), 1.3 * np.float64(ty_)
    tx = np.clip(t[:, 0] / t[:, 2], -limx, limx) * t[:, 2]
    ty = np.clip(t[:, 1] / t[:, 2], -limy, limy) * t[:, 2]
    tz = t[:, 2]
    J = np.zeros((len(p), 2, 3))
    J[:, 0, 0], J[:, 0, 2] = fx / tz, -fx * tx / tz ** 2
    J[:, 1, 1], J[:, 1, 2] = fy / tz, -fy * ty / tz ** 2
    c = np.asarray(cov3D, np.float64)
    S = np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], 1)
    Mx = J @ Rv
    return Mx @ S @ np.transpose(Mx, (0, 2, 1))


def compensation(fw, means3D, viewmatrix, tanfovx, tanfovy, cov3D_precomp=None):
    """dict(s, r, a, b, c, d1) per Gaussian in float64 (a, b, c: the dilated covariance S')."""
    cov3D = cov3D_precomp if cov3D_precomp is not None else fw["cov3D"]
    S2 = screen_cov64(means3D, viewmatrix, fw["W"], fw["H"], tanfovx, tanfovy, cov3D)
    a0, b, c0 = S2[:, 0, 0], S2[:, 0, 1], S2[:, 1, 1]
    a, c = a0 + 0.3, c0 + 0.3
    d0, d1 = a0 * c0 - b * b, a * c - b * b
    r = d0 / d1
    return dict(s=np.sqrt(np.maximum(CLAMP, r)), r=r, a=a, b=b, c=c, d1=d1)


def forward(means3D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, bg, antialiasing=True, **kw):
    """gs_oracle.forward() with the anti-aliased projection: fw["conic_opacity"][:, 3] = o_eff, fw["aa"] = compensation()."""
    stages_only = kw.pop("stages_only", False)
    if not antialiasing:
        return O.forward(means3D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, bg, stages_only=stages_only, **kw)
    fw = O.forward(means3D, opacities, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, bg, stages_only=True, **kw)
    comp = compensation(fw, means3D, viewmatrix, tanfovx, tanfovy, kw.get("cov3D_precomp"))
    vis = fw["radii"] > 0
    o = np.asarray(opacities, np.float32).reshape(-1).astype(np.float64)
    fw["conic_opacity"][vis, 3] = (o * comp["s"])[vis].astype(np.float32)
    fw["aa"], fw["opacities"] = comp, np.asarray(opacities, np.float32).reshape(-1)
    if stages_only:
        return fw
    # the oracle's blend on the compensated state (gs_oracle.forward's last step)
    L = O.lib()
    F, N = fw["F"], W * H
    colors = O._f32(kw.get("colors_precomp")) if kw.get("colors_precomp") is not None else fw["rgb"]
    feature = O._f32(kw.get("feature"))
    fw["final_T"] = np.zeros(N, np.float32)
    fw["n_contrib"] = np.zeros(N, np.uint32)
    fw["out_color"] = np.zeros((3, H, W), np.float32)
    fw["out_feature"] = np.zeros((F, H, W), np.float32) if F else np.zeros((1,), np.float32)
    L.gso_render_forward(C.c_int(W), C.c_int(H), C.c_int(F), O._p(fw["ranges"]), O._p(fw["point_list"]), O._p(fw["means2D"]),
                         O._p(colors), O._p(feature), O._p(fw["conic_opacity"]), O._p(O._f32(bg).reshape(-1)), O._p(fw["final_T"]),
                         O._p(fw["n_contrib"]), O._p(fw["out_color"]), O._p(fw["out_feature"]))
    return fw


def conic_gradient(comp, Ga, Gb, Gc):
    """[P,3] (dL/dconic.x, .y halved, .w) that the oracle's preprocess backward (backward.cu:199-210) maps to the covariance
    gradient (Ga, Gb (b one variable), Gc)."""
    a, b, c, D = comp["a"], comp["b"], comp["c"], comp["d1"]
    k = 1.0 / (D * D + 1e-7)
    A = np.zeros((len(a), 3, 3))
    A[:, 0] = np.stack([-c * c, 2 * b * c, -b * b], 1)
    A[:, 1] = np.stack([2 * b * c, -2 * (D + 2 * b * b), 2 * a * b], 1)
    A[:, 2] = np.stack([-b * b, 2 * a * b, -a * a], 1)
    A *= k[:, None, None]
    return np.linalg.solve(A, np.stack([Ga, Gb, Gc], 1)[:, :, None])[:, :, 0]


def compensation_backward(fw, g_eff):
    """(dL/do [P], extra dL/dconic [P,4]) of the compensation, given g_eff = dL/do_eff [P]."""
    comp = fw["aa"]
    P = len(g_eff)
    vis = fw["radii"] > 0
    s, r, d1 = comp["s"], comp["r"], comp["d1"]
    g = np.where(vis, np.asarray(g_eff, np.float64).reshape(-1), 0.0)
    go = g * fw["opacities"].astype(np.float64)
    live = vis & (r > CLAMP)
    Ga = np.where(live, go * ((comp["c"] - 0.3) - r * comp["c"]) / (2 * s * d1), 0.0)
    Gc = np.where(live, go * ((comp["a"] - 0.3) - r * comp["a"]) / (2 * s * d1), 0.0)
    Gb = np.where(live, go * (-comp["b"] * (1 - r)) / (s * d1), 0.0)
    dconic = np.zeros((P, 4))
    if live.any():
        x = conic_gradient({k: v[live] for k, v in comp.items()}, Ga[live], Gb[live], Gc[live])
        dconic[live, 0], dconic[live, 1], dconic[live, 3] = x[:, 0], x[:, 1], x[:, 2]
    return (s * g).astype(np.float32), dconic


def preprocess_backward(fw, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy, dL_dmean2D, dL_dconic, dL_dcolor, dL_dopacity_eff,
                        scales=None, rotations=None, cov3D_precomp=None, shs=None, sh_degree=0, scale_modifier=1.0, **_):
    """The per-Gaussian backward of the anti-aliased projection: the oracle's gso_preprocess_backward on the blend's conic
    gradient plus the compensation's, and dL/do.  Returns dict(dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations,
    dL_dopacity)."""
    P, W, H = fw["P"], fw["W"], fw["H"]
    M = 0 if shs is None else np.asarray(shs).shape[1]
    dL_dopacity, extra = compensation_backward(fw, dL_dopacity_eff)
    dconic = (np.asarray(dL_dconic, np.float64).reshape(P, 4) + extra).astype(np.float32)
    out = dict(dL_dmeans3D=np.zeros((P, 3), np.float32), dL_dcov3D=np.zeros((P, 6), np.float32),
               dL_dsh=np.zeros((P, M, 3), np.float32), dL_dscales=np.zeros((P, 3), np.float32),
               dL_drotations=np.zeros((P, 4), np.float32), dL_dopacity=dL_dopacity.reshape(P, 1))
    f32 = O._f32
    cov3D = f32(cov3D_precomp) if cov3D_precomp is not None else fw["cov3D"]
    O.lib().gso_preprocess_backward(
        C.c_int(P), C.c_int(sh_degree), C.c_int(M), O._p(f32(means3D)), O._p(fw["radii"]), O._p(f32(shs)), O._p(fw["clamped"]),
        O._p(f32(scales)), O._p(f32(rotations)), C.c_float(scale_modifier), O._p(cov3D), O._p(f32(viewmatrix).reshape(-1)),
        O._p(f32(projmatrix).reshape(-1)), C.c_int(W), C.c_int(H), C.c_float(tanfovx), C.c_float(tanfovy), O._p(f32(campos).reshape(-1)),
        O._p(f32(dL_dmean2D)), O._p(dconic), O._p(f32(dL_dcolor)), O._p(out["dL_dmeans3D"]), O._p(out["dL_dcov3D"]), O._p(out["dL_dsh"]),
        O._p(out["dL_dscales"]), O._p(out["dL_drotations"]))
    return out


def backward(fw, dL_dcolor, dL_dfeature, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy, bg, antialiasing=True, **kw):
    """gs_oracle.backward() of an anti-aliased forward(): dL_dopacity is dL/do of the raw opacity, dL_dopacity_eff the blend's."""
    if not antialiasing:
        return O.backward(fw, dL_dcolor, dL_dfeature, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy, bg, **kw)
    L = O.lib()
    P, W, H, F, M = fw["P"], fw["W"], fw["H"], fw["F"], fw["M"]
    f32 = O._f32
    feature = f32(kw.get("feature"))
    colors = f32(kw.get("colors_precomp")) if kw.get("colors_precomp") is not None else fw["rgb"]
    g = dict(dL_dmeans2D=np.zeros((P, 3), np.float32), dL_dconic=np.zeros((P, 4), np.float32),
             dL_dopacity_eff=np.zeros((P, 1), np.float32), dL_dcolors=np.zeros((P, 3), np.float32),
             dL_dfeature=np.zeros((P, F), np.float32) if F else np.zeros((1,), np.float32))
    L.gso_render_backward(C.c_int(P), C.c_int(W), C.c_int(H), C.c_int(F), O._p(fw["ranges"]), O._p(fw["point_list"]),
                          O._p(f32(bg).reshape(-1)), O._p(fw["means2D"]), O._p(fw["conic_opacity"]), O._p(colors), O._p(feature),
                          O._p(fw["final_T"]), O._p(fw["n_contrib"]), O._p(f32(dL_dcolor)), O._p(f32(dL_dfeature) if F else None),
                          O._p(g["dL_dmeans2D"]), O._p(g["dL_dconic"]), O._p(g["dL_dopacity_eff"]), O._p(g["dL_dcolors"]),
                          O._p(g["dL_dfeature"]))
    g.update(preprocess_backward(fw, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy, g["dL_dmeans2D"], g["dL_dconic"],
                                 g["dL_dcolors"], g["dL_dopacity_eff"], **kw))
    return g
