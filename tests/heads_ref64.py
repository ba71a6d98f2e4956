"""Float64 reference of the pointwise heads (DESIGN rows f2, f4, f9), with a first-order bound of fp32 evaluation.

Every value is an `E` of project_ref64: its float64 value `v` and `e`, a first-order bound (units of u = 2^-24) of the error
fp32 evaluation of the same expression accumulates from exact fp32 inputs.  A kernel value x is within bound when
|x - v| <= KAPPA[q] u e.  Each function follows its kernel's operation order; a reduction of n terms is bounded as in
camera_ref64: the terms' own bounds plus `depth` u |term| for each term, `depth` being the longest chain of fp32 additions
the kernel's reduction shape (sequential loop, warp-shuffle tree, the chain of `red_add` atomics) can put a term through.

* `activate` / `activate_backward` (activate.cu): means + offsets, min(exp(s + ds), scale_max), q / max(|q|, 1e-12),
  sigmoid, and feature rows x / (|x| + 1e-12), forward and backward.  Where exp(s + ds) lies within BAND u e of scale_max,
  or |q| within BAND u e of 1e-12, fp32 may take the other branch of the clamp: such an element is `border` and unchecked.
  expf is taken as 2 ulp (CUDA's bound); -v past fp32 exp's overflow gives sigmoid 0 exactly, as the kernel does.
* `loss_heads` (loss_heads.cuh): the colour L2 cotangent 2 (x - g) / (3 N) and S_rgb = sum (x - g)^2, and the cosine head
  with ATen's gradient, d cos / dx = y / (cx cy) - cos x / (|x| cx), cx = max(|x|, eps), for every |x| > 0.  The clamps
  max(|x|, eps) and max(|y|, eps) are 1-Lipschitz and the gradient is continuous at |x| = eps, so those decisions need no
  band; |x| = 0 is exact for fp32 inputs whose squares do not underflow.  Norms whose square overflows fp32 (|x| >~ 1e19)
  are out of scope.
* `ssim_forward` / `ssim_backward` (ssim.cu): the two separable 11-tap passes (each a sequential loop over the taps, with
  the window's fp32-rounded weights as rounded constants), the cancellation in E[x^2] - mu^2, S, the three partials and the
  per-view sums {sum |x - g|, sum S}; the backward convolves the partials, adds the sign term, cot_in_scale cot_in and the
  per-view scales.  sign(x - g) is exact for fp32 inputs.

`mutate` breaks one convention on purpose (MUTATIONS): tests/test_heads_ref64_cpu.py shows each moves a checked element past
twice its bound.
"""
import math

import numpy as np

from project_ref64 import E, U, sqrt, where, within

f32 = np.float32
BAND = 4.0
FLT_MAX = float(np.finfo(f32).max)
COS_EPS = float(f32(1e-8))     # the fp32 constants the kernels compare against
ROT_EPS = float(f32(1e-12))
FEAT_EPS = float(f32(1e-12))
SS_TW, SS_TH, SS_R = 32, 16, 5
GAUSS = np.array([math.exp(-(i - 5) ** 2 / 4.5) for i in range(11)])
GAUSS = GAUSS / GAUSS.sum()
MUTATIONS = ("cos_k0_below_eps", "rgb_one_third", "ssim_halo_shift", "ssim_c1_c2_swapped", "ssim_exg_no_2", "sigmoid_bwd_x",
             "feat_eps_in_sqrt")
# an element is within bound when |x - v| <= KAPPA[q] u e: 4x the largest |x - v| / (u e) measured against the kernels over
# every case of tests/test_heads_ref64_gpu.py (H100 80GB HBM3; the table is in its docstring).  The accumulators' bounds
# (S_rgb, S_cos, sum_l1, sum_S) charge every term the whole chain of atomics, which the measured sums stay far below.
KAPPA = dict(means=4.0, scales=4.0, rot=2.3, opac=2.9, feature=1.7,
             dL_scales=3.0, dL_rot=1.95, dL_opac=2.9, dL_feature=1.4,
             cot_color=3.0, cot_feature=1.5, S_rgb=0.58, S_cos=0.062,
             dS_dmu=0.63, dS_dxx=0.69, dS_dxg=0.7, sum_l1=0.39, sum_S=0.089, ssim_cot=1.92)


def x_(a):
    """exact fp32 input"""
    return E(np.asarray(a, f32).astype(np.float64))


def const(c):
    """a constant the kernel holds rounded to fp32"""
    return E(c, abs(c))


def _arr(a):
    """an E whose e and d are arrays of v's shape"""
    z = 0 * a.v
    return E(a.v, a.e + z, a.d + z)


def chain_sum(t, axis, depth):
    """sum of the E terms t along axis, for any fp32 order whose longest chain of additions is `depth`"""
    t = _arr(t)
    return E(t.v.sum(axis), t.e.sum(axis) + depth * np.abs(t.v).sum(axis), t.d.sum(axis))


def expand(a, axis):
    return E(np.expand_dims(a.v, axis), np.expand_dims(a.e + 0 * a.v, axis), np.expand_dims(a.d + 0 * a.v, axis))


def exp_(a, ulp=2.0):
    y = np.exp(a.v)
    return E(y, y * a.e + ulp * y, y * a.d)


def clamp_min(a, lo):
    """max(a, lo): 1-Lipschitz, so a's bound carries over whichever side fp32 lands on"""
    return E(np.maximum(a.v, lo), a.e + 0 * a.v, a.d + 0 * a.v)


def ratio(got, ref):
    """|got - v| / (u e) elementwise: within bound when <= KAPPA[q]"""
    return np.abs(np.asarray(got, np.float64) - ref.v) / (U * (ref.e + 0 * ref.v) + 1e-300)


# --------------------------------------------------------------------------- f2 activations
def _plus(a, d):
    return x_(a) if d is None else x_(a) + x_(d)


def _rows_depth(F):
    """the row sums of feature_rows (ceil(F / G) lanes' loops + the shuffle tree) and of the vec4 path (4 + its tree) both
    stay within F additions"""
    return max(int(F), 1)


def activate(means=None, d_means=None, rot=None, d_rot=None, scales=None, d_scales=None, opac=None, feature=None,
             scale_mode=1, scale_max=0.05, opacity_mode=1, rot_normalize=True, feature_normalize=True, mutate=()):
    """-> dict of name -> E, and 'border_scales' / 'border_rot' masks (elementwise / per row)"""
    out = {}
    if means is not None:
        out["means"] = _plus(means, d_means)
    if scales is not None:
        v = _plus(scales, d_scales)
        if scale_mode == 1:
            smax = float(f32(scale_max))
            y = exp_(v)
            out["border_scales"] = within(y, smax, BAND)
            v = where(y.v <= smax, y, smax)
        out["scales"] = v
    if rot is not None:
        q = [_plus(rot[:, k], None if d_rot is None else d_rot[:, k]) for k in range(4)]
        if rot_normalize:
            ss = q[0] * q[0]
            for k in range(1, 4):
                ss = ss + q[k] * q[k]
            n = sqrt(ss)
            d = clamp_min(n, ROT_EPS)
            out["rot"] = [qk / d for qk in q]
            out["border_rot"] = within(n, ROT_EPS, BAND)
        else:
            out["rot"] = q
    if opac is not None:
        o = x_(opac)
        if opacity_mode == 1:
            ex = exp_(-o)
            y = 1.0 / (1.0 + ex)
            o = where(ex.v > FLT_MAX, 0.0, y)
        out["opac"] = o
    if feature is not None and feature.shape[1] > 0:
        x = x_(feature)
        if feature_normalize:
            n = _feature_norm(x, mutate)
            out["feature"] = x / expand(n[1], 1)
        else:
            out["feature"] = x
    return out


def _feature_norm(x, mutate):
    """(|x|, |x| + eps) per row"""
    ss = chain_sum(x * x, 1, _rows_depth(x.v.shape[1]))
    if "feat_eps_in_sqrt" in mutate:
        n = sqrt(ss + FEAT_EPS)
        return n, n
    n = sqrt(ss)
    return n, n + FEAT_EPS


def activate_backward(means=None, d_means=None, rot=None, d_rot=None, scales=None, d_scales=None, opac=None, feature=None,
                      g_means=None, g_rot=None, g_scales=None, g_opac=None, g_feature=None,
                      scale_mode=1, scale_max=0.05, opacity_mode=1, rot_normalize=True, feature_normalize=True, mutate=()):
    """-> dict dL_means, dL_scales, dL_rot (list of 4), dL_opac, dL_feature (E each), border_scales / border_rot"""
    out = {}
    if g_means is not None:
        out["dL_means"] = x_(g_means)
    if g_scales is not None:
        g = x_(g_scales)
        if scale_mode == 1:
            smax = float(f32(scale_max))
            y = exp_(_plus(scales, d_scales))
            out["border_scales"] = within(y, smax, BAND)
            g = where(y.v <= smax, g * y, 0.0)
        out["dL_scales"] = g
    if g_rot is not None:
        q = [_plus(rot[:, k], None if d_rot is None else d_rot[:, k]) for k in range(4)]
        g = [x_(g_rot[:, k]) for k in range(4)]
        if rot_normalize:
            ss, gq = q[0] * q[0], g[0] * q[0]
            for k in range(1, 4):
                ss, gq = ss + q[k] * q[k], gq + g[k] * q[k]
            n = sqrt(ss)
            d = clamp_min(n, ROT_EPS)
            live = n.v >= ROT_EPS
            k2 = where(live, gq / (d * d * where(live, n, 1.0)), 0.0)
            g = [gk / d - qk * k2 for gk, qk in zip(g, q)]
            out["border_rot"] = within(n, ROT_EPS, BAND)
        out["dL_rot"] = g
    if g_opac is not None:
        g = x_(g_opac)
        if opacity_mode == 1:
            o = x_(opac)
            ex = exp_(-o)
            y = where(ex.v > FLT_MAX, 0.0, 1.0 / (1.0 + ex))
            if "sigmoid_bwd_x" in mutate:
                y = o
            g = (g * (1.0 - y)) * y
        out["dL_opac"] = g
    if g_feature is not None and feature is not None and feature.shape[1] > 0:
        x, g = x_(feature), x_(g_feature)
        if feature_normalize:
            n, d = _feature_norm(x, mutate)
            gx = chain_sum(g * x, 1, _rows_depth(x.v.shape[1]))
            live = n.v > 0
            k = expand(where(live, gx / (d * d * where(live, n, 1.0)), 0.0), 1)
            out["dL_feature"] = g / expand(d, 1) - x * k
        else:
            out["dL_feature"] = g
    return out


# --------------------------------------------------------------------------- f4 colour L2 + cosine embedding
def heads_depth(N):
    """loss_heads.cu's accumulators past a pixel's own thread: the warp's shuffle tree (5), then one red_add per warp"""
    return 5 + -(-int(N) // 32)


def _flat(a, V):
    a = _arr(a)
    return E(a.v.reshape(V, -1), a.e.reshape(V, -1), a.d.reshape(V, -1))


def loss_heads(color=None, tgt_color=None, feature=None, tgt_feature=None, eps=COS_EPS, depth=None, mutate=()):
    """color / tgt_color [V,3,N], feature / tgt_feature [V,F,N] (fp32, either pair None).  depth: the accumulators' chain past
    the pixel's thread (default heads_depth(N)); S_rgb adds the 3 channels.  -> dict cot_color [V,3,N], S_rgb [V],
    cot_feature [V,F,N], S_cos [V] (E each), cos [V,N]"""
    out = {}
    N = (color if color is not None else feature).shape[-1]
    depth = heads_depth(N) if depth is None else depth
    invN = const(1.0 / N)
    if color is not None:
        d = x_(color) - x_(tgt_color)
        c23 = const(1.0 / 3.0 if "rgb_one_third" in mutate else 2.0 / 3.0)
        out["cot_color"] = (c23 * invN) * d
        out["S_rgb"] = chain_sum(_flat(d * d, d.v.shape[0]), 1, 3 + depth)
    if feature is not None and feature.shape[1] > 0:
        F = feature.shape[1]
        x, y = x_(feature), x_(tgt_feature)
        xy, xx, yy = (chain_sum(a * b, 1, F) for a, b in ((x, y), (x, x), (y, y)))
        nx, ny = sqrt(xx), sqrt(yy)
        cx, cy = clamp_min(nx, eps), clamp_min(ny, eps)
        inv_nn = 1.0 / (cx * cy)
        cos = xy * inv_nn
        live = nx.v > 0
        if "cos_k0_below_eps" in mutate:
            live = nx.v > eps
        k = where(live, cos / (where(live, nx, 1.0) * cx), 0.0)
        out["cot_feature"] = (-1.0 * invN) * (y * expand(inv_nn, 1) - expand(k, 1) * x)
        out["cos"] = cos
        out["S_cos"] = chain_sum(cos, 1, depth)
    return out


# --------------------------------------------------------------------------- f9 L1 + SSIM
def _shift(a, dy, dx):
    """b[..., i, j] = a[..., i + dy, j + dx], zero outside the image"""
    def sh(z):
        z = np.asarray(z + 0 * a.v, np.float64)
        H, W = z.shape[-2:]
        o = np.zeros_like(z)
        ys, yd = (slice(dy, H), slice(0, H - dy)) if dy >= 0 else (slice(0, H + dy), slice(-dy, H))
        xs, xd = (slice(dx, W), slice(0, W - dx)) if dx >= 0 else (slice(0, W + dx), slice(-dx, W))
        o[..., yd, xd] = z[..., ys, xs]
        return o
    return E(sh(a.v), sh(a.e), sh(a.d))


def _pass(a, axis, xs=None):
    """one 11-tap pass along axis (-1: the rows, horizontal; -2: the columns), taps in order k = 0..10 as the kernel's
    `acc += w * v` from 0.  xs (with a): the second factor of the w * x * x and w * x * g products."""
    acc = None
    for k in range(11):
        o = k - SS_R
        s = _shift(a, 0, o) if axis == -1 else _shift(a, o, 0)
        t = const(GAUSS[k]) * s
        if xs is not None:
            t = t * (_shift(xs, 0, o) if axis == -1 else _shift(xs, o, 0))
        acc = t if acc is None else acc + t
    return acc


def _hpass(a, mutate=(), xs=None):
    h = _pass(a, -1, xs)
    if "ssim_halo_shift" in mutate:
        # a tile's halo loaded one pixel to the right: the horizontal sums of the first column of every tile but the first
        sh = _pass(_shift(a, 0, 1), -1, None if xs is None else _shift(xs, 0, 1))
        W = a.v.shape[-1]
        cols = np.arange(SS_TW, W, SS_TW)
        h = _arr(h)
        sh = _arr(sh)
        h.v[..., cols] = sh.v[..., cols]
        h.e[..., cols] = sh.e[..., cols]
    return h


def ssim_depth(C, H, W):
    """ssim_fwd_kernel: 2 rows per thread, the warp's shuffle tree (5), one red_add per warp: 8 warps x the view's tiles"""
    return 2 + 5 + 8 * C * -(-W // SS_TW) * -(-H // SS_TH)


def ssim_forward(x, g, mutate=()):
    """x, g [V,C,H,W] fp32.  -> dict dS_dmu, dS_dxx, dS_dxg [V,C,H,W] (the kernel's terms planes), S, sum_l1 [V], sum_S [V]"""
    X, G = x_(x), x_(g)
    V, C, H, W = X.v.shape
    hz = [_hpass(X, mutate), _hpass(G, mutate), _hpass(X, mutate, X), _hpass(G, mutate, G), _hpass(X, mutate, G)]
    m = [_pass(h, -2) for h in hz]
    mux, mug = m[0], m[1]
    sxx, sgg, sxg = m[2] - mux * mux, m[3] - mug * mug, m[4] - mux * mug
    c1, c2 = E(1e-4, 3e-4), E(9e-4, 3 * 9e-4)  # 0.01f * 0.01f, 0.03f * 0.03f: two rounded factors and a rounded product
    if "ssim_c1_c2_swapped" in mutate:
        c1, c2 = c2, c1
    A = 2.0 * mux * mug + c1
    B = 2.0 * sxg + c2
    Cc = mux * mux + mug * mug + c1
    D = sxx + sgg + c2
    inv_cd = 1.0 / (Cc * D)
    S = A * B * inv_cd
    out = dict(S=S)
    out["dS_dmu"] = 2.0 * mug * (B - A) * inv_cd - 2.0 * mux * S * (1.0 / Cc - 1.0 / D)
    out["dS_dxx"] = -1.0 * S / D
    out["dS_dxg"] = (1.0 if "ssim_exg_no_2" in mutate else 2.0) * A * inv_cd
    dep = ssim_depth(C, H, W)
    ad = X - G
    out["sum_l1"] = chain_sum(_flat(E(np.abs(ad.v), ad.e, ad.d), V), 1, dep)
    out["sum_S"] = chain_sum(_flat(S, V), 1, dep)
    return out


def ssim_backward(x, g, terms, scale=None, cot_in=None, cot_in_scale=None, mutate=()):
    """cot_out [V,C,H,W] = cot_in_scale cot_in + scale[v,0] sign(x - g) / N + scale[v,1] d ssim / dx.  terms: the three
    partials, either a dict of E as ssim_forward returns or fp32 arrays [V,3,C,H,W] (the kernel's own planes, exact);
    scale [V,2] fp32 or None (1), cot_in [V,C,H,W] or None, cot_in_scale [V] or None (1)."""
    X, G = x_(x), x_(g)
    V, C, H, W = X.v.shape
    if isinstance(terms, dict):
        T = [terms[k] for k in ("dS_dmu", "dS_dxx", "dS_dxg")]
    else:
        T = [x_(terms[:, t]) for t in range(3)]
    m0, m1, m2 = (_pass(_hpass(t, mutate), -2) for t in T)
    inv_n = const(1.0 / (C * H * W))
    sc = np.ones((V, 2), f32) if scale is None else np.asarray(scale, f32)
    g_l1 = E(sc[:, 0].astype(np.float64)) * inv_n
    g_ss = E(sc[:, 1].astype(np.float64)) * inv_n
    g_l1, g_ss = (E(a.v[:, None, None, None], (a.e + 0 * a.v)[:, None, None, None]) for a in (g_l1, g_ss))
    sgn = np.sign(X.v - G.v)
    val = g_l1 * sgn + g_ss * (m0 + 2.0 * X * m1 + G * m2)
    if cot_in is not None:
        s_in = np.ones(V) if cot_in_scale is None else np.asarray(cot_in_scale, f32).astype(np.float64)
        val = val + E(s_in[:, None, None, None]) * x_(cot_in)
    return val
