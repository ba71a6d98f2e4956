"""A numpy restatement of MCMC density control (include/mgs_rasterizer.h, mgs_mcmc_relocate / mgs_mcmc_perturb).

The generator (Philox4x32-10), the dead test, the weights, the integer draw and the counts are restated bit for bit; the
relocation maths and the position noise in float64.  gsplat_double_sum is gsplat's relocation formula as it writes it, a
double sum over i = 1..n and k = 0..i-1, which the hockey-stick identity collapses into relocation_maths' single sum.
"""
import math

import numpy as np

MASK = np.uint64(0xFFFFFFFF)
TAG_RELOCATE, TAG_PERTURB = 0, 1
N_MAX = 51
EPS = 2.0 ** -23


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Random123's philox4x32 with 10 rounds on broadcast uint32 counters and a two-word key: four uint32 arrays"""
    c = [np.asarray(v, np.uint64) & MASK for v in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & MASK, np.uint64(k1) & MASK
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & MASK, (k1 + np.uint64(0xBB67AE85)) & MASK
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & MASK]
    return [v.astype(np.uint32) for v in c]


def draws(seed, offset, slots, tag):
    """the four words of each slot at the generator state {seed, offset}"""
    seed, offset = int(seed) & (2 ** 64 - 1), int(offset) & (2 ** 64 - 1)
    return philox4x32_10(np.asarray(slots, np.uint64), offset & 0xFFFFFFFF, offset >> 32, tag, seed & 0xFFFFFFFF, seed >> 32)


def mulhi64(a, b):
    """the high 64 bits of the 128-bit products a b (uint64 arrays)"""
    a, b = np.asarray(a, np.uint64), np.asarray(b, np.uint64)
    s = np.uint64(32)
    al, ah, bl, bh = a & MASK, a >> s, b & MASK, b >> s
    ll, lh, hl, hh = al * bl, al * bh, ah * bl, ah * bh
    mid = (ll >> s) + (lh & MASK) + (hl & MASK)
    return hh + (lh >> s) + (hl >> s) + (mid >> s)


def dead_threshold(min_opacity):
    mo = float(np.float32(min_opacity))
    return np.float32(math.log(mo / (1.0 - mo)))


def weights(x, t):
    """w_i = floor(2^24 sigmoid_f64(x_i)) where x_i > t, else 0 (NaN included)"""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        o = 1.0 / (1.0 + np.exp(-x.astype(np.float64)))
        w = np.where(x > t, np.floor(o * 2.0 ** 24), 0.0)
    return w.astype(np.uint64)


def draw(x, P_old, P, seed, offset, min_opacity=0.005):
    """(source [P] int64, m [P_old] int64, relocated) of the definition: the integer part of a relocation"""
    x = np.asarray(x, np.float32)
    t = dead_threshold(min_opacity)
    S = np.cumsum(weights(x[:P_old], t), dtype=np.uint64)
    T = S[-1] if P_old else np.uint64(0)
    dest = np.concatenate([x[:P_old] <= t, np.ones(P - P_old, bool)])
    source = np.full(P, -1, np.int64)
    if T > 0:
        j = np.nonzero(dest)[0]
        w0, w1, _, _ = draws(seed, offset, j, TAG_RELOCATE)
        r64 = w0.astype(np.uint64) | (w1.astype(np.uint64) << np.uint64(32))
        source[j] = np.searchsorted(S, mulhi64(r64, T), side="right")
    m = np.bincount(source[source >= 0], minlength=P_old).astype(np.int64)
    return source, m, int((source >= 0).sum())


_BINOM = np.array([[float(math.comb(n, j)) for j in range(N_MAX + 1)] for n in range(N_MAX + 1)])


def relocation_maths(o, n):
    """(o', s'/s) of the definition in float64: o' = -expm1(log1p(-o)/n), s'/s = o / sum_j C(n,j) (-1)^(j-1) o'^j / sqrt(j)"""
    o, n = np.asarray(o, np.float64), np.asarray(n, np.int64)
    a = -np.expm1(np.log1p(-o) / n)
    den = np.zeros_like(a)
    for j in range(1, N_MAX + 1):
        term = _BINOM[n, j] * a ** j / math.sqrt(j) * (1.0 if j % 2 else -1.0)
        den += np.where(j <= n, term, 0.0)
    return a, o / den


def gsplat_double_sum(o, n):
    """gsplat's relocation formula as written: o' = 1 - (1 - o)^(1/n), s'/s = o / sum_{i=1..n} sum_{k=0..i-1}
    C(i-1,k) (-1)^k o'^(k+1) / sqrt(k+1), scalar o and n"""
    a = 1.0 - (1.0 - o) ** (1.0 / n)
    den = 0.0
    for i in range(1, n + 1):
        for k in range(i):
            den += math.comb(i - 1, k) * (-1.0) ** k * a ** (k + 1) / math.sqrt(k + 1)
    return a, o / den


def relocate(params, P_old, seed, offset, min_opacity=0.005):
    """the expected result of mgs_mcmc_relocate: params a dict of float32 arrays [P, ...] with keys pts_xyz, rotations,
    scales (log), opacity (logits, [P]) and any further rows.  Returns (new params, source, relocated, touched [P] bool:
    sources and filled destinations, where every moment is zero), the new opacity logits and log scales of the sources
    as float64 before their final rounding under "x64" and "ls64"."""
    x = params["opacity"].reshape(-1)
    P = x.shape[0]
    source, m, relocated = draw(x, P_old, P, seed, offset, min_opacity)
    out = {k: v.copy() for k, v in params.items()}
    src = np.nonzero(m > 0)[0]
    o = 1.0 / (1.0 + np.exp(-x[src].astype(np.float64)))
    a, ratio = relocation_maths(o, np.minimum(m[src] + 1, N_MAX))
    a = np.clip(a, float(np.float32(min_opacity)), 1.0 - EPS)
    x64 = np.log(a / (1.0 - a))
    ls64 = np.log(np.exp(params["scales"][src].astype(np.float64)) * ratio[:, None])
    out["opacity"].reshape(-1)[src] = x64.astype(np.float32)
    out["scales"][src] = ls64.astype(np.float32)
    j = np.nonzero(source >= 0)[0]
    for k in out:
        out[k][j] = out[k][source[j]]
    touched = np.zeros(P, bool)
    touched[src] = True
    touched[j] = True
    return out, source, relocated, touched, {"src": src, "x64": x64, "ls64": ls64}


def normals(seed, offset, P):
    """z [P,3] float64 from the float32 uniforms the definition's Box-Muller takes"""
    w0, w1, w2, w3 = draws(seed, offset, np.arange(P), TAG_PERTURB)
    f = np.float32(2.0 ** -32)
    u = [(w.astype(np.float32) + np.float32(1.0)) * f if k % 2 == 0 else w.astype(np.float32) * f
         for k, w in enumerate((w0, w1, w2, w3))]
    r0, r1 = np.sqrt(-2.0 * np.log(u[0].astype(np.float64))), np.sqrt(-2.0 * np.log(u[2].astype(np.float64)))
    a0, a1 = 2.0 * np.pi * u[1].astype(np.float64), 2.0 * np.pi * u[3].astype(np.float64)
    return np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1)], 1)


def covariance(quats, log_scales):
    """Sigma = R(q^) diag(s^2) R(q^)^T in float64, q^ = q / max(|q|, 1e-12), (r, x, y, z)"""
    q = quats.astype(np.float64)
    q = q / np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-12)
    r, x, y, z = q.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                  2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                  2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    s2 = np.exp(2.0 * log_scales.astype(np.float64))
    return np.einsum("pij,pj,pkj->pik", R, s2, R)


def perturb(means, quats, log_scales, x, scale, seed, offset):
    """the expected means after mgs_mcmc_perturb, in float64"""
    P = means.shape[0]
    o = 1.0 / (1.0 + np.exp(-x.reshape(-1).astype(np.float64)))
    g = 1.0 / (1.0 + np.exp(-100.0 * ((1.0 - o) - 0.995)))
    d = np.einsum("pij,pj->pi", covariance(quats, log_scales), normals(seed, offset, P)) * (g * float(scale))[:, None]
    return means.astype(np.float64) + d
