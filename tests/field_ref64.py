"""Float64 torch restatement of the field query (include/mgs_rasterizer.h, mgs_field_query), brute force over every
(point, Gaussian) pair with the same cutoff; gradients by autograd.

    m_i(x) = |S_i^-1 R(q_i / |q_i|) (x - mu_i)|^2,   g_i(x) = o_i exp(-m_i / 2) where that is >= 1/255 (the fp32 constant the
    kernels compare with), else 0;   density = sum_i g_i,   features[c] = sum_i g_i f_i[c].

A Gaussian with o <= 1/255, a scale <= 0 or a non-finite input contributes nothing.  A pair whose float64 m lies within
AMBIGUOUS relative of the cutoff 2 ln(255 o) may fall on either side of it in fp32: `ambiguous_points` flags the points that
have one, and the tests query only the others.

`bounded` restates field.cu pair by pair in closed form (no autograd), following its operation order, and gives every
value a first-order bound B of its fp32 evaluation in units of u = 2^-24 (the convention of project_ref64.E and
heads_ref64): each fp32 operation adds |result| to the operands' propagated bounds.

* Prep (field_prep_kernel, field_bwd_gauss_kernel): rsqrtf of |q|^2 (2 ulp), q^ = q inv, frame_row, A_k = R_k / s_k.
* eval_pair: d = x - mu, u_k = A_k . d, m, expf(-m / 2) (2 ulp), g = o E and the test g >= 1/255.
* Sums in the lane (density, dL/dpoints).  A bin lists its Gaussians in ascending id and a listed Gaussian without support
  at the point adds an exact zero, so the lane's sum is the sequential sum of the point's live pairs in ascending id: a
  term of live rank r among n goes through n - max(r, 1) roundings.  The order is recovered exactly; no longest-chain
  assumption is needed.
* Tensor-core sums (features, GEMM 1, GEMM 2): each product carries SPLIT u |a b| for the truncated 3xTF32 split (each
  operand to 2^-20 relative, the lo*lo term dropped), and each of the three mma_tf32 of a step charges MMA u times its
  operands.  The forward's features follow the lane order above (3 mma per live pair, one more for the first); GEMM 1 runs
  over the channel k-steps; GEMM 2 over the four 8-query k-steps of the item.
* Per-Gaussian sums (dL/dmu, dL/dA_k, dL/do, dL/df): warp_sum16 (5 levels), then one red.global.add per item that lists
  the Gaussian, in any order.  The number of such items is not visible from outside; it is at most the Gaussian's number
  of live pairs N, so every term is charged 5 + N (GEMM 2: 12 MMA + N) roundings.
* Cutoff decisions: a pair whose float64 g is within BAND u B of 1/255 may fall on either side in fp32.  The reference takes
  the float64 decision, carries the pair's whole contribution to every element it feeds (its term in the density, the
  features, dL/dpoints, the per-Gaussian sums and GEMM 2) as a separate absolute bound D that KAPPA does not scale, and
  counts the pair as live in the chain lengths and in B.  An element is then within bound when |x - v| <= KAPPA u B + D.
  Gaussians without support and non-finite points get exactly zero with zero bound.

`mutate` breaks one convention on purpose (MUTATIONS); tests/test_field_ref64_cpu.py shows each moves a checked element past
twice its bound.  The cutoff's `>=` (a kernel `>` differs only where fp32 g rounds to exactly 1/255, which is inside the
either-side band by construction) and the support box's slack (it only guards pairs inside that band) cannot move a value
past the bound; `support_reach` checks the box against the band instead, and its mutation `no_box_slack` is shown to miss.
"""
import numpy as np
import torch

THRESH = float(np.float32(1.0) / np.float32(255.0))  # mgs::ALPHA_MIN
AMBIGUOUS = 1e-5


def rotation_rows(q):
    """R(q^) [P,3,3] with row k the direction scale k stretches (the rasterizer's R, Sigma = R^T S^2 R)"""
    q = q / q.norm(dim=1, keepdim=True)
    r, x, y, z = q.unbind(1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)], 1),
        torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)], 1),
        torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)], 1)], 1)


def valid(means, scales, rotations, opacity):
    o = opacity.reshape(-1)
    fin = torch.isfinite(means).all(1) & torch.isfinite(scales).all(1) & torch.isfinite(rotations).all(1) & torch.isfinite(o)
    return fin & (scales > 0).all(1) & (o > THRESH) & (rotations.norm(dim=1) > 0)


def _mahalanobis(x, means, scales, rotations):
    A = rotation_rows(rotations) / scales[:, :, None]           # [P,3,3]
    d = x[:, None, :] - means[None]                               # [Q,P,3]
    u = torch.einsum("qpj,pkj->qpk", d, A)
    return (u * u).sum(-1)                                        # [Q,P]


def field(points, means, scales, rotations, opacity, features=None, chunk=2048):
    """density [Q] and features [Q,C] (or None), float64, differentiable in every argument"""
    ok = valid(means.detach(), scales.detach(), rotations.detach(), opacity.detach())
    o = opacity.reshape(-1)
    idx = torch.nonzero(ok).reshape(-1)
    mu, s, q, o = means[idx], scales[idx], rotations[idx], o[idx]
    f = features[idx] if features is not None else None
    dens, feats = [], []
    for a in range(0, points.shape[0], chunk):
        x = points[a:a + chunk]
        g = o[None] * torch.exp(-0.5 * _mahalanobis(x, mu, s, q))
        g = torch.where(g >= THRESH, g, torch.zeros_like(g))
        dens.append(g.sum(1))
        if f is not None:
            feats.append(g @ f)
    return torch.cat(dens), (torch.cat(feats) if f is not None else None)


def ambiguous_points(points, means, scales, rotations, opacity, chunk=2048):
    """[Q] bool: the point has a pair with a valid Gaussian whose m is within AMBIGUOUS relative of the cutoff"""
    with torch.no_grad():
        ok = valid(means, scales, rotations, opacity)
        idx = torch.nonzero(ok).reshape(-1)
        o = opacity.reshape(-1)[idx].double()
        cut = -2.0 * torch.log(THRESH / o)
        out = []
        for a in range(0, points.shape[0], chunk):
            m = _mahalanobis(points[a:a + chunk].double(), means[idx].double(), scales[idx].double(), rotations[idx].double())
            out.append(((m - cut[None]).abs() <= AMBIGUOUS * cut[None]).any(1))
        return torch.cat(out) if out else torch.zeros(0, dtype=torch.bool)


def support_box(means, scales, rotations, opacity):
    """[P,3] half-extent of the support m <= 2 ln(255 o) along the world axes: sqrt(2 ln(255 o) Sigma_kk)"""
    R = rotation_rows(rotations)
    sig = ((scales[:, :, None] ** 2) * R ** 2).sum(1)            # Sigma_jj = sum_k s_k^2 R_kj^2
    cut = -2.0 * torch.log(THRESH / opacity.reshape(-1))
    return torch.sqrt(cut[:, None] * sig)


def rel_l2(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    den = b.norm()
    return float((a - b).norm() / den) if den > 0 else float((a - b).norm())


# ------------------------------------------------------------------------------------------------ bounded restatement
U = 2.0 ** -24
BAND = 4.0
EXP_ULP = 2.0        # expf, CUDA's bound
RSQRT_ULP = 2.0      # rsqrtf
SPLIT = 48.0         # 3xTF32 product error in u |a b|
MMA = 2.0            # per mma_tf32 of a chain, in u times |accumulator| + sum |products| (truncating alignment)
WARP_LEVELS = 5      # warp_sum16's additions per term
GEMM2_MMA = 12       # GEMM 2 per item: four 8-query k-steps of three mma_tf32
FQ_CH = 32           # Gaussians per chunk of a bin list
MUTATIONS = ("unnormalised_q", "r_transposed", "exp_m", "dmu_sign", "dq_no_projection", "ds_no_inv_s", "plain_tf32",
             "drop_last_chunk", "no_box_slack")
QUANTITIES = ("density", "features", "points", "means", "scales", "rot", "opacity", "feat")
# an element is within bound when |x - v| <= KAPPA[q] u B: 4x the largest |x - v| / (u B) measured against the kernels over
# every case of tests/test_field_ref64_gpu.py (H100 80GB HBM3; the measured worsts are in its docstring)
KAPPA = dict(density=2.3, features=1.7, points=0.95, means=0.85, scales=0.84, rot=0.53, opacity=0.94, feat=1.06)


class T:
    """a float64 tensor v with its first-order fp32 bound e (units of u) and an absolute bound d inherited from the
    either-side pairs it sums (not scaled by KAPPA)"""
    __slots__ = ("v", "e", "d")

    def __init__(self, v, e=None, d=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e
        self.d = torch.zeros_like(v) if d is None else d

    def __add__(self, o):
        o = _t(o)
        v = self.v + o.v
        return T(v, self.e + o.e + v.abs(), self.d + o.d)

    def __sub__(self, o):
        return self + (-_t(o))

    def __rsub__(self, o):
        return _t(o) + (-self)

    def __neg__(self):
        return T(-self.v, self.e, self.d)

    def __mul__(self, o):
        o = _t(o)
        v = self.v * o.v
        a, b = self.v.abs(), o.v.abs()
        return T(v, a * o.e + b * self.e + v.abs(), a * o.d + b * self.d)

    def __truediv__(self, o):
        o = _t(o)
        v = self.v / o.v
        return T(v, (self.e + v.abs() * o.e) / o.v.abs() + v.abs(), (self.d + v.abs() * o.d) / o.v.abs())

    def scale(self, c):
        """times a power of two: exact"""
        return T(self.v * c, self.e * abs(c), self.d * abs(c))


def _t(x):
    return x if isinstance(x, T) else T(torch.as_tensor(x, dtype=torch.float64))


def _exp(a, ulp=EXP_ULP):
    y = torch.exp(a.v)
    return T(y, y * a.e + ulp * y)


def _rsqrt(a):
    y = torch.rsqrt(a.v)
    return T(y, 0.5 * y / a.v * a.e + RSQRT_ULP * y)


def _dot3(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _frame_rows(q):
    r, x, y, z = q
    two = lambda a: a.scale(2.0)  # noqa: E731
    return [[1.0 - two(y * y + z * z), two(x * y + r * z), two(x * z - r * y)],
            [two(x * y - r * z), 1.0 - two(x * x + z * z), two(y * z + r * x)],
            [two(x * z + r * y), two(y * z - r * x), 1.0 - two(x * x + y * y)]]


def _frame_row_bwd(q, gs):
    """dL/dq^ of sum_k g_k . R_k(q^), accumulated row by row as frame_row_bwd"""
    r, x, y, z = q
    d = [None] * 4

    def acc(c, t):
        d[c] = t if d[c] is None else d[c] + t

    gx, gy, gz = gs[0]
    acc(0, (z * gy - y * gz).scale(2.0))
    acc(1, (y * gy + z * gz).scale(2.0))
    acc(2, (y * gx).scale(-4.0) + (x * gy - r * gz).scale(2.0))
    acc(3, (z * gx).scale(-4.0) + (r * gy + x * gz).scale(2.0))
    gx, gy, gz = gs[1]
    acc(0, (x * gz - z * gx).scale(2.0))
    acc(1, (x * gy).scale(-4.0) + (y * gx + r * gz).scale(2.0))
    acc(2, (x * gx + z * gz).scale(2.0))
    acc(3, (z * gy).scale(-4.0) + (y * gz - r * gx).scale(2.0))
    gx, gy, gz = gs[2]
    acc(0, (y * gx - x * gy).scale(2.0))
    acc(1, (x * gz).scale(-4.0) + (z * gx - r * gy).scale(2.0))
    acc(2, (y * gz).scale(-4.0) + (r * gx + z * gy).scale(2.0))
    acc(3, (x * gx + y * gy).scale(2.0))
    return d


def _tf32(a):
    """round to 10 mantissa bits (plain TF32 operands)"""
    m, e = torch.frexp(a)
    return torch.ldexp(torch.round(m * 2048.0) / 2048.0, e)


def _prep(means, scales, rotations, opacity, mutate):
    """per Gaussian with support (index idx): q^, inv, A_k, mu, o, s as T"""
    ok = valid(means, scales, rotations, opacity)
    idx = torch.nonzero(ok).reshape(-1)
    r = [T(rotations[idx, c].double()) for c in range(4)]
    inv = _rsqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3])
    q = r if "unnormalised_q" in mutate else [rc * inv for rc in r]
    R = _frame_rows(q)
    if "r_transposed" in mutate:
        R = [[R[j][k] for j in range(3)] for k in range(3)]
    s = [T(scales[idx, k].double()) for k in range(3)]
    A = [[R[k][j] / s[k] for j in range(3)] for k in range(3)]
    mu = [means[idx, k].double() for k in range(3)]
    o = opacity.reshape(-1)[idx].double()
    return dict(idx=idx, q=q, inv=inv, A=A, s=s, mu=mu, o=o)


def _kernel_box(means, scales, rotations, opacity, slack=True):
    """[P,3] field_prep_kernel's half-extent sqrt(tau Sigma_kk) (1.0001) + 1e-7 with tau = 2 ln(255 o) (1.001) + 1e-4"""
    R = rotation_rows(rotations.double())
    sig = ((scales.double()[:, :, None] ** 2) * R ** 2).sum(1)
    cut = 2.0 * torch.log(255.0 * opacity.reshape(-1).double())
    if not slack:
        return torch.sqrt(cut[:, None] * sig)
    return torch.sqrt((cut * 1.001 + 1e-4)[:, None] * sig) * 1.0001 + 1e-7


def support_reach(points, means, scales, rotations, opacity, mutate=(), chunk=4096):
    """The pairs fp32 may keep (live, or within the either-side band) whose point lies outside the Gaussian's support box
    as field_prep_kernel widens it: [K,2] (point, Gaussian) indices; empty when the box is sound for these points."""
    with torch.no_grad():
        box = _kernel_box(means, scales, rotations, opacity, slack="no_box_slack" not in mutate)
        out = []
        for a in range(0, points.shape[0], chunk):
            r = _pairs(points[a:a + chunk], _prep(means, scales, rotations, opacity, ()), ())
            keep = r["live"] | r["either"]
            idx = r["idx"]
            x = points[a:a + chunk].double()
            far = ((x[:, None, :] - means[idx].double()[None]).abs() > box[idx][None]).any(-1) & keep
            pq, pg = torch.nonzero(far, as_tuple=True)
            out.append(torch.stack([pq + a, idx[pg]], 1))
        return torch.cat(out) if out else torch.zeros(0, 2, dtype=torch.long)


def _pairs(x, G, mutate):
    """the chunk's pairs [q,P']: d, u, E, g as T and the live / either-side masks"""
    x = x.double()
    fin = torch.isfinite(x).all(1, keepdim=True)
    x = torch.where(fin, x, torch.zeros_like(x))
    d = []
    for j in range(3):
        v = x[:, j:j + 1] - G["mu"][j][None]
        d.append(T(v, v.abs()))
    A = [[T(a.v[None], a.e[None]) for a in row] for row in G["A"]]
    u = [_dot3(A[k], d) for k in range(3)]
    m = u[0] * u[0] + u[1] * u[1] + u[2] * u[2]
    E = _exp(-m) if "exp_m" in mutate else _exp(m.scale(-0.5))
    g = T(G["o"][None]) * E
    live = fin & (g.v >= THRESH)
    either = fin & ((g.v - THRESH).abs() <= BAND * U * g.e)
    return dict(d=d, u=u, E=E, g=g, A=A, live=live, either=either, idx=G["idx"])


def _gate(t, live, either):
    """a per-pair term: its value where the pair is live, its bound where it is live or either-side (a kept either-side
    pair adds its fp32 term), and its whole size where it is either-side"""
    zero = torch.zeros_like(t.v)
    return torch.where(live, t.v, zero), torch.where(live | either, t.e, zero), torch.where(either, t.v.abs(), zero)


def bounded(points, means, scales, rotations, opacity, features=None, grad_density=None, grad_features=None, mutate=(),
            pairs_per_chunk=1 << 22):
    """The field query and, with a cotangent, its gradients, each as (value, bound B in u), float64 on points' device:
    density [Q], features [Q,C], points [Q,3], means [P,3], scales [P,3], rot [P,4], opacity [P], feat [P,C].  The
    cotangents are grad_density [Q] and grad_features [Q,C] (None for zero).  Each entry is (value, B, D): an element x is
    within bound when |x - value| <= KAPPA u B + D, D being the either-side pairs' share.  Also 'live' [Q]: each point's
    live and either-side pairs (its list of Gaussians with support there)."""
    mutate = set(mutate)
    dev = points.device
    Q, P = points.shape[0], means.shape[0]
    C = features.shape[1] if features is not None else 0
    G = _prep(means, scales, rotations, opacity, mutate)
    idx = G["idx"]
    Pv = idx.numel()
    f = features[idx].double() if C else None
    grads = grad_density is not None or (C and grad_features is not None)
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)  # noqa: E731
    out = dict(density=(z(Q), z(Q), z(Q)), live=torch.zeros(Q, dtype=torch.long, device=dev))
    if C:
        out["features"] = (z(Q, C), z(Q, C), z(Q, C))
    if grads:
        out["points"] = (z(Q, 3), z(Q, 3), z(Q, 3))
        acc_v, acc_e, acc_d, acc_a = z(13, Pv), z(13, Pv), z(13, Pv), z(13, Pv)   # dA_k (9), dmu (3), do; sum |term|
        npair = z(Pv)
        if C:
            fv, fe, fd, fa = z(Pv, C), z(Pv, C), z(Pv, C), z(Pv, C)
    step = max(1, pairs_per_chunk // max(Pv, 1))
    for a in range(0, Q if Pv else 0, step):
        b = min(Q, a + step)
        r = _pairs(points[a:b], G, mutate)
        live, either = r["live"], r["either"]
        inlist = live | either
        rank = torch.cumsum(inlist.to(torch.long), 1) - 1
        n = inlist.sum(1, keepdim=True)
        if "drop_last_chunk" in mutate:
            live = live & ~((n > FQ_CH) & (rank >= FQ_CH * ((n - 1) // FQ_CH)))
        depth = torch.where(inlist, n - rank.clamp(min=1), torch.zeros_like(rank)).double()
        out["live"][a:b] = n[:, 0]
        gv, ge, allow = _gate(r["g"], live, either)
        out["density"][0][a:b] = gv.sum(1)
        out["density"][1][a:b] = (ge + gv * depth).sum(1)
        out["density"][2][a:b] = allow.sum(1)
        if C:
            w, fw = (_tf32(gv), _tf32(f)) if "plain_tf32" in mutate else (gv, f)
            out["features"][0][a:b] = w @ fw
            out["features"][1][a:b] = (ge + gv * (SPLIT + 3 * MMA * (depth + 1))) @ f.abs()
            out["features"][2][a:b] = allow @ f.abs()
        if not grads:
            continue
        dD = grad_density[a:b].double() if grad_density is not None else z(b - a)
        dg = T(dD[:, None].expand(-1, Pv))
        if C and grad_features is not None:
            dF = grad_features[a:b].double()
            nks = -(-C // 8) if C <= 32 else 4 * -(-C // 32)
            D1 = dF @ f.t()
            dgv = dD[:, None] + D1
            dg = T(dgv, (SPLIT + 3 * MMA * nks) * (dF.abs() @ f.abs().t()) + dgv.abs())
            fv += gv.t() @ dF
            fe += (ge + SPLIT * gv).t() @ dF.abs()
            fd += allow.t() @ dF.abs()
            fa += gv.t() @ dF.abs()
        t = -(dg * r["g"])
        # pass C: dL/du_k = t u_k, dL/dA_kj = dL/du_k d_j, dL/dx = sum_k dL/du_k A_k, dL/dmu = -dL/dx, dL/do = dg E
        ck = [t * r["u"][k] for k in range(3)]
        vx = [ck[0] * r["A"][0][j] + ck[1] * r["A"][1][j] + ck[2] * r["A"][2][j] for j in range(3)]
        terms = ([ck[k] * r["d"][j] for k in range(3) for j in range(3)] +
                 [vx[j] if "dmu_sign" in mutate else -vx[j] for j in range(3)] + [dg * r["E"]])
        for j in range(3):
            v, bb, dd = _gate(vx[j], live, either)
            out["points"][0][a:b, j] = v.sum(1)
            out["points"][1][a:b, j] = (bb + v.abs() * depth).sum(1)
            out["points"][2][a:b, j] = dd.sum(1)
        for i, tm in enumerate(terms):
            v, bb, dd = _gate(tm, live, either)
            acc_v[i] += v.sum(0)
            acc_e[i] += bb.sum(0)
            acc_d[i] += dd.sum(0)
            acc_a[i] += v.abs().sum(0)
        npair += inlist.sum(0).double()
    if not grads:
        return out
    # per-Gaussian sums: warp_sum16 then the chain of red.global.add over the items (at most npair of them)
    Gs = T(acc_v, acc_e + (WARP_LEVELS + npair)[None] * acc_a, acc_d)
    row = lambda i: T(Gs.v[i], Gs.e[i], Gs.d[i])  # noqa: E731
    dA = [[row(3 * k + j) for j in range(3)] for k in range(3)]
    dmu = [row(9 + j) for j in range(3)]
    do = row(12)
    s, A, q, inv = G["s"], G["A"], G["q"], G["inv"]
    ds = [-_dot3(dA[k], A[k]) if "ds_no_inv_s" in mutate else (-_dot3(dA[k], A[k])) / s[k] for k in range(3)]
    gs = [[dA[k][j] / s[k] for j in range(3)] for k in range(3)]
    dqh = _frame_row_bwd(q, gs)
    if "dq_no_projection" in mutate:
        dq = [dqh[c] * inv for c in range(4)]
    else:
        qd = q[0] * dqh[0] + q[1] * dqh[1] + q[2] * dqh[2] + q[3] * dqh[3]
        dq = [(dqh[c] - q[c] * qd) * inv for c in range(4)]

    def full(cols, width):
        v, e, d = z(P, width), z(P, width), z(P, width)
        v[idx] = torch.stack([c.v for c in cols], 1)
        e[idx] = torch.stack([c.e for c in cols], 1)
        d[idx] = torch.stack([c.d for c in cols], 1)
        return v, e, d

    out["means"] = full(dmu, 3)
    out["scales"] = full(ds, 3)
    out["rot"] = full(dq, 4)
    out["opacity"] = tuple(t[:, 0] for t in full([do], 1))
    if C:
        v, e, d = z(P, C), z(P, C), z(P, C)
        if grad_features is not None:
            v[idx] = fv
            e[idx] = fe + (GEMM2_MMA * MMA + npair)[:, None] * fa
            d[idx] = fd
        out["feat"] = (v, e, d)
    return out


def ratio(got, ref, B, D=0.0, quantity=None):
    """|got - ref| / (KAPPA[quantity] u B + D) elementwise: within bound when <= 1.  Without a quantity it is the measured
    ratio max(|got - ref| - D, 0) / (u B), the rounding part in units of the bound, from which KAPPA is set.  Where the
    bound is 0 the element must be exact (ratio 0, else inf); a non-finite got is inf."""
    got = got.double()
    err = (got - ref).abs()
    if quantity is None:
        err = (err - D).clamp(min=0.0)
        r = err / (U * B)
    else:
        r = err / (KAPPA[quantity] * U * B + D)
    r = torch.where(err == 0, torch.zeros_like(r), r)
    return torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
