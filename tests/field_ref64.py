"""Float64 torch restatement of the field query (include/mgs_rasterizer.h, mgs_field_query), brute force over every
(point, Gaussian) pair with the same cutoff; gradients by autograd.

    m_i(x) = |S_i^-1 R(q_i / |q_i|) (x - mu_i)|^2,   g_i(x) = o_i exp(-m_i / 2) where that is >= 1/255 (the fp32 constant the
    kernels compare with), else 0;   density = sum_i g_i,   features[c] = sum_i g_i f_i[c].

A Gaussian with o <= 1/255, a scale <= 0 or a non-finite input contributes nothing.  A pair whose float64 m lies within
AMBIGUOUS relative of the cutoff 2 ln(255 o) may fall on either side of it in fp32: `ambiguous_points` flags the points that
have one, and the tests query only the others.
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
