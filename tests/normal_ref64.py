"""Float64 restatement of the per-Gaussian surface normal (include/mgs_rasterizer.h, mgs_view_normal) and of its quaternion
gradient, in numpy.  Quaternions are (r, x, y, z).

    k   = argmin_j scales[j]            (lowest index on ties)
    q^  = q / |q|
    a   = R(q^) e_k                     (world space; Sigma a = s_k^2 a)
    s   = +1 if a . (campos - mean) >= 0 else -1
    n   = s a
    dL/dq = (I - q^ q^T) / |q| . J_k(q^)^T . sum_v s_v dL/dn_v
"""
import numpy as np


def shortest_axis(scales):
    return np.argmin(np.asarray(scales, np.float64), axis=1)  # numpy's argmin returns the first minimum


def rotation_matrix(q):
    """R(q) [P,3,3] for unit quaternions q [P,4]"""
    r, x, y, z = (q[:, i] for i in range(4))
    R = np.empty((q.shape[0], 3, 3))
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - r * z); R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y); R[:, 2, 1] = 2 * (y * z + r * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def axis(scales, rotations, argmax=False, row=False, normalize=True):
    """(a [P,3], k [P], q^ [P,4], |q| [P]).  argmax / row / normalize=False are the broken conventions the tests rule out."""
    q = np.asarray(rotations, np.float64)
    n = np.linalg.norm(q, axis=1)
    qh = q / n[:, None] if normalize else q
    k = np.argmax(np.asarray(scales, np.float64), axis=1) if argmax else shortest_axis(scales)
    R = rotation_matrix(qh)
    i = np.arange(q.shape[0])
    a = R[i, k, :] if row else R[i, :, k]
    return a, k, qh, n


def facing(a, means3D, campos):
    d = np.einsum("pi,pi->p", a, np.asarray(campos, np.float64)[None, :] - np.asarray(means3D, np.float64))
    return np.where(d >= 0, 1.0, -1.0), d


def normals(means3D, scales, rotations, campos, flip=True, **kw):
    """n [P,3] of one view, and the facing dot product [P] (sign decisions within rounding of 0 are not determined)"""
    a, _, _, _ = axis(scales, rotations, **kw)
    s, d = facing(a, means3D, campos)
    return (a * s[:, None] if flip else a), d


def axis_jacobian(qh, k):
    """J [P,3,4]: d (R(q^) e_k) / d q^"""
    r, x, y, z = (qh[:, i] for i in range(4))
    o = np.zeros_like(r)
    J0 = np.stack([np.stack([o, o, -4 * y, -4 * z], 1), np.stack([2 * z, 2 * y, 2 * x, 2 * r], 1),
                   np.stack([-2 * y, 2 * z, -2 * r, 2 * x], 1)], 1)
    J1 = np.stack([np.stack([-2 * z, 2 * y, 2 * x, -2 * r], 1), np.stack([o, -4 * x, o, -4 * z], 1),
                   np.stack([2 * x, 2 * r, 2 * z, 2 * y], 1)], 1)
    J2 = np.stack([np.stack([2 * y, 2 * z, 2 * r, 2 * x], 1), np.stack([-2 * x, -2 * r, 2 * z, 2 * y], 1),
                   np.stack([o, -4 * x, -4 * y, o], 1)], 1)
    return np.where((k == 0)[:, None, None], J0, np.where((k == 1)[:, None, None], J1, J2))


def rotation_grad(means3D, scales, rotations, campos_per_view, dL_dn_per_view, normalization_jacobian=True):
    """dL/dq [P,4] from the views' dL/dn [V][P,3] and camera centres [V][3]"""
    a, k, qh, n = axis(scales, rotations)
    g = np.zeros_like(a)
    for cp, dn in zip(campos_per_view, dL_dn_per_view):
        s, _ = facing(a, means3D, cp)
        g += s[:, None] * np.asarray(dn, np.float64)
    d = np.einsum("pij,pi->pj", axis_jacobian(qh, k), g)  # dL/dq^
    if not normalization_jacobian:
        return d
    return (d - qh * np.einsum("pi,pi->p", qh, d)[:, None]) / n[:, None]
