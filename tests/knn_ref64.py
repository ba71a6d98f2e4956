"""float64 restatement of the k-nearest-neighbour definition (include/mgs_rasterizer.h, mgs_knn), by brute force: for each
query the k nearest reference points by squared distance, ascending by (d2, index); queries None: the points themselves,
each without its own index; a point with a non-finite coordinate is never a neighbour, a non-finite query gets only
padding; missing slots are index -1, d2 = +inf."""
import numpy as np


def knn_ref64(points, k, queries=None, extra=1, chunk=256):
    """(index [Q,k+extra] int64, d2 [Q,k+extra] float64): the k nearest and `extra` more, so that a caller can see the
    margin between the k-th and the (k+1)-th distance"""
    P = np.asarray(points, np.float64).reshape(-1, 3)
    self_mode = queries is None
    Qp = P if self_mode else np.asarray(queries, np.float64).reshape(-1, 3)
    ok_p = np.isfinite(P).all(1)
    ok_q = np.isfinite(Qp).all(1)
    m = k + extra
    index = np.full((len(Qp), m), -1, np.int64)
    dist = np.full((len(Qp), m), np.inf)
    Pf = np.where(ok_p[:, None], P, 0.0)
    ids = np.arange(len(P))
    for q0 in range(0, len(Qp), chunk):
        q = np.where(ok_q[q0:q0 + chunk, None], Qp[q0:q0 + chunk], 0.0)
        d2 = ((q[:, None, :] - Pf[None, :, :]) ** 2).sum(-1)
        bad = np.broadcast_to(~ok_p[None, :], d2.shape).copy()
        bad |= ~ok_q[q0:q0 + chunk, None]
        if self_mode:
            r = np.arange(q0, q0 + len(q))
            bad[r - q0, r] = True
        d2 = np.where(bad, np.inf, d2)
        order = np.lexsort((np.broadcast_to(ids, d2.shape), d2), axis=1)[:, :m]  # by d2, then index
        dd = np.take_along_axis(d2, order, 1)
        valid = np.isfinite(dd)
        index[q0:q0 + len(q), :order.shape[1]] = np.where(valid, order, -1)
        dist[q0:q0 + len(q), :order.shape[1]] = np.where(valid, dd, np.inf)
    return index, dist


def decided(dist, k, rel=1e-5):
    """rows whose k-th and (k+1)-th distances are more than `rel` relative apart (or whose k-th or (k+1)-th slot is padding)"""
    a, b = dist[:, k - 1], dist[:, k]
    with np.errstate(invalid="ignore"):
        return ~np.isfinite(a) | ~np.isfinite(b) | (b - a > rel * np.maximum(np.abs(b), 1e-30))


def dist_cuda2_ref64(points):
    """simple-knn's distCUDA2 value, exactly: the mean of each point's three nearest squared distances"""
    _, d = knn_ref64(points, 3, extra=0)
    return d.mean(1)


def start_level(points, k, bits=21):
    """The search's start level, restated with the kernel's fp32 grid (a cubic grid of 2^bits fine cells along the longest
    axis of the finite points' box; level L groups 2^L fine cells a side) and the occupied cells counted with np.unique:
    the first level whose mean occupancy reaches max(k, 8), or the level below it when that one's mean is nearer to the
    target as a ratio.  Returns (level, mean occupancy of each level)."""
    p = np.asarray(points, np.float32).reshape(-1, 3)
    p = p[np.isfinite(p).all(1)]
    lo, hi = p.min(0), p.max(0)
    emax = np.float32((hi - lo).max())
    inv = np.float32(2 ** bits) / emax if emax > 0 else np.float32(0)
    top = 2 ** bits - 1

    def cell(x, gmax):
        return np.clip(np.floor((x - lo) * inv), 0, gmax).astype(np.int64)

    gmax = cell(hi[None, :], top)[0]
    c = cell(p, gmax)
    n = len(p)
    mean = np.array([n / len(np.unique(c >> L, axis=0)) for L in range(bits + 1)])
    target = max(k, 8)
    L0 = next((L for L in range(bits + 1) if mean[L] >= target), bits)
    if L0 > 0 and target / mean[L0 - 1] < mean[L0] / target:
        L0 -= 1
    return L0, mean
