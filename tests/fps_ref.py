"""Farthest-point sampling in float32 numpy (include/mgs_rasterizer.h, mgs_fps): the definition restated op for op, so that
its picks and distances are bitwise those of the kernel.  numpy rounds every float32 operation and never contracts
((dx*dx) + (dy*dy)) + (dz*dz) into an FMA, as the kernel's __fsub_rn / __fmul_rn / __fadd_rn do not."""
import numpy as np


def d2_f32(p, s):
    """the definition's D from every row of p [N,3] float32 to s [3] float32"""
    dx, dy, dz = (p[:, k] - s[k] for k in range(3))
    return (dx * dx + dy * dy) + dz * dz


def fps_ref_cloud(points, n, start=None):
    """one cloud points [L,3] (already cut to its length): (index [n] int64, dist2 [n] float32)"""
    p = np.ascontiguousarray(points, np.float32)
    finite = np.isfinite(p).all(1)
    d = np.where(finite, np.float32(np.inf), np.float32(-1.0)).astype(np.float32)  # -1: picked or not available
    index = np.full(n, -1, np.int64)
    dist2 = np.full(n, np.inf, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(n):
            if t == 0 and start is not None and 0 <= start < len(p) and finite[start]:
                s = int(start)
            else:
                s = int(np.argmax(d)) if len(d) else 0  # the first of equal maxima: the lower index
                if len(d) == 0 or d[s] < 0:
                    break
            index[t], dist2[t] = s, d[s]
            d[s] = -1.0
            d = np.where(d >= 0, np.minimum(d, d2_f32(p, p[s])), d)
    return index, dist2


def fps_ref(points, n, lengths=None, start=None):
    """points [B,P,3] with lengths [B] (clamped to 0 .. P) and start [B], each None to omit: (index [B,n], dist2 [B,n])"""
    points = np.asarray(points, np.float32)
    B, P = points.shape[:2]
    index = np.full((B, n), -1, np.int64)
    dist2 = np.full((B, n), np.inf, np.float32)
    for b in range(B):
        L = P if lengths is None else int(min(max(int(lengths[b]), 0), P))
        index[b], dist2[b] = fps_ref_cloud(points[b, :L], n, None if start is None else int(start[b]))
    return index, dist2


def fps_loop(points, n, start=None):
    """the definition as a literal per-point Python loop over one cloud, in Python floats rounded to float32 after every
    operation (the check of fps_ref_cloud)"""
    f = np.float32
    p = [tuple(f(c) for c in row) for row in np.asarray(points, np.float32)]
    ok = [all(np.isfinite(c) for c in row) for row in p]
    d = [f(np.inf) if o else None for o in ok]
    index, dist2 = [], []
    for t in range(n):
        if t == 0 and start is not None and 0 <= start < len(p) and ok[start]:
            s = start
        else:
            s = None
            for i in range(len(p)):
                if d[i] is not None and (s is None or d[i] > d[s]):
                    s = i
            if s is None:
                break
        index.append(s)
        dist2.append(d[s])
        d[s] = None
        for i in range(len(p)):
            if d[i] is None:
                continue
            dx, dy, dz = (f(p[i][k] - p[s][k]) for k in range(3))
            D = f(f(f(dx * dx) + f(dy * dy)) + f(dz * dz))
            d[i] = min(d[i], D)
    index += [-1] * (n - len(index))
    dist2 += [f(np.inf)] * (n - len(dist2))
    return np.array(index, np.int64), np.array(dist2, np.float32)
