"""A numpy restatement of default density control (include/mgs_rasterizer.h, mgs_densify_stats / mgs_densify_count /
mgs_densify_emit).

The statistics are restated in float32, one correctly rounded operation at a time, so the device must match them bit for
bit.  The refinement's decisions, order, copied rows, moments and children's log scales are restated exactly; the
children's means in float64 from the same float32 uniforms.  The generator (Philox4x32-10) and the Box-Muller normals are
mcmc_ref64's: the children draw at tags 2 and 3 where MCMC's perturbation draws at tag 1.
"""
import math

import numpy as np

import mcmc_ref64 as M

TAG_CHILD = 2
LOG_1_6 = math.log(1.6)
F32 = np.float32


def stats(grad2d, count, radius, viewspace_grad, radii, sizes, scale=1.0):
    """the statistics after one mgs_densify_stats call: (grad2d, count, radius), the inputs left unchanged.
    viewspace_grad [V,P,3] or [P,3] float32, radii [V,P] or [P] int32, sizes V ints."""
    P = grad2d.shape[0]
    vg = np.asarray(viewspace_grad, F32).reshape(-1, P, 3)
    rd = np.asarray(radii, np.int32).reshape(-1, P)
    g, c, r = grad2d.astype(F32).copy(), count.astype(np.int32).copy(), radius.astype(F32).copy()
    sc = F32(scale)
    with np.errstate(over="ignore", invalid="ignore"):
        for v in range(vg.shape[0]):
            m = rd[v] > 0
            gx, gy = vg[v, :, 0], vg[v, :, 1]
            n = np.sqrt(gx * gx + gy * gy)
            g = np.where(m, g + n * sc, g)
            c = np.where(m, c + 1, c).astype(np.int32)
            r = np.where(m, np.maximum(r, rd[v].astype(F32) / F32(sizes[v])), r)
    return g, c, r


def thresholds(scene_scale, grow_scale3d=0.01, prune_scale3d=0.1, prune_opacity=0.005):
    """(t_small, t_big, t_opa): fp32 of the fp64 log / logit of the definition"""
    return (F32(math.log(grow_scale3d * scene_scale)), F32(math.log(prune_scale3d * scene_scale)),
            F32(math.log(prune_opacity / (1.0 - prune_opacity))))


def largest(ls):
    """the largest log scale per row, a NaN operand ignored (fmaxf)"""
    return np.fmax(np.fmax(ls[:, 0], ls[:, 1]), ls[:, 2])


def child_scales(ls):
    return (ls.astype(np.float64) - LOG_1_6).astype(F32)


def classify(log_scales, opacity, grad2d, count, radius, scene_scale, grad_threshold=2e-4, grow_scale3d=0.01,
             grow_scale2d=None, prune_opacity=0.005, prune_scale3d=0.1, prune_scale2d=None, prune_too_big=False):
    """per-Gaussian bool arrays {keep, clone_kept, child_kept, clone, split} of the definition"""
    t_small, t_big, t_opa = thresholds(scene_scale, grow_scale3d, prune_scale3d, prune_opacity)
    ls = np.asarray(log_scales, F32)
    x = np.asarray(opacity, F32).reshape(-1)
    r = np.asarray(radius, F32)
    with np.errstate(invalid="ignore", divide="ignore"):
        L, Lc = largest(ls), largest(child_scales(ls))
        high = grad2d.astype(F32) / np.maximum(count, 1).astype(F32) > F32(grad_threshold)
        small = L <= t_small
        clone = high & small
        split = (high & ~small) | (r > F32(grow_scale2d) if grow_scale2d is not None else False)

        def pruned(L_):
            big = (L_ > t_big) | (r > F32(prune_scale2d) if prune_scale2d is not None else False)
            return (x < t_opa) | (big if prune_too_big else False)

        gone = pruned(L)
        return {"keep": ~split & ~gone, "clone_kept": clone & ~gone, "child_kept": split & ~pruned(Lc),
                "clone": clone, "split": split}


def child_normals(seed, offset, P, b):
    """z [P,3] float64 of child b of every Gaussian: mcmc_ref64.normals' Box-Muller on the words of counter
    {i, offset, tag 2 + b} (mcmc_ref64.normals draws at its module's TAG_PERTURB, set here for the call)"""
    saved = M.TAG_PERTURB
    M.TAG_PERTURB = TAG_CHILD + b
    try:
        return M.normals(seed, offset, P)
    finally:
        M.TAG_PERTURB = saved


def rotation(quats):
    """R(q^) [N,3,3] in float64, q^ = q / max(|q|, 1e-12), (r, x, y, z)"""
    q = quats.astype(np.float64)
    q = q / np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-12)
    r, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def refine(params, moments, grad2d, count, radius, seed, offset, normals=None, **rule):
    """the expected result of mgs_densify_count + mgs_densify_emit.  params: a dict of float32 arrays [P, ...] with keys
    pts_xyz, rotations, scales (log), opacity (logits) and any further rows; moments: {name: [arrays shaped like
    params[name]]}.  normals(b) -> z [P,3] replaces the Philox normals of child b (None: child_normals).  Returns (new
    params, new moments, source, counts (n_new, cloned, split, pruned), {"mean64": the children's means [2 S,3] in float64,
    "children": the slice of the children's rows}); the children's means in new params are mean64 rounded to float32."""
    P = params["pts_xyz"].shape[0]
    f = classify(params["scales"], params["opacity"], grad2d, count, radius, **rule)
    ik, ic, ich = (np.nonzero(f[k])[0] for k in ("keep", "clone_kept", "child_kept"))
    source = np.concatenate([ik, ic, ich, ich]).astype(np.int64)
    out = {k: v[source].copy() for k, v in params.items()}
    children = slice(len(ik) + len(ic), len(source))
    out["scales"][children] = np.tile(child_scales(params["scales"][ich]), (2, 1))
    R = rotation(params["rotations"][ich])
    s = np.exp(params["scales"][ich].astype(np.float64))
    mu = params["pts_xyz"][ich].astype(np.float64)
    mean64 = []
    for b in range(2):
        z = (normals(b) if normals is not None else child_normals(seed, offset, P, b))[ich]
        mean64.append(mu + np.einsum("nij,nj->ni", R, s * z))
    mean64 = np.concatenate(mean64) if len(ich) else np.zeros((0, 3))
    out["pts_xyz"][children] = mean64.astype(F32)
    n_new = len(source)
    new_moments = {}
    for k, vs in moments.items():
        new_moments[k] = []
        for v in vs:
            m = np.zeros((n_new,) + v.shape[1:], F32)
            m[:len(ik)] = v[ik]
            new_moments[k].append(m)
    cloned, split = int(f["clone"].sum()), int(f["split"].sum())
    counts = (n_new, cloned, split, P + cloned + split - n_new)
    return out, new_moments, source, counts, {"mean64": mean64, "children": children}
