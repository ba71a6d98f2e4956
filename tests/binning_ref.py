"""The binning state as it should be, in numpy: which tile instances a view keeps when its binning state holds `capacity`
slots, and in which order (binning.cu emit_tiles_kernel, the stable tile sort, ranges_pack_kernel).

Input: the projection's records read back from the geometry state (radii, means2D, depths; a culled Gaussian has radius
0 and depth +inf), the image size and the capacity.  The statement:

* emission order is the depth order: ascending depth bits, ties by ascending Gaussian id, culled Gaussians last;
* within one Gaussian its instances follow its tile rectangle row-major (y outer, x inner); the rectangle is
  mgs_common.cuh's tile_rect, restated in float32;
* an instance is kept iff its emission position is below the capacity (a Gaussian can keep part of its rectangle);
* the kept instances take a stable sort by tile id;
* status = {R, R > capacity}; point_list and tile_ids hold the first min(R, capacity) slots; ranges [T, 2] holds each
  tile's [begin, end) in them, {0, 0} for a tile without instances.

`mutate` (a set of names, MUTATIONS) breaks one of these on purpose: tests/test_binning_ref_cpu.py shows each changes the
result on at least one case, so a kernel doing the same would fail its comparison on the GPU.
"""
import numpy as np

TILE = 16
# id_order: emit (and cut) in Gaussian-id order instead of depth order; whole: keep only Gaussians whose whole rectangle
# fits below the capacity; col_major: emit a rectangle column-major; ties_desc: equal depths in descending id order;
# no_clamp: the last tile's range ends at R instead of min(R, capacity)
MUTATIONS = ("id_order", "whole", "col_major", "ties_desc", "no_clamp")


def _f32_int(v):
    """(int) of a float32 as the device converts it: toward zero, saturating at the int range."""
    v = np.asarray(v, np.float64)
    return np.trunc(np.clip(v, -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)


def tile_rect(means2D, radii, gx, gy):
    """(x0, y0, x1, y1) of every Gaussian's tile rectangle [x0, x1) x [y0, y1), as mgs_common.cuh tile_rect computes it
    in float32: (px - r) / 16 and (px + r + 16 - 1) / 16, each operation rounded, truncated to int, clamped to [0, g]."""
    m = np.asarray(means2D, np.float32).reshape(-1, 2)
    r = np.asarray(radii).astype(np.float32)
    t, one = np.float32(TILE), np.float32(1)
    out = []
    for c, g in ((0, gx), (1, gy)):
        p = m[:, c]
        lo = _f32_int((p - r) / t)
        hi = _f32_int((((p + r) + t) - one) / t)
        out.append((np.minimum(g, np.maximum(0, lo)), np.minimum(g, np.maximum(0, hi))))
    (x0, x1), (y0, y1) = out
    return x0, y0, x1, y1


def emission(radii, means2D, depths, W, H, mutate=()):
    """Every instance in emission order: (tile id [R], Gaussian id [R]), and each Gaussian's emission offset and count
    (offset [P], count [P]; offset is where its first instance lands)."""
    radii = np.asarray(radii).astype(np.int64)
    P = radii.shape[0]
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    x0, y0, x1, y1 = tile_rect(means2D, radii, gx, gy)
    live = radii > 0
    w = np.where(live, np.maximum(x1 - x0, 0), 0)
    h = np.where(live, np.maximum(y1 - y0, 0), 0)
    count = w * h
    bits = np.asarray(depths, np.float32).view(np.uint32).astype(np.int64)
    ids = np.arange(P)
    if "id_order" in mutate:
        order = ids
    else:
        tie = -ids if "ties_desc" in mutate else ids
        order = np.lexsort((tie, bits, ~live))  # the last key is the primary one
    c = count[order]
    start = np.cumsum(c) - c
    offset = np.zeros(P, np.int64)
    offset[order] = start
    R = int(c.sum())
    gid = np.repeat(order, c)
    k = np.arange(R) - np.repeat(start, c)
    if "col_major" in mutate:
        hh = np.repeat(h[order], c)
        lx, ly = k // np.maximum(hh, 1), k % np.maximum(hh, 1)
    else:
        ww = np.repeat(w[order], c)
        lx, ly = k % np.maximum(ww, 1), k // np.maximum(ww, 1)
    tile = (np.repeat(y0[order], c) + ly) * gx + np.repeat(x0[order], c) + lx
    return tile.astype(np.int64), gid.astype(np.int64), offset, count


def reference(radii, means2D, depths, W, H, capacity, mutate=()):
    """The binning state of one view with `capacity` slots: dict(status, point_list, tile_ids, ranges), plus R and the
    emission (offset, count) per Gaussian for building capacities."""
    tile, gid, offset, count = emission(radii, means2D, depths, W, H, mutate)
    R = tile.shape[0]
    cap = int(capacity)
    n = min(R, cap)
    keep = np.arange(R) < n
    if "whole" in mutate:
        keep = (offset[gid] + count[gid]) <= cap
    tk, gk = tile[keep], gid[keep]
    s = np.argsort(tk, kind="stable")
    tile_ids, point_list = tk[s], gk[s]
    T = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    ranges = np.zeros((T, 2), np.int64)
    if tile_ids.size:
        present = np.unique(tile_ids)
        ranges[present, 0] = np.searchsorted(tile_ids, present, "left")
        ranges[present, 1] = np.searchsorted(tile_ids, present, "right")
        if "no_clamp" in mutate:
            ranges[tile_ids[-1], 1] = R
    return dict(status=np.array([R, int(R > cap)], np.int64), point_list=point_list.astype(np.uint32),
                tile_ids=tile_ids.astype(np.uint32), ranges=ranges.astype(np.uint32), R=R, offset=offset, count=count)


def compare(got, want):
    """The fields of `got` (status, point_list, tile_ids, ranges; numpy) that differ from `want`, with the first difference."""
    bad = []
    for k in ("status", "point_list", "tile_ids", "ranges"):
        a, b = np.asarray(got[k]).astype(np.int64), np.asarray(want[k]).astype(np.int64)
        if a.shape != b.shape:
            bad.append(f"{k}: shape {a.shape} != {b.shape}")
        elif not np.array_equal(a, b):
            i = np.argwhere(a != b)[0]
            bad.append(f"{k}: {int((a != b).sum())} entries differ, first at {tuple(int(x) for x in i)}: "
                       f"{a[tuple(i)]} != {b[tuple(i)]}")
    return bad
