"""Vectorised restatement of marching cubes (include/mgs_rasterizer.h, mgs_marching_cubes_count / _emit), in torch so that
the same code runs on the CPU for the tests and on the device for tools/bench_mesh.py.  The case table is read from
manigaussian_b200/csrc/mc_table.cuh, the one place it lives, so that the reference and the kernels cannot drift apart.

* A grid point is valid when its value is finite and, with a weight, its weight is > 0.  A cell (the cube of 8 points with
  lower corner (i, j, k)) with an invalid corner emits nothing; corner c is below when value < level, bit c of the case.
* The edge from point a to a + e_axis gets a vertex when a cell around it uses it (MC_EDGE_MASK of the cell's case).
  Vertices are ordered by (a in x-major order, axis); t = (level - v_a) / (v_b - v_a) and p = c_a + t (c_b - c_a) per
  coordinate, each operation a separate float32 op (no FMA), colours likewise with the same t.
* Faces: the table's triangles of each cell, cells in x-major order.
"""
import os
import re

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = os.path.join(ROOT, "manigaussian_b200", "csrc", "mc_table.cuh")


def _array(text, name):
    body = re.search(name + r"\[[^=]*=\s*\{(.*?)\n\};", text, re.S).group(1)
    body = re.sub(r"//[^\n]*", "", body)
    return [int(x) for x in re.findall(r"-?\d+", body)]


def load_table():
    """(edge_mask [256] int64, tri_count [256] int64, tris [256, MC_MAX_TRIS, 3] int64, -1 padded)"""
    text = open(TABLE).read()
    max_t = int(re.search(r"MC_MAX_TRIS = (\d+);", text).group(1))
    mask = np.array(_array(text, "MC_EDGE_MASK"), np.int64)
    count = np.array(_array(text, "MC_TRI_COUNT"), np.int64)
    tris = np.array(_array(text, "MC_TRIS"), np.int64).reshape(256, max_t, 3)
    assert mask.shape == (256,) and count.shape == (256,)
    return mask, count, tris


MASK, COUNT, TRIS = load_table()


def edge_corners(e):
    """(a, b) corners of edge e (a the lower), as mc_table.cuh numbers them"""
    axis, s = divmod(e, 4)
    others = [k for k in range(3) if k != axis]
    a = ((s & 1) << others[0]) | (((s >> 1) & 1) << others[1])
    return a, a | (1 << axis)


def corner_offset(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def axis_centres(bounds, n):
    """per axis the float32 voxel centres lo + (i + 1/2) ((hi - lo) / n), formed in float64 (voxel_centres)"""
    b = [float(v) for v in bounds]
    return [(torch.tensor(b[k], dtype=torch.float64) + (torch.arange(n[k], dtype=torch.float64) + 0.5) * ((b[k + 3] - b[k]) / n[k])
             ).to(torch.float32) for k in range(3)]


def marching_cubes(values, level, bounds, weight=None, color=None):
    """{"vertices": [Nv,3] float32, "faces": [Nf,3] int64, "colors": [Nv,C] float32 or None} of values [X,Y,Z] (torch,
    any device), as the kernels define them"""
    dev = values.device
    X, Y, Z = values.shape
    C = None if color is None else color.shape[0]
    empty = {"vertices": torch.zeros(0, 3, device=dev), "faces": torch.zeros(0, 3, dtype=torch.int64, device=dev),
             "colors": None if color is None else torch.zeros(0, C, device=dev)}
    if min(X, Y, Z) < 2:
        return empty
    lvl = float(np.float32(level))
    valid = torch.isfinite(values)
    if weight is not None:
        valid &= weight > 0
    below = values < lvl
    mask_t, count_t, tris_t = (torch.as_tensor(a, device=dev) for a in (MASK, COUNT, TRIS))
    # cases of the cells, indexed by their lower corner over [X-1, Y-1, Z-1]
    case = torch.zeros((X - 1, Y - 1, Z - 1), dtype=torch.int64, device=dev)
    ok = torch.ones((X - 1, Y - 1, Z - 1), dtype=torch.bool, device=dev)
    for c in range(8):
        dx, dy, dz = corner_offset(c)
        sl = (slice(dx, X - 1 + dx), slice(dy, Y - 1 + dy), slice(dz, Z - 1 + dz))
        case |= below[sl].to(torch.int64) << c
        ok &= valid[sl]
    case = torch.where(ok, case, torch.zeros_like(case))
    cmask = mask_t[case]
    # edge-used bits per point and axis: OR over the <= 4 cells around the edge
    used = torch.zeros((X, Y, Z, 3), dtype=torch.bool, device=dev)
    for e in range(12):
        a, _ = edge_corners(e)
        axis = e // 4
        ox, oy, oz = corner_offset(a)
        bit = ((cmask >> e) & 1).bool()
        used[ox:X - 1 + ox, oy:Y - 1 + oy, oz:Z - 1 + oz, axis] |= bit
    flat_used = used.reshape(-1)
    vid = torch.cumsum(flat_used.to(torch.int64), 0) - 1  # id of each (point, axis) slot that is used
    slots = torch.nonzero(flat_used).squeeze(1)
    pt, axis = slots // 3, slots % 3
    i, j, k = pt // (Y * Z), (pt // Z) % Y, pt % Z
    ib, jb, kb = i + (axis == 0).long(), j + (axis == 1).long(), k + (axis == 2).long()
    vals = values.reshape(-1)
    va, vb = vals[pt], vals[(ib * Y + jb) * Z + kb]
    lv = torch.full_like(va, lvl)
    t = (lv - va) / (vb - va)
    cx, cy, cz = (c.to(dev) for c in axis_centres(bounds, (X, Y, Z)))
    ca = torch.stack([cx[i], cy[j], cz[k]], -1)
    cb = torch.stack([cx[ib], cy[jb], cz[kb]], -1)
    verts = ca + t[:, None] * (cb - ca)
    colors = None
    if color is not None:
        col = color.reshape(C, -1)
        qa, qb = col[:, pt].T, col[:, (ib * Y + jb) * Z + kb].T
        colors = qa + t[:, None] * (qb - qa)
    # faces: cells in x-major order, the table's triangles of each
    cell_idx = torch.nonzero(count_t[case].reshape(-1) > 0).squeeze(1)
    cc = case.reshape(-1)[cell_idx]
    n = count_t[cc]
    rep_cell = torch.repeat_interleave(cell_idx, n)
    rep_case = torch.repeat_interleave(cc, n)
    start = torch.cumsum(n, 0) - n
    tri_no = torch.arange(int(n.sum()), device=dev) - torch.repeat_interleave(start, n)
    edges = tris_t[rep_case, tri_no]  # [Nf,3]
    ci, cj, ck = rep_cell // ((Y - 1) * (Z - 1)), (rep_cell // (Z - 1)) % (Y - 1), rep_cell % (Z - 1)
    lower = torch.tensor([edge_corners(e)[0] for e in range(12)], device=dev)[edges]
    ex, ey, ez = lower & 1, (lower >> 1) & 1, (lower >> 2) & 1
    owner = ((ci[:, None] + ex) * Y + cj[:, None] + ey) * Z + ck[:, None] + ez
    faces = vid[owner * 3 + edges // 4]
    return {"vertices": verts, "faces": faces, "colors": colors}
