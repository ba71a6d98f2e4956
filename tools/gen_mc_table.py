"""Generate the marching-cubes case table (manigaussian_b200/csrc/mc_table.cuh).

    python tools/gen_mc_table.py        # rewrites the header

The table is derived, not copied: for each of the 256 below/above patterns of a cell's corners,
  1. every face gets the segments that separate its below corners from its above corners.  A face with two crossed
     edges has one segment.  An ambiguous face (diagonal corners alike, four crossed edges) always cuts off its two below
     corners.  That rule reads only the face's own four corners, so both cells that share a face split it the same way;
  2. each segment is directed so that (q - p) x m points to the below side, m the face's outward normal.  That is the
     boundary orientation of a surface whose normal points toward increasing value;
  3. the directed segments chain into closed loops, one per surface sheet in the cell, each triangulated from its
     first vertex.  The triangulation uses no diagonal between two edges of an ambiguous face, so that the pair cannot
     be a diagonal in both cells that share the face as well.
tests/test_mesh_cpu.py proves the result: face consistency over every pattern of two neighbouring cells, separation,
orientation and closed reference meshes.
"""
import itertools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "manigaussian_b200", "csrc", "mc_table.cuh")


def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.float64)


def edge_corners(e):
    """the endpoints (a, b) of edge e, a the lower one: edge 4 axis + s runs along axis from the corner whose other two
    bits are s's bits in increasing axis order"""
    axis, s = divmod(e, 4)
    others = [k for k in range(3) if k != axis]
    a = ((s & 1) << others[0]) | (((s >> 1) & 1) << others[1])
    return a, a | (1 << axis)


def edge_of(a, b):
    for e in range(12):
        if set(edge_corners(e)) == {a, b}:
            return e
    raise ValueError((a, b))


def faces():
    """(outward normal, corners in cyclic order) of the six faces"""
    out = []
    for axis in range(3):
        u, v = [k for k in range(3) if k != axis]
        for side in (0, 1):
            base = side << axis
            cyc = [base, base | (1 << u), base | (1 << u) | (1 << v), base | (1 << v)]
            m = np.zeros(3)
            m[axis] = 1.0 if side else -1.0
            out.append((m, cyc))
    return out


FACES = faces()
MID = [0.5 * (corner_pos(a) + corner_pos(b)) for a, b in (edge_corners(e) for e in range(12))]


def face_segments(case, m, cyc):
    """directed segments (p, q) of one face, and whether the face is ambiguous"""
    below = [(case >> c) & 1 for c in cyc]
    edges = [edge_of(cyc[k], cyc[(k + 1) % 4]) for k in range(4)]  # edges[k] joins cyc[k] and cyc[k + 1]
    crossed = [below[k] != below[(k + 1) % 4] for k in range(4)]
    segs = []
    n = sum(crossed)
    if n == 2:
        p, q = [edges[k] for k in range(4) if crossed[k]]
        ref = next(cyc[k] for k in range(4) if below[k])
        segs.append((p, q, ref))
    elif n == 4:
        for k in range(4):
            if below[k]:
                segs.append((edges[(k - 1) % 4], edges[k], cyc[k]))
    out = []
    for p, q, ref in segs:
        side = np.cross(MID[q] - MID[p], m)
        mid = 0.5 * (MID[p] + MID[q])
        out.append((p, q) if np.dot(side, corner_pos(ref) - mid) > 0 else (q, p))
    return out, n == 4, edges


def triangulations(loop):
    """every triangulation of a polygon (vertex lists), the fan from loop[0] first"""
    if len(loop) == 3:
        yield [tuple(loop)]
        return
    a, b = loop[0], loop[-1]
    # the triangle on edge (a, b) has apex loop[k]; recurse on the two sides
    for k in range(1, len(loop) - 1):
        left, right = loop[:k + 1], loop[k:]
        for tl in (triangulations(left) if len(left) >= 3 else [[]]):
            for tr in (triangulations(right) if len(right) >= 3 else [[]]):
                yield tl + tr + [(a, loop[k], b)]


def case_triangles(case):
    nxt = {}
    bad = set()
    for m, cyc in FACES:
        segs, amb, edges = face_segments(case, m, cyc)
        for p, q in segs:
            assert p not in nxt, (case, p)
            nxt[p] = q
        if amb:
            bad |= {frozenset(pq) for pq in itertools.combinations(edges, 2)}
    crossed = [e for e in range(12) if ((case >> edge_corners(e)[0]) & 1) != ((case >> edge_corners(e)[1]) & 1)]
    assert sorted(nxt) == crossed and sorted(nxt.values()) == crossed, case
    tris, seen = [], set()
    for e in crossed:
        if e in seen:
            continue
        loop = [e]
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
        seen |= set(loop)
        boundary = {frozenset((loop[k], loop[(k + 1) % len(loop)])) for k in range(len(loop))}
        for tr in triangulations(loop):
            diags = {frozenset(pq) for t in tr for pq in itertools.combinations(t, 2)} - boundary
            if not (diags & bad):
                break
        else:
            raise RuntimeError(f"case {case}: no triangulation of {loop} avoids the ambiguous faces")
        # keep the loop's orientation: (a, apex, b) with a = loop[0], b = loop[-1] runs against the loop; reorient each
        # triangle to follow the loop's cyclic order
        pos = {v: k for k, v in enumerate(loop)}
        for t in tr:
            t = sorted(t, key=lambda v: pos[v])
            tris.append(tuple(t))
    return tris, crossed


def build():
    rows = [case_triangles(c) for c in range(256)]
    max_t = max(len(t) for t, _ in rows)
    return rows, max_t


def render(rows, max_t):
    lines = [
        "// Marching-cubes case table (include/mgs_rasterizer.h, mgs_marching_cubes_count), generated by tools/gen_mc_table.py:",
        "// do not edit.  tests/mc_ref.py reads it from this file.",
        "//",
        "// Corner c of a cell sits at grid offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along (x, y, z); the case index has bit c",
        "// set when corner c is below the level.  Edge 4 a + s runs along axis a (0 = x, 1 = y, 2 = z) from the corner whose",
        "// other two offsets are s's bits, the lower axis first: edge 0 is (0, 1), 4 is (0, 2), 8 is (0, 4).",
        "// MC_EDGE_MASK[case]: bit e = edge e is crossed.  MC_TRI_COUNT[case] triangles, MC_TRIS[case][3 t + k] the edges of",
        "// triangle t, each normal (v1 - v0) x (v2 - v0) toward increasing value.  An ambiguous face cuts off its below corners.",
        "#pragma once",
        "#include <cstdint>",
        "",
        "namespace mgs {",
        "",
        f"constexpr int MC_MAX_TRIS = {max_t};",
        "",
        "__device__ const uint16_t MC_EDGE_MASK[256] = {",
    ]
    masks = [sum(1 << e for e in crossed) for _, crossed in rows]
    for k in range(0, 256, 16):
        lines.append("\t" + ", ".join(str(m) for m in masks[k:k + 16]) + ",")
    lines += ["};", "", "__device__ const uint8_t MC_TRI_COUNT[256] = {"]
    counts = [len(t) for t, _ in rows]
    for k in range(0, 256, 32):
        lines.append("\t" + ", ".join(str(c) for c in counts[k:k + 32]) + ",")
    lines += ["};", "", "__device__ const int8_t MC_TRIS[256][3 * MC_MAX_TRIS] = {"]
    for c, (tris, _) in enumerate(rows):
        flat = [e for t in tris for e in t] + [-1] * (3 * (max_t - len(tris)))
        lines.append("\t{ " + ", ".join(str(e) for e in flat) + " },  // %d" % c)
    lines += ["};", "", "}  // namespace mgs", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    rows, max_t = build()
    text = render(rows, max_t)
    if "--check" in sys.argv:
        sys.exit(0 if open(OUT).read() == text else 1)
    with open(OUT, "w") as fh:
        fh.write(text)
    print(OUT, "max triangles per case:", max_t)
