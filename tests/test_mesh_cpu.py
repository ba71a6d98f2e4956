"""Meshes and TSDF volumes without a GPU: the marching-cubes table (manigaussian_b200/csrc/mc_table.cuh) and its reference
(tests/mc_ref.py), the float64 fusion reference (tests/tsdf_ref64.py), the C ABI and the Python surface.

* Table consistency, exhaustively: for two cells sharing a face along each axis and all 2^12 below/above patterns of their
  12 grid points, the triangle edges each cell leaves on the shared face are the same segments, run in opposite
  directions.  Every case's triangles use exactly its crossed edges and separate its below corners from its above corners.
* Reference meshes: an analytic sphere SDF gives a closed 2-manifold (by vertex ids) with Euler characteristic 2 and
  positive signed volume, its vertices within the linear-interpolation bound of the sphere; a torus gives 0; random
  smooth fields with many ambiguous faces give closed meshes where the level set stays inside the grid.
* Reference fusion of one pinhole view of a fronto-parallel plane equals the closed form.
* The C ABI's declarations, exports, state size and argument errors, calls that enqueue nothing, and every refusal of
  gaussian_renderer.tsdf_fuse and marching_cubes.
"""
import ctypes
import itertools
import math
import os
import re

import numpy as np
import pytest
import torch

import mc_ref as M
import tsdf_ref64 as T64
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR

FACE_AXES = (0, 1, 2)


def _tri_edges(case, lower):
    """the directed triangle edges of one cell's case as ((point, axis), (point, axis)) pairs, lower its lower corner"""
    out = []
    for t in range(M.COUNT[case]):
        ids = []
        for e in M.TRIS[case, t]:
            a, _ = M.edge_corners(int(e))
            off = M.corner_offset(a)
            ids.append((tuple(lower[q] + off[q] for q in range(3)), int(e) // 4))
        out += [(ids[0], ids[1]), (ids[1], ids[2]), (ids[2], ids[0])]
    return out


def _on_plane(edge, axis, coord):
    (p, ax) = edge
    return ax != axis and p[axis] == coord


@pytest.mark.parametrize("axis", FACE_AXES)
def test_shared_faces_are_split_the_same_way_from_both_cells(axis):
    pts = [p for p in itertools.product(*[range(3 if q == axis else 2) for q in range(3)])]
    lower_b = tuple(1 if q == axis else 0 for q in range(3))
    for bits in range(1 << 12):
        below = {p: (bits >> k) & 1 for k, p in enumerate(pts)}

        def case_of(lower):
            return sum(below[tuple(lower[q] + M.corner_offset(c)[q] for q in range(3))] << c for c in range(8))

        seg = []
        for lower in ((0, 0, 0), lower_b):
            e = [(a, b) for a, b in _tri_edges(case_of(lower), lower) if _on_plane(a, axis, 1) and _on_plane(b, axis, 1)]
            seg.append(e)
        a, b = seg
        assert sorted(a) == sorted((q, p) for p, q in b), (axis, bits)
        assert len(set(a)) == len(a)


def _face_of(e):
    """the faces (axis, side) that local edge e lies on"""
    a, _ = M.edge_corners(e)
    off = M.corner_offset(a)
    return {(q, off[q]) for q in range(3) if q != e // 4}


@pytest.mark.parametrize("case", range(256))
def test_every_case_separates_its_below_corners_from_its_above_corners(case):
    crossed = {e for e in range(12) if ((case >> M.edge_corners(e)[0]) & 1) != ((case >> M.edge_corners(e)[1]) & 1)}
    assert M.MASK[case] == sum(1 << e for e in crossed)
    tris = [tuple(int(e) for e in M.TRIS[case, t]) for t in range(M.COUNT[case])]
    assert {e for t in tris for e in t} == crossed
    assert all((M.TRIS[case, M.COUNT[case]:] == -1).ravel())
    # every edge of the triangle set is used twice (inside the cell, in opposite directions) or once (its boundary)
    count = {}
    for t in tris:
        for p, q in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            count[(p, q)] = count.get((p, q), 0) + 1
    boundary = []
    for (p, q), n in count.items():
        assert n == 1, (case, p, q)
        if (q, p) not in count:
            boundary.append((p, q))
    # the boundary lies on the faces and pairs up each face's crossed edges: a path along the cube's edges between two
    # corners then crosses the surface an odd number of times exactly when their signs differ
    for axis, side in itertools.product(range(3), (0, 1)):
        on = [(p, q) for p, q in boundary if (axis, side) in _face_of(p) & _face_of(q)]
        face_crossed = {e for e in crossed if (axis, side) in _face_of(e)}
        assert sorted(x for s in on for x in s) == sorted(face_crossed), (case, axis, side)
    assert len(boundary) == sum(len({e for e in crossed if f in _face_of(e)}) for f in itertools.product(range(3), (0, 1))) // 2


def test_one_below_corner_faces_away_from_it():
    # case 1: corner 0 below, the vertices on its three edges at t = 1/2; the normal points toward increasing value
    v = {e: 0.5 * (np.array(M.corner_offset(M.edge_corners(e)[0])) + np.array(M.corner_offset(M.edge_corners(e)[1])))
         for e in range(12)}
    for case in range(256):
        for t in range(M.COUNT[case]):
            a, b, c = (v[int(e)] for e in M.TRIS[case, t])
            n = np.cross(b - a, c - a)
            if bin(case).count("1") == 1:
                corner = np.array(M.corner_offset(case.bit_length() - 1), np.float64)
                assert np.dot(n, (a + b + c) / 3 - corner) > 0, case


def test_the_table_is_the_generators_output():
    import subprocess
    import sys
    rc = subprocess.run([sys.executable, os.path.join(util.ROOT, "tools", "gen_mc_table.py"), "--check"]).returncode
    assert rc == 0


# --------------------------------------------------------------------------- reference meshes
def _manifold(v, f):
    """(closed: every vertex pair of a triangle edge in exactly two triangles, Euler characteristic, every vertex used)"""
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = torch.minimum(e[:, 0], e[:, 1]) * (1 << 32) + torch.maximum(e[:, 0], e[:, 1])
    uniq, cnt = torch.unique(key, return_counts=True)
    used = torch.unique(f)
    return bool((cnt == 2).all()), len(used) - len(uniq) + len(f), len(used) == len(v)


def _centres(bounds, n):
    cs = M.axis_centres(bounds, (n, n, n))
    return torch.meshgrid(*[c.double() for c in cs], indexing="ij")


def _signed_volume(v, f):
    a, b, c = (v[f[:, k]].double() for k in range(3))
    return float((a * torch.cross(b, c, dim=1)).sum()) / 6


def test_sphere_is_closed_with_euler_characteristic_2_and_within_the_interpolation_bound():
    bounds, n, R = (-1, -1, -1, 1, 1, 1), 48, 0.7
    x, y, z = _centres(bounds, n)
    sdf = (torch.sqrt(x * x + y * y + z * z) - R).float()
    out = M.marching_cubes(sdf, 0.0, bounds)
    v, f = out["vertices"], out["faces"]
    closed, chi, used = _manifold(v, f)
    assert closed and chi == 2 and used
    assert _signed_volume(v, f) > 0.95 * 4 / 3 * math.pi * R ** 3  # positive: the normals point out of the surface
    # along an edge f = |x| - R is convex with f'' <= 1 / |x| <= 1 / (R - h): the linear interpolant's root x_v has
    # |f(x_v)| <= h^2 / (8 (R - h)), and |f(x_v)| is the vertex's distance to the sphere
    h = 2.0 / n
    err = (v.double().norm(dim=1) - R).abs().max()
    assert float(err) <= h * h / (8 * (R - h)) + 1e-6


def test_torus_has_euler_characteristic_0():
    bounds, n = (-1, -1, -1, 1, 1, 1), 48
    x, y, z = _centres(bounds, n)
    f = (torch.sqrt((torch.sqrt(x * x + y * y) - 0.55) ** 2 + z * z) - 0.25).float()
    out = M.marching_cubes(f, 0.0, bounds)
    closed, chi, used = _manifold(out["vertices"], out["faces"])
    assert closed and chi == 0 and used and _signed_volume(out["vertices"], out["faces"]) > 0


def _ambiguous_faces(case_grid):
    """the number of cell faces whose four corners alternate in sign"""
    n = 0
    for a, b, c, d in ((0, 1, 3, 2), (4, 5, 7, 6), (0, 1, 5, 4), (2, 3, 7, 6), (0, 2, 6, 4), (1, 3, 7, 5)):
        bit = lambda k: (case_grid >> k) & 1  # noqa: E731
        n += int(((bit(a) == bit(c)) & (bit(b) == bit(d)) & (bit(a) != bit(b))).sum())
    return n


@pytest.mark.parametrize("seed", range(4))
def test_random_smooth_fields_give_closed_meshes(seed):
    g = torch.Generator().manual_seed(seed)
    r = torch.randn(1, 1, 7, 9, 8, generator=g, dtype=torch.float64)
    fld = torch.nn.functional.interpolate(r, size=(36, 40, 33), mode="trilinear", align_corners=True)[0, 0].float()
    fld[[0, -1]] = 1.0
    fld[:, [0, -1]] = 1.0
    fld[:, :, [0, -1]] = 1.0  # the level set stays inside the grid
    for level, weight in ((0.0, None), (0.2, torch.rand(fld.shape, generator=g) > 0.0)):
        out = M.marching_cubes(fld, level, (0, 0, 0, 3.6, 4.0, 3.3), weight=weight)
        closed, _, used = _manifold(out["vertices"], out["faces"])
        assert closed and used and len(out["faces"]) > 1000
    case = torch.zeros(35, 39, 32, dtype=torch.int64)
    for c in range(8):
        dx, dy, dz = M.corner_offset(c)
        case |= (fld[dx:35 + dx, dy:39 + dy, dz:32 + dz] < 0).long() << c
    assert _ambiguous_faces(case) > 20


def test_vertices_are_shared_ordered_and_colours_follow_t():
    rng = np.random.default_rng(2)
    vals = torch.tensor(rng.standard_normal((5, 6, 4)), dtype=torch.float32)
    col = torch.tensor(rng.standard_normal((2, 5, 6, 4)), dtype=torch.float32)
    out = M.marching_cubes(vals, 0.1, (0, 0, 0, 1, 1, 1), color=col)
    v, f, c = out["vertices"], out["faces"], out["colors"]
    assert len(torch.unique(v, dim=0)) == len(v) and set(torch.unique(f).tolist()) == set(range(len(v)))
    # interpolation written op for op: the colour of a vertex is qa + t (qb - qa) with t from the values
    assert c.shape == (len(v), 2) and torch.isfinite(c).all()
    # a side below 2 gives an empty mesh
    assert len(M.marching_cubes(vals[:1], 0.0, (0, 0, 0, 1, 1, 1))["faces"]) == 0


# --------------------------------------------------------------------------- reference fusion
def test_reference_fusion_of_a_plane_matches_the_closed_form():
    from manigaussian_b200 import scenes
    cam = scenes.make_camera(64, 48, 0, 4)
    view = dict(viewmatrix=np.asarray(cam["viewmatrix"], np.float64).reshape(-1), projmatrix=np.asarray(cam["projmatrix"], np.float64).reshape(-1),
                W=64, H=48, tanfovx=float(cam["tanfovx"]), tanfovy=float(cam["tanfovy"]))
    bounds, n = tuple(float(x) for x in scenes.SCENE_BOUNDS), 24
    pts = torch.stack([c.reshape(-1) for c in torch.meshgrid(*M.axis_centres(bounds, (n, n, n)), indexing="ij")], -1).numpy()
    D, trunc = float(np.float32(1.7)), 0.08  # the depth image holds D in float32
    depth = np.full((1, 48, 64), D, np.float32)
    ts, w, _, border = T64.fuse(pts, [view], depth, trunc)
    want_ts, want_w = T64.plane_closed_form(pts, view, D, trunc)
    import visibility_ref64 as V64
    uv, _, ok = V64.project(pts, view)
    inside = V64.in_view(uv, ok, 64, 48) & ~border
    assert inside.sum() > 1000 and ((want_w > 0) & inside).sum() > 100
    assert np.array_equal(w[inside], want_w[inside]) and np.abs(ts[inside] - want_ts[inside]).max() < 1e-12
    assert (w[~V64.in_view(uv, ok, 64, 48)] == 0).all() and (ts[w == 0] == 1).all()
    # continuing from a state equals one call over both views
    a = T64.fuse(pts, [view, view], np.concatenate([depth, depth * 1.01]), trunc)
    b = T64.fuse(pts, [view], depth * 1.01, trunc, state=T64.fuse(pts, [view], depth, trunc)[:3])
    assert all(np.array_equal(x, y) for x, y in zip(a[:2], b[:2]))


# --------------------------------------------------------------------------- C ABI
SYMS = ("mgs_tsdf_fuse", "mgs_marching_cubes_state_bytes", "mgs_marching_cubes_count", "mgs_marching_cubes_emit")


def test_header_declares_and_the_library_exports_the_mesh_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    L = _binding.lib()
    for sym in SYMS:
        assert re.fullmatch(r"mgs_[a-z_]+", sym)
        assert re.search(r"\b%s\s*\(" % sym, hdr) and sym in _binding.EXPORTED_SYMBOLS and hasattr(L, sym)
    assert L.mgs_abi_version() == 400


def test_state_bytes_grow_with_the_grid():
    L = _binding.lib()
    sizes = [L.mgs_marching_cubes_state_bytes(n, n, n) for n in (2, 16, 64, 128)]
    assert all(b > a for a, b in zip(sizes, sizes[1:]))
    assert L.mgs_marching_cubes_state_bytes(64, 64, 64) >= 18 * 64 ** 3
    assert L.mgs_marching_cubes_state_bytes(512, 512, 512) < 19 * 512 ** 3


_S = 4096  # a non-NULL address: every call below fails before it could be used


def _views(V=1, W=8, H=6):
    views = (_binding.View * V)()
    for v in views:
        v.width, v.height, v.tan_fovx, v.tan_fovy = W, H, 0.5, 0.5
        v.viewmatrix, v.projmatrix = _S, _S
    return views


def _bounds(b=(0, 0, 0, 1, 1, 1)):
    return (ctypes.c_double * 6)(*b)


def _fuse(V=1, views=None, fisheye=None, depth=_S, C=0, color=None, bounds="ok", X=4, Y=4, Z=4, trunc=0.1, tsdf=_S, weight=_S,
          cvol=None):
    L = _binding.lib()
    views = _views(max(V, 1)) if views is None else views
    b = _bounds() if bounds == "ok" else bounds
    return L.mgs_tsdf_fuse(V, views, None, None, fisheye, None, depth, C, color, b, X, Y, Z, trunc, tsdf, weight, cvol, 0, None)


@pytest.mark.parametrize("case,msg", [
    ("V0", "at least one view"),
    ("no_matrix", "matrices"),
    ("size", "bad size"),
    ("mixed_size", "same width and height"),
    ("fisheye", "theta_max"),
    ("X0", "X, Y and Z must be > 0"),
    ("Zneg", "X, Y and Z must be > 0"),
    ("trunc0", "trunc must be finite and > 0"),
    ("trunc_nan", "trunc must be finite and > 0"),
    ("trunc_inf", "trunc must be finite and > 0"),
    ("C33", "C must be in [0, 32]"),
    ("Cneg", "C must be in [0, 32]"),
    ("no_bounds", "bounds are required"),
    ("flat_bounds", "bounds must be finite and increasing"),
    ("nan_bounds", "bounds must be finite and increasing"),
    ("no_depth", "depth, tsdf and weight are required"),
    ("no_tsdf", "depth, tsdf and weight are required"),
    ("no_weight", "depth, tsdf and weight are required"),
    ("no_color", "color and color_volume are required"),
    ("no_color_volume", "color and color_volume are required"),
])
def test_fusion_argument_errors_return_before_anything_is_enqueued(case, msg):
    kw = {}
    if case == "V0":
        kw["V"] = 0
    elif case == "no_matrix":
        kw["views"] = _views()
        kw["views"][0].viewmatrix = None
    elif case == "size":
        kw["views"] = _views(W=0)
    elif case == "mixed_size":
        kw["views"] = _views(2)
        kw["views"][1].height = 7
        kw["V"] = 2
    elif case == "fisheye":
        fe = (_binding.ViewFisheye * 1)()
        fe[0].fisheye, fe[0].theta_max = 1, 2.0
        kw["fisheye"] = fe
    elif case == "X0":
        kw["X"] = 0
    elif case == "Zneg":
        kw["Z"] = -3
    elif case.startswith("trunc"):
        kw["trunc"] = {"trunc0": 0.0, "trunc_nan": float("nan"), "trunc_inf": float("inf")}[case]
    elif case == "C33":
        kw.update(C=33, color=_S, cvol=_S)
    elif case == "Cneg":
        kw["C"] = -1
    elif case == "no_bounds":
        kw["bounds"] = None
    elif case == "flat_bounds":
        kw["bounds"] = _bounds((0, 0, 0, 1, 0, 1))
    elif case == "nan_bounds":
        kw["bounds"] = _bounds((0, 0, float("nan"), 1, 1, 1))
    elif case == "no_depth":
        kw["depth"] = None
    elif case == "no_tsdf":
        kw["tsdf"] = None
    elif case == "no_weight":
        kw["weight"] = None
    elif case == "no_color":
        kw.update(C=3, cvol=_S)
    elif case == "no_color_volume":
        kw.update(C=3, color=_S)
    rc = _fuse(**kw)
    assert rc == -1 and msg in _binding.last_error(), (rc, _binding.last_error())


@pytest.mark.parametrize("call,args,msg", [
    ("count", (_S, -1, 4, 4, _S, None, 0.0, _S), "X, Y and Z must be >= 0"),
    ("count", (None, 4, 4, 4, _S, None, 0.0, _S), "state, values and out_counts are required"),
    ("count", (_S, 4, 4, 4, None, None, 0.0, _S), "state, values and out_counts are required"),
    ("count", (_S, 4, 4, 4, _S, None, 0.0, None), "state, values and out_counts are required"),
    ("emit", (_S, 4, -4, 4, _S, 0.0, "ok", 0, None, _S, _S, None), "X, Y and Z must be >= 0"),
    ("emit", (_S, 4, 4, 4, _S, 0.0, "ok", 33, _S, _S, _S, _S), "C must be in [0, 32]"),
    ("emit", (_S, 4, 4, 4, _S, 0.0, None, 0, None, _S, _S, None), "bounds are required"),
    ("emit", (_S, 4, 4, 4, _S, 0.0, (0, 0, 0, 1, 1, -1), 0, None, _S, _S, None), "finite and increasing"),
    ("emit", (None, 4, 4, 4, _S, 0.0, "ok", 0, None, _S, _S, None), "are required"),
    ("emit", (_S, 4, 4, 4, _S, 0.0, "ok", 0, None, None, _S, None), "are required"),
    ("emit", (_S, 4, 4, 4, _S, 0.0, "ok", 0, None, _S, None, None), "are required"),
    ("emit", (_S, 4, 4, 4, _S, 0.0, "ok", 2, None, _S, _S, _S), "color and out_colors are required"),
    ("emit", (_S, 4, 4, 4, _S, 0.0, "ok", 2, _S, _S, _S, None), "color and out_colors are required"),
])
def test_marching_cubes_argument_errors_return_before_anything_is_enqueued(call, args, msg):
    L = _binding.lib()
    if call == "count":
        rc = L.mgs_marching_cubes_count(*args, 0, None)
    else:
        a = list(args)
        a[6] = _bounds() if a[6] == "ok" else (None if a[6] is None else _bounds(a[6]))
        rc = L.mgs_marching_cubes_emit(*a, 0, None)
    assert rc == -1 and msg in _binding.last_error(), (rc, _binding.last_error())


@pytest.mark.parametrize("shape", [(1, 5, 5), (5, 0, 5), (5, 5, 1), (0, 0, 0)])
def test_grids_without_a_cell_enqueue_nothing(shape):
    L = _binding.lib()
    # NULL everything and no device touched: these return before anything is looked up or launched
    assert L.mgs_marching_cubes_count(None, *shape, None, None, 0.0, None, 0, None) == 0
    assert L.mgs_marching_cubes_emit(None, *shape, None, 0.0, None, 0, None, None, None, None, 0, None) == 0


# --------------------------------------------------------------------------- Python surface
def _settings(V=2, W=8, H=6, device="cpu"):
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    return [GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4, device=device), torch.eye(4, device=device), 0,
                                          torch.zeros(3), False, False, False) for _ in range(V)]


_B = (0, 0, 0, 1, 1, 1)


def _volume(C=0, n=(4, 4, 4)):
    return {"tsdf": torch.ones(n), "weight": torch.zeros(n), "color": torch.zeros((C,) + n) if C else None}


@pytest.mark.parametrize("kw,match", [
    (dict(cameras=[]), "at least one view"),
    (dict(), "expected a CUDA viewmatrix"),
    (dict(cameras=_settings(1) + _settings(1, W=9)), "same size"),
    (dict(bounds=(0, 0, 0, 1, 1)), "bounds must be"),
    (dict(bounds=(0, 1, 0, 1, 1, 1)), "bounds must be"),
    (dict(resolution=0), "resolution must be"),
    (dict(resolution=(4, 4)), "resolution must be"),
    (dict(trunc=0.0), "trunc must be a finite number > 0"),
    (dict(trunc=-1.0), "trunc must be a finite number > 0"),
    (dict(trunc=float("inf")), "trunc must be a finite number > 0"),
    (dict(trunc=True), "trunc must be a finite number > 0"),
    (dict(depth=torch.zeros(2, 6, 9)), r"depth: expected \[2,6,8\]"),
    (dict(depth=torch.zeros(3, 6, 8)), r"depth: expected \[2,6,8\]"),
    (dict(depth=torch.zeros(2, 6, 8, dtype=torch.float64)), "depth: expected float32"),
    (dict(depth=np.zeros((2, 6, 8), np.float32)), r"depth: expected \[2,6,8\]"),
    (dict(color=torch.zeros(2, 3, 6, 9)), r"color: expected \[2,\.,6,8\]"),
    (dict(color=torch.zeros(2, 3, 6, 8, dtype=torch.float16)), "color: expected float32"),
    (dict(color=torch.zeros(2, 33, 6, 8)), "1 to 32 channels"),
    (dict(color=torch.zeros(2, 0, 6, 8)), "1 to 32 channels"),
    (dict(volume={"tsdf": torch.ones(4, 4, 4)}), "volume: expected an earlier result"),
    (dict(volume=_volume(n=(4, 4, 5))), r"volume\['tsdf'\]: expected \[4,4,4\]"),
    (dict(volume=dict(_volume(), weight=torch.zeros(4, 4, 4, dtype=torch.float64))), r"volume\['weight'\]: expected float32"),
    (dict(volume=_volume(C=3)), "both be given or both be None"),
    (dict(volume=_volume(), color=torch.zeros(2, 3, 6, 8)), "both be given or both be None"),
    (dict(volume=_volume(C=2), color=torch.zeros(2, 3, 6, 8)), r"volume\['color'\]: expected \[3,4,4,4\]"),
    (dict(volume=dict(_volume(), tsdf=torch.ones(4, 4, 4).transpose(0, 1))), "contiguous"),
])
def test_tsdf_fuse_rejects_bad_arguments(kw, match):
    args = dict(cameras=_settings(), depth=torch.zeros(2, 6, 8), bounds=_B, resolution=4, trunc=0.1)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        GR.tsdf_fuse(**args)


def test_marching_cubes_has_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.marching_cubes(torch.zeros(3, 3, 3), 0.0, _B)


@pytest.mark.parametrize("kw,match", [
    (dict(values=torch.zeros(3, 3)), r"values: expected \[X,Y,Z\]"),
    (dict(values=[[[0.0]]]), r"values: expected \[X,Y,Z\]"),
    (dict(values=torch.zeros(3, 3, 3, dtype=torch.float64)), "values: expected float32"),
    (dict(level=float("nan")), "level must be a finite number"),
    (dict(level="0"), "level must be a finite number"),
    (dict(bounds=(0, 0, 0, 1, 1)), "bounds must be"),
    (dict(bounds=(0, 0, 1, 1, 1, 1)), "bounds must be"),
    (dict(weight=torch.zeros(3, 3, 4)), r"weight: expected \[3,3,3\]"),
    (dict(weight=torch.zeros(3, 3, 3, dtype=torch.int32)), "weight: expected float32"),
    (dict(color=torch.zeros(3, 3, 3)), r"color: expected \[\.,3,3,3\]"),
    (dict(color=torch.zeros(33, 3, 3, 3)), "1 to 32 channels"),
    (dict(color=torch.zeros(0, 3, 3, 3)), "1 to 32 channels"),
])
def test_marching_cubes_rejects_bad_arguments(kw, match):
    args = dict(values=torch.zeros(3, 3, 3), level=0.0, bounds=_B)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        GR.marching_cubes(**args)
