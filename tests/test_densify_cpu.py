"""Default density control without a GPU: the numpy restatement (tests/densify_ref64.py) against an independent torch
transcription of gsplat's DefaultStrategy duplicate / split / remove sequence with the same normals injected, its edge
cases, the C ABI's declarations and argument errors through ctypes, and the Python surface's refusals
(gaussian_renderer.densify_stats / densify_and_prune / densify_reset_opacity)."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import densify_ref64 as D
import mcmc_ref64 as M
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR


# --------------------------------------------------------------------------- gsplat, transcribed in torch (float64)
def _rotmat(q):
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


def gsplat_refine(params, moments, grads, radii, z, scene_scale, grow_grad2d=2e-4, grow_scale3d=0.01, grow_scale2d=None,
                  prune_opa=0.005, prune_scale3d=0.1, prune_scale2d=None, prune_too_big=False):
    """gsplat's DefaultStrategy._grow_gs (duplicate, then split) and _prune_gs (remove) as its ops write them, on float64
    tensors, with the split's torch.randn(2, N, 3) replaced by z[:, sel] (z [2,P,3]).  A row "index" carries each row's
    parent.  Returns (params, moments) as numpy."""
    p = {k: torch.from_numpy(v).double() for k, v in params.items()}
    P = p["pts_xyz"].shape[0]
    p["index"] = torch.arange(P, dtype=torch.float64)
    m = {k: [torch.from_numpy(v).double() for v in vs] for k, vs in moments.items()}
    radii = torch.from_numpy(radii).double()
    z = torch.from_numpy(z)

    is_grad_high = torch.from_numpy(grads).double() > grow_grad2d
    is_small = torch.exp(p["scales"]).max(dim=-1).values <= grow_scale3d * scene_scale
    is_dupli = is_grad_high & is_small
    is_split = is_grad_high & ~is_small
    if grow_scale2d is not None:
        is_split |= radii > grow_scale2d
    # duplicate
    sel = torch.where(is_dupli)[0]
    p = {k: torch.cat([v, v[sel]]) for k, v in p.items()}
    m = {k: [torch.cat([v, torch.zeros_like(v[sel])]) for v in vs] for k, vs in m.items()}
    radii = torch.cat([radii, radii[sel]])
    is_split = torch.cat([is_split, torch.zeros(len(sel), dtype=torch.bool)])
    # split
    sel, rest = torch.where(is_split)[0], torch.where(~is_split)[0]
    scales = torch.exp(p["scales"][sel])
    quats = torch.nn.functional.normalize(p["rotations"][sel], dim=-1)
    samples = torch.einsum("nij,nj,bnj->bni", _rotmat(quats), scales, z[:, sel])
    for k, v in p.items():
        if k == "pts_xyz":
            new = (v[sel] + samples).reshape(-1, 3)
        elif k == "scales":
            new = torch.log(scales / 1.6).repeat(2, 1)
        else:
            new = v[sel].repeat([2] + [1] * (v.dim() - 1))
        p[k] = torch.cat([v[rest], new])
    m = {k: [torch.cat([v[rest], torch.zeros((2 * len(sel),) + v.shape[1:], dtype=v.dtype)]) for v in vs] for k, vs in m.items()}
    radii = torch.cat([radii[rest], radii[sel].repeat(2)])
    # prune
    is_prune = torch.sigmoid(p["opacity"].flatten()) < prune_opa
    if prune_too_big:
        is_too_big = torch.exp(p["scales"]).max(dim=-1).values > prune_scale3d * scene_scale
        if prune_scale2d is not None:
            is_too_big |= radii > prune_scale2d
        is_prune |= is_too_big
    keep = ~is_prune
    return ({k: v[keep].numpy() for k, v in p.items()}, {k: [v[keep].numpy() for v in vs] for k, vs in m.items()})


def _cloud(P, seed, opacity_shape=None):
    rng = np.random.default_rng(seed)
    p = {"pts_xyz": rng.normal(0, 1, (P, 3)), "rotations": rng.normal(0, 1, (P, 4)),
         "scales": rng.uniform(-7.0, -1.0, (P, 3)), "opacity": rng.uniform(-8.0, 4.0, opacity_shape or (P,)),
         "sh": rng.normal(0, 1, (P, 16, 3)), "feat": rng.normal(0, 1, (P, 5))}
    p = {k: v.astype(np.float32) for k, v in p.items()}
    moments = {k: [rng.uniform(0.5, 1.5, v.shape).astype(np.float32) for _ in range(2)] for k, v in p.items()}
    count = rng.integers(0, 5, P).astype(np.int32)
    grad2d = (rng.uniform(0, 4e-4, P) * np.maximum(count, 1)).astype(np.float32)
    radius = rng.uniform(0, 0.2, P).astype(np.float32)
    return p, moments, grad2d, count, radius


RULES = [dict(scene_scale=1.0),
         dict(scene_scale=2.5, grow_scale2d=0.15),
         dict(scene_scale=1.0, prune_too_big=True, prune_scale3d=0.2, prune_opacity=0.02),
         dict(scene_scale=0.5, grow_scale2d=0.1, prune_too_big=True, prune_scale2d=0.18, grad_threshold=1e-4)]


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("opacity_shape", [None, "col"])
def test_restatement_matches_gsplats_ops(rule, opacity_shape):
    P = 3000
    params, moments, grad2d, count, radius = _cloud(P, 7, (P, 1) if opacity_shape else None)
    z = np.random.default_rng(8).normal(0, 1, (2, P, 3))
    out, mom, source, counts, ex = D.refine(params, moments, grad2d, count, radius, seed=0, offset=0,
                                            normals=lambda b: z[b], **rule)
    g = {"grow_grad2d": rule.get("grad_threshold", 2e-4), "prune_opa": rule.get("prune_opacity", 0.005)}
    g.update({k: v for k, v in rule.items() if k not in ("grad_threshold", "prune_opacity")})
    want, want_m = gsplat_refine(params, moments, (grad2d / np.maximum(count, 1)).astype(np.float64), radius, z, **g)
    # the same rows in the same order
    assert np.array_equal(source, want["index"].astype(np.int64))
    n_new, cloned, split, pruned = counts
    assert n_new == len(source) and n_new == P + cloned + split - pruned
    assert cloned > 0 and split > 0 and pruned > 0
    ch = ex["children"]
    for k in ("rotations", "opacity", "sh", "feat"):
        assert np.array_equal(out[k], want[k].astype(np.float32)), k
    assert np.array_equal(out["pts_xyz"][:ch.start], want["pts_xyz"][:ch.start].astype(np.float32))
    assert np.array_equal(out["scales"][:ch.start], want["scales"][:ch.start].astype(np.float32))
    assert np.allclose(out["scales"][ch], want["scales"][ch], rtol=1e-6, atol=0)  # log(s / 1.6) vs ls - log(1.6)
    assert np.allclose(ex["mean64"], want["pts_xyz"][ch], rtol=0, atol=1e-12)
    for k in mom:
        for a, b in zip(mom[k], want_m[k]):
            assert np.array_equal(a, b.astype(np.float32)), k


def test_edge_cases():
    """row 0 both cloned and split, 1 with count 0, 2 and 3 NaN, 4 untouched, 5 transparent, 6 split with children that
    are still too big, which only prune_too_big removes"""
    ls = np.array([[-6, -6, -6], [-6, -6, -6], [np.nan, -6, -6], [np.nan, np.nan, np.nan], [-3, -3, -3], [-3, -3, -3],
                   [-1, -2, -2]], np.float32)
    x = np.array([1, 1, 1, np.nan, 1, -9, 1], np.float32)
    grad2d = np.array([1e-3, 3e-4, 1e-3, 1e-3, 0, 1e-3, 1e-3], np.float32)
    count = np.array([1, 0, 1, 1, 3, 1, 1], np.int32)
    radius = np.array([0.5, 0, 0, 0, 0.01, 0, 0], np.float32)
    f = D.classify(ls, x, grad2d, count, radius, scene_scale=1.0, grow_scale2d=0.3)
    # 0: high, small and a large radius: cloned and split, the original replaced by its clone and two children
    assert f["clone"][0] and f["split"][0] and not f["keep"][0] and f["clone_kept"][0] and f["child_kept"][0]
    # 1: count 0 divides by 1: 3e-4 > 2e-4
    assert f["clone"][1] and f["keep"][1]
    # 2: a NaN axis is ignored, so L = -6 <= log(0.01): cloned
    assert f["clone"][2] and not f["split"][2]
    # 3: every axis NaN: L is NaN, not small, so split; a NaN logit is not below t_opa, so nothing is pruned
    assert f["split"][3] and not f["clone"][3] and f["child_kept"][3]
    assert f["keep"][4] and not (f["clone"][4] or f["split"][4])
    assert f["split"][5] and not (f["keep"][5] or f["child_kept"][5])  # transparent: every row pruned
    # 6: L = -1 > log(0.1) = -2.30: too big, its children (L = -1.47) too
    f2 = D.classify(ls, x, grad2d, count, radius, scene_scale=1.0, prune_too_big=True)
    assert f2["split"][6] and not f2["child_kept"][6]
    assert f2["keep"][4] and not f2["keep"][6] and f["child_kept"][6]  # exp(-3) < 0.1: not too big


def test_nothing_selected_and_everything_pruned():
    params, moments, grad2d, count, radius = _cloud(200, 3)
    out, mom, source, counts, _ = D.refine(params, moments, np.zeros_like(grad2d), count, radius, 0, 0, scene_scale=1.0,
                                           prune_opacity=1e-9)
    assert counts == (200, 0, 0, 0) and np.array_equal(source, np.arange(200))
    for k in params:
        assert np.array_equal(out[k], params[k])
        for a, b in zip(mom[k], moments[k]):
            assert np.array_equal(a, b)
    params["opacity"][:] = -20.0
    out, mom, source, counts, _ = D.refine(params, moments, grad2d, count, radius, 0, 0, scene_scale=1.0)
    assert counts[0] == 0 and len(source) == 0 and counts[3] == 200 + counts[1] + counts[2]
    assert all(v.shape[0] == 0 for v in out.values())


def test_children_draw_at_their_own_tags():
    z0, z1 = D.child_normals(5, 9, 1000, 0), D.child_normals(5, 9, 1000, 1)
    zp = M.normals(5, 9, 1000)
    assert M.TAG_PERTURB == 1  # restored
    assert not np.allclose(z0, zp) and not np.allclose(z1, zp) and not np.allclose(z0, z1)
    w = M.draws(5, 9, np.arange(1000), 3)
    u1 = (w[0].astype(np.float32) + np.float32(1.0)) * np.float32(2.0 ** -32)
    u2 = w[1].astype(np.float32) * np.float32(2.0 ** -32)
    assert np.allclose(z1[:, 0], np.sqrt(-2.0 * np.log(u1.astype(np.float64))) * np.cos(2 * np.pi * u2.astype(np.float64)))


def test_stats_restatement():
    rng = np.random.default_rng(2)
    V, P = 4, 500
    g = rng.normal(0, 1e-3, (V, P, 3)).astype(np.float32)
    radii = rng.integers(-1, 30, (V, P)).astype(np.int32)
    sizes = [640, 480, 800, 100]
    z = (np.zeros(P, np.float32), np.zeros(P, np.int32), np.zeros(P, np.float32))
    gd, c, r = D.stats(*z, g, radii, sizes, scale=4.0)
    m = radii > 0
    assert np.array_equal(c, m.sum(0))
    want = (np.hypot(g[..., 0].astype(np.float64), g[..., 1].astype(np.float64)) * m).sum(0) * 4.0
    assert np.allclose(gd, want, rtol=1e-6, atol=0)
    assert np.array_equal(r, np.max(np.where(m, radii / np.array(sizes, np.float32)[:, None], 0), 0).astype(np.float32))
    # one call over V views equals successive calls over the views in order
    s = z
    for v in range(V):
        s = D.stats(*s, g[v], radii[v], sizes[v:v + 1], scale=4.0)
    assert all(np.array_equal(a, b) for a, b in zip(s, (gd, c, r)))


# --------------------------------------------------------------------------- C ABI
_SYMS = ("mgs_densify_stats", "mgs_densify_state_bytes", "mgs_densify_count", "mgs_densify_emit")


def test_header_declares_and_the_library_exports_the_densify_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    for sym in _SYMS:
        assert re.search(r"\b%s\s*\(" % sym, hdr)
        assert sym in _binding.EXPORTED_SYMBOLS
        assert hasattr(_binding.lib(), sym)


_S = 4096  # a non-NULL address: every call below fails before it could be used


def _stats(**kw):
    a = dict(V=2, P=10, grad=_S, radii=_S, sizes=(ctypes.c_int * 2)(640, 480), scale=1.0, scale_device=None, grad2d=_S,
             count=_S, radius=_S)
    a.update(kw)
    return _binding.lib().mgs_densify_stats(a["V"], a["P"], a["grad"], a["radii"], a["sizes"], a["scale"], a["scale_device"],
                                            a["grad2d"], a["count"], a["radius"], 0, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(V=-1), "V and P must be >= 0"),
    (dict(P=-1), "V and P must be >= 0"),
    (dict(grad=None), "are required"),
    (dict(radii=None), "are required"),
    (dict(sizes=None), "are required"),
    (dict(grad2d=None), "are required"),
    (dict(count=None), "are required"),
    (dict(radius=None), "are required"),
    (dict(sizes=(ctypes.c_int * 2)(640, 0)), "every size must be > 0"),
    (dict(scale=float("inf")), "scale must be finite"),
    (dict(scale=float("nan")), "scale must be finite"),
])
def test_stats_argument_errors_return_their_code_without_touching_a_gpu(kw, msg):
    assert _stats(**kw) == -1
    assert msg in _binding.last_error()


def test_stats_with_nothing_to_do_returns_without_touching_a_gpu():
    assert _stats(V=0, grad=None) == 0 and _stats(P=0, radius=None) == 0


def _count(**kw):
    a = dict(state=_S, P=10, ls=_S, x=_S, grad2d=_S, count=_S, radius=_S, scene_scale=1.0, grad_threshold=2e-4,
             grow_scale3d=0.01, grow_scale2d=math.inf, prune_opacity=0.005, prune_scale3d=0.1, prune_scale2d=math.inf,
             too_big=0, out=_S)
    a.update(kw)
    return _binding.lib().mgs_densify_count(a["state"], a["P"], a["ls"], a["x"], a["grad2d"], a["count"], a["radius"],
                                            a["scene_scale"], a["grad_threshold"], a["grow_scale3d"], a["grow_scale2d"],
                                            a["prune_opacity"], a["prune_scale3d"], a["prune_scale2d"], a["too_big"], a["out"],
                                            0, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(P=-1), "P must be >= 0"),
    (dict(state=None), "state and out_counts are required"),
    (dict(out=None), "state and out_counts are required"),
    (dict(ls=None), "required with P > 0"),
    (dict(x=None), "required with P > 0"),
    (dict(grad2d=None), "required with P > 0"),
    (dict(count=None), "required with P > 0"),
    (dict(radius=None), "required with P > 0"),
    (dict(scene_scale=0.0), "must be finite and > 0"),
    (dict(scene_scale=math.inf), "must be finite and > 0"),
    (dict(grow_scale3d=-1.0), "must be finite and > 0"),
    (dict(prune_scale3d=math.nan), "must be finite and > 0"),
    (dict(prune_opacity=0.0), "prune_opacity must be in (0, 1)"),
    (dict(prune_opacity=1.0), "prune_opacity must be in (0, 1)"),
    (dict(grad_threshold=math.nan), "must not be NaN"),
    (dict(grow_scale2d=math.nan), "must not be NaN"),
    (dict(prune_scale2d=math.nan), "must not be NaN"),
])
def test_count_argument_errors_return_their_code_without_touching_a_gpu(kw, msg):
    assert _count(**kw) == -1
    assert msg in _binding.last_error()


def _lists(n, width=3, ptr=_S):
    return n, (ctypes.c_void_p * max(n, 1))(*([ptr] * n)), (ctypes.c_int * max(n, 1))(*([width] * n))


def _emit(**kw):
    a = dict(state=_S, P=10, n_new=12, old=(_S,) * 4, rows=_lists(2), moments=_lists(4), new=(_S,) * 4,
             new_rows=_lists(2)[1], new_moments=_lists(4)[1], rng=_S, source=_S)
    a.update(kw)
    return _binding.lib().mgs_densify_emit(a["state"], a["P"], a["n_new"], *a["old"], *a["rows"], *a["moments"], *a["new"],
                                           a["new_rows"], a["new_moments"], a["rng"], a["source"], 0, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(P=-1), "P and n_new must be >= 0"),
    (dict(n_new=-1), "P and n_new must be >= 0"),
    (dict(P=0), "n_new must be 0 with P = 0"),
    (dict(state=None), "state and rng are required"),
    (dict(rng=None), "state and rng are required"),
    (dict(old=(_S, None, _S, _S)), "are required with P > 0"),
    (dict(new=(_S, _S, _S, None)), "are required with n_new > 0"),
    (dict(source=None), "are required with n_new > 0"),
    (dict(rows=_lists(17)), "rows: the count must be in [0, 16]"),
    (dict(moments=_lists(65)), "moments: the count must be in [0, 64]"),
    (dict(rows=(2, None, None)), "rows: the pointer and width arrays are required"),
    (dict(moments=_lists(4, width=0)), "moments: every width must be > 0"),
    (dict(rows=_lists(2, ptr=None)), "rows: every pointer is required"),
    (dict(new_rows=None), "rows: every new pointer is required"),
    (dict(new_moments=_lists(4, ptr=None)[1]), "moments: every new pointer is required"),
])
def test_emit_argument_errors_return_their_code_without_touching_a_gpu(kw, msg):
    assert _emit(**kw) == -1
    assert msg in _binding.last_error()


# --------------------------------------------------------------------------- Python surface
def _params(P=8, **over):
    p = {"pts_xyz": torch.zeros(P, 3), "rotations": torch.zeros(P, 4), "scales": torch.zeros(P, 3), "opacity": torch.zeros(P)}
    p.update(over)
    return p


_RNG = torch.zeros(2, dtype=torch.int64)


@pytest.mark.parametrize("case,match", [
    (dict(stats={}), "stats: expected a dict with keys"),
    (dict(stats=dict(GR.densify_state(8, "cpu"), count=torch.zeros(8))), r"stats\['count'\]: expected a contiguous torch.int32"),
    (dict(stats=GR.densify_state(7, "cpu")), r"stats\['grad2d'\]: expected a contiguous torch.float32 \[8\]"),
    (dict(viewspace_grad=torch.zeros(2, 8, 2)), r"viewspace_grad: expected \[V,P,3\] or \[P,3\]"),
    (dict(viewspace_grad=[0.0]), r"viewspace_grad: expected"),
    (dict(viewspace_grad=torch.zeros(2, 8, 3, dtype=torch.float64)), "viewspace_grad: expected float32"),
    (dict(radii=torch.zeros(8, dtype=torch.int32)), r"radii: expected \[2,8\], got"),
    (dict(radii=torch.zeros(2, 8, dtype=torch.int64)), "radii: expected int32"),
    (dict(sizes=[640]), "sizes: expected 2 positive ints"),
    (dict(sizes=[640, 0]), "sizes: expected 2 positive ints"),
    (dict(sizes=[640, 480.0]), "sizes: expected 2 positive ints"),
    (dict(sizes=None), "sizes: expected ints, a CameraBatch"),
    (dict(scale=float("nan")), "scale: expected a finite number"),
    (dict(scale=torch.ones(2)), "scale: expected a float32 tensor of one element"),
])
def test_densify_stats_rejects_bad_arguments(case, match):
    kw = dict(stats=GR.densify_state(8, "cpu"), viewspace_grad=torch.zeros(2, 8, 3), radii=torch.zeros(2, 8, dtype=torch.int32),
              sizes=[640, 480])
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.densify_stats(**kw)


def test_densify_stats_sizes_from_cameras_and_settings():
    from manigaussian_b200.cameras import camera_batch
    cams = camera_batch(torch.eye(4).repeat(3, 1, 1), np.tile(np.array([[50.0, 0, 32], [0, 50.0, 24], [0, 0, 1]]), (3, 1, 1)),
                        64, 48)
    assert GR._densify_sizes("w", cams, 3) == [64] * 3
    assert GR._densify_sizes("w", [cams.settings(k, torch.zeros(3), 0, False) for k in range(3)], 3) == [64] * 3
    assert GR._densify_sizes("w", 100, 2) == [100, 100]


@pytest.mark.parametrize("case,match", [
    (dict(params={"pts_xyz": torch.zeros(8, 3)}), "expected a dict with keys"),
    (dict(params=_params(rotations=torch.zeros(8, 3))), r"rotations'\]: expected \[8,4\]"),
    (dict(params=_params(sh=torch.zeros(9, 16, 3))), r"sh'\]: expected \[8, ...\]"),
    (dict(params=_params(**{f"f{k}": torch.zeros(8, 2) for k in range(17)})), "at most 16 rows"),
    (dict(stats=GR.densify_state(9, "cpu")), r"stats\['grad2d'\]: expected a contiguous torch.float32 \[8\]"),
    (dict(scene_scale=0.0), "scene_scale must be a finite number > 0"),
    (dict(scene_scale=None), "scene_scale must be a finite number > 0"),
    (dict(grow_scale3d=-1.0), "grow_scale3d must be a finite number > 0"),
    (dict(prune_scale3d=math.inf), "prune_scale3d must be a finite number > 0"),
    (dict(prune_opacity=0.0), r"prune_opacity must be a number in \(0, 1\)"),
    (dict(grad_threshold=math.nan), "grad_threshold must be a number"),
    (dict(grow_scale2d="0.1"), "grow_scale2d must be a number or None"),
    (dict(prune_scale2d=math.nan), "prune_scale2d must be a number or None"),
    (dict(rng=torch.zeros(2, dtype=torch.int32)), r"rng: expected a contiguous int64 \[2\]"),
])
def test_densify_and_prune_rejects_bad_arguments(case, match):
    kw = dict(params=_params(), stats=GR.densify_state(8, "cpu"), scene_scale=1.0, rng=_RNG)
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.densify_and_prune(**kw)


def test_densify_and_prune_refuses_non_leaf_params_and_too_many_moments():
    leaf = torch.zeros(8, 3, requires_grad=True)
    with pytest.raises(ValueError, match="pts_xyz'\\] is not a leaf"):
        GR.densify_and_prune(_params(pts_xyz=leaf * 2.0), GR.densify_state(8, "cpu"), torch.optim.Adam([leaf]), scene_scale=1.0,
                             rng=_RNG)
    p = {k: torch.nn.Parameter(v) for k, v in _params(**{f"f{k}": torch.zeros(8, 2) for k in range(16)}).items()}
    opt = torch.optim.Adam(list(p.values()))
    for v in p.values():
        opt.state[v] = {"step": torch.zeros(()), "exp_avg": torch.zeros_like(v), "exp_avg_sq": torch.zeros_like(v),
                        "max_exp_avg_sq": torch.zeros_like(v), "other": torch.zeros_like(v)}
    with pytest.raises(ValueError, match="at most 64 moment tensors, got 80"):
        GR.densify_and_prune(p, GR.densify_state(8, "cpu"), opt, scene_scale=1.0, rng=_RNG)


def test_densify_has_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.densify_and_prune(_params(), GR.densify_state(8, "cpu"), scene_scale=1.0, rng=_RNG)
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.densify_stats(GR.densify_state(8, "cpu"), torch.zeros(8, 3), torch.zeros(8, dtype=torch.int32), 64)


def test_densify_reset_opacity():
    x = torch.nn.Parameter(torch.tensor([-9.0, -4.0, 0.0, 3.0, float("nan")]))
    other = torch.nn.Parameter(torch.ones(5, 3))
    opt = torch.optim.Adam([x, other])
    x.grad, other.grad = torch.ones(5), torch.ones(5, 3)
    opt.step()
    t = np.float32(math.log(0.01 / 0.99))
    x0 = x.detach().numpy().copy()
    out = GR.densify_reset_opacity({"opacity": x, "pts_xyz": other}, opt, value=0.01)
    assert out is x
    got = x.detach().numpy()
    assert np.array_equal(got[:4], np.minimum(x0[:4], t)) and (got[2:4] == t).all() and got[0] == x0[0]
    assert np.isnan(got[4])
    assert (opt.state[x]["exp_avg"] == 0).all() and (opt.state[x]["exp_avg_sq"] == 0).all()
    assert (opt.state[other]["exp_avg"] != 0).all() and float(opt.state[x]["step"]) == 1.0
    for bad in (0.0, 1.0, True):
        with pytest.raises(ValueError, match=r"value must be a number in \(0, 1\)"):
            GR.densify_reset_opacity({"opacity": x}, value=bad)
    with pytest.raises(ValueError, match="expected a dict with key opacity"):
        GR.densify_reset_opacity({"pts_xyz": other})
