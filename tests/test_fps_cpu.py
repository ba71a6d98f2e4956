"""Farthest-point sampling without a GPU: the float32 reference (tests/fps_ref.py) against a literal per-point Python loop on
tiny clouds and the definition's consequences, the C ABI's declarations, exports, state size and argument errors, calls
that enqueue nothing, and the Python surface's refusals (gaussian_renderer.farthest_point_sample)."""
import os
import re

import numpy as np
import pytest
import torch

import fps_ref as R
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR


def _tiny(kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.random((40, 3)).astype(np.float32)
    if kind == "lattice":  # many equal distances: the ties decide
        return (rng.integers(0, 3, (40, 3)) * 0.5).astype(np.float32)
    if kind == "duplicates":
        p = rng.random((30, 3)).astype(np.float32)
        p[10:20] = p[3]
        return p
    p = rng.normal(0, 1, (40, 3)).astype(np.float32)  # non-finite rows
    p[[0, 5, 17], [0, 2, 1]] = [np.nan, np.inf, -np.inf]
    return p


@pytest.mark.parametrize("kind", ["uniform", "lattice", "duplicates", "non_finite"])
@pytest.mark.parametrize("start", [None, 7, 0, 99, 5])
def test_reference_matches_the_literal_loop(kind, start):
    p = _tiny(kind, seed=len(kind))
    for n in (1, 12, len(p), len(p) + 5):
        idx, d2 = R.fps_ref_cloud(p, n, start)
        widx, wd2 = R.fps_loop(p, n, start)
        assert idx.tolist() == widx.tolist()
        assert d2.tobytes() == wd2.tobytes()


def test_reference_consequences():
    p = _tiny("duplicates", 3)
    idx, d2 = R.fps_ref_cloud(p, len(p) + 3)
    valid = idx >= 0
    assert valid.sum() == len(p) and len(set(idx[valid].tolist())) == len(p)
    assert np.isinf(d2[0]) and (np.diff(d2[1:len(p)]) <= 0).all()
    # the ten copies of point 3 at d2 = 0, in ascending index, once every distinct position is taken
    zero = idx[valid][d2[valid] == 0]
    assert zero.tolist() == sorted(zero.tolist()) and len(zero) == 10
    assert (idx[len(p):] == -1).all() and np.isinf(d2[len(p):]).all()


def test_reference_start_and_lowest_finite_point():
    p = _tiny("non_finite", 1)
    assert R.fps_ref_cloud(p, 1)[0][0] == 1          # point 0 is not finite
    assert R.fps_ref_cloud(p, 1, start=9)[0][0] == 9
    assert R.fps_ref_cloud(p, 1, start=5)[0][0] == 1  # a non-finite start falls back
    assert R.fps_ref_cloud(p, 1, start=-2)[0][0] == 1


def test_reference_batch_is_the_rows_cut_to_their_lengths():
    rng = np.random.default_rng(4)
    pts = rng.random((3, 50, 3)).astype(np.float32)
    lengths, start = np.array([50, 17, -3]), np.array([4, 30, 0])
    idx, d2 = R.fps_ref(pts, 20, lengths, start)
    for b, L in enumerate((50, 17, 0)):
        wi, wd = R.fps_ref_cloud(pts[b, :L], 20, start[b])
        assert idx[b].tolist() == wi.tolist() and d2[b].tobytes() == wd.tobytes()
    assert (idx[2] == -1).all()


# --------------------------------------------------------------------------- C ABI
def test_header_declares_and_the_library_exports_the_fps_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    for sym in ("mgs_fps_state_bytes", "mgs_fps"):
        assert re.search(r"\b%s\s*\(" % sym, hdr)
        assert sym in _binding.EXPORTED_SYMBOLS
        assert hasattr(_binding.lib(), sym)


def test_state_bytes_grow_with_b_and_p():
    L = _binding.lib()
    base = L.mgs_fps_state_bytes(1, 1000)
    assert L.mgs_fps_state_bytes(2, 1000) > base and L.mgs_fps_state_bytes(1, 2000) > base
    assert L.mgs_fps_state_bytes(4, 500_000) >= 4 * 500_000 * 16  # the streaming tier's {x, y, z, d} copy
    assert L.mgs_fps_state_bytes(0, 0) > 0


_S = 4096  # a non-NULL address: every call below fails before it could be used


@pytest.mark.parametrize("args,msg", [
    ((_S, -1, 10, 4, _S, None, None, _S, _S), "must be >= 0"),
    ((_S, 1, -1, 4, _S, None, None, _S, _S), "must be >= 0"),
    ((_S, 1, 10, -1, _S, None, None, _S, _S), "must be >= 0"),
    ((None, 1, 10, 4, _S, None, None, _S, _S), "required"),
    ((_S, 1, 10, 4, _S, None, None, None, _S), "required"),
    ((_S, 1, 10, 4, _S, None, None, _S, None), "required"),
    ((_S, 1, 10, 4, None, _S, _S, _S, _S), "points are required"),
])
def test_argument_errors_return_their_code_without_touching_a_gpu(args, msg):
    L = _binding.lib()
    assert L.mgs_fps(*args, 0, None) == -1
    assert msg in _binding.last_error()


def test_no_clouds_or_no_picks_enqueue_nothing():
    L = _binding.lib()
    # NULL everything, and no device touched: these return before anything is looked up or launched
    assert L.mgs_fps(None, 0, 10, 4, None, None, None, None, None, 0, None) == 0
    assert L.mgs_fps(None, 3, 10, 0, None, None, None, None, None, 0, None) == 0
    assert L.mgs_fps(None, 0, 0, 0, None, None, None, None, None, 0, None) == 0


# --------------------------------------------------------------------------- Python surface
_I = torch.zeros(2, dtype=torch.int64)


@pytest.mark.parametrize("case,match", [
    (dict(points=torch.zeros(5, 3, dtype=torch.float64)), "float32"),
    (dict(points=torch.zeros(5, 2)), r"\[P,3\] or \[B,P,3\]"),
    (dict(points=torch.zeros(2, 5, 3, 1)), r"\[P,3\] or \[B,P,3\]"),
    (dict(points=[[0.0, 0.0, 0.0]]), r"\[P,3\] or \[B,P,3\]"),
    (dict(points=torch.zeros(2, 5, 3), lengths=torch.zeros(2, dtype=torch.int32)), "lengths: expected int64"),
    (dict(points=torch.zeros(2, 5, 3), lengths=torch.zeros(3, dtype=torch.int64)), r"lengths: expected \[2\]"),
    (dict(points=torch.zeros(2, 5, 3), start=torch.zeros(2, 1, dtype=torch.int64)), r"start: expected \[2\]"),
    (dict(points=torch.zeros(5, 3), start=_I), r"start: expected \[\] or \[1\]"),
    (dict(points=torch.zeros(2, 5, 3), start=[0, 1]), "start: expected int64"),
    (dict(points=torch.zeros(5, 3), n=-1), "int >= 0"),
    (dict(points=torch.zeros(5, 3), n=2.0), "int >= 0"),
    (dict(points=torch.zeros(5, 3), n=True), "int >= 0"),
])
def test_farthest_point_sample_rejects_bad_arguments(case, match):
    kw = dict(n=3)
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.farthest_point_sample(**kw)


def test_farthest_point_sample_has_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.farthest_point_sample(torch.rand(10, 3), 3)
