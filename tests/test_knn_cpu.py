"""k nearest neighbours without a GPU: the float64 reference (tests/knn_ref64.py) against scipy's cKDTree on random,
clustered and duplicate-heavy clouds, its ordering, self, padding and non-finite rules, the C ABI's declarations, exports and
argument errors, and the Python surface's refusals (gaussian_renderer.knn, simple_knn._C.distCUDA2)."""
import os
import re

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import knn_ref64 as K64
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR


def _cloud(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.random((n, 3))
    if kind == "clustered":
        centres = rng.random((8, 3)) * 10.0
        return centres[rng.integers(0, 8, n)] + rng.normal(0.0, 0.05, (n, 3))
    # duplicate-heavy: a third of the points on one point, the rest on a coarse lattice (many equal distances)
    p = rng.integers(0, 6, (n, 3)).astype(np.float64) * 0.25
    p[: n // 3] = (0.5, 0.5, 0.5)
    return p


@pytest.mark.parametrize("kind", ["uniform", "clustered", "duplicates"])
@pytest.mark.parametrize("k", [1, 3, 20])
def test_reference_matches_ckdtree_on_the_points_themselves(kind, k):
    p = _cloud(kind, 700, seed=k)
    idx, d2 = K64.knn_ref64(p, k)
    # cKDTree counts the query point itself: its first hit is at distance 0 (itself or a duplicate), so drop one zero
    dt, it = cKDTree(p).query(p, k + 2)
    np.testing.assert_allclose(d2[:, :k], dt[:, 1:k + 1] ** 2, rtol=1e-12, atol=1e-12)
    assert (idx[:, :k] != np.arange(len(p))[:, None]).all()
    ok = K64.decided(d2, k)
    for i in np.flatnonzero(ok)[:200]:
        want = set(it[i, :k + 1]) - {i}
        if len(want) == k + 1:  # i was not among cKDTree's hits: drop its farthest
            want = set(it[i, :k])
        assert set(idx[i, :k]) == want


@pytest.mark.parametrize("kind", ["uniform", "clustered"])
def test_reference_matches_ckdtree_for_distinct_queries(kind):
    p = _cloud(kind, 600, seed=3)
    q = np.concatenate([_cloud(kind, 200, seed=4), np.random.default_rng(5).normal(0, 50.0, (20, 3))])
    idx, d2 = K64.knn_ref64(p, 8, queries=q)
    dt, it = cKDTree(p).query(q, 9)
    np.testing.assert_allclose(d2, dt ** 2, rtol=1e-12)
    ok = K64.decided(d2, 8)
    assert ok.mean() > 0.9
    for i in np.flatnonzero(ok):
        assert set(idx[i, :8]) == set(it[i, :8])


def test_reference_orders_by_distance_then_index_and_pads():
    p = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 0], [-1, 0, 0], [0, 2, 0]], np.float64)
    idx, d2 = K64.knn_ref64(p, 5, extra=0)
    assert idx[0].tolist() == [2, 1, 3, 4, -1]          # the duplicate at 0 first, then the tie 1 / 3 by index
    assert d2[0].tolist() == [0.0, 1.0, 1.0, 4.0, np.inf]
    assert idx[2].tolist() == [0, 1, 3, 4, -1]
    idx, d2 = K64.knn_ref64(p[:0], 2, queries=p[:2], extra=0)  # no points: every slot padded
    assert (idx == -1).all() and np.isinf(d2).all()


def test_reference_non_finite_points_are_never_neighbours_and_non_finite_queries_are_padded():
    p = np.array([[0, 0, 0], [np.nan, 0, 0], [0, np.inf, 0], [3, 0, 0]], np.float64)
    idx, d2 = K64.knn_ref64(p, 3, extra=0)
    assert idx[0].tolist() == [3, -1, -1] and d2[0, 0] == 9.0
    assert (idx[1] == -1).all() and (idx[2] == -1).all()
    idx, _ = K64.knn_ref64(p, 2, queries=np.array([[1, 0, 0], [0, 0, -np.inf]]), extra=0)
    assert idx[0].tolist() == [0, 3] and (idx[1] == -1).all()


def test_dist_cuda2_reference_is_the_mean_of_three_squared_distances():
    p = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [0, 0, 3], [10, 10, 10]], np.float64)
    assert K64.dist_cuda2_ref64(p)[0] == pytest.approx((1 + 4 + 9) / 3)


# --------------------------------------------------------------------------- C ABI
def test_header_declares_and_the_library_exports_the_knn_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    for sym in ("mgs_knn_state_bytes", "mgs_knn"):
        assert re.search(r"\b%s\s*\(" % sym, hdr)
        assert sym in _binding.EXPORTED_SYMBOLS
        assert hasattr(_binding.lib(), sym)
    L = _binding.lib()
    small = L.mgs_knn_state_bytes(100, 100)
    if small == 0:  # no CUDA device: CUB's scratch size cannot be queried, and the call says so
        assert "mgs_knn_state_bytes" in _binding.last_error()
    else:
        assert L.mgs_knn_state_bytes(1000, 1000) > small >= 100 * (8 + 8 + 4 + 4 + 16)


_S = 4096  # a non-NULL address: every call below fails before it could be used


@pytest.mark.parametrize("args,code,msg", [
    ((_S, 10, 10, 33, _S, None, _S, _S), -2, "at most 32"),
    ((_S, 10, 10, 0, _S, None, _S, _S), -1, "k must be"),
    ((_S, -1, 10, 3, _S, _S, _S, _S), -1, "must be >= 0"),
    ((_S, 10, -1, 3, _S, _S, _S, _S), -1, "must be >= 0"),
    ((_S, 10, 5, 3, _S, None, _S, _S), -1, "Q must equal N"),
    ((None, 10, 10, 3, _S, None, _S, _S), -1, "required"),
    ((_S, 10, 10, 3, _S, None, None, _S), -1, "required"),
    ((_S, 10, 10, 3, _S, None, _S, None), -1, "required"),
    ((_S, 10, 4, 3, None, _S, _S, _S), -1, "points are required"),
])
def test_argument_errors_return_their_code_without_touching_a_gpu(args, code, msg):
    L = _binding.lib()
    assert L.mgs_knn(*args, 0, None) == code
    assert msg in _binding.last_error()


def test_zero_queries_is_a_no_op():
    L = _binding.lib()
    assert L.mgs_knn(None, 0, 0, 3, None, None, None, None, 0, None) == 0
    assert L.mgs_knn(None, 10, 0, 3, _S, None, None, None, 0, None) == 0  # an empty queries tensor has no address


def test_start_level_restatement_counts_occupied_cells():
    # 1000 points on a 10^3 lattice with unit spacing: the fine cell is 9 / 2^21, so a level-L cell spans 2^L 9 / 2^21
    p = np.stack(np.meshgrid(*[np.arange(10.0)] * 3, indexing="ij"), -1).reshape(-1, 3)
    level, mean = K64.start_level(p, 8)
    assert mean[0] == 1.0 and mean[21] == 1000.0
    assert 8 / 8 ** 0.5 <= mean[level] <= 8 * 8 ** 0.5


# --------------------------------------------------------------------------- Python surface
@pytest.mark.parametrize("case,match", [
    (dict(points=torch.zeros(5, 3, dtype=torch.float64)), "float32"),
    (dict(points=torch.zeros(5, 2)), r"\[\.,3\]"),
    (dict(points=torch.zeros(5, 3), queries=torch.zeros(5, 3, dtype=torch.float16)), "float32"),
    (dict(points=torch.zeros(5, 3), queries=torch.zeros(5)), r"\[\.,3\]"),
    (dict(points=torch.zeros(5, 3), k=0), "1 .. 32"),
    (dict(points=torch.zeros(5, 3), k=33), "1 .. 32"),
    (dict(points=torch.zeros(5, 3), k=2.0), "1 .. 32"),
])
def test_knn_rejects_bad_arguments(case, match):
    kw = dict(k=3)
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.knn(**kw)


def test_knn_and_dist_cuda2_have_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.knn(torch.rand(10, 3), 3)
    from simple_knn._C import distCUDA2
    with pytest.raises(RuntimeError, match="no CPU path"):
        distCUDA2(torch.rand(10, 3))


def test_dist_cuda2_import_path_and_its_refusals():
    import simple_knn
    from simple_knn._C import distCUDA2
    assert simple_knn.distCUDA2 is distCUDA2
    with pytest.raises(ValueError, match="at least 4"):
        distCUDA2(torch.rand(3, 3))
    with pytest.raises(ValueError, match=r"\[P,3\]"):
        distCUDA2(torch.rand(8, 2))
