"""Farthest-point sampling on the GPU (fps.cu, mgs_fps, gaussian_renderer.farthest_point_sample).

Every result is compared bitwise, index and dist2, with the float32 reference (tests/fps_ref.py).
1. Every tier the host can choose, at a size just below and just above each threshold (2,048 .. 131,072 points, the
   register tiers' cluster sizes 1 .. 16, then the streaming tier), on uniform, surface (the depth image of test_knn_gpu.py,
   unprojected) and cluster-with-far-outliers clouds; and 500k points with n = 1024.
2. Edge cases: 20k duplicates of one point, non-finite points, n above the finite count, start valid, out of range and on a
   non-finite point, P = 0, B = 0 and n = 0.
3. A ragged batch equals separate calls on its slices row by row; repeated calls are bitwise equal; a CUDA graph replayed on
   new point values gives the new answer; a call on a non-current device works.
"""
import functools

import numpy as np
import pytest
import torch

import fps_ref as R
from test_knn_gpu import _surface

pytestmark = pytest.mark.gpu

# one size at and one above each capacity the host chooses from: 512 threads x 4 points x C CTAs (C = 1 .. 8), 512 x 16 x
# C (C = 4, 8, 16), then the streaming tier
THRESHOLDS = [2048, 4096, 8192, 16384, 32768, 65536, 131072]
SIZES = [s + o for s in THRESHOLDS for o in (0, 1)]


@functools.lru_cache(maxsize=None)
def _big_surface(side):
    return _surface(W=side, H=side)


def _cloud(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.random((n, 3)).astype(np.float32)
    if kind == "surface":
        side = 384 if n <= 384 * 384 else 708
        return _big_surface(side)[:n].copy()
    # a tight cluster and a few far outliers
    p = rng.normal(0.0, 0.01, (n, 3))
    p[: max(n // 100, 5)] = rng.normal(0.0, 1.0, (max(n // 100, 5), 3)) * 1e3
    return p.astype(np.float32)


def _fps(p, n, lengths=None, start=None):
    from manigaussian_b200 import gaussian_renderer as GR
    t = lambda x: None if x is None else torch.as_tensor(np.asarray(x), dtype=torch.int64).cuda()  # noqa: E731
    out = GR.farthest_point_sample(torch.from_numpy(np.ascontiguousarray(p)).cuda(), n, t(lengths), t(start))
    return out["index"].cpu().numpy(), out["dist2"].cpu().numpy()


def _same(got, want):
    (gi, gd), (wi, wd) = got, want
    assert gi.shape == wi.shape and gd.shape == wd.shape
    bad = np.flatnonzero((gi != wi).reshape(-1) | (gd.view(np.uint32) != wd.view(np.uint32)).reshape(-1))
    assert bad.size == 0, f"first difference at flat slot {bad[0]}: {gi.reshape(-1)[bad[0]]} / {gd.reshape(-1)[bad[0]]} " \
                          f"against {wi.reshape(-1)[bad[0]]} / {wd.reshape(-1)[bad[0]]}"


def _consequences(idx, d2):
    v = idx[idx >= 0]
    assert len(set(v.tolist())) == len(v)
    assert (idx[len(v):] == -1).all() and np.isinf(d2[len(v):]).all()
    assert np.isinf(d2[0]) and (np.diff(d2[1:len(v)]) <= 0).all()


@pytest.mark.parametrize("kind", ["uniform", "surface", "outliers"])
@pytest.mark.parametrize("P", SIZES)
def test_every_tier_matches_the_reference(kind, P):
    p = _cloud(kind, P, seed=P)
    got = _fps(p, 256)
    _same(got, R.fps_ref_cloud(p, 256))
    _consequences(*got)


@pytest.mark.parametrize("kind", ["uniform", "surface", "outliers"])
def test_c3_size_matches_the_reference(kind):
    p = _cloud(kind, 500_000, seed=1)
    got = _fps(p, 1024)
    _same(got, R.fps_ref_cloud(p, 1024))
    _consequences(*got)


def test_twenty_thousand_duplicates_of_one_point():
    p = np.tile(np.float32([[0.25, -0.5, 1.0]]), (20000, 1))
    idx, d2 = _fps(p, 300)
    assert idx.tolist() == list(range(300))
    assert np.isinf(d2[0]) and (d2[1:] == 0).all()
    # duplicates among distinct points come last, at 0, in ascending index
    q = np.concatenate([np.random.default_rng(2).random((100, 3)).astype(np.float32), p[:50]])
    got = _fps(q, 160)
    _same(got, R.fps_ref_cloud(q, 160))
    assert got[0][101:151].tolist() == list(range(101, 150)) + [-1] and (got[1][101:150] == 0).all()


@pytest.mark.parametrize("P", [3000, 40000, 200000])
def test_non_finite_points_are_never_picked(P):
    rng = np.random.default_rng(3)
    p = rng.random((P, 3)).astype(np.float32)
    p[rng.integers(0, P, P // 15), rng.integers(0, 3, P // 15)] = np.float32(np.nan)
    p[rng.integers(0, P, P // 60), 1] = np.float32(np.inf)
    p[0, 2] = -np.inf
    got = _fps(p, 512)
    _same(got, R.fps_ref_cloud(p, 512))
    assert np.isfinite(p[got[0]]).all()


@pytest.mark.parametrize("P", [100, 20000, 150000])
def test_n_above_the_finite_count_pads(P):
    rng = np.random.default_rng(4)
    p = rng.random((P, 3)).astype(np.float32)
    p[rng.choice(P, P // 10, replace=False), 0] = np.float32(np.nan)
    finite = int(np.isfinite(p).all(1).sum())
    n = finite + 37 if P <= 20000 else 600
    if P > 20000:
        p = p[:600]
        finite = int(np.isfinite(p).all(1).sum())
        p = np.concatenate([p, np.full((P - 600, 3), np.nan, np.float32)])
    got = _fps(p, n)
    _same(got, R.fps_ref_cloud(p, n))
    assert (got[0][finite:] == -1).all() and np.isinf(got[1][finite:]).all()
    assert sorted(got[0][:finite].tolist()) == np.flatnonzero(np.isfinite(p).all(1)).tolist()


@pytest.mark.parametrize("P", [1000, 50000, 140000])
def test_start_valid_out_of_range_and_non_finite(P):
    rng = np.random.default_rng(5)
    p = rng.random((P, 3)).astype(np.float32)
    p[0] = np.nan
    p[17, 1] = np.inf
    for s in (123, P - 1, -1, P, 1 << 40, 17, 0):
        got = _fps(p, 64, start=[s])
        _same(got, R.fps_ref_cloud(p, 64, s))
        assert got[0][0] == (s if s in (123, P - 1) else 1)


def test_ragged_batch_equals_separate_calls_on_the_slices():
    rng = np.random.default_rng(6)
    B, P, n = 32, 10_500, 1024
    pts = rng.random((B, P, 3)).astype(np.float32)
    lengths = rng.integers(9_000, P + 1, B)
    lengths[3], lengths[4], lengths[5] = 0, P + 100, -7
    lengths[6] = 500  # fewer points than picks
    start = rng.integers(0, 9_000, B)
    start[7] = -1
    idx, d2 = _fps(pts, n, lengths, start)
    assert idx.shape == (B, n)
    for b in range(B):
        L = min(max(int(lengths[b]), 0), P)
        row = _fps(pts[b, :L], n, start=[start[b]])
        _same((idx[b], d2[b]), row)
        _same(row, R.fps_ref_cloud(pts[b, :L], n, int(start[b])))
    # a batch of clouds large enough for the streaming tier
    big = np.stack([_cloud("uniform", 140000, seed=s) for s in (1, 2)])
    got = _fps(big, 300, lengths=[140000, 135000], start=[9, 10])
    _same(got, R.fps_ref(big, 300, [140000, 135000], [9, 10]))


def test_repeated_calls_are_bitwise_equal():
    for P in (16384, 300000):
        p = _cloud("outliers", P, seed=8)
        a, b = _fps(p, 512), _fps(p, 512)
        _same(a, b)


def test_shapes_empty_inputs_and_detached_outputs():
    from manigaussian_b200 import gaussian_renderer as GR
    p = torch.rand(3, 100, 3, device="cuda", requires_grad=True)
    out = GR.farthest_point_sample(p, 5)
    assert out["index"].shape == (3, 5) and out["index"].dtype == torch.int64 and out["dist2"].dtype == torch.float32
    assert not out["index"].requires_grad and not out["dist2"].requires_grad
    out = GR.farthest_point_sample(p[0], 5, start=torch.tensor(4, device="cuda"))
    assert out["index"].shape == (5,) and out["index"][0].item() == 4
    out = GR.farthest_point_sample(torch.zeros(2, 0, 3, device="cuda"), 4)  # P = 0: every slot padded
    assert (out["index"] == -1).all() and torch.isinf(out["dist2"]).all()
    assert GR.farthest_point_sample(torch.zeros(0, 10, 3, device="cuda"), 4)["index"].shape == (0, 4)
    assert GR.farthest_point_sample(p, 0)["index"].shape == (3, 0)
    with pytest.raises(ValueError, match="lengths"):
        GR.farthest_point_sample(p, 4, lengths=torch.zeros(3, dtype=torch.int64))


def test_cuda_graph_replay_on_new_point_values():
    from manigaussian_b200 import gaussian_renderer as GR
    for P in (10000, 200000):
        p = torch.from_numpy(_cloud("uniform", P, seed=5)).cuda()
        GR.farthest_point_sample(p, 256)  # warm-up outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cap = GR.farthest_point_sample(p, 256)
        new = _cloud("outliers", P, seed=6)
        p.copy_(torch.from_numpy(new))
        graph.replay()
        torch.cuda.synchronize()
        _same((cap["index"].cpu().numpy(), cap["dist2"].cpu().numpy()), R.fps_ref_cloud(new, 256))


def test_a_call_on_a_non_current_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import gaussian_renderer as GR
    p = _cloud("uniform", 20000, seed=9)
    d1 = torch.device("cuda:1")
    out = GR.farthest_point_sample(torch.from_numpy(p).to(d1), 128)
    assert out["index"].device == d1
    _same((out["index"].cpu().numpy(), out["dist2"].cpu().numpy()), R.fps_ref_cloud(p, 128))
