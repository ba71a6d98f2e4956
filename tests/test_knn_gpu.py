"""k nearest neighbours on the GPU (knn.cu, mgs_knn, gaussian_renderer.knn, simple_knn._C.distCUDA2).

1. Against the float64 reference (tests/knn_ref64.py) for k = 1, 3, 20, 32 on uniform, surface (a depth image of the
   scenes.py scene rendered by this package and unprojected, pixels without depth on one point) and cluster-with-outliers
   clouds: the index set wherever the k-th and (k+1)-th float64 distances are more than 1e-5 relative apart, dist2 to 1e-6
   relative, dist2 equal to the fp32 recomputation from the index, rows ascending by (d2, index).
2. Edge cases: N = k + 1, 20k duplicates of one point, distinct queries (some far outside the box), non-finite points and
   queries, no points, fewer valid points than k.
3. c3 size (500k points, k = 20) against cKDTree on a sample of queries; distCUDA2 against the reference.
4. CUDA-graph capture replayed on new point values gives the new answer; a call on a non-current device works.
"""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import knn_ref64 as K64
import util  # noqa: F401  (sys.path)

pytestmark = pytest.mark.gpu


def _surface(W=128, H=128, P=16384, seed=0):
    """ManiGaussian's cloud: the front camera's depth image of the scene unprojected, one point per pixel; pixels without
    depth (alpha < 0.5) land on the camera centre"""
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200 import scenes
    cam = scenes.make_camera(W, H, 0, 4)
    g = scenes.make_gaussians(P, seed=seed)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    s = R.GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], t(np.zeros(3)), 1.0, t(cam["viewmatrix"]),
                                        t(cam["projmatrix"]), g["sh_degree"], t(cam["campos"]), False, False, False)
    outs, _ = R.rasterize_views_raw([s], t(g["means3D"]), None, None, t(g["opacities"]), t(g["scales"]), t(g["rotations"]), 1.0,
                                    None, t(g["shs"]), g["sh_degree"], False, return_depth=True, return_alpha=True)
    torch.cuda.synchronize()
    depth, alpha = (outs[0][i].double().reshape(H, W).cpu().numpy() for i in (7, 8))
    z = np.where(alpha > 0.5, depth / np.maximum(alpha, 1e-12), 0.0)
    fx = W / (2.0 * cam["tanfovx"])
    fy = H / (2.0 * cam["tanfovy"])
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    pc = np.stack([(u - (W - 1) / 2.0) / fx * z, (v - (H - 1) / 2.0) / fy * z, z, np.ones_like(z)], -1).reshape(-1, 4)
    pw = pc @ np.linalg.inv(np.asarray(cam["viewmatrix"], np.float64))
    return pw[:, :3].astype(np.float32)


def _cloud(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.random((n, 3)).astype(np.float32)
    if kind == "surface":
        return _surface()
    # a tight cluster and a few far outliers
    p = rng.normal(0.0, 0.01, (n, 3))
    p[: max(n // 100, 5)] = rng.normal(0.0, 1.0, (max(n // 100, 5), 3)) * 1e3
    return p.astype(np.float32)


def _check(p, k, queries=None, out=None):
    """the kernel's answer against the float64 reference (the rules of the module docstring)"""
    from manigaussian_b200 import gaussian_renderer as GR
    if out is None:
        out = GR.knn(torch.from_numpy(p).cuda(), k, None if queries is None else torch.from_numpy(queries).cuda())
    idx, d2 = out["index"].cpu().numpy(), out["dist2"].cpu().numpy()
    ridx, rd2 = K64.knn_ref64(p, k, queries=queries)
    assert idx.shape == (len(p) if queries is None else len(queries), k) and out["index"].dtype == torch.int64
    assert ((idx == -1) == (ridx[:, :k] == -1)).all(), "padding differs"
    np.testing.assert_allclose(d2, rd2[:, :k], rtol=1e-6, atol=1e-30)
    ok = K64.decided(rd2, k)
    assert ok.mean() > 0.5
    assert (np.sort(idx[ok], 1) == np.sort(ridx[ok, :k], 1)).all()
    # fp32 recomputation from the index, and the (d2, index) order
    q = p if queries is None else queries
    valid = idx >= 0
    re = ((q[:, None, :] - p[np.where(valid, idx, 0)]) ** 2).sum(-1, dtype=np.float32)
    np.testing.assert_allclose(d2[valid], re[valid], rtol=4e-7, atol=0)
    a, b = d2[:, :-1], d2[:, 1:]
    ia, ib = idx[:, :-1], idx[:, 1:]
    assert ((a < b) | ((a == b) & ((ia < ib) | (ib == -1)))).all()
    if queries is None:
        assert (idx != np.arange(len(p))[:, None]).all()
    return idx, d2


@pytest.mark.parametrize("kind", ["uniform", "surface", "outliers"])
@pytest.mark.parametrize("k", [1, 3, 8, 12, 20, 32])  # every list bucket (K = 4, 8, 16, 32), k below and at its size
def test_points_themselves_match_the_reference(kind, k):
    _check(_cloud(kind, 6000, seed=k), k)


@pytest.mark.parametrize("k", [1, 3, 8, 12, 20, 32])
def test_n_is_k_plus_one(k):
    p = np.random.default_rng(k).random((k + 1, 3)).astype(np.float32)
    idx, d2 = _check(p, k)
    for i in range(k + 1):
        assert sorted(idx[i]) == [j for j in range(k + 1) if j != i]


def test_distinct_queries_including_far_outside_the_box():
    rng = np.random.default_rng(7)
    p = _cloud("uniform", 5000, seed=1)
    q = np.concatenate([rng.random((3000, 3)), rng.normal(0.0, 1.0, (200, 3)) * 100.0, [[1e4, -1e4, 3e3]]]).astype(np.float32)
    for k in (1, 3, 5, 8, 12, 16, 20, 32):
        _check(p, k, queries=q)


def test_twenty_thousand_duplicates_of_one_point():
    from manigaussian_b200 import gaussian_renderer as GR
    n, k = 20000, 20
    p = np.tile(np.float32([[0.25, -0.5, 1.0]]), (n, 1))
    out = GR.knn(torch.from_numpy(p).cuda(), k)
    idx, d2 = out["index"].cpu().numpy(), out["dist2"].cpu().numpy()
    assert (d2 == 0).all()
    lowest = np.arange(k + 1)
    for i in (0, 1, 7, 20, 21, 5000, n - 1):
        assert idx[i].tolist() == [j for j in lowest if j != i][:k]
    # the same duplicates inside a surface cloud (its pixels without depth already coincide)
    s = _surface()
    _check(np.concatenate([s, p[:3000]]), k)


def test_non_finite_points_and_queries():
    rng = np.random.default_rng(3)
    p = rng.random((3000, 3)).astype(np.float32)
    p[rng.integers(0, 3000, 200), rng.integers(0, 3, 200)] = np.float32(np.nan)
    p[rng.integers(0, 3000, 50), 1] = np.float32(np.inf)
    q = rng.random((500, 3)).astype(np.float32)
    q[::7, 2] = -np.inf
    q[::11, 0] = np.nan
    for k in (3, 20):
        _check(p, k)
        idx, _ = _check(p, k, queries=q)
        assert (idx[::7] == -1).all() and (idx[::11] == -1).all()


def test_zero_queries_return_empty_outputs():
    from manigaussian_b200 import gaussian_renderer as GR
    out = GR.knn(torch.rand(50, 3, device="cuda"), 4, torch.empty(0, 3, device="cuda"))
    assert out["index"].shape == (0, 4) and out["dist2"].shape == (0, 4)


@pytest.mark.parametrize("kind", ["uniform", "surface", "outliers"])
@pytest.mark.parametrize("k", [3, 20])
def test_start_level_holds_about_max_k_8_points_per_occupied_cell(kind, k):
    """the grid record the call leaves at the start of its state (KnnGrid in knn.cu: lo[3], inv, gmax[3], level, nvalid)
    against the restatement with np.unique cell counts"""
    from manigaussian_b200 import _binding
    p = _cloud(kind, 20000, seed=k)
    L = _binding.lib()
    pt = torch.from_numpy(p).cuda()
    idx = torch.empty((len(p), k), dtype=torch.int64, device="cuda")
    d2 = torch.empty((len(p), k), dtype=torch.float32, device="cuda")
    state = torch.zeros(int(L.mgs_knn_state_bytes(len(p), len(p))), dtype=torch.uint8, device="cuda")
    assert L.mgs_knn(state.data_ptr(), len(p), len(p), k, pt.data_ptr(), None, idx.data_ptr(), d2.data_ptr(), 0,
                     torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    level, nvalid = state[28:36].view(torch.int32).tolist()
    want, mean = K64.start_level(p, k)
    assert nvalid == len(p) and level == want
    target = max(k, 8)
    assert target / 8 ** 0.5 <= mean[level] <= target * 8 ** 0.5


def test_no_points_and_too_few_points_pad():
    from manigaussian_b200 import gaussian_renderer as GR
    q = torch.rand(70, 3, device="cuda")
    out = GR.knn(torch.zeros(0, 3, device="cuda"), 5, q)
    assert (out["index"] == -1).all() and torch.isinf(out["dist2"]).all()
    p = np.random.default_rng(0).random((6, 3)).astype(np.float32)
    p[2] = np.nan
    idx, d2 = _check(p, 8)
    assert (idx[:, 4:] == -1).all() and np.isinf(d2[:, 4:]).all()
    out = GR.knn(torch.zeros(0, 3, device="cuda"), 5)
    assert out["index"].shape == (0, 5)


def test_c3_size_against_ckdtree():
    from manigaussian_b200 import gaussian_renderer as GR
    rng = np.random.default_rng(11)
    n, k = 500_000, 20
    p = (rng.random((n, 3)) * np.float32([1.0, 1.0, 1.0])).astype(np.float32)
    out = GR.knn(torch.from_numpy(p).cuda(), k)
    idx, d2 = out["index"].cpu().numpy(), out["dist2"].cpu().numpy()
    sample = rng.choice(n, 3000, replace=False)
    dt, it = cKDTree(p.astype(np.float64)).query(p[sample].astype(np.float64), k + 2)
    dt, it = dt[:, 1:] ** 2, it[:, 1:]  # drop the point itself (no duplicates in a uniform random cloud)
    np.testing.assert_allclose(d2[sample], dt[:, :k], rtol=1e-6)
    ok = K64.decided(dt, k)
    assert ok.mean() > 0.95
    assert (np.sort(idx[sample][ok], 1) == np.sort(it[ok, :k], 1)).all()


def test_dist_cuda2_matches_the_reference():
    from simple_knn._C import distCUDA2
    for kind in ("uniform", "surface"):
        p = _cloud(kind, 8000, seed=2)
        got = distCUDA2(torch.from_numpy(p).cuda())
        assert got.shape == (len(p),) and got.dtype == torch.float32
        np.testing.assert_allclose(got.cpu().numpy(), K64.dist_cuda2_ref64(p), rtol=2e-6, atol=1e-30)


def test_inputs_that_require_grad_are_detached_and_mixed_devices_are_refused():
    from manigaussian_b200 import gaussian_renderer as GR
    p = torch.rand(100, 3, device="cuda", requires_grad=True)
    out = GR.knn(p, 4)
    assert not out["index"].requires_grad and not out["dist2"].requires_grad
    with pytest.raises(ValueError, match="queries"):
        GR.knn(p, 4, torch.rand(5, 3))


def test_cuda_graph_replay_on_new_point_values():
    from manigaussian_b200 import gaussian_renderer as GR
    rng = np.random.default_rng(5)
    p = torch.from_numpy(_cloud("uniform", 4000, seed=5)).cuda()
    q = torch.from_numpy(rng.random((1000, 3)).astype(np.float32)).cuda()
    GR.knn(p, 20, q)  # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = GR.knn(p, 20, q)
    new = _cloud("outliers", 4000, seed=6)
    p.copy_(torch.from_numpy(new))
    q.copy_(torch.from_numpy(new[:1000] + np.float32(1e-3)))
    graph.replay()
    torch.cuda.synchronize()
    _check(new, 20, queries=new[:1000] + np.float32(1e-3), out=cap)


def test_a_call_on_a_non_current_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import gaussian_renderer as GR
    p = _cloud("uniform", 3000, seed=9)
    d1 = torch.device("cuda:1")
    out = GR.knn(torch.from_numpy(p).to(d1), 8)
    assert out["index"].device == d1
    _check(p, 8, out={k: v for k, v in out.items()})
