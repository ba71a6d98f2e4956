"""Default density control on the GPU (densify.cu, mgs_densify_stats / _count / _emit, gaussian_renderer.densify_stats /
densify_and_prune / densify_reset_opacity), against the numpy restatement in tests/densify_ref64.py.

1. Statistics bitwise equal to the float32 restatement at P = 1, 1k and 1M with V = 1, 4 and 8 and some radii <= 0, from
   random gradients and from real render_views / render backwards; a CUDA-graph replay equals the eager calls.
2. Refinement: source, counts and order, every copied row and moment, the children's log scales and the zero moments
   bitwise; the children's means within float32 rounding of the float64 values from the same uniforms; SH and feature
   rows travel, the optimizer holds the new tensors and steps on them; repeatability and the generator's offset; nothing
   to do, everything pruned and an empty cloud.
3. The views split over two simulated ranks, the statistics reduced as INTEGRATION.md §24 documents: the same refinement.
"""
import math

import numpy as np
import pytest
import torch

import densify_ref64 as D
from manigaussian_b200 import gaussian_renderer as GR

pytestmark = pytest.mark.gpu


def _stats_inputs(V, P, seed):
    rng = np.random.default_rng(seed)
    g = rng.normal(0, 1e-3, (V, P, 3)).astype(np.float32)
    radii = rng.integers(-2, 40, (V, P)).astype(np.int32)
    radii[rng.random((V, P)) < 0.3] = 0
    sizes = [int(s) for s in rng.integers(64, 1024, V)]
    start = (rng.uniform(0, 1e-2, P).astype(np.float32), rng.integers(0, 9, P).astype(np.int32),
             rng.uniform(0, 0.1, P).astype(np.float32))
    return g, radii, sizes, start


def _dev_stats(start):
    return {k: torch.from_numpy(v.copy()).cuda() for k, v in zip(("grad2d", "count", "radius"), start)}


def _host(stats):
    return tuple(stats[k].cpu().numpy() for k in ("grad2d", "count", "radius"))


def _bitwise(a, b):
    return all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(a, b))


@pytest.mark.parametrize("P", [1, 1000, 1_000_000])
@pytest.mark.parametrize("V", [1, 4, 8])
def test_stats_are_bitwise_equal_to_the_restatement(P, V):
    g, radii, sizes, start = _stats_inputs(V, P, P + V)
    stats = _dev_stats(start)
    GR.densify_stats(stats, torch.from_numpy(g).cuda(), torch.from_numpy(radii).cuda(), sizes, scale=float(V))
    want = D.stats(*start, g, radii, sizes, scale=float(V))
    assert _bitwise(_host(stats), want)
    # a second step with the scale on the device, and a [P,3] call for one view
    GR.densify_stats(stats, torch.from_numpy(g).cuda(), torch.from_numpy(radii).cuda(), sizes,
                     scale=torch.tensor([0.5], device="cuda"))
    want = D.stats(*want, g, radii, sizes, scale=0.5)
    assert _bitwise(_host(stats), want)
    GR.densify_stats(stats, torch.from_numpy(g[0]).cuda(), torch.from_numpy(radii[0]).cuda(), sizes[0])
    assert _bitwise(_host(stats), D.stats(*want, g[0], radii[0], sizes[:1]))


def _scene(P, seed):
    rng = np.random.default_rng(seed)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    xyz = np.concatenate([rng.uniform(-0.6, 0.6, (P, 2)), rng.uniform(1.5, 2.5, (P, 1))], 1)
    xyz[rng.random(P) < 0.1, 2] = -1.0  # behind every camera: radius 0
    q = rng.normal(0, 1, (P, 4))
    return {"pts_xyz": t(xyz), "rotations": t(q / np.linalg.norm(q, axis=1, keepdims=True)),
            "scales": t(rng.uniform(-5.0, -3.0, (P, 3))), "opacity": t(rng.uniform(-2.0, 3.0, (P, 1))),
            "rgb": t(rng.uniform(0, 1, (P, 3)))}


def _cameras(V, W=96, H=80):
    from manigaussian_b200.cameras import camera_batch
    w2c = torch.eye(4, device="cuda").repeat(V, 1, 1)
    for v in range(V):
        w2c[v, 0, 3] = 0.15 * math.cos(2 * math.pi * v / V)
        w2c[v, 1, 3] = 0.15 * math.sin(2 * math.pi * v / V)
    K = np.tile(np.array([[70.0, 0, W / 2], [0, 70.0, H / 2], [0, 0, 1]], np.float32), (V, 1, 1))
    return camera_batch(w2c, K, W, H)


def _render_grads(cams, s, seed):
    p = {k: v.clone().requires_grad_(True) for k, v in s.items()}
    out = GR.render_views(cams, p["pts_xyz"], p["rotations"], torch.exp(p["scales"]), torch.sigmoid(p["opacity"]),
                          pts_rgb=p["rgb"])
    gen = torch.Generator(device="cuda").manual_seed(seed)
    (out["render"] * torch.randn(out["render"].shape, generator=gen, device="cuda")).mean().backward()
    return out["viewspace_points"].grad, out["radii"]


@pytest.mark.parametrize("V", [1, 4, 8])
def test_stats_from_a_real_render_views_backward(V):
    P = 20_000
    cams = _cameras(V)
    grad, radii = _render_grads(cams, _scene(P, V), V)
    assert grad.shape == (V, P, 3) and radii.dtype == torch.int32
    r = radii.cpu().numpy()
    assert (r > 0).any() and (r == 0).any()
    stats = GR.densify_state(P, "cuda")
    GR.densify_stats(stats, grad, radii, cams, scale=float(V))
    want = D.stats(*(np.zeros(P, np.float32), np.zeros(P, np.int32), np.zeros(P, np.float32)), grad.cpu().numpy(), r,
                   [96] * V, scale=float(V))
    assert _bitwise(_host(stats), want)
    assert (want[0] > 0).any()


def test_stats_from_render():
    P = 20_000
    cams = _cameras(3)
    s = _scene(P, 5)
    p = {k: v.clone().requires_grad_(True) for k, v in s.items()}
    out = GR.render({"novel_view": cams.as_novel_view()}, 1, p["pts_xyz"], p["rotations"], torch.exp(p["scales"]),
                    torch.sigmoid(p["opacity"]), [0, 0, 0], pts_rgb=p["rgb"])
    out["render"].square().mean().backward()
    grad, radii = out["viewspace_points"].grad, out["radii"]
    assert grad.shape == (P, 3)
    stats = GR.densify_state(P, "cuda")
    GR.densify_stats(stats, grad, radii, [cams.settings(1, torch.zeros(3, device="cuda"), 0, False)])
    want = D.stats(np.zeros(P, np.float32), np.zeros(P, np.int32), np.zeros(P, np.float32), grad.cpu().numpy(),
                   radii.cpu().numpy(), [96])
    assert _bitwise(_host(stats), want) and (want[1] > 0).any()


def test_a_captured_stats_graph_replayed_k_times_equals_k_eager_calls():
    k, V, P = 3, 4, 50_000
    g, radii, sizes, start = _stats_inputs(V, P, 3)
    gd, rd = torch.from_numpy(g).cuda(), torch.from_numpy(radii).cuda()
    scale = torch.tensor([4.0], device="cuda")
    eager, graphed = _dev_stats(start), _dev_stats(start)
    for _ in range(k):
        GR.densify_stats(eager, gd, rd, sizes, scale)
    GR.densify_stats(_dev_stats(start), gd, rd, sizes, scale)  # loads the module outside the capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        GR.densify_stats(graphed, gd, rd, sizes, scale)
    for _ in range(k):
        graph.replay()
    torch.cuda.synchronize()
    assert _bitwise(_host(graphed), _host(eager))


# --------------------------------------------------------------------------- refinement
def _cloud(P, seed, nan_rows=True):
    rng = np.random.default_rng(seed)
    p = {"pts_xyz": rng.normal(0, 1, (P, 3)), "rotations": rng.normal(0, 1, (P, 4)),
         "scales": rng.uniform(-7.0, -1.0, (P, 3)), "opacity": rng.uniform(-8.0, 4.0, (P, 1)),
         "sh": rng.normal(0, 1, (P, 16, 3)), "feat": rng.normal(0, 1, (P, 32)), "tag": rng.normal(0, 1, (P, 5))}
    p = {k: v.astype(np.float32) for k, v in p.items()}
    count = rng.integers(0, 5, P).astype(np.int32)
    grad2d = (rng.uniform(0, 4e-4, P) * np.maximum(count, 1)).astype(np.float32)
    radius = rng.uniform(0, 0.2, P).astype(np.float32)
    if nan_rows and P >= 10:
        p["scales"][3, 0] = np.nan
        p["scales"][5] = np.nan
        p["opacity"][7] = np.nan
    return p, (grad2d, count, radius)


def _to_device(host, st):
    params = {k: torch.nn.Parameter(torch.from_numpy(v.copy()).cuda()) for k, v in host.items()}
    stats = {k: torch.from_numpy(v.copy()).cuda() for k, v in zip(("grad2d", "count", "radius"), st)}
    return params, stats


def _adam(params, seed):
    opt = torch.optim.Adam(list(params.values()), lr=1e-3)
    g = torch.Generator(device="cuda").manual_seed(seed)
    for p in params.values():
        opt.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.rand(p.shape, generator=g, device="cuda") + 0.5,
                        "exp_avg_sq": torch.rand(p.shape, generator=g, device="cuda") + 0.5}
    return opt


RULES = [dict(scene_scale=1.0, grow_scale2d=0.15),
         dict(scene_scale=0.5, grow_scale2d=0.1, prune_too_big=True, prune_scale2d=0.18, grad_threshold=1e-4)]


@pytest.mark.parametrize("P", [1, 1000, 1_000_000])
@pytest.mark.parametrize("rule", RULES)
def test_refinement_matches_the_reference(P, rule):
    seed, offset = 40 + P, 11
    host, st = _cloud(P, P)
    if P == 1:
        st = (np.array([1e-3], np.float32), np.array([1], np.int32), np.array([0.5], np.float32))
        host["opacity"][:] = 2.0
    params, stats = _to_device(host, st)
    opt = _adam(params, seed)
    moments0 = {k: [opt.state[p][s].cpu().numpy() for s in ("exp_avg", "exp_avg_sq")] for k, p in params.items()}
    rng = torch.tensor([seed, offset], dtype=torch.int64, device="cuda")
    out = GR.densify_and_prune(params, stats, opt, rng=rng, **rule)
    torch.cuda.synchronize()

    want, want_m, source, counts, ex = D.refine(host, moments0, *st, seed, offset, **rule)
    assert tuple(out["counts"].values()) == counts and list(out["counts"]) == ["n_new", "cloned", "split", "pruned"]
    assert counts[1] + counts[2] > 0
    assert np.array_equal(out["source"].cpu().numpy(), source)
    assert rng.cpu().tolist() == [seed, offset + 1]
    got = {k: v.detach().cpu().numpy() for k, v in params.items()}
    ch = ex["children"]
    for k in host:
        assert got[k].shape == want[k].shape, k
        if k != "pts_xyz":
            assert np.array_equal(got[k].view(np.int32), want[k].view(np.int32)), k  # copies and children's log scales
    assert np.array_equal(got["pts_xyz"][:ch.start], want["pts_xyz"][:ch.start])
    mu = np.tile(host["pts_xyz"][source[ch][: (ch.stop - ch.start) // 2]], (2, 1)).astype(np.float64)
    fin = np.isfinite(ex["mean64"]).all(1)  # a NaN log scale gives NaN children
    assert np.array_equal(np.isfinite(got["pts_xyz"][ch]).all(1), fin)
    m64, mu, gm = ex["mean64"][fin], mu[fin], got["pts_xyz"][ch][fin]
    d = np.abs(m64 - mu).max(1, keepdims=True)
    assert (np.abs(gm - m64) <= 1e-4 * d + 4 * np.spacing(np.abs(mu).astype(np.float32))).all()
    # the optimizer holds the params dict's new tensors; kept originals keep their moments, new rows are zero
    assert {id(p) for g in opt.param_groups for p in g["params"]} == {id(p) for p in params.values()}
    for k, p in params.items():
        assert p.is_leaf and p.requires_grad and isinstance(p, torch.nn.Parameter)
        for s, w in zip(("exp_avg", "exp_avg_sq"), want_m[k]):
            assert np.array_equal(opt.state[p][s].cpu().numpy(), w), (k, s)
        assert float(opt.state[p]["step"]) == 3.0
    # fresh zero statistics of the new length
    for k, t in stats.items():
        assert t.shape == (counts[0],) and not t.any(), k


def test_repeatable_and_the_optimizer_steps_on_the_new_tensors():
    results = []
    for _ in range(2):
        host, st = _cloud(100_000, 3, nan_rows=False)  # NaN children would not compare equal
        params, stats = _to_device(host, st)
        opt = _adam(params, 3)
        rng = torch.tensor([9, 2], dtype=torch.int64, device="cuda")
        out = GR.densify_and_prune(params, stats, opt, scene_scale=1.0, grow_scale2d=0.15, rng=rng)
        assert rng.cpu().tolist() == [9, 3]
        results.append([out["source"].cpu()] + [p.detach().cpu() for p in params.values()] +
                       [opt.state[p][s].cpu() for p in params.values() for s in ("exp_avg", "exp_avg_sq")])
    for a, b in zip(*results):
        assert torch.equal(a, b)
    n = out["counts"]["n_new"]
    before = {k: p.detach().clone() for k, p in params.items()}
    for p in params.values():
        p.grad = torch.ones_like(p)
    opt.step()
    for k, p in params.items():
        assert p.shape[0] == n and not torch.equal(p.detach(), before[k]), k
        assert opt.state[p]["exp_avg"].shape == p.shape


def test_nothing_to_do_everything_pruned_and_an_empty_cloud():
    host, st = _cloud(5000, 4, nan_rows=False)
    host["opacity"][:] = 1.0
    params, stats = _to_device(host, (np.zeros_like(st[0]), st[1], st[2]))
    opt = _adam(params, 4)
    ids = {k: id(p) for k, p in params.items()}
    rng = torch.tensor([1, 0], dtype=torch.int64, device="cuda")
    out = GR.densify_and_prune(params, stats, opt, scene_scale=1.0, rng=rng)
    assert out["counts"] == {"n_new": 5000, "cloned": 0, "split": 0, "pruned": 0}
    assert {k: id(p) for k, p in params.items()} == ids and rng.cpu().tolist() == [1, 1]
    assert torch.equal(out["source"].cpu(), torch.arange(5000)) and not stats["radius"].any()
    # everything pruned
    params["opacity"].data.fill_(-20.0)
    stats["grad2d"].fill_(1.0)
    out = GR.densify_and_prune(params, stats, opt, scene_scale=1.0, rng=rng)
    assert out["counts"]["n_new"] == 0 and out["counts"]["pruned"] == 5000 + out["counts"]["split"] + out["counts"]["cloned"]
    assert all(p.shape[0] == 0 for p in params.values()) and out["source"].shape == (0,) and rng.cpu().tolist() == [1, 2]
    assert all(opt.state[p]["exp_avg"].shape[0] == 0 for p in params.values())
    # and the empty cloud
    out = GR.densify_and_prune(params, stats, opt, scene_scale=1.0, rng=rng)
    assert out["counts"] == {"n_new": 0, "cloned": 0, "split": 0, "pruned": 0}


def test_two_ranks_that_reduce_their_statistics_make_the_same_refinement():
    V, P = 8, 30_000
    cams = _cameras(V)
    s = _scene(P, 12)
    grad, radii = _render_grads(cams, s, 12)
    one = GR.densify_state(P, "cuda")
    GR.densify_stats(one, grad, radii, cams, scale=float(V))
    ranks = []
    for views in (slice(0, 4), slice(4, 8)):
        st = GR.densify_state(P, "cuda")
        GR.densify_stats(st, grad[views], radii[views], [96] * 4, scale=float(V))
        ranks.append(st)
    reduced = {"grad2d": ranks[0]["grad2d"] + ranks[1]["grad2d"], "count": ranks[0]["count"] + ranks[1]["count"],
               "radius": torch.maximum(ranks[0]["radius"], ranks[1]["radius"])}
    assert torch.equal(reduced["count"], one["count"]) and torch.equal(reduced["radius"], one["radius"])
    # a threshold half way between two neighbouring per-Gaussian means, so the ranks' differently ordered sums (last-bit
    # differences) cannot fall on either side of it
    seen = one["count"] > 0
    r = torch.sort(one["grad2d"][seen] / one["count"][seen].float()).values
    k = int(0.8 * r.numel())
    threshold = float(0.5 * (r[k] + r[k + 1]))
    outs = []
    for stats in (one, reduced):
        params = {k: v.clone() for k, v in s.items()}
        out = GR.densify_and_prune(params, stats, scene_scale=1.0, grad_threshold=threshold,
                                   rng=torch.tensor([5, 0], dtype=torch.int64, device="cuda"))
        outs.append((out, params))
    (a, pa), (b, pb) = outs
    assert a["counts"] == b["counts"] and a["counts"]["cloned"] + a["counts"]["split"] > 0
    assert torch.equal(a["source"], b["source"])
    for k in pa:
        assert torch.equal(pa[k], pb[k]), k


def test_reset_opacity_on_the_device():
    params, _ = _to_device(*_cloud(10_000, 6, nan_rows=False))
    opt = _adam(params, 6)
    x0 = params["opacity"].detach().clone()
    GR.densify_reset_opacity(params, opt, value=0.01)
    t = float(np.float32(math.log(0.01 / 0.99)))
    assert torch.equal(params["opacity"].detach(), torch.clamp(x0, max=t))
    assert not opt.state[params["opacity"]]["exp_avg"].any() and opt.state[params["sh"]]["exp_avg"].all()
