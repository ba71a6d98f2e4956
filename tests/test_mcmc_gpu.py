"""MCMC density control on the GPU (mcmc.cu, mgs_mcmc_relocate / mgs_mcmc_perturb, gaussian_renderer.mcmc_relocate /
mcmc_perturb), against the numpy restatement in tests/mcmc_ref64.py.

1. Relocation at P = 1, 1k and 1M with 0 %, 10 % and 100 % dead, with and without growth, and with few live Gaussians:
   sources, counts and `source` bitwise; relocated opacity and scale rows within the float32 rounding of the float64
   reference; every other row and moment bitwise unchanged, the moments zero exactly at the sources and destinations; the
   params dict and the optimizer's tensors swapped on growth.
2. A chi-square test of 10^6 draws against w / T; coincident copies render the alpha of their source.
3. Perturbation against the float64 restatement on the same draws, every other input bitwise unchanged.
4. Repeated calls are bitwise equal; a CUDA graph of perturbation and relocation replayed k times equals k eager calls; a
   call on a non-current device works.
"""
import numpy as np
import pytest
import torch

import mcmc_ref64 as R
from manigaussian_b200 import gaussian_renderer as GR

pytestmark = pytest.mark.gpu


def _unambiguous(x):
    """x with every entry nudged until 2^24 sigmoid(x) is not within 1e-6 of an integer: the weight's floor then does not
    depend on the last bit of exp, which the device and numpy may round differently"""
    x = x.copy()
    for _ in range(8):
        f = (1.0 / (1.0 + np.exp(-x.astype(np.float64)))) * 2.0 ** 24
        near = np.abs(f - np.round(f)) < 1e-6
        if not near.any():
            break
        x[near] = np.nextafter(x[near], np.float32(np.inf))
    return x


def _cloud(P, dead, seed, alive=None):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-4.0, 6.0, P).astype(np.float32)
    nd = int(round(dead * P)) if alive is None else P - alive
    dead_idx = rng.permutation(P)[:nd]
    x[dead_idx] = rng.uniform(-12.0, R.dead_threshold(0.005), nd).astype(np.float32)
    if nd:
        x[dead_idx[0]] = R.dead_threshold(0.005)  # exactly at the threshold: dead
    return {"pts_xyz": rng.normal(0, 1, (P, 3)).astype(np.float32),
            "rotations": rng.normal(0, 1, (P, 4)).astype(np.float32),
            "scales": rng.uniform(-6.0, -1.0, (P, 3)).astype(np.float32),
            "opacity": _unambiguous(x),
            "sh": rng.normal(0, 1, (P, 16, 3)).astype(np.float32),
            "feat": rng.normal(0, 1, (P, 5)).astype(np.float32)}  # 5 floats a row: the copy's scalar path


def _to_params(np_params):
    return {k: torch.nn.Parameter(torch.from_numpy(v.copy()).cuda()) for k, v in np_params.items()}


def _adam(params, seed):
    opt = torch.optim.Adam(list(params.values()), lr=1e-3)
    g = torch.Generator(device="cuda").manual_seed(seed)
    for p in params.values():
        opt.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.rand(p.shape, generator=g, device="cuda") + 0.5,
                        "exp_avg_sq": torch.rand(p.shape, generator=g, device="cuda") + 0.5}
    return opt


def _ulps(a, b):
    return np.abs(a.astype(np.float32).view(np.int32).astype(np.int64) - b.astype(np.float32).view(np.int32).astype(np.int64))


CASES = [(P, dead, grow) for P in (1, 1000, 1_000_000) for dead in (0.0, 0.1, 1.0) for grow in (False, True)]


@pytest.mark.parametrize("P,dead,grow,alive", [c + (None,) for c in CASES] + [(1000, None, False, 3), (1000, None, True, 1)])
def test_relocation_matches_the_reference(P, dead, grow, alive):
    seed, offset = 1234 + P, 17
    host = _cloud(P, dead, seed=P, alive=alive)
    params = _to_params(host)
    opt = _adam(params, seed)
    moments0 = {k: {s: v.detach().cpu().numpy() for s, v in opt.state[p].items() if s != "step"} for k, p in params.items()}
    n = P + max(1, P // 20) if grow else None
    Pn = P if n is None else n
    rng = torch.tensor([seed, offset], dtype=torch.int64, device="cuda")
    out = GR.mcmc_relocate(params, optimizer=opt, n=n, rng=rng)
    torch.cuda.synchronize()

    expect = {k: np.concatenate([v, np.zeros((Pn - P,) + v.shape[1:], np.float32)]) for k, v in host.items()}
    expect["opacity"][P:] = R.dead_threshold(0.005)
    want, source, relocated, touched, ref = R.relocate(expect, P, seed, offset)
    assert np.array_equal(out["source"].cpu().numpy(), source)
    assert int(out["relocated"].item()) == relocated
    assert rng.cpu().tolist() == [seed, offset + 1]
    got = {k: v.detach().cpu().numpy() for k, v in params.items()}
    src = ref["src"]
    for k in ("pts_xyz", "rotations", "sh", "feat"):
        assert np.array_equal(got[k], want[k]), k
    # the sources' new opacity and scales: the float64 values rounded once to float32
    assert (_ulps(got["opacity"][src], ref["x64"]) <= 1).all()
    assert (_ulps(got["scales"][src], ref["ls64"]) <= 1).all()
    keep = ~touched
    for k in ("opacity", "scales"):
        assert np.array_equal(got[k][keep], want[k][keep]), k
        j = np.nonzero(source >= 0)[0]
        assert np.array_equal(got[k][j], got[k][source[j]]), k  # every destination a bitwise copy of its source
    # the optimizer holds the params dict's tensors, with moments zero exactly at the sources and destinations
    assert {id(p) for g in opt.param_groups for p in g["params"]} == {id(p) for p in params.values()}
    for k, p in params.items():
        assert tuple(p.shape[:1]) == (Pn,) and p.is_leaf and p.requires_grad
        st = opt.state[p]
        for s, v0 in moments0[k].items():
            v = st[s].cpu().numpy()
            v0 = np.concatenate([v0, np.zeros((Pn - P,) + v0.shape[1:], np.float32)])
            assert np.array_equal(v[keep], v0[keep]), (k, s)
            assert (v[touched] == 0).all(), (k, s)
        assert float(st["step"]) == 3.0


def test_draw_frequencies_follow_the_weights():
    """10^6 appended rows drawn from 1000 live Gaussians: chi-square of the counts against 10^6 w / T"""
    from scipy.stats import chi2
    P_old, D = 1000, 1_000_000
    host = _cloud(P_old, 0.0, seed=5)
    params = _to_params(host)
    rng = torch.tensor([99, 0], dtype=torch.int64, device="cuda")
    out = GR.mcmc_relocate(params, n=P_old + D, rng=rng)
    src = out["source"].cpu().numpy()
    assert (src[:P_old] == -1).all() and int(out["relocated"].item()) == D
    counts = np.bincount(src[P_old:], minlength=P_old)
    w = R.weights(host["opacity"], R.dead_threshold(0.005)).astype(np.float64)
    e = D * w / w.sum()
    stat = ((counts - e) ** 2 / e).sum()
    assert chi2.sf(stat, P_old - 1) > 1e-3, stat
    assert np.array_equal(src, R.draw(np.concatenate([host["opacity"], np.zeros(D, np.float32)]), P_old, P_old + D, 99, 0)[0])


def test_coincident_copies_render_the_alpha_of_their_source():
    """isolated Gaussians, each on the optical axis of its own camera (so its mean projects onto the centre pixel), split
    into n <= 4 copies: the centre pixel's alpha 1 - (1 - o')^n equals the source's o"""
    from manigaussian_b200.cameras import camera_batch
    A, Dd, W = 4, 6, 65
    rng_np = np.random.default_rng(3)
    xs = np.arange(A, dtype=np.float32) * 3.0
    o = rng_np.uniform(0.5, 0.95, A)
    x_alive = np.log(o) - np.log1p(-o)
    host = {"pts_xyz": np.concatenate([np.stack([xs, np.zeros(A), np.full(A, 2.0)], 1), np.tile([-10.0, 0.0, -5.0], (Dd, 1))]),
            "rotations": np.tile([1.0, 0.0, 0.0, 0.0], (A + Dd, 1)),
            "scales": np.log(np.full((A + Dd, 3), 0.3)),
            "opacity": np.concatenate([x_alive, np.full(Dd, -10.0)])}
    host = {k: v.astype(np.float32) for k, v in host.items()}
    host["opacity"] = _unambiguous(host["opacity"])
    seed = next(s for s in range(1000) if R.draw(host["opacity"], A + Dd, A + Dd, s, 0)[1].max() <= 3)
    w2c = torch.eye(4, device="cuda").repeat(A, 1, 1)
    w2c[:, 0, 3] = -torch.from_numpy(xs).cuda()
    K = np.tile(np.array([[64.0, 0, W / 2], [0, 64.0, W / 2], [0, 0, 1]], np.float32), (A, 1, 1))
    cams = camera_batch(w2c, K, W, W)

    def alpha(p):
        q = p["rotations"] / p["rotations"].norm(dim=1, keepdim=True)
        o = GR.render_views(cams, p["pts_xyz"], q, p["scales"].exp(), torch.sigmoid(p["opacity"])[:, None],
                            pts_rgb=torch.ones_like(p["pts_xyz"]), return_alpha=True)
        return o["alpha"][:, W // 2, W // 2].detach().cpu().numpy()

    params = {k: torch.from_numpy(v).cuda() for k, v in host.items()}
    before = alpha(params)
    assert np.allclose(before, 1.0 / (1.0 + np.exp(-host["opacity"][:A].astype(np.float64))), rtol=0, atol=1e-5)
    out = GR.mcmc_relocate(params, rng=torch.tensor([seed, 0], dtype=torch.int64, device="cuda"))
    assert int(out["relocated"].item()) == Dd
    after = alpha(params)
    assert np.abs(after - before).max() <= 1e-5, (before, after)


def _perturb_inputs(P, seed):
    rng = np.random.default_rng(seed)
    return {"pts_xyz": rng.normal(0, 1, (P, 3)).astype(np.float32), "rotations": rng.normal(0, 1, (P, 4)).astype(np.float32),
            "scales": rng.uniform(-5.0, -1.0, (P, 3)).astype(np.float32), "opacity": rng.uniform(-9.0, 2.0, P).astype(np.float32)}


@pytest.mark.parametrize("P", [1, 1000, 100_000])
def test_perturb_matches_the_float64_restatement(P):
    host = _perturb_inputs(P, P)
    t = {k: torch.from_numpy(v.copy()).cuda() for k, v in host.items()}
    scale = torch.tensor([5e5 * 1.6e-4], device="cuda")
    rng = torch.tensor([7, 41], dtype=torch.int64, device="cuda")
    GR.mcmc_perturb(t["pts_xyz"], t["rotations"], t["scales"], t["opacity"], scale, rng)
    got = t["pts_xyz"].cpu().numpy()
    want = R.perturb(host["pts_xyz"], host["rotations"], host["scales"], host["opacity"], float(scale), 7, 41)
    d = np.abs(want - host["pts_xyz"]).max(1, keepdims=True)
    assert (np.abs(got - want) <= 1e-4 * d + 4 * np.spacing(np.abs(host["pts_xyz"]))).all()
    assert (np.abs(got - host["pts_xyz"]) > 0).any() or P == 1
    for k in ("rotations", "scales", "opacity"):
        assert np.array_equal(t[k].cpu().numpy(), host[k]), k
    assert rng.cpu().tolist() == [7, 42]


def test_two_identical_calls_are_bitwise_equal():
    results = []
    for _ in range(2):
        params = _to_params(_cloud(50_000, 0.1, seed=8))
        opt = _adam(params, 8)
        rng = torch.tensor([3, 5], dtype=torch.int64, device="cuda")
        GR.mcmc_perturb(params["pts_xyz"], params["rotations"], params["scales"], params["opacity"], 0.05, rng)
        out = GR.mcmc_relocate(params, optimizer=opt, rng=rng)
        results.append([out["source"].cpu(), out["relocated"].cpu()] + [p.detach().cpu() for p in params.values()] +
                       [opt.state[p]["exp_avg"].cpu() for p in params.values()])
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_a_captured_graph_replayed_k_times_equals_k_eager_calls():
    k, P = 3, 20_000
    host = _cloud(P, 0.1, seed=11)

    def setup():
        params = {n: torch.from_numpy(v.copy()).cuda() for n, v in host.items()}
        return params, torch.tensor([21, 0], dtype=torch.int64, device="cuda"), torch.tensor([0.02], device="cuda")

    def step(params, rng, scale):
        GR.mcmc_perturb(params["pts_xyz"], params["rotations"], params["scales"], params["opacity"], scale, rng)
        # every step kills some Gaussians so that each replay relocates
        params["opacity"][::97] = -20.0
        return GR.mcmc_relocate(params, rng=rng)

    eager, rng_e, scale_e = setup()
    for _ in range(k):
        out_e = step(eager, rng_e, scale_e)
    graphed, rng_g, scale_g = setup()
    warm = {n: v.clone() for n, v in graphed.items()}
    step(warm, rng_g.clone(), scale_g)  # loads the modules and caches the scan's size outside the capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out_g = step(graphed, rng_g, scale_g)
    for _ in range(k):
        g.replay()
    torch.cuda.synchronize()
    assert rng_g.cpu().tolist() == rng_e.cpu().tolist() == [21, 2 * k]
    for n in host:
        assert torch.equal(graphed[n], eager[n]), n
    assert torch.equal(out_g["source"], out_e["source"]) and torch.equal(out_g["relocated"], out_e["relocated"])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_non_current_device():
    host = _cloud(10_000, 0.1, seed=12)
    params = {k: torch.from_numpy(v.copy()).to("cuda:1") for k, v in host.items()}
    rng = torch.tensor([4, 9], dtype=torch.int64, device="cuda:1")
    GR.mcmc_perturb(params["pts_xyz"], params["rotations"], params["scales"], params["opacity"], 0.01, rng)
    out = GR.mcmc_relocate(params, rng=rng)
    torch.cuda.synchronize(1)
    assert rng.cpu().tolist() == [4, 11]
    want = R.draw(host["opacity"], 10_000, 10_000, 4, 10)[0]
    assert np.array_equal(out["source"].cpu().numpy(), want)
