"""The bounded float64 visibility reference (visibility_ref64.bounded) proves itself without a GPU.

* With the decisions it takes, its T equals visibility_grad_ref64's screen-space transmittance, and its duv and blend-stage
  rows gb equal that function's torch float64 autograd gradients (gb in the blend backward's units: W/2 and H/2 on the
  mean, the half-weight b slot), to 1e-12 of each array's scale, on a synthetic view built for the edges and on the golden
  scenes' oracle states.
* The fp32 decision replay: the tile at u = 15.5 and one ulp either side, at -0.5 and at W - 0.5 - ulp (where u + 0.5f
  stays below W, except in a one-pixel view where it rounds to W and the clamp keeps column 0); the cut at d equal to a list depth and one ulp either side, and over a
  run of equal depths.
* Its bounds are tight enough to matter: each mutation in visibility_ref64.MUTATIONS moves a checked element of T, duv or
  gb past twice its bound.
"""
import os

import numpy as np
import pytest
import torch

import blend_ref64 as R64
import visibility_grad_ref64 as VG
import visibility_ref64 as V64
from test_blend_ref64_cpu import GOLDEN, _golden, oracle_state

f32 = np.float32
D64 = torch.float64


def _conics(rng, P, lo, hi):
    s = rng.uniform(lo, hi, (P, 2))
    th = rng.uniform(0, np.pi, P)
    c, n = np.cos(th), np.sin(th)
    a = c * c * s[:, 0] ** 2 + n * n * s[:, 1] ** 2 + 0.3
    b = c * n * (s[:, 0] ** 2 - s[:, 1] ** 2)
    d = n * n * s[:, 0] ** 2 + c * c * s[:, 1] ** 2 + 0.3
    det = a * d - b * b
    return np.stack([d / det, -b / det, a / det], 1)


def synthetic(seed=0, W=48, H=40, P=400, Q=900):
    """A view whose tiles list the Gaussians near them in (fp32 depth, id) order, and points at the edges: on the tile seams
    and one ulp either side, at -0.5 and W - 0.5 - ulp, at Gaussian centres with d equal to that Gaussian's depth and one
    ulp either side, behind opaque stacks that reach the stop; opacities at 1/255 and a few ulps above, and under the 0.99
    clamp; runs of equal depths."""
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-4, [W + 4, H + 4], (P, 2)).astype(f32)
    co = np.concatenate([_conics(rng, P, 1.5, 8.0), rng.uniform(0.05, 0.98, (P, 1))], 1).astype(f32)
    a255 = f32(1) / f32(255)
    co[:6, 3] = [a255, np.nextafter(a255, f32(1)), a255 * f32(1.0000003), 0.995, 0.9999, 1.0]
    co[6:60, 3] = rng.uniform(0.9, 1.0, 54)                   # opaque stacks reach the stop
    co[60:90, :3] = _conics(rng, 30, 20.0, 30.0)              # wide and faint: alpha near 1/255 far from the centre
    co[60:90, 3] = a255 * rng.uniform(1.0, 3.0, 30)
    dep = rng.uniform(1.0, 5.0, P).astype(f32)
    dep[100:110] = dep[100]                                   # a run of equal depths
    st = dict(W=W, H=H, means2D=mu, conic_opacity=co, depths=dep)
    uv = rng.uniform(-0.5, [W - 0.5, H - 0.5], (Q, 2)).astype(f32)
    d = rng.uniform(0.5, 6.0, Q).astype(f32)
    seam = [f32(15.5), np.nextafter(f32(15.5), f32(0)), np.nextafter(f32(15.5), f32(99)), f32(31.5), f32(-0.5),
            np.nextafter(f32(W - 0.5), f32(0))]
    uv[:6, 0] = seam
    uv[6:12, 1] = seam[:5] + [np.nextafter(f32(H - 0.5), f32(0))]
    g = rng.choice(np.arange(60), 60, replace=False)
    uv[12:72] = mu[g] + rng.normal(0, 0.5, (60, 2)).astype(f32)
    d[12:72] = dep[g]
    d[72:132] = np.nextafter(dep[g], f32(0))
    d[132:192] = np.nextafter(dep[g], f32(9))
    uv[72:192] = np.concatenate([uv[12:72], uv[12:72]])
    d[192:200] = dep[100]
    d[200:400] = 9.0                                          # behind everything
    mu[:6] = rng.uniform(2.0, [W - 2.0, H - 2.0], (6, 2)).astype(f32)
    uv[200:206] = mu[:6]                                      # alpha = o exactly: at 1/255 the pair is either-side
    uv = np.clip(uv, -0.5, np.nextafter(f32([W - 0.5, H - 0.5]), f32(0))).astype(f32)
    # each tile lists the Gaussians whose centre lies within 10 px of it, in (fp32 depth, id) order
    gx, gy = (W + 15) // 16, (H + 15) // 16
    order = np.lexsort((np.arange(P), dep))
    lists = []
    for t in range(gx * gy):
        x0, y0 = 16 * (t % gx), 16 * (t // gx)
        near = (mu[order, 0] > x0 - 10) & (mu[order, 0] < x0 + 26) & (mu[order, 1] > y0 - 10) & (mu[order, 1] < y0 + 26)
        lists.append(order[near])
    ends = np.cumsum([len(x) for x in lists])
    st["point_list"] = np.concatenate(lists).astype(np.uint32)
    st["ranges"] = np.stack([ends - [len(x) for x in lists], ends], 1).astype(np.uint32)
    gT = rng.standard_normal(Q).astype(f32)
    gT[::7] = 0.0
    return st, uv, d, np.ones(Q, bool), gT


def _golden_case(path):
    _, inp, fw, _ = _golden(path)
    st = dict(oracle_state(inp, fw), depths=np.asarray(fw["depths"], f32))
    W, H = inp["W"], inp["H"]
    rng = np.random.default_rng(3)
    Q = 800
    uv = rng.uniform(-0.5, [W - 0.5, H - 0.5], (Q, 2)).astype(f32)
    fin = np.asarray(st["depths"])[np.isfinite(st["depths"])]
    d = rng.uniform(fin.min() * 0.9, fin.max() * 1.1, Q).astype(f32)
    return st, uv, d, np.ones(Q, bool), rng.standard_normal(Q).astype(f32)


def _autograd(st, uv, acc, gT):
    """T, dL/duv and dL/d(mean, conic, opacity) of L = sum g_T T with the decisions `acc`"""
    uvl = torch.tensor(uv.astype(np.float64), requires_grad=True)
    mu = torch.tensor(np.asarray(st["means2D"], np.float64), requires_grad=True)
    co = np.asarray(st["conic_opacity"], np.float64)
    conic = torch.tensor(co[:, :3], requires_grad=True)
    op = torch.tensor(co[:, 3], requires_grad=True)
    T = VG.screen_transmittance(uvl, mu, conic, op, acc)
    (T * torch.tensor(gT.astype(np.float64))).sum().backward()
    return T.detach().numpy(), uvl.grad.numpy(), mu.grad.numpy(), conic.grad.numpy(), op.grad.numpy()


def _close(a, b, tag):
    scale = max(float(np.abs(b).max()), 1e-300)
    err = float(np.abs(a - b).max()) / scale
    assert err <= 1e-12, (tag, err)


CASES = ["synthetic0", "synthetic1"] + [os.path.basename(p)[:-4] for p in GOLDEN]


def _case(name):
    if name.startswith("synthetic"):
        return synthetic(seed=int(name[-1]))
    return _golden_case(next(p for p in GOLDEN if os.path.basename(p)[:-4] == name))


@pytest.mark.parametrize("name", CASES)
def test_bounded_equals_the_autograd_reference_with_the_same_decisions(name):
    st, uv, d, inside, gT = _case(name)
    ref = V64.bounded(st, uv, d, inside, gT)
    T, duv, dmu, dconic, dop = _autograd(st, uv, ref["accepted"], gT)
    W, H = st["W"], st["H"]
    _close(ref["T"][0], T, "T")
    _close(ref["duv"][0], duv, "duv")
    gb = ref["gb"][0]
    for i, want in enumerate((0.5 * W * dmu[:, 0], 0.5 * H * dmu[:, 1], dconic[:, 0], 0.5 * dconic[:, 1], dconic[:, 2], dop)):
        _close(gb[:, i], want, ("gb", i))
    assert ref["checked"] == inside.sum() and ref["pairs"] > 0
    assert (ref["T"][0] < 0.5).any() and (ref["T"][0] == 1).any()
    if name.startswith("synthetic"):
        # the scene reaches the edges it is built for
        assert (ref["T"][0] < 2 * R64.T_STOP).any()
        assert ref["either"] > 0


def test_the_tile_is_replayed_in_fp32():
    W, H = 48, 40
    ulp = lambda x, to: np.nextafter(f32(x), f32(to))  # noqa: E731
    u = np.array([15.5, ulp(15.5, 0), ulp(15.5, 99), -0.5, ulp(W - 0.5, 0), ulp(31.5, 0), 31.5], f32)
    uv = np.stack([u, np.full_like(u, ulp(H - 0.5, 0))], 1)
    row = 2 * 3                                               # the last tile row of a 48 x 40 view
    assert (V64.tile_of32(uv, W, H) - row).tolist() == [1, 0, 1, 0, 2, 1, 2]
    assert (V64.tile_of32(uv, W, H, mutate={"tile_floor_u"}) - row).tolist()[:3] == [0, 0, 0]
    # at W - 0.5 - ulp, u + 0.5f stays below W when W - 0.5 and W share a binade; in a one-pixel view it rounds to W = 1,
    # and the clamp keeps the pixel in column 0
    assert f32(u[4]) + f32(0.5) < f32(W)
    half = ulp(0.5, 0)
    assert half + f32(0.5) == f32(1.0) and np.float64(half) + 0.5 < 1.0
    assert V64.tile_of32(np.array([[half, half]], f32), 1, 1).tolist() == [0]


def test_the_cut_is_replayed_in_fp32():
    dep = np.array([1.0, 2.0, 2.0, 2.0, 3.0, 4.0], f32)
    st = dict(depths=dep, point_list=np.arange(6, dtype=np.uint32), ranges=np.array([[0, 6]], np.uint32))
    two = f32(2.0)
    d = np.array([two, np.nextafter(two, f32(0)), np.nextafter(two, f32(9)), f32(0.5), f32(9.0), f32(4.0)], f32)
    _, cut = V64.cut_of(st, np.zeros(len(d), np.int64), d)
    assert cut.tolist() == [1, 1, 4, 0, 6, 5]
    _, le = V64.cut_of(st, np.zeros(len(d), np.int64), d, mutate={"cut_le"})
    assert le.tolist() == [4, 1, 4, 0, 6, 6]


@pytest.mark.parametrize("mutation", V64.MUTATIONS)
def test_each_mutation_moves_a_checked_element_past_twice_its_bound(mutation):
    worst = 0.0
    for seed in (0, 1):
        st, uv, d, inside, gT = synthetic(seed)
        ref = V64.bounded(st, uv, d, inside, gT)
        mut = V64.bounded(st, uv, d, inside, gT, T_out=ref["T"][0], mutate={mutation})
        for q in ("T", "duv", "gb"):
            worst = max(worst, float(V64.ratio(mut[q][0], ref[q], q).max()))
    assert worst > 2.0, (mutation, worst)
