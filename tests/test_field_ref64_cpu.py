"""The bounded float64 field reference (field_ref64.bounded) proves itself without a GPU.

* Its values equal field_ref64.field, and its gradients that function's torch float64 autograd gradients, to 1e-12
  relative, on random clouds, flat Gaussians (1e-4 next to 0.05), quaternions with |q| from 0.05 to 20, Gaussians without
  support (o at and below 1/255, zero, negative and non-finite scales, a non-finite mean), non-finite points, and points on
  the support edge.
* A float32 evaluation of the density in the kernel's operation order lands within the bound.
* Its bounds are tight enough to matter: each mutation in field_ref64.MUTATIONS moves a checked element past twice its
  KAPPA bound, except `no_box_slack`, which changes no value (it only guards pairs inside the either-side band) and is shown
  to leave such a pair outside the support box instead.
"""
import numpy as np
import pytest
import torch

import field_ref64 as F64

f32 = np.float32
T255 = F64.THRESH


def _f(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=f32))


def _cloud(P, C, seed, spread=0.3, qnorm=(0.5, 2.0)):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(P, 4))
    q *= (rng.uniform(*qnorm, (P, 1)) / np.linalg.norm(q, axis=1, keepdims=True))
    cl = dict(means=_f(rng.uniform(-spread, spread, (P, 3))), scales=_f(rng.uniform(0.03, 0.15, (P, 3))), rot=_f(q),
              opac=_f(rng.uniform(0.05, 0.99, P)), feat=_f(rng.normal(0, 1, (P, C))) if C else None)
    return cl


def _special(cl):
    """Gaussians without support, flat Gaussians and a needle in place of the first ones"""
    m, s, r, o = cl["means"], cl["scales"], cl["rot"], cl["opac"]
    o[0] = T255
    o[1] = 0.002
    s[2, 1] = 0.0
    s[3, 0] = -0.01
    s[4, 2] = float("inf")
    m[5, 1] = float("nan")
    o[6] = float("nan")
    s[7:12] = torch.tensor([0.05, 0.04, 1e-4])
    o[7:12] = 0.9
    s[12] = torch.tensor([0.05, 5e-6, 5e-6])
    o[12] = 0.8
    return cl


def _points(cl, Q, seed, spread=0.35):
    rng = np.random.default_rng(seed)
    x = _f(rng.uniform(-spread, spread, (Q, 3)))
    near = cl["means"][13:13 + Q // 4] + _f(rng.normal(0, 0.02, (min(Q // 4, cl["means"].shape[0] - 13), 3)))
    x[:near.shape[0]] = near
    return x


def _edge_points(cl, ids, outside=False):
    """one point per Gaussian id on its support edge along its first frame axis (m = cut, rounded to fp32), slightly
    outside it with `outside`"""
    R = F64.rotation_rows(cl["rot"].double())
    cut = 2.0 * torch.log(255.0 * cl["opac"].double())
    pts = []
    for i in ids:
        k = 1.0 + 3e-7 if outside else 1.0
        pts.append(cl["means"][i].double() + k * torch.sqrt(cut[i]) * cl["scales"][i, 0].double() * R[i, 0])
    return torch.stack(pts).float()


def _box_extremes(cl, ids, k=1.0 + 5e-7):
    """per Gaussian id the support's extreme points along each world axis, pushed out by k: there the support touches its
    axis-aligned box, so these pairs lie outside the exact box and inside the either-side band"""
    R = F64.rotation_rows(cl["rot"].double())
    S = R.transpose(1, 2) @ (cl["scales"].double()[:, :, None] ** 2 * R)
    cut = 2.0 * torch.log(255.0 * cl["opac"].double())
    pts = [cl["means"][i].double() + k * torch.sqrt(cut[i]) * S[i, :, j] / torch.sqrt(S[i, j, j]) for i in ids for j in range(3)]
    return torch.stack(pts).float()


def _autograd(x, cl, gd, gf):
    leaves = [t.double().requires_grad_(True) for t in (x, cl["means"], cl["scales"], cl["rot"], cl["opac"])]
    fe = cl["feat"].double().requires_grad_(True) if cl["feat"] is not None else None
    fin = torch.isfinite(leaves[0].detach()).all(1)
    xs = torch.where(fin[:, None], leaves[0], torch.zeros_like(leaves[0]))
    d, f = F64.field(xs, *leaves[1:], fe)
    d = torch.where(fin, d, torch.zeros_like(d))
    loss = (d * gd.double()).sum()
    if f is not None:
        f = torch.where(fin[:, None], f, torch.zeros_like(f))
        loss = loss + (f * gf.double()).sum()
    loss.backward()
    g = dict(points=leaves[0].grad, means=leaves[1].grad, scales=leaves[2].grad, rot=leaves[3].grad, opacity=leaves[4].grad)
    if fe is not None:
        g["feat"] = fe.grad
    return d.detach(), (f.detach() if f is not None else None), g


def _close(got, want, tol=1e-12):
    scale = max(float(want.abs().max()) if want.numel() else 0.0, 1e-300)
    err = float((got - want).abs().max()) if want.numel() else 0.0
    assert err <= tol * scale, err / scale


def _case(name):
    C = dict(random=5, flat=3, qnorm=8, special=33, edge=1)[name]
    cl = _cloud(64, C, seed=len(name), qnorm=(0.05, 20.0) if name == "qnorm" else (0.5, 2.0))
    if name in ("flat", "special"):
        cl = _special(cl)
    x = _points(cl, 120, seed=len(name) + 1)
    if name == "flat":
        x = torch.cat([x, cl["means"][7:12], cl["means"][7:12] + torch.tensor([0.0, 0.0, 1e-4])])
    if name == "special":
        x[5] = torch.tensor([float("nan"), 0.0, 0.0])
        x[6] = torch.tensor([0.0, float("inf"), 0.0])
        x[7] = torch.tensor([0.0, 0.0, -float("inf")])
    if name == "edge":
        x = torch.cat([x, _edge_points(cl, range(13, 40))])
    rng = np.random.default_rng(len(name) + 2)
    gd = _f(rng.normal(size=x.shape[0]))
    gf = _f(rng.normal(size=(x.shape[0], C)))
    return cl, x, gd, gf


@pytest.mark.parametrize("name", ["random", "flat", "qnorm", "special", "edge"])
def test_bounded_values_and_gradients_equal_float64_autograd(name):
    cl, x, gd, gf = _case(name)
    ref = F64.bounded(x, cl["means"], cl["scales"], cl["rot"], cl["opac"], cl["feat"], gd, gf if cl["feat"] is not None else None)
    d, f, g = _autograd(x, cl, gd, gf)
    _close(ref["density"][0], d)
    if f is not None:
        _close(ref["features"][0], f)
    for k, want in g.items():
        _close(ref[k][0], want.reshape(ref[k][0].shape))
    for k in ref:
        if k != "live":
            v, B, D = ref[k]
            assert torch.isfinite(v).all() and torch.isfinite(B).all() and (B >= 0).all() and (D >= 0).all(), k
    if name == "special":
        for k in ("means", "scales", "rot", "opacity", "feat"):
            assert all(torch.count_nonzero(t[:7]) == 0 for t in ref[k]), k
        for k in ("density", "features", "points"):
            assert all(torch.count_nonzero(t[5:8]) == 0 for t in ref[k]), k
    assert (ref["density"][0] > 0).float().mean() > 0.3  # the points sample the cloud


def _density_fp32(x, cl):
    """the lane's density in float32, in field.cu's order (ascending Gaussian id)"""
    ok = F64.valid(cl["means"], cl["scales"], cl["rot"], cl["opac"])
    r = cl["rot"][ok]
    inv = torch.rsqrt((r * r).sum(1))
    q = r * inv[:, None]
    A = F64.rotation_rows(q) / cl["scales"][ok][:, :, None]
    d = x[:, None, :] - cl["means"][ok][None]
    u = (A[None] * d[:, :, None, :]).sum(-1)
    g = cl["opac"][ok][None] * torch.exp(-0.5 * (u * u).sum(-1))
    g = torch.where(g >= T255, g, torch.zeros_like(g))
    dens = torch.zeros(x.shape[0])
    for j in range(g.shape[1]):
        dens = dens + g[:, j]
    return dens


def test_float32_density_lands_within_the_bound():
    cl, x, _, _ = _case("random")
    ref = F64.bounded(x, cl["means"], cl["scales"], cl["rot"], cl["opac"])
    assert float(F64.ratio(_density_fp32(x, cl), *ref["density"]).max()) <= 1.0  # the measured ratio, KAPPA 1


def _mutation_scene():
    """a cloud with flat Gaussians, a needle, |q| away from 1, and 40 Gaussians over one tight cluster (a live list of 40,
    so the last 32-Gaussian chunk is not the first)"""
    cl = _special(_cloud(96, 8, seed=7, qnorm=(0.3, 3.0)))
    cl["means"][40:80] = _f(np.random.default_rng(8).normal(0, 0.01, (40, 3)))
    cl["scales"][40:80] = 0.2
    x = torch.cat([_points(cl, 100, seed=9), _f(np.random.default_rng(10).normal(0, 0.01, (8, 3)))])
    rng = np.random.default_rng(11)
    return cl, x, _f(rng.normal(size=x.shape[0])), _f(rng.normal(size=(x.shape[0], 8)))


@pytest.mark.parametrize("mutation", [m for m in F64.MUTATIONS if m != "no_box_slack"])
def test_every_mutation_moves_a_checked_element_past_twice_its_bound(mutation):
    cl, x, gd, gf = _mutation_scene()
    args = (x, cl["means"], cl["scales"], cl["rot"], cl["opac"], cl["feat"], gd, gf)
    ref = F64.bounded(*args)
    assert int(ref["live"].max()) > 32
    mut = F64.bounded(*args, mutate={mutation})
    worst = {q: float(F64.ratio(mut[q][0], *ref[q], quantity=q).max()) for q in F64.QUANTITIES}
    assert max(worst.values()) > 2.0, worst


def test_the_support_box_holds_every_pair_fp32_may_keep_and_misses_them_without_its_slack():
    cl = _cloud(64, 0, seed=12)
    cl["opac"][20] = T255 * (1 + 2 ** -22)   # two ulps above the cutoff: its whole support is inside the either-side band
    x = torch.cat([_points(cl, 200, seed=13), _edge_points(cl, range(13, 30)), _box_extremes(cl, range(13, 30)),
                   cl["means"][20:21] + 1e-5])
    args = (x, cl["means"], cl["scales"], cl["rot"], cl["opac"])
    ref = F64.bounded(*args)
    assert bool((F64.ratio(ref["density"][0], *ref["density"]) == 0).all())
    assert F64.support_reach(*args).shape[0] == 0
    assert F64.support_reach(*args, mutate={"no_box_slack"}).shape[0] > 0
