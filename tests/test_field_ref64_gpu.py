"""The field query on the GPU element by element against the bounded float64 reference (field_ref64.bounded): every element
of the density, the features and the six gradients within KAPPA u B, through field_query_raw / field_query_backward_raw
and through query_field / voxelize, on scenes built for the kernel's edges.  Pairs on the cutoff are kept: the reference's
either-side rule bounds them.

* Channel widths that pick each instantiation (NFT 0/1/2/4, VEC and padded rows, GRP with remainder groups of 1 and 15),
  and C = 8 and 32 with rows 4 bytes off 16-byte alignment.
* Bin lists of 1, 31, 32, 33, 64, 65 and 1000 Gaussians (a tight cluster of points inside overlapping Gaussians; the live
  list length is asserted from the reference), and bins holding 1, 31, 32, 33 and 65 points.
* Degenerate bounding boxes: coincident points, points on a plane and on a line, one outlier 10^3 away, and points on a
  lattice through bin faces and the box maximum.
* Non-finite points (NaN, +-inf) among finite ones: exact zeros, and the finite points' density bitwise unchanged.
* Gaussians whose support reaches the points only through the box's slack or covers the whole box, o at 1/255 and one and
  two ulps above, flat Gaussians and 1e4-anisotropic needles, zero, negative and non-finite scales and a non-finite mean,
  with points on the support edges.
* Q in {1, 33, 6000} by P in {1, 2048}, and the 100^3 grid over SCENE_BOUNDS with 16k Gaussians on a sampled subset.
* Every requested-gradient subset of field_query_backward_raw, zero and absent cotangents, and query_field with only the
  points or only the features requiring grad; voxelize's backward, and its channel-first raw backward against the
  point-major one.

Measured worst (|x - v| - D) / (u B) per quantity over every case, on an NVIDIA H100 80GB HBM3 at a 700 W power limit
(printed at the end of a `-s` run); field_ref64.KAPPA is 4x these:

    density 0.580   features 0.417   points 0.237   means 0.213   scales 0.211   rot 0.134   opacity 0.235   feat 0.265

The file runs in about 15 s on that GPU.
"""
import numpy as np
import pytest
import torch

import field_ref64 as F64
from manigaussian_b200 import gaussian_renderer as GR
from manigaussian_b200 import rasterizer as R
from manigaussian_b200 import scenes

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
NEEDS = ("points", "means", "scales", "rot", "opacity", "feat")
ALL = (True,) * 6
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nfield_ref64 worst |x - v| / (u B): " + ", ".join(f"{q}={WORST.get(q, 0.0):.4g}" for q in F64.QUANTITIES))


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def _cloud(P, C, seed=0, unaligned=False):
    g = scenes.make_gaussians(P, seed=seed)
    rng = np.random.default_rng(seed + 1)
    cl = dict(means=_t(g["means3D"]), rot=_t(g["rotations"] * rng.uniform(0.5, 2.0, (P, 1))), scales=_t(g["scales"]),
              opac=_t(np.maximum(g["opacities"], 0.05)), feat=None)
    if C:
        f = _t(rng.normal(0, 1, (P, C)))
        if unaligned:
            buf = torch.empty(P * C + 1, dtype=torch.float32, device=DEV)[1:]
            buf.copy_(f.reshape(-1))
            f = buf.view(P, C)
            assert f.data_ptr() % 16 != 0
        cl["feat"] = f
    return cl


def _random_points(Q, seed):
    rng = np.random.default_rng(seed)
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    return _t(lo + (hi - lo) * rng.random((Q, 3)))


def _cot(Q, C, seed, mask=None):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    gd = torch.randn(Q, generator=gen).to(DEV)
    gf = torch.randn(Q, max(C, 1), generator=gen)[:, :C].contiguous().to(DEV)
    if mask is not None:
        gd, gf = gd * mask, gf * mask[:, None]
    return gd, gf


def _within(name, got, ref, sel=None):
    v, B, D = ref
    if sel is not None:
        got, v, B, D = got[sel], v[sel], B[sel], D[sel]
    raw = F64.ratio(got, v, B, D)
    WORST[name] = max(WORST.get(name, 0.0), float(raw.max()) if raw.numel() else 0.0)
    r = F64.ratio(got, v, B, D, name)
    worst = float(r.max()) if r.numel() else 0.0
    assert worst <= 1.0, (name, worst, int(r.argmax()))


def _check(pts, cl, gd=None, gf=None, needs=ALL, channel_first=False, sel=None):
    """raw forward and backward against the reference; returns (density, features, gradients, reference)"""
    C = cl["feat"].shape[1] if cl["feat"] is not None else 0
    args = (cl["means"], cl["scales"], cl["rot"], cl["opac"])
    dens, feat, st, ps, _ = R.field_query_raw(pts, *args, cl["feat"], channel_first=channel_first)
    rp = pts if sel is None else pts[sel]
    rgd = None if gd is None else (gd if sel is None else gd[sel])
    rgf = None if gf is None else (gf if sel is None else gf[sel])
    ref = F64.bounded(rp, *args, cl["feat"], rgd, rgf)
    _within("density", dens if sel is None else dens[sel], ref["density"])
    if C:
        fq = feat.t() if channel_first else feat
        _within("features", fq if sel is None else fq[sel], ref["features"])
    if gd is None and gf is None:
        return dens, feat, None, ref
    cot_f = gf.t().contiguous() if (channel_first and gf is not None) else gf
    g = R.field_query_backward_raw(st, ps, pts, cl["scales"], cl["rot"], cl["feat"], gd, cot_f if C else None,
                                   channel_first=channel_first, needs=needs)
    for k, (n, x) in enumerate(zip(NEEDS, g)):
        if not needs[k] or (n == "feat" and not C):
            assert x is None, n
            continue
        if n == "points":
            if sel is not None:
                off = torch.ones(pts.shape[0], dtype=torch.bool, device=DEV)
                off[sel] = False
                assert torch.count_nonzero(x[off]) == 0
                x = x[sel]
        _within(n, x, ref[n])
    return dens, feat, g, ref


def _full(pts, cl, seed=0, **kw):
    C = cl["feat"].shape[1] if cl["feat"] is not None else 0
    gd, gf = _cot(pts.shape[0], C, seed)
    return _check(pts, cl, gd, gf if C else None, **kw)


# ---------------------------------------------------------------------------------------------------- channel widths
@pytest.mark.parametrize("C,unaligned", [(c, False) for c in (0, 1, 3, 8, 12, 16, 31, 32, 33, 47, 64, 96, 130, 512)] +
                         [(8, True), (32, True)])
def test_channel_widths_within_bound(C, unaligned):
    cl = _cloud(2048, C, seed=C + 100, unaligned=unaligned)
    pts = _random_points(6000 if C <= 130 else 1500, seed=C)
    dens, _, _, ref = _full(pts, cl, seed=C)
    assert (dens > 0).float().mean() > 0.5


# ---------------------------------------------------------------------------------------------------- bin lists and items
@pytest.mark.parametrize("n", [1, 31, 32, 33, 64, 65, 1000])
def test_bin_lists_at_the_chunk_boundaries(n):
    rng = np.random.default_rng(n)
    P = n + 300
    means = np.concatenate([rng.normal(0, 0.01, (n, 3)), rng.uniform(3, 4, (300, 3))])  # the 300 never reach the cluster
    q = rng.normal(size=(P, 4))
    cl = dict(means=_t(means), rot=_t(q), scales=_t(rng.uniform(0.2, 0.4, (P, 3))), opac=_t(rng.uniform(0.3, 0.9, P)),
              feat=_t(rng.normal(size=(P, 16))))
    pts = _t(rng.normal(0, 0.005, (40, 3)))
    _, _, _, ref = _full(pts, cl, seed=n)
    assert (ref["live"] == n).all()  # every cluster point sees every cluster Gaussian: its bin lists all n


@pytest.mark.parametrize("k", [1, 31, 32, 33, 65])
def test_warp_items_at_the_item_boundaries(k):
    cl = _cloud(2048, 12, seed=k)
    rng = np.random.default_rng(k)
    c = scenes.make_gaussians(1, seed=k)["means3D"][0]
    pts = _t(np.concatenate([c + rng.normal(0, 1e-3, (k, 3)), c[None] + 0.6]))
    _full(pts, cl, seed=k)


# ---------------------------------------------------------------------------------------------------- degenerate boxes
def _degenerate(kind, rng, c):
    if kind == "coincident":
        return np.repeat(c[None], 50, 0)
    if kind == "plane":
        x = c + rng.uniform(-0.2, 0.2, (300, 3))
        x[:, 2] = c[2]
        return x
    if kind == "line":
        x = np.repeat(c[None], 300, 0)
        x[:, 0] += rng.uniform(-0.2, 0.2, 300)
        return x
    if kind == "outlier":
        return np.concatenate([c + rng.uniform(-0.1, 0.1, (500, 3)), c[None] + 1e3])
    # a lattice of step 1/16 (exact in fp32) through the bin faces and the box maximum
    g = np.arange(17, dtype=np.float64) / 16.0 * 0.5
    return c + np.stack(np.meshgrid(g, g, g[:5], indexing="ij"), -1).reshape(-1, 3)


@pytest.mark.parametrize("kind", ["coincident", "plane", "line", "outlier", "lattice"])
def test_degenerate_bounding_boxes(kind):
    cl = _cloud(2048, 8, seed=21)
    c = np.round(scenes.make_gaussians(1, seed=3)["means3D"][0] * 16) / 16
    pts = _t(_degenerate(kind, np.random.default_rng(5), c))
    _full(pts, cl, seed=5)


def test_non_finite_points_are_exact_zeros_and_change_nothing_else():
    cl = _cloud(2048, 32, seed=22)
    fin = _random_points(2000, seed=22)
    bad = torch.tensor([[float("nan"), 0.0, 0.0], [0.0, float("inf"), 0.0], [0.0, 0.0, -float("inf")],
                        [float("inf"), float("nan"), -float("inf")]], device=DEV).repeat(10, 1)
    pts = torch.cat([fin[:700], bad[:20], fin[700:], bad[20:]])
    isbad = ~torch.isfinite(pts).all(1)
    dens, feat, g, _ = _full(pts, cl, seed=22)
    assert torch.count_nonzero(dens[isbad]) == 0 and torch.count_nonzero(feat[isbad]) == 0
    assert torch.count_nonzero(g[0][isbad]) == 0
    alone = R.field_query_raw(fin, cl["means"], cl["scales"], cl["rot"], cl["opac"], cl["feat"])[0]
    assert torch.equal(dens[~isbad], alone)


# ---------------------------------------------------------------------------------------------------- Gaussians
def _edge(means, scales, rot, opac, ids, k=1.0):
    Rm = F64.rotation_rows(rot.double())
    cut = 2.0 * torch.log(255.0 * opac.double())
    return torch.stack([means[i].double() + k * torch.sqrt(cut[i]) * scales[i, 0].double() * Rm[i, 0] for i in ids]).float()


def test_special_gaussians_and_points_on_the_cutoff():
    rng = np.random.default_rng(30)
    cl = _cloud(2048, 12, seed=30)
    m, s, o = cl["means"], cl["scales"], cl["opac"]
    T = np.float32(F64.THRESH)
    o[0], o[1], o[2] = float(T), float(np.nextafter(T, np.float32(1))), float(np.nextafter(np.nextafter(T, np.float32(1)), np.float32(1)))
    s[3, 1] = 0.0
    s[4, 0] = -0.01
    s[5, 2] = float("inf")
    s[6, 0] = float("nan")
    m[7, 1] = float("nan")
    s[8:200:4] = torch.tensor([0.05, 0.04, 1e-4], device=DEV)       # flat
    o[8:200:4] = 0.9
    s[9:200:8] = torch.tensor([0.05, 5e-6, 5e-6], device=DEV)       # needles, 1e4 anisotropic
    o[9:200:8] = 0.8
    s[10] = 10.0                                                    # a support larger than every box here
    pts = torch.cat([m[:200] + _t(rng.normal(0, 0.01, (200, 3))), m[8:200:4], m[9:200:8] + _t(rng.normal(0, 1e-5, (24, 3))),
                     _edge(m, s, cl["rot"], o, range(11, 200, 3)), _edge(m, s, cl["rot"], o, range(11, 200, 3), 1 + 3e-7),
                     _edge(m, s, cl["rot"], o, range(8, 200, 4))])
    pts = pts[torch.isfinite(pts).all(1)]
    # a Gaussian that reaches the points' box only through the slack of its support box
    box_lo = pts.min(0).values.double()
    r = F64._kernel_box(m[12:13], s[12:13], cl["rot"][12:13], o[12:13])[0]
    exact = F64._kernel_box(m[12:13], s[12:13], cl["rot"][12:13], o[12:13], slack=False)[0]
    m[12] = (box_lo - 0.5 * (r + exact)).float()
    assert F64.support_reach(pts, m, s, cl["rot"], o).shape[0] == 0
    _, _, g, ref = _full(pts, cl, seed=30)
    for x in g[1:]:
        assert torch.count_nonzero(x[:8]) == 0  # no support: every gradient exactly zero


@pytest.mark.parametrize("Q,P", [(1, 1), (33, 1), (6000, 1), (1, 2048), (33, 2048), (6000, 2048)])
def test_query_and_cloud_sizes(Q, P):
    cl = _cloud(P, 5, seed=Q + P)
    if P == 1:
        cl["scales"][:] = 0.5
    pts = _random_points(Q, seed=Q) if Q > 1 else cl["means"][:1] + 0.01
    _full(pts, cl, seed=Q)


def test_grid_over_scene_bounds_with_16k_gaussians():
    cl = _cloud(16384, 3, seed=4)
    pts, _ = GR.voxel_centres(scenes.SCENE_BOUNDS, 100, DEV)
    sub = torch.from_numpy(np.random.default_rng(4).choice(pts.shape[0], 12000, replace=False)).to(DEV)
    mask = torch.zeros(pts.shape[0], device=DEV)
    mask[sub] = 1.0
    gd, gf = _cot(pts.shape[0], 3, 4, mask)
    _check(pts, cl, gd, gf, sel=sub)


# ---------------------------------------------------------------------------------------------------- requested gradients
SUBSETS = [tuple(i == k for i in range(6)) for k in range(6)] + [ALL, (True, False, False, False, False, True),
                                                               (False, True, True, True, True, False)]


@pytest.mark.parametrize("needs", SUBSETS, ids=lambda n: "".join("x" if b else "-" for b in n))
def test_every_requested_gradient_subset(needs):
    cl = _cloud(2048, 12, seed=40)
    pts = _random_points(3000, seed=40)
    _full(pts, cl, seed=40, needs=needs)


@pytest.mark.parametrize("cot", ["density_none", "density_zero", "features_none", "features_zero"])
def test_zero_and_absent_cotangents(cot):
    cl = _cloud(2048, 40, seed=41)
    pts = _random_points(3000, seed=41)
    gd, gf = _cot(pts.shape[0], 40, 41)
    if cot.startswith("density"):
        gd = None if cot.endswith("none") else torch.zeros_like(gd)
    else:
        gf = None if cot.endswith("none") else torch.zeros_like(gf)
    _check(pts, cl, gd, gf)


@pytest.mark.parametrize("leaf", ["points", "features"])
def test_query_field_with_one_leaf_requiring_grad(leaf):
    cl = _cloud(2048, 12, seed=42)
    pts = _random_points(3000, seed=42)
    gd, gf = _cot(pts.shape[0], 12, 42)
    x = pts.clone().requires_grad_(leaf == "points")
    f = cl["feat"].clone().requires_grad_(leaf == "features")
    out = GR.query_field(x, cl["means"], cl["rot"], cl["scales"], cl["opac"], f)
    ((out["density"] * gd).sum() + (out["features"] * gf).sum()).backward()
    needs = tuple(n == {"points": "points", "features": "feat"}[leaf] for n in NEEDS)
    _, _, g, ref = _check(pts, cl, gd, gf, needs=needs)
    name = "points" if leaf == "points" else "feat"
    _within(name, x.grad if leaf == "points" else f.grad, ref[name])
    assert sum(t is not None for t in g) == 1


# ---------------------------------------------------------------------------------------------------- voxelize
def test_voxelize_backward_within_bound():
    cl = _cloud(2048, 5, seed=50)
    n = 40
    pts, _ = GR.voxel_centres(scenes.SCENE_BOUNDS, n, DEV)
    leaves = [cl[k].clone().requires_grad_(True) for k in ("means", "rot", "scales", "opac", "feat")]
    vox = GR.voxelize(scenes.SCENE_BOUNDS, n, *leaves)
    gen = torch.Generator(device="cpu").manual_seed(50)
    cd = torch.randn(n, n, n, generator=gen).to(DEV)
    cf = torch.randn(5, n, n, n, generator=gen).to(DEV)
    ((vox["density"] * cd).sum() + (vox["features"] * cf).sum()).backward()
    gd, gf = cd.reshape(-1), cf.reshape(5, -1).t().contiguous()
    ref = F64.bounded(pts, cl["means"], cl["scales"], cl["rot"], cl["opac"], cl["feat"], gd, gf)
    _within("density", vox["density"].reshape(-1), ref["density"])
    _within("features", vox["features"].reshape(5, -1).t(), ref["features"])
    for name, leaf in zip(("means", "rot", "scales", "opacity", "feat"), leaves):
        _within(name, leaf.grad.reshape(ref[name][0].shape), ref[name])
    # the raw channel-first backward and the point-major one on the transposed cotangent, each within bound
    _check(pts, cl, gd, gf, channel_first=True)
    _check(pts, cl, gd, gf, channel_first=False)
