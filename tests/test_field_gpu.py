"""The field query on the GPU against the float64 reference (field_ref64): density and features within 1e-5 relative L2,
and the gradients of points, means, scales, rotations, opacities and features within 1e-4, on random points, a 100^3 grid
over SCENE_BOUNDS, far and duplicate points, points at a mean, Gaussians without support and flat Gaussians.  Points
with an ambiguous pair (field_ref64.ambiguous_points) are left out of every query.  Also: binning invariance, voxelize's
layout, and no growth of device memory over repeated calls."""
import numpy as np
import pytest
import torch

import field_ref64 as F64
from manigaussian_b200 import gaussian_renderer as GR
from manigaussian_b200 import scenes

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
VAL_TOL, GRAD_TOL = 1e-5, 1e-4


def _cloud(P, C, seed=0, special=False, unaligned=False):
    g = scenes.make_gaussians(P, seed=seed)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)
    rng = np.random.default_rng(seed + 1)
    cl = dict(pts_xyz=t(g["means3D"]), rotations=t(g["rotations"] * rng.uniform(0.5, 2.0, (P, 1))), scales=t(g["scales"]),
              opacity=t(np.maximum(g["opacities"], 0.05)))
    if special:
        # below the opacity cutoff, a zero scale, a negative scale, and flat Gaussians (1e-4 next to 0.05) facing every way
        cl["opacity"][0:8] = 1.0 / 255.0
        cl["opacity"][8:16] = 0.002
        cl["scales"][16:24, 1] = 0.0
        cl["scales"][24:32, 0] = -0.01
        cl["scales"][32:P:5] = torch.tensor([0.05, 0.04, 1e-4], device=DEV)
        cl["opacity"][32:P:5] = 0.9
    cl["features"] = None
    if C:
        f = torch.from_numpy(rng.normal(0, 1, (P, C)).astype(np.float32)).to(DEV)
        if unaligned:
            buf = torch.empty(P * C + 1, dtype=torch.float32, device=DEV)[1:]  # rows start 4 bytes off 16-byte alignment
            buf.copy_(f.reshape(-1))
            f = buf.view(P, C)
            assert f.is_contiguous() and f.data_ptr() % 16 != 0
        cl["features"] = f
    return cl


def _keep_unambiguous(points, cl):
    amb = F64.ambiguous_points(points, cl["pts_xyz"], cl["scales"], cl["rotations"], cl["opacity"])
    return points[~amb]


def _leaves(points, cl):
    xs = [points] + [cl[k] for k in ("pts_xyz", "rotations", "scales", "opacity")] + ([cl["features"]] if cl["features"] is not None else [])
    return [x.detach().clone().requires_grad_(True) for x in xs]


def _ref(points, leaves):
    """the reference on leaves in query_field's order (points, means, rotations, scales, opacity[, features])"""
    return F64.field(points, leaves[1], leaves[3], leaves[2], leaves[4], leaves[5] if len(leaves) > 5 else None)


def _check(points, cl, seed=0, grads=True, cot_mask=None):
    """query_field against the reference, values and (with random cotangents, zero outside cot_mask) every gradient"""
    leaves = _leaves(points, cl)
    C = cl["features"].shape[1] if cl["features"] is not None else 0
    out = GR.query_field(*leaves[:5], leaves[5] if C else None)
    ref_leaves = [x.detach().double().requires_grad_(True) for x in leaves]
    rd, rf = _ref(ref_leaves[0], ref_leaves)
    sel = slice(None) if cot_mask is None else cot_mask
    assert F64.rel_l2(out["density"][sel], rd[sel]) < VAL_TOL
    if C:
        assert out["features"].shape == (points.shape[0], C)
        assert F64.rel_l2(out["features"][sel], rf[sel]) < VAL_TOL
    if not grads:
        return out
    gen = torch.Generator(device="cpu").manual_seed(seed)
    gd = torch.randn(points.shape[0], generator=gen, dtype=torch.float64).to(DEV)
    gf = torch.randn(points.shape[0], max(C, 1), generator=gen, dtype=torch.float64).to(DEV)[:, :C]
    if cot_mask is not None:
        gd = gd * cot_mask
        gf = gf * cot_mask[:, None]
    loss = (out["density"] * gd.float()).sum() + ((out["features"] * gf.float()).sum() if C else 0)
    loss.backward()
    rloss = (rd * gd).sum() + ((rf * gf).sum() if C else 0)
    rloss.backward()
    names = ("points", "means", "rotations", "scales", "opacity", "features")
    for n, a, b in zip(names, leaves, ref_leaves):
        assert a.grad is not None, n
        err = F64.rel_l2(a.grad, b.grad)
        assert err < GRAD_TOL, (n, err)
    return out


@pytest.mark.parametrize("C,unaligned", [(0, False), (3, False), (32, False), (32, True), (64, False), (130, False), (8, True)])
def test_random_points_match_the_float64_reference(C, unaligned):
    cl = _cloud(2048, C, seed=C, unaligned=unaligned)
    rng = np.random.default_rng(11 + C)
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    pts = torch.from_numpy((lo + (hi - lo) * rng.random((6000, 3))).astype(np.float32)).to(DEV)
    pts = _keep_unambiguous(pts, cl)
    out = _check(pts, cl, seed=C)
    assert (out["density"] > 0).float().mean() > 0.5  # the points sample the cloud, not empty space


def test_grid_over_scene_bounds_with_16k_gaussians():
    cl = _cloud(16384, 3, seed=4)
    pts, n = GR.voxel_centres(scenes.SCENE_BOUNDS, 100, DEV)
    # the reference at a random subset of the 10^6 voxels; the cotangents vanish elsewhere, so every gradient is exact there
    rng = np.random.default_rng(4)
    sub = torch.from_numpy(rng.choice(pts.shape[0], 12000, replace=False)).to(DEV)
    amb = F64.ambiguous_points(pts[sub], cl["pts_xyz"], cl["scales"], cl["rotations"], cl["opacity"])
    sub = sub[~amb]
    mask = torch.zeros(pts.shape[0], dtype=torch.float64, device=DEV)
    mask[sub] = 1.0
    leaves = _leaves(pts, cl)
    out = GR.query_field(*leaves)
    ref_leaves = [x.detach().double().requires_grad_(True) for x in leaves]
    rd, rf = _ref(ref_leaves[0][sub], ref_leaves)
    assert F64.rel_l2(out["density"][sub], rd) < VAL_TOL
    assert F64.rel_l2(out["features"][sub], rf) < VAL_TOL
    gen = torch.Generator(device="cpu").manual_seed(9)
    gd = torch.randn(pts.shape[0], generator=gen, dtype=torch.float64).to(DEV) * mask
    gf = torch.randn(pts.shape[0], 3, generator=gen, dtype=torch.float64).to(DEV) * mask[:, None]
    ((out["density"] * gd.float()).sum() + (out["features"] * gf.float()).sum()).backward()
    ((rd * gd[sub]).sum() + (rf * gf[sub]).sum()).backward()
    for n_, a, b in zip(("points", "means", "rotations", "scales", "opacity", "features"), leaves, ref_leaves):
        assert F64.rel_l2(a.grad, b.grad) < GRAD_TOL, n_
    # voxelize is the same query, channel first
    vox = GR.voxelize(scenes.SCENE_BOUNDS, 100, *[x.detach() for x in leaves[1:]])
    assert vox["density"].shape == (100, 100, 100) and vox["features"].shape == (3, 100, 100, 100)
    assert vox["features"].is_contiguous()
    assert torch.equal(vox["density"].reshape(-1), out["density"].detach())
    assert F64.rel_l2(vox["features"].reshape(3, -1).t(), out["features"].detach()) < 1e-6


def test_far_points_are_exact_zeros():
    cl = _cloud(1024, 32, seed=2)
    pts = torch.tensor([[5.0, 5.0, 5.0], [-3.0, 0.0, 1.0], [0.2, 0.0, 9.0]], device=DEV).repeat(40, 1)
    pts = pts + 0.01 * torch.arange(120, device=DEV, dtype=torch.float32)[:, None]
    leaves = _leaves(pts, cl)
    out = GR.query_field(*leaves)
    assert torch.count_nonzero(out["density"]) == 0 and torch.count_nonzero(out["features"]) == 0
    (out["density"].sum() + out["features"].sum()).backward()
    for x in leaves:
        assert torch.count_nonzero(x.grad) == 0


def test_duplicate_points_and_points_at_means():
    cl = _cloud(2048, 32, seed=3)
    at_means = _keep_unambiguous(cl["pts_xyz"][:200], cl)
    base = torch.cat([at_means, _keep_unambiguous(cl["pts_xyz"][100:300] + 0.003, cl)])
    pts = torch.cat([base, base, base[:50]])
    out = _check(pts, cl, seed=3)
    n = base.shape[0]
    assert torch.equal(out["density"][:n], out["density"][n:2 * n])
    assert torch.equal(out["features"][:n], out["features"][n:2 * n])
    assert (out["density"][:at_means.shape[0]] >= 0.05 * (1 - 1e-6)).all()  # a mean carries at least its own opacity


def test_gaussians_without_support_and_flat_gaussians():
    cl = _cloud(2048, 32, seed=5, special=True)
    rng = np.random.default_rng(5)
    near = cl["pts_xyz"][:400] + torch.from_numpy(rng.normal(0, 0.01, (400, 3)).astype(np.float32)).to(DEV)
    flat = cl["pts_xyz"][32:2048:5][:300]
    pts = torch.cat([near, flat, flat + torch.tensor([0.0, 0.0, 1e-4], device=DEV)])
    pts = _keep_unambiguous(pts, cl)
    leaves = _leaves(pts, cl)
    _check(pts, cl, seed=5)
    out = GR.query_field(*leaves)
    (out["density"].sum() + out["features"].sum()).backward()
    for x in leaves[1:]:
        assert torch.count_nonzero(x.grad[:32]) == 0  # no support: zero gradients


def test_results_do_not_depend_on_the_binning():
    cl = _cloud(4096, 32, seed=6)
    rng = np.random.default_rng(6)
    few = _keep_unambiguous(cl["pts_xyz"][:20] + torch.from_numpy(rng.normal(0, 0.01, (20, 3)).astype(np.float32)).to(DEV), cl)
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    many = torch.from_numpy((lo + (hi - lo) * rng.random((200000, 3))).astype(np.float32)).to(DEV)
    alone = GR.query_field(few, cl["pts_xyz"], cl["rotations"], cl["scales"], cl["opacity"], cl["features"])  # one bin
    spread = GR.query_field(torch.cat([many[:1000], few, many[1000:]]), cl["pts_xyz"], cl["rotations"], cl["scales"], cl["opacity"],
                            cl["features"])
    k = few.shape[0]
    assert (alone["density"] > 0).all()
    assert torch.equal(spread["density"][1000:1000 + k], alone["density"])  # lane sums in ascending Gaussian id either way
    assert F64.rel_l2(spread["features"][1000:1000 + k], alone["features"]) < 1e-6


def test_repeated_calls_do_not_grow_device_memory():
    cl = _cloud(4096, 32, seed=7)
    leaves = _leaves(torch.rand(50000, 3, device=DEV), cl)

    def step():
        out = GR.query_field(*leaves)
        (out["density"].sum() + out["features"].square().sum()).backward()
        for x in leaves:
            x.grad = None

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(DEV)
    for _ in range(20):
        step()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) == before
