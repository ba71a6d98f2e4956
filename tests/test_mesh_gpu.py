"""TSDF fusion and marching cubes on the GPU (tsdf.cu, marching_cubes.cu; gaussian_renderer.tsdf_fuse / marching_cubes).

1. Fusion against the float64 reference (tests/tsdf_ref64.py) for each camera model and in one call mixing all four, with
   C = 0, 3 and 32: on every voxel the reference does not flag as border, tsdf within 1e-5, weight exactly and colour within
   1e-5; the border voxels are a small, reported fraction.
2. Fusion invariants, bit for bit: repeatability, one call against a split into volume= calls (across the 64-view launch
   chunk too), voxels no view updates left unchanged, and a CUDA-graph capture replayed on new depth images.
3. Marching cubes against tests/mc_ref.py bit for bit (vertex bytes, faces, colours and their order): a fused TSDF with its
   weight mask and colour, voxelize's density of a random cloud, random fields with invalid points, one-cell and empty grids.
4. Accuracy: analytic depth images of a sphere and a box from 24 views per camera model, fused and extracted, give a closed
   mesh whose vertices lie within one voxel of the true surface (within trunc of the box's convex edges, where projective
   fusion rounds them).
5. End to end: a Gaussian cloud sampled on a sphere, rendered with planar depth in 12 views, depth / alpha fused where
   alpha > 0.99, gives a closed mesh near the sphere.
6. A 512^3 fusion of 64 views against the reference on sampled voxels, and a call on a non-current device.
"""

import numpy as np
import pytest
import torch

import mc_ref as M
import tsdf_ref64 as T64
import util
from manigaussian_b200 import scenes
from test_planar_depth_gpu import MODELS, _model_kw

pytestmark = pytest.mark.gpu

CENTRE = np.asarray(scenes.SCENE_CENTER, np.float64)
R_SPHERE = 0.3
BOUNDS = tuple(float(x) for x in np.concatenate([CENTRE - 0.45, CENTRE + 0.45]))


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as RS
    RS.reset_capacity_estimates()
    yield
    RS.reset_capacity_estimates()


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def _camera(W, H, view, num_views, height=0.4, radius=1.6):
    return dict(W=W, H=H, cam=scenes.make_camera(W, H, view, num_views, radius=radius, height=height))


def _setting(inp, model):
    """GaussianRasterizationSettings and the reference's view dict of one camera model on a scenes camera"""
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    kw, view = _model_kw(inp, model)
    cam = inp["cam"]
    tx, ty = kw.pop("tanfovx", cam["tanfovx"]), kw.pop("tanfovy", cam["tanfovy"])
    pm = kw.pop("projmatrix", None)
    pm = cam["projmatrix"] if pm is None else pm
    z3 = torch.zeros(3, device="cuda")
    return GaussianRasterizationSettings(inp["H"], inp["W"], tx, ty, z3, 1.0, _t(cam["viewmatrix"]), _t(pm), 0, _t(cam["campos"]),
                                         False, False, False, **kw), view


def _ring(W, H, models, heights=(0.4,), per_ring=None):
    """views on rings around the scene centre, the camera models cycling through `models`"""
    per_ring = per_ring or len(models)
    out = []
    for r, h in enumerate(heights):
        for k in range(per_ring):
            inp = _camera(W, H, k + 0.5 * r, per_ring, height=h)
            out.append(_setting(inp, models[(r * per_ring + k) % len(models)]))
    return [s for s, _ in out], [v for _, v in out]


def _sphere_depth(views, centre=CENTRE, R=R_SPHERE):
    """[V,H,W] view-space z of the first hit of each pixel centre's ray with the sphere (0 where it misses), through each
    view's own lens (camera_rays)"""
    from manigaussian_b200 import gaussian_renderer as GR
    rays = GR.camera_rays(views)
    o, d = rays["origin"].double(), rays["direction"].double()
    oc = o - torch.tensor(centre, device="cuda")
    a, b, c = (d * d).sum(-1), 2 * (d * oc).sum(-1), (oc * oc).sum(-1) - R * R
    disc = b * b - 4 * a * c
    z = (-b - torch.sqrt(disc.clamp_min(0))) / (2 * a)
    return torch.where(rays["valid"] & (disc > 0) & (z > 0), z, torch.zeros_like(z)).float()


def _box_depth(views, lo, hi):
    from manigaussian_b200 import gaussian_renderer as GR
    rays = GR.camera_rays(views)
    o, d = rays["origin"].double(), rays["direction"].double()
    lo_t, hi_t = (torch.tensor(x, device="cuda", dtype=torch.float64) for x in (lo, hi))
    with torch.no_grad():
        t1, t2 = (lo_t - o) / d, (hi_t - o) / d
        near = torch.minimum(t1, t2).amax(-1)
        far = torch.maximum(t1, t2).amin(-1)
    hit = rays["valid"] & (near <= far) & (near > 0)
    return torch.where(hit, near, torch.zeros_like(near)).float()


def _points(bounds, n):
    cs = M.axis_centres(bounds, n)
    return torch.stack([c.reshape(-1) for c in torch.meshgrid(*cs, indexing="ij")], -1).numpy()


def _manifold(v, f):
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = torch.minimum(e[:, 0], e[:, 1]) * (1 << 32) + torch.maximum(e[:, 0], e[:, 1])
    _, cnt = torch.unique(key, return_counts=True)
    used = torch.unique(f)
    return bool((cnt == 2).all()), len(used) == len(v)


def _bits(x):
    return x.contiguous().view(torch.int32) if x.dtype == torch.float32 else x


def _same_mesh(got, want):
    for k in ("vertices", "faces", "colors"):
        a, b = got[k], want[k]
        if b is None:
            assert a is None, k
            continue
        assert a.shape == b.shape, (k, a.shape, b.shape)
        assert torch.equal(_bits(a.cpu()), _bits(b.cpu())), k


# --------------------------------------------------------------------------- 1. against the float64 reference
CASES = [(m, 3) for m in MODELS] + [("mixed", 0), ("mixed", 32)]


@pytest.mark.parametrize("model,C", CASES)
def test_fusion_matches_the_float64_reference(model, C):
    from manigaussian_b200 import gaussian_renderer as GR
    models = MODELS if model == "mixed" else (model,)
    views, refs = _ring(80, 60, models, heights=(0.4, -0.6), per_ring=4)
    depth = _sphere_depth(views)
    rng = np.random.default_rng(C)
    color = _t(rng.random((len(views), C, 60, 80))) if C else None
    n, trunc = (28, 30, 26), 0.06
    out = GR.tsdf_fuse(views, depth, BOUNDS, n, trunc, color=color)
    ts, w, col, border = T64.fuse(_points(BOUNDS, n), refs, depth.cpu().numpy(), trunc, None if color is None else color.cpu().numpy())
    keep = ~border
    frac = 1 - keep.mean()
    gw, gt = out["weight"].cpu().numpy().reshape(-1), out["tsdf"].cpu().numpy().reshape(-1)
    print(f"{model} C={C}: border voxels {100 * frac:.3f} %, observed {(w > 0).mean() * 100:.1f} %, weights differ on "
          f"{int((gw != w).sum())} voxels ({int(((gw != w) & keep).sum())} not border), max tsdf error off the border "
          f"{np.abs(gt - ts)[keep].max():.3g}")
    assert np.array_equal(gw[keep], w[keep])
    assert np.abs(gt[keep] - ts[keep]).max() <= 1e-5
    assert frac < 0.02 and (w[keep] > 0).sum() > 2000
    if C:
        gc = out["color"].cpu().numpy().reshape(C, -1).T
        assert out["color"].shape == (C,) + n and np.abs(gc[keep] - col[keep]).max() <= 1e-5
    else:
        assert out["color"] is None


# --------------------------------------------------------------------------- 2. invariants
def test_fusion_is_repeatable_split_invariant_and_leaves_unseen_voxels_alone():
    from manigaussian_b200 import gaussian_renderer as GR
    views, _ = _ring(48, 36, MODELS, heights=(0.4, -0.5, 1.2), per_ring=24)  # 72 views: two launches of up to 64
    depth = _sphere_depth(views)
    color = _t(np.random.default_rng(1).random((len(views), 3, 36, 48)))
    n, trunc = (20, 22, 18), 0.05
    a = GR.tsdf_fuse(views, depth, BOUNDS, n, trunc, color=color)
    b = GR.tsdf_fuse(views, depth, BOUNDS, n, trunc, color=color)
    for k in a:
        assert torch.equal(_bits(a[k]), _bits(b[k])), k
    for cut in ((5,), (64,), (3, 40, 70)):
        vol = None
        for lo, hi in zip((0,) + cut, cut + (len(views),)):
            vol = GR.tsdf_fuse(views[lo:hi], depth[lo:hi].contiguous(), BOUNDS, n, trunc, color=color[lo:hi].contiguous(), volume=vol)
        for k in a:
            assert torch.equal(_bits(a[k]), _bits(vol[k])), (cut, k)
    # a voxel no view updates keeps its bits, even when they are not a fresh volume's
    g = torch.Generator(device="cuda").manual_seed(3)
    init = {"tsdf": torch.randn(n, device="cuda", generator=g), "weight": torch.rand(n, device="cuda", generator=g) * 3,
            "color": torch.randn((3,) + n, device="cuda", generator=g)}
    before = {k: v.clone() for k, v in init.items()}
    init["tsdf"].view(-1)[:7] = float("nan")
    before["tsdf"].view(-1)[:7] = float("nan")
    out = GR.tsdf_fuse(views[:3], depth[:3].contiguous(), BOUNDS, n, trunc, color=color[:3].contiguous(), volume=init)
    assert out is init
    same = out["weight"] == before["weight"]
    assert int(same.sum()) > 0 and int((~same).sum()) > 0
    assert torch.equal(_bits(out["tsdf"])[same], _bits(before["tsdf"])[same])
    assert torch.equal(_bits(out["color"])[:, same], _bits(before["color"])[:, same])


def test_fusion_captures_in_a_cuda_graph():
    from manigaussian_b200 import gaussian_renderer as GR
    views, _ = _ring(48, 36, MODELS, per_ring=4)
    depth = _sphere_depth(views)
    n = (16, 16, 16)
    vol = {"tsdf": torch.ones(n, device="cuda"), "weight": torch.zeros(n, device="cuda"), "color": None}
    src = depth.clone()

    def step():
        vol["tsdf"].fill_(1.0)
        vol["weight"].zero_()
        GR.tsdf_fuse(views, src, BOUNDS, n, 0.06, volume=vol)

    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        step()
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    src.copy_(_sphere_depth(views, R=0.25))
    graph.replay()
    torch.cuda.synchronize()
    want = GR.tsdf_fuse(views, src, BOUNDS, n, 0.06)
    assert torch.equal(_bits(vol["tsdf"]), _bits(want["tsdf"])) and torch.equal(vol["weight"], want["weight"])


# --------------------------------------------------------------------------- 3. marching cubes against mc_ref
def _mc_both(values, level, bounds, weight=None, color=None):
    from manigaussian_b200 import gaussian_renderer as GR
    got = GR.marching_cubes(values, level, bounds, weight=weight, color=color)
    want = M.marching_cubes(values.cpu(), level, bounds, None if weight is None else weight.cpu(),
                            None if color is None else color.cpu())
    _same_mesh(got, want)
    again = GR.marching_cubes(values, level, bounds, weight=weight, color=color)
    _same_mesh(again, got)
    return got


def test_marching_cubes_of_a_fused_tsdf_with_weights_and_colour():
    from manigaussian_b200 import gaussian_renderer as GR
    views, _ = _ring(96, 72, MODELS, heights=(0.4, -0.6, 1.3), per_ring=6)
    depth = _sphere_depth(views)
    color = _t(np.random.default_rng(4).random((len(views), 3, 72, 96)))
    n = (40, 44, 36)
    vol = GR.tsdf_fuse(views, depth, BOUNDS, n, 0.07, color=color)
    got = _mc_both(vol["tsdf"], 0.0, BOUNDS, weight=vol["weight"], color=vol["color"])
    assert len(got["faces"]) > 1000 and got["colors"].shape == (len(got["vertices"]), 3)


def test_marching_cubes_of_a_voxelized_density():
    from manigaussian_b200 import gaussian_renderer as GR
    g = util.make_inputs(P=3000, W=8, H=8, seed=6)["g"]
    den = GR.voxelize(tuple(float(x) for x in scenes.SCENE_BOUNDS), 48, _t(g["means3D"]), _t(g["rotations"]), _t(g["scales"]),
                      _t(g["opacities"]))["density"]
    level = float(den.max()) * 0.3
    got = _mc_both(den.contiguous(), level, tuple(float(x) for x in scenes.SCENE_BOUNDS))
    assert len(got["faces"]) > 100


@pytest.mark.parametrize("seed", range(3))
def test_marching_cubes_of_random_fields(seed):
    g = torch.Generator().manual_seed(seed)
    r = torch.randn(1, 1, 9, 7, 11, generator=g, dtype=torch.float64)
    f = torch.nn.functional.interpolate(r, size=(37, 29, 45), mode="trilinear", align_corners=True)[0, 0].float()
    f.view(-1)[torch.randint(0, f.numel(), (40,), generator=g)] = float("nan")
    w = (torch.rand(f.shape, generator=g) > 0.02).float()
    col = torch.randn(5, *f.shape, generator=g)
    b = (-1.0, 0.5, 2.0, 1.5, 2.0, 4.5)
    got = _mc_both(f.cuda(), 0.1, b, weight=w.cuda(), color=col.cuda())
    assert len(got["faces"]) > 1000
    _mc_both(f.cuda(), -0.2, b)
    # a value exactly at the level: zero-area triangles are kept, as the reference keeps them
    q = torch.round(f * 4) / 4
    _mc_both(q.cuda(), 0.25, b)


def test_marching_cubes_of_one_cell_and_empty_grids():
    from manigaussian_b200 import gaussian_renderer as GR
    b = (0, 0, 0, 1, 1, 1)
    for case in (1, 0x69, 0x3c, 0x7e, 0xff, 0):
        v = torch.tensor([1.0 - 2.0 * ((case >> c) & 1) for c in range(8)]).reshape(2, 2, 2)
        v = v.permute(2, 1, 0).contiguous()  # corner c at (c & 1, (c >> 1) & 1, (c >> 2) & 1)
        got = _mc_both(v.cuda(), 0.0, b)
        assert len(got["faces"]) == int(M.COUNT[case])
    for shape in ((1, 4, 4), (4, 1, 4), (3, 3, 0)):
        out = GR.marching_cubes(torch.zeros(shape, device="cuda"), 0.0, b, color=torch.zeros((2,) + shape, device="cuda"))
        assert out["vertices"].shape == (0, 3) and out["faces"].shape == (0, 3) and out["colors"].shape == (0, 2)
    out = GR.marching_cubes(torch.ones(5, 5, 5, device="cuda"), 0.0, b)
    assert out["vertices"].shape == (0, 3) and out["colors"] is None


# --------------------------------------------------------------------------- 4. accuracy
def _box_sdf(p, lo, hi):
    c, h = (lo + hi) / 2, (hi - lo) / 2
    q = np.abs(p - c) - h
    return np.linalg.norm(np.maximum(q, 0), axis=1) + np.minimum(q.max(1), 0)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("shape", ["sphere", "box"])
def test_fused_analytic_shapes_give_closed_meshes_within_a_voxel(model, shape):
    """Where every grid point's fused tsdf has the sign of the true signed distance, each vertex lies on a grid edge the
    surface crosses, so within one voxel of it.  Along a box's convex edges a view behind the edge sees a voxel just
    outside it through less than trunc of box and counts it negative (projective TSDF): there, within trunc of an edge,
    the bound is trunc."""
    from manigaussian_b200 import gaussian_renderer as GR
    views, _ = _ring(160, 120, (model,), heights=(-0.9, 0.4, 1.5), per_ring=8)  # 24 views
    lo, hi = CENTRE - np.array([0.25, 0.2, 0.15]), CENTRE + np.array([0.2, 0.25, 0.3])
    depth = _sphere_depth(views) if shape == "sphere" else _box_depth(views, lo, hi)
    n = 64
    voxel = (BOUNDS[3] - BOUNDS[0]) / n
    trunc = 4 * voxel
    vol = GR.tsdf_fuse(views, depth, BOUNDS, n, trunc)
    mesh = GR.marching_cubes(vol["tsdf"], 0.0, BOUNDS, weight=vol["weight"])
    v, f = mesh["vertices"], mesh["faces"]
    closed, used = _manifold(v, f)
    assert closed and used and len(f) > 1000, (model, shape, len(f))
    p = v.cpu().double().numpy()
    if shape == "sphere":
        dist, edge = np.abs(np.linalg.norm(p - CENTRE, axis=1) - R_SPHERE), np.zeros(len(p), bool)
    else:
        dist = np.abs(_box_sdf(p, lo, hi))
        q = np.abs(np.abs(p - (lo + hi) / 2) - (hi - lo) / 2)
        edge = (q < trunc).sum(1) >= 2  # within trunc of two faces: near an edge
    far = dist[~edge].max()
    print(f"{shape} {model}: {len(f)} faces, max distance {far / voxel:.3f} voxel, {dist[edge].max(initial=0) / voxel:.3f} "
          f"voxel near the edges")
    assert far <= voxel and dist[edge].max(initial=0) <= trunc


# --------------------------------------------------------------------------- 5. end to end
def test_rendered_planar_depth_of_a_gaussian_sphere_fuses_into_a_closed_mesh_near_it():
    """Gaussians on the sphere |x - c| = 0.3, flat along its normal (sigma 0.008 along the surface, 0.001 across), rendered
    with planar depth in 12 views; depth / alpha is fused where alpha > 0.99.  Fusion with nearest-pixel depth places the
    zero crossing within one voxel (0.014) of the surface the depth images show (test 4).  Those images lie within one more
    voxel of the sphere: a pixel's depth / alpha blends the tangent planes of the Gaussians covering it, whose centres lie
    up to 3 sigma = 0.024 apart on the sphere, and a tangent plane leaves the sphere by d^2 / (2 R) <= 0.001 at distance
    d = 0.024 on a face-on pixel but by up to d tan(angle) toward the silhouette.  So every vertex is within 2 voxels."""
    from manigaussian_b200 import gaussian_renderer as GR
    rng = np.random.default_rng(8)
    P = 40000
    nrm = rng.standard_normal((P, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    xyz = CENTRE + R_SPHERE * nrm
    # the rotation taking +z to the normal: q = normalize(1 + n_z, -n_y, n_x, 0)
    q = np.stack([1 + nrm[:, 2], -nrm[:, 1], nrm[:, 0], np.zeros(P)], -1)
    q[nrm[:, 2] < -0.999] = (0.0, 1.0, 0.0, 0.0)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    scales = np.tile([0.008, 0.008, 0.001], (P, 1))
    views, _ = _ring(128, 96, ("pinhole",), heights=(-0.8, 0.4, 1.4), per_ring=4)
    out = GR.render_views(views, _t(xyz), _t(q), _t(scales), _t(np.full((P, 1), 0.95)), pts_rgb=_t(np.zeros((P, 3))),
                          return_depth=True, return_alpha=True, planar_depth=True)
    depth, alpha = out["depth"].reshape(12, 96, 128), out["alpha"].reshape(12, 96, 128)
    z = torch.where(alpha > 0.99, depth / alpha, torch.zeros_like(depth)).detach().contiguous()
    assert float((alpha > 0.99).float().mean()) > 0.1
    n = 64
    voxel = (BOUNDS[3] - BOUNDS[0]) / n
    vol = GR.tsdf_fuse(views, z, BOUNDS, n, 4 * voxel)
    mesh = GR.marching_cubes(vol["tsdf"], 0.0, BOUNDS, weight=vol["weight"])
    closed, used = _manifold(mesh["vertices"], mesh["faces"])
    assert closed and used and len(mesh["faces"]) > 1000
    d = np.abs(np.linalg.norm(mesh["vertices"].cpu().double().numpy() - CENTRE, axis=1) - R_SPHERE)
    print(f"end to end: {len(mesh['faces'])} faces, max distance {d.max() / voxel:.3f} voxel")
    assert d.max() <= 2 * voxel


# --------------------------------------------------------------------------- 6. large and cross-device
def test_fusion_at_512_cubed_with_64_views_matches_the_reference_on_sampled_voxels():
    from manigaussian_b200 import gaussian_renderer as GR
    views, refs = _ring(640, 480, ("pinhole", "distorted"), heights=(-0.7, 0.4, 1.3), per_ring=22)
    views, refs = views[:64], refs[:64]
    depth = _sphere_depth(views)
    n, trunc = 512, 0.02
    vol = GR.tsdf_fuse(views, depth, BOUNDS, n, trunc)
    # 20,000 voxels anywhere and 20,000 within 2 trunc of the surface
    rng = np.random.default_rng(9)
    cs = [c.numpy() for c in M.axis_centres(BOUNDS, (n, n, n))]
    ijk = rng.integers(0, n, (400000, 3))
    pts = np.stack([cs[q][ijk[:, q]] for q in range(3)], -1)
    near = np.abs(np.linalg.norm(pts - CENTRE, axis=1) - R_SPHERE) < 2 * trunc
    pick = np.concatenate([np.arange(20000), rng.choice(np.nonzero(near)[0], 20000, replace=False)])
    idx = (ijk[pick, 0] * n + ijk[pick, 1]) * n + ijk[pick, 2]
    ts, w, _, border = T64.fuse(pts[pick], refs, depth.cpu().numpy(), trunc)
    keep = ~border
    gi = torch.as_tensor(idx, device="cuda")
    gw, gt = vol["weight"].view(-1)[gi].cpu().numpy(), vol["tsdf"].view(-1)[gi].cpu().numpy()
    # 64 views of 640 x 480: a voxel seen by many views is more often within a band of some pixel border
    print(f"512^3: border {100 * (1 - keep.mean()):.3f} % of {len(idx)} sampled voxels, weights differ on "
          f"{int((gw != w).sum())} ({int(((gw != w) & keep).sum())} not border)")
    assert np.array_equal(gw[keep], w[keep])
    assert np.abs(gt[keep] - ts[keep]).max() <= 1e-5
    assert keep.mean() > 0.6 and (w[keep] > 0).sum() > 10000


def test_a_call_on_a_non_current_device_gives_the_same_volume_and_mesh():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import gaussian_renderer as GR
    views, _ = _ring(64, 48, MODELS, per_ring=4)
    depth = _sphere_depth(views)
    ref = GR.tsdf_fuse(views, depth, BOUNDS, 32, 0.06)
    ref_mesh = GR.marching_cubes(ref["tsdf"], 0.0, BOUNDS, weight=ref["weight"])
    d1 = torch.device("cuda:1")
    mv = lambda x: x.to(d1) if torch.is_tensor(x) else x  # noqa: E731
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    views1 = [GaussianRasterizationSettings(*[mv(x) for x in s], orthographic=s.orthographic, fisheye=s.fisheye,
                                            distortion=s.distortion) for s in views]
    with torch.cuda.device(0):
        got = GR.tsdf_fuse(views1, depth.to(d1), BOUNDS, 32, 0.06)
        mesh = GR.marching_cubes(got["tsdf"], 0.0, BOUNDS, weight=got["weight"])
    assert got["tsdf"].device == d1 and torch.equal(got["tsdf"].cpu(), ref["tsdf"].cpu())
    _same_mesh(mesh, ref_mesh)
