"""Point visibility on the GPU (visibility.cu, mgs_visibility_views, gaussian_renderer.point_visibility).

1. Against the float64 reference (tests/visibility_ref64.py) for pinhole, orthographic, fisheye and distorted views, one call
   mixing all four, a device field-of-view camera and the anti-aliased mode: uv and depth against the reference's
   projection, in_view away from the image edges, and T at the kernel's (u, v, d) on the view's own projected and sorted
   state (read back from a render of the same view), excluding points with a borderline decision.
2. Against the render, bit for bit: points on the pixel centres' rays, far behind the scene, give T == final_T.
3. Scale: 100^3 voxel centres x 4 views at c3's size (500k Gaussians), against the reference on a seeded subsample; Q not a
   multiple of 32, every point in one tile, points outside every view, a view that no Gaussian reaches.
4. CUDA-graph capture and replay give the eager outputs; a call on a non-current device gives the same outputs.
"""
import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
import visibility_ref64 as V64
from test_planar_depth_gpu import MODELS, _inputs, _model_kw, _settings, _t

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _states(views, g, aa=False, tan_fov=None):
    """per view the projected and sorted state of a render of the same views (the visibility call's front end)"""
    from manigaussian_b200 import rasterizer as R
    P = g["means3D"].shape[0]
    outs, _ = R.rasterize_views_raw(views, _t(g["means3D"]), None, None, _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]),
                                    1.0, None, _t(g["shs"]), g["sh_degree"], False, return_alpha=True, antialiasing=aa,
                                    tan_fov=tan_fov)
    torch.cuda.synchronize()
    sts = []
    for s, o in zip(views, outs):
        assert not o.overflowed()
        W, H = int(s.image_width), int(s.image_height)
        cap, Rn = int(o[0]), o.num_rendered()
        T = ((W + 15) // 16) * ((H + 15) // 16)

        def arr(which, name, state, a0, a1, dtype, count):
            off = R.state_array(which, name, state, a0, a1) - state.data_ptr()
            n = count * torch.empty((), dtype=dtype).element_size()
            return state[off:off + n].view(dtype).cpu().numpy()

        sts.append(dict(
            W=W, H=H,
            means2D=arr("geometry", "means2D", o[4], P, 0, torch.float32, 2 * P).reshape(P, 2),
            conic_opacity=arr("geometry", "conic_opacity", o[4], P, 0, torch.float32, 4 * P).reshape(P, 4),
            depths=arr("geometry", "depths", o[4], P, 0, torch.float32, P),
            point_list=arr("binning", "point_list", o[5], cap, 0, torch.int32, Rn).view(np.uint32),
            ranges=arr("image", "ranges", o[6], W, H, torch.int32, 2 * T).view(np.uint32).reshape(T, 2),
            final_T=arr("image", "final_T", o[6], W, H, torch.float32, W * H).reshape(H, W)))
    return sts


def _points(g, Q, seed=0):
    """points near the cloud's Gaussians (on, in front of and behind surfaces), a spread around it, and a few far away"""
    rng = np.random.default_rng(seed)
    m = np.asarray(g["means3D"], np.float64)
    near = m[rng.integers(0, len(m), Q - Q // 4)] + 0.05 * rng.standard_normal((Q - Q // 4, 3))
    lo, hi = m.min(0), m.max(0)
    spread = rng.uniform(lo - 0.5 * (hi - lo), hi + 0.5 * (hi - lo), (Q // 4, 3))
    pts = np.concatenate([near, spread]).astype(np.float32)
    pts[:5] = [[0, 0, -50], [1e4, 0, 0], [0, 1e4, 0], [-1e4, -1e4, 1e4], [np.nan, 0, 0]]
    return pts


def _check_view(st, view, pts, uv, depth, inv, T, tag):
    """uv / depth / in_view against the reference's projection, T against the reference at the kernel's own (u, v, d)"""
    ruv, rd, rok = V64.project(pts.astype(np.float64), view)
    ok = rok & np.isfinite(uv[:, 0])
    W, H = st["W"], st["H"]
    # the cull of the map: equal away from its threshold (near plane)
    clear = ~(np.abs(np.nan_to_num(rd, nan=1e9) - 0.2) < 1e-4)
    assert np.array_equal(np.isfinite(uv[clear, 0]), rok[clear]), tag
    assert np.abs(uv[ok] - ruv[ok]).max() <= 1e-3 + 1e-5 * np.abs(ruv[ok]).max(), tag
    assert np.allclose(depth[ok], rd[ok], rtol=1e-5, atol=1e-5), tag
    rin = V64.in_view(ruv, rok, W, H)
    edge = np.zeros(len(pts), bool)
    with np.errstate(invalid="ignore"):
        for c, S in ((0, W), (1, H)):
            edge |= (np.abs(ruv[:, c] + 0.5) < 1e-3) | (np.abs(ruv[:, c] - (S - 0.5)) < 1e-3)
    assert np.array_equal(inv[clear & ~edge], rin[clear & ~edge]), tag
    assert (T[~inv] == 1.0).all(), tag
    rT, border = V64.transmittance(st, uv.astype(np.float64), depth.astype(np.float64), inv)
    keep = inv & ~border
    print(f"[{tag}] {inv.sum()} points in view, {keep.sum()} clear of every decision band")
    assert keep.sum() > 0.6 * inv.sum() and inv.sum() > 0, (tag, keep.sum(), inv.sum())
    err = np.abs(T[keep] - rT[keep])
    assert (err <= 2e-6 + 1e-4 * rT[keep]).all(), (tag, float(err.max()))
    return keep.sum()


def _run(views, g, pts, aa=False, tan_fov=None):
    from manigaussian_b200 import rasterizer as R
    out = R.visibility_views_raw(views, _t(g["means3D"]), _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]), 1.0, None,
                                 _t(pts), antialiasing=aa, tan_fov=tan_fov)
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in out]


# --------------------------------------------------------------------------- 1. against the reference
@pytest.mark.parametrize("model,aa", [(m, False) for m in MODELS] + [("pinhole", True), ("fisheye", True)])
def test_matches_the_float64_reference(model, aa):
    inps, g = _inputs(4000, 96, 64, 0, 1)
    views = [_settings(inps[0], 0, model, aa)]
    pts = _points(g, 3001)
    uv, depth, inv, T = _run(views, g, pts, aa)
    st = _states(views, g, aa)[0]
    _check_view(st, _model_kw(inps[0], model)[1], pts, uv[0], depth[0], inv[0].astype(bool), T[0], (model, aa))
    live = inv[0].astype(bool)
    assert (T[0][live] < 0.5).any() and (T[0][live] == 1).any()


def test_one_call_mixing_all_four_models_and_a_device_fov():
    inps, g = _inputs(4000, 80, 72, 0, 4)
    views = [_settings(inps[v], 0, m) for v, m in enumerate(MODELS)]
    pts = _points(g, 2500, seed=1)
    got = _run(views, g, pts)
    sts = _states(views, g)
    for v, m in enumerate(MODELS):
        _check_view(sts[v], _model_kw(inps[v], m)[1], pts, got[0][v], got[1][v], got[2][v].astype(bool), got[3][v], m)
        # each view alone gives the same outputs
        one = _run([views[v]], g, pts)
        for a, b in zip(got, one):
            assert np.array_equal(a[v], b[0], equal_nan=True)
    # the field of view on the device gives the host one's outputs
    tf = torch.tensor([[float(s.tanfovx), float(s.tanfovy)] for s in views], device="cuda")
    dev = _run(views, g, pts, tan_fov=tf)
    for a, b in zip(got, dev):
        assert np.array_equal(a, b, equal_nan=True)


def test_point_visibility_takes_a_camera_batch_with_a_learnable_fov():
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import camera_batch
    from test_camera_grad_gpu import _intr, _scene, _w2c
    V, W, H = 3, 96, 80
    sc = _scene(5000, sh=False, seed=4)
    K = torch.tensor(_intr(V, W, H), dtype=torch.float32, device="cuda").requires_grad_()
    cams = camera_batch(_w2c(V, seed=V), K, W, H)
    pts = sc["pts_xyz"][:2000].detach() + 0.02 * torch.randn(2000, 3, device="cuda")
    out = GR.point_visibility(cams, pts, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"])
    assert out["uv"].shape == (V, 2000, 2) and out["in_view"].dtype == torch.bool
    assert not any(t.requires_grad for t in out.values())
    # the same cameras with the field of view held on the host: the same map up to the matrices' rounding
    hcams = camera_batch(_w2c(V, seed=V), K.detach(), W, H)
    ref = GR.point_visibility(hcams, pts, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"])
    both = out["in_view"] & ref["in_view"]
    assert float(both.float().sum()) >= 0.99 * float(ref["in_view"].float().sum())
    assert torch.allclose(out["uv"][both], ref["uv"][both], rtol=0, atol=1e-3)
    assert float((out["transmittance"][both] - ref["transmittance"][both]).abs().mean()) < 1e-3
    assert bool((out["transmittance"][out["in_view"]] < 0.5).any())
    one = GR.point_visibility(cams, pts, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], view_ids=[2])
    assert torch.equal(one["transmittance"][0], out["transmittance"][2])


# --------------------------------------------------------------------------- 2. against the render, bit for bit
def _pixel_rays(view, W, H, z):
    """float64 world points at view-space depth z whose float64 projection is each pixel centre (Newton on the reference)"""
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).T
    c2w = np.linalg.inv(vm)
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    target = np.stack([xx.ravel(), yy.ravel()], 1)
    ortho = bool(view.get("ortho"))
    fx, fy = W / (2 * view["tanfovx"]), H / (2 * view["tanfovy"])
    t = np.stack([(target[:, 0] - (W - 1) / 2) / fx * (1 if ortho else z), (target[:, 1] - (H - 1) / 2) / fy * (1 if ortho else z),
                  np.full(len(target), z)], 1)

    def world(tt):
        return tt @ c2w[:3, :3].T + c2w[:3, 3]

    for _ in range(8):
        uv, _, _ = V64.project(world(t), view)
        h = 1e-6 * (1 if ortho else z)
        J = np.empty((len(t), 2, 2))
        for k in range(2):
            dt = t.copy()
            dt[:, k] += h
            J[:, :, k] = (V64.project(world(dt), view)[0] - uv) / h
        t[:, :2] += np.linalg.solve(J, (target - uv)[:, :, None])[:, :, 0]
    return world(t), target


@pytest.mark.parametrize("model", MODELS)
def test_pixel_centres_behind_the_scene_give_final_T_bit_for_bit(model):
    from manigaussian_b200 import rasterizer as R
    W, H = 64, 48
    inps, g = _inputs(3000, W, H, 0, 1, seed=7)
    views = [_settings(inps[0], 0, model)]
    view = _model_kw(inps[0], model)[1]
    st = _states(views, g)[0]
    z = float(st["depths"][np.isfinite(st["depths"])].max()) * 1.05 + 0.1
    pts, target = _pixel_rays(view, W, H, z)
    p32 = pts.astype(np.float32)
    # a few rounds of fp32 Newton on the kernel's own uv, so that most points land exactly on their pixel centre
    for _ in range(3):
        uv = _run(views, g, p32)[0][0].astype(np.float64)
        miss = np.any(uv != target, 1)
        if not miss.any():
            break
        uv64, _, _ = V64.project(p32.astype(np.float64), view)
        eps = 1e-4
        dj = []
        for k in range(3):
            d = p32.astype(np.float64).copy()
            d[:, k] += eps
            dj.append((V64.project(d, view)[0] - uv64) / eps)
        Jw = np.stack(dj, 2)  # [Q,2,3]
        corr = np.einsum("qij,qj->qi", np.linalg.pinv(Jw), target - uv)
        p32 = np.where(miss[:, None], (p32.astype(np.float64) + corr).astype(np.float32), p32)
    uv, depth, inv, T = (x[0] for x in _run(views, g, p32))
    exact = np.all(uv.astype(np.float64) == target, 1) & inv.astype(bool) & (depth > st["depths"][np.isfinite(st["depths"])].max())
    print(f"[{model}] {exact.sum()} of {W * H} pixel centres hit exactly")
    assert exact.sum() >= 0.3 * W * H
    fT = st["final_T"].ravel()
    assert np.array_equal(T[exact].view(np.uint32), fT[exact].view(np.uint32))
    assert (fT[exact] < 1).sum() > exact.sum() // 4
    R.reset_capacity_estimates()


# --------------------------------------------------------------------------- 3. scale and edges
def test_voxel_centres_at_c3_size_match_the_reference_on_a_subsample():
    import bench
    from manigaussian_b200 import GaussianRasterizationSettings, gaussian_renderer as GR, scenes
    wl = bench.WORKLOADS["c3"]
    P, V, W, H = wl["P"], wl["views"], wl["W"], wl["H"]
    g = scenes.make_gaussians(P, F=0, sh_degree=bench.SH_DEGREE, seed=1234)
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, _t(c["viewmatrix"]), _t(c["projmatrix"]),
                                           bench.SH_DEGREE, _t(c["campos"]), False, False, False) for c in cams]
    pts, _ = GR.voxel_centres(scenes.SCENE_BOUNDS, 100, "cuda")
    out = GR.point_visibility(views, pts, _t(g["means3D"]), _t(g["rotations"]), _t(g["scales"]), _t(g["opacities"]))
    sts = _states(views, g)
    rng = np.random.default_rng(2)
    p = pts.cpu().numpy()
    for v, c in enumerate(cams):
        sub = rng.choice(len(p), 400, replace=False)
        view = dict(viewmatrix=np.asarray(c["viewmatrix"], np.float64).reshape(-1),
                    projmatrix=np.asarray(c["projmatrix"], np.float64).reshape(-1), W=W, H=H, tanfovx=float(c["tanfovx"]),
                    tanfovy=float(c["tanfovy"]))
        _check_view(sts[v], view, p[sub], out["uv"][v, sub].cpu().numpy(), out["depth"][v, sub].cpu().numpy(),
                    out["in_view"][v, sub].cpu().numpy(), out["transmittance"][v, sub].cpu().numpy(), ("c3", v))
        assert float(out["in_view"][v].float().mean()) > 0.5


def test_edges_ragged_q_one_tile_outside_and_an_empty_view():
    inps, g = _inputs(3000, 96, 64, 0, 2)
    views = [_settings(inps[0], 0), _settings(inps[1], 0)]
    st = _states(views, g)
    view0 = _model_kw(inps[0], "pinhole")[1]
    # Q not a multiple of 32, and every point of one call in a single tile (a pixel ray, at depths through the scene)
    for Q in (1, 31, 33, 1000, 4099):
        pts = _points(g, max(Q, 8), seed=Q)[-Q:]
        uv, depth, inv, T = _run(views, g, pts)
        for v in range(2):
            if inv[v].sum() >= 5:
                _check_view(st[v], _model_kw(inps[v], "pinhole")[1], pts, uv[v], depth[v], inv[v].astype(bool), T[v], (Q, v))
    ray, _ = _pixel_rays(view0, 96, 64, 1.0)
    centre = ray[64 // 2 * 96 + 96 // 2]
    vm = np.asarray(view0["viewmatrix"], np.float64).reshape(4, 4).T
    cam = np.linalg.inv(vm)[:3, 3]
    s = np.linspace(0.3, 8.0, 3000)[:, None]
    pts = (cam + s * (centre - cam)).astype(np.float32)
    uv, depth, inv, T = _run(views[:1], g, pts)
    tiles = V64.tile_of(uv[0].astype(np.float64), 96, 64)
    assert inv[0].all() and len(set(tiles.tolist())) == 1
    _check_view(st[0], view0, pts, uv[0], depth[0], inv[0].astype(bool), T[0], "one tile")
    # fp32 moves the ray's screen position by ~1e-5 px along it: T may rise by that much
    assert np.all(np.diff(T[0]) <= 1e-6) and T[0][0] == 1.0 and T[0][-1] < 1.0
    # points outside every view
    far = np.array([[0, 0, -100], [100, 100, 100], [-1e3, 0, 0]], np.float32).repeat(40, 0)
    uv, depth, inv, T = _run(views, g, far)
    assert not inv.any() and (T == 1.0).all()
    # a view that no Gaussian reaches: the cloud sits behind its camera
    moved = dict(g, means3D=(np.asarray(g["means3D"]) * 0.01 + np.array([0, 0, -50], np.float32)).astype(np.float32))
    pts = _points(g, 500)
    uv, depth, inv, T = _run(views, moved, pts)
    assert inv.any() and (T == 1.0).all()


# --------------------------------------------------------------------------- 4. graph capture, other device
def test_cuda_graph_capture_and_replay_give_the_eager_outputs():
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(4000, 96, 64, 0, 2)
    views = [_settings(inps[0], 0, "pinhole"), _settings(inps[1], 0, "fisheye")]
    m, o, s, r = _t(g["means3D"]), _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"])
    pts = _t(_points(g, 2000))
    eager = GR.point_visibility(views, pts, m, r, s, o)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        GR.point_visibility(views, pts, m, r, s, o)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = GR.point_visibility(views, pts, m, r, s, o)
    pts.copy_(pts.flip(0))
    graph.replay()
    torch.cuda.synchronize()
    flipped = GR.point_visibility(views, pts, m, r, s, o)
    for k in eager:
        a, b = torch.nan_to_num(cap[k].float(), 7.0), torch.nan_to_num(flipped[k].float(), 7.0)
        assert torch.equal(a, b), k
        assert torch.equal(torch.nan_to_num(eager[k].float(), 7.0).flip(1), a), k


def test_a_call_on_a_non_current_device_gives_the_same_outputs():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(3000, 96, 64, 0, 1)
    views = [_settings(inps[0], 0)]
    pts = _points(g, 1500)
    ref = GR.point_visibility(views, _t(pts), *[x for x in (_t(g["means3D"]), _t(g["rotations"]), _t(g["scales"]), _t(g["opacities"]))])
    d1 = torch.device("cuda:1")
    mv = lambda x: x.to(d1)  # noqa: E731
    s1 = views[0]._replace(bg=mv(views[0].bg), viewmatrix=mv(views[0].viewmatrix), projmatrix=mv(views[0].projmatrix),
                           campos=mv(views[0].campos))
    with torch.cuda.device(0):
        got = GR.point_visibility([s1], mv(_t(pts)), mv(_t(g["means3D"])), mv(_t(g["rotations"])), mv(_t(g["scales"])),
                                  mv(_t(g["opacities"])))
    for k in ref:
        assert got[k].device == d1
        assert torch.equal(torch.nan_to_num(got[k].cpu().float(), 7.0), torch.nan_to_num(ref[k].cpu().float(), 7.0)), k
