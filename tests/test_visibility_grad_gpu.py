"""The point-visibility backward on the GPU (visibility.cu, mgs_visibility_views_backward, point_visibility(differentiable=True)).

1. Against the float64 reference (tests/visibility_grad_ref64.py) per camera model, with and without the anti-aliased mode,
   with a device field of view and in one call mixing all four models: the gradients of a random weighted sum of T, uv and
   depth (T's weights zero on points with a borderline decision, uv's and depth's arbitrary where the cull fails) to the
   points, means, scales, rotations, opacities, view and projection matrices and tan_fov, within rel-L2 1e-4.
2. Against the render: points at pixel centres behind the scene have T == final_T, so the cloud's gradients of sum c T match
   render_views(return_alpha=True)'s backward of -sum c alpha at those pixels.
3. The default path is unchanged; only the requested gradients are computed; Q = 0, points behind the camera or outside
   every view, a view no Gaussian reaches, ragged Q, and 100^3 voxel centres at c3 size against the reference on a subsample.
4. CUDA-graph capture of forward + backward and replay on new values; a non-current device.
"""
import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
import visibility_grad_ref64 as VG
from test_planar_depth_gpu import MODELS, _inputs, _model_kw, _settings, _t
from test_visibility_gpu import _pixel_rays, _points, _states

pytestmark = pytest.mark.gpu
D64 = torch.float64
TOL = 1e-4


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _rel(got, ref):
    got, ref = (x.detach().cpu().numpy() if torch.is_tensor(x) else x for x in (got, ref))
    got, ref = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
    return float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))


def _cotangents(uv, inv, border, seed):
    """T's weights on in-view points clear of every decision band; uv's and depth's everywhere (NaN outputs ignore theirs)"""
    rng = np.random.default_rng(seed)
    V, Q = inv.shape
    cT = rng.standard_normal((V, Q)) * (inv & ~border)
    cuv = rng.standard_normal((V, Q, 2)) * 0.01
    cd = rng.standard_normal((V, Q)) * 0.1
    return cT.astype(np.float32), cuv.astype(np.float32), cd.astype(np.float32)


def _gpu(views, g, pts, cot, aa=False, tan_fov=None, want_points=True, want_cloud=True, camera=True):
    from manigaussian_b200 import rasterizer as R
    m, o, s, r = _t(g["means3D"]), _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"])
    uv, d, inv, T, state = R.visibility_views_raw(views, m, o, s, r, 1.0, None, _t(pts), antialiasing=aa, tan_fov=tan_fov,
                                                  keep_state=True)
    out = R.visibility_views_backward_raw(state, _t(pts), m, o, s, r, 1.0, None, T, *(_t(c) if c is not None else None for c in cot),
                                          want_points=want_points, want_cloud=want_cloud, camera_grads=camera)
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (uv, d, inv, T)], out


def _reference(refviews, g, pts, accs, cot, aa=False, device_fov=False):
    """float64 gradients of the weighted sum: points, means, scales, rotations, opacities, then per view vm, pm, tan_fov"""
    # a non-finite point receives nothing: it enters as a masked zero row
    fin = np.isfinite(np.asarray(pts, np.float64)).all(1)
    pts = np.where(fin[:, None], np.asarray(pts, np.float64), 0.0)
    leaves = [torch.tensor(np.asarray(x, np.float64), requires_grad=True)
              for x in (pts, g["means3D"], g["scales"], g["rotations"], g["opacities"])]
    cams = []
    total = 0.0
    for v, (view, acc) in enumerate(zip(refviews, accs)):
        vm = torch.tensor(np.asarray(view["viewmatrix"], np.float64), requires_grad=True)
        pm = torch.tensor(np.asarray(view["projmatrix"], np.float64), requires_grad=True)
        tf = torch.tensor([view["tanfovx"], view["tanfovy"]], dtype=D64, requires_grad=True)
        cams += [vm, pm, tf]
        w = dict(view, viewmatrix=vm, projmatrix=pm, tanfovx=tf[0] if device_fov else view["tanfovx"],
                 tanfovy=tf[1] if device_fov else view["tanfovy"])
        uv, d, T = VG.outputs(leaves[0], leaves[1], leaves[4], w, acc, scales=leaves[2], rotations=leaves[3], antialias=aa)
        ok = torch.isfinite(uv[:, 0]) & VG.F64.valid(leaves[0].detach(), view) & torch.as_tensor(fin)
        cT, cuv, cd = (torch.tensor(np.asarray(c[v], np.float64)) for c in cot)
        total = total + (cT * T).sum() + (cuv[ok] * uv[ok]).sum() + (cd[ok] * d[ok]).sum()
    gr = torch.autograd.grad(total, leaves + cams, allow_unused=True)
    # a fisheye or distorted view's screen means do not read its projection matrix: its gradient is 0
    return [np.zeros(x.shape) if g_ is None else g_.numpy() for x, g_ in zip(leaves + cams, gr)]


def _compare(views, refviews, g, pts, aa=False, tan_fov=None, tag=""):
    from manigaussian_b200 import rasterizer as R
    (uv, d, inv, T), _ = _gpu(views, g, pts, (None, None, None), aa=aa, tan_fov=tan_fov, camera=False, want_cloud=False)
    sts = _states(views, g, aa, tan_fov)
    accs, borders = [], []
    for v in range(len(views)):
        acc, border = VG.decisions(sts[v], uv[v].astype(np.float64), d[v].astype(np.float64), inv[v].astype(bool))
        accs.append(acc)
        borders.append(border)
    inv = inv.astype(bool)
    cot = _cotangents(uv, inv, np.stack(borders), seed=len(pts))
    R.reset_capacity_estimates()
    _, (dp, dm, dop, ds, dr, cam) = _gpu(views, g, pts, cot, aa=aa, tan_fov=tan_fov)
    ref = _reference(refviews, g, pts, accs, cot, aa=aa, device_fov=tan_fov is not None)
    errs = dict(points=_rel(dp, ref[0]), means=_rel(dm, ref[1]), scales=_rel(ds, ref[2]), rotations=_rel(dr, ref[3]),
                opacities=_rel(dop, ref[4]))
    V = len(views)
    errs["viewmatrix"] = _rel(cam[0], np.stack([ref[5 + 3 * v] for v in range(V)]))
    errs["projmatrix"] = _rel(cam[1], np.stack([ref[6 + 3 * v] for v in range(V)]))
    if tan_fov is not None:
        errs["tan_fov"] = _rel(cam[3], np.stack([ref[7 + 3 * v] for v in range(V)]))
    assert (cam[2].cpu().numpy() == 0).all()  # no SHs: no camera-centre term
    print(f"[{tag}] {int(inv.sum())} in view, rel-L2 " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert e <= TOL, (tag, k, e)
    return errs


# --------------------------------------------------------------------------- 1. against the reference
@pytest.mark.parametrize("model,aa", [(m, False) for m in MODELS] + [("pinhole", True), ("fisheye", True)])
def test_gradients_match_the_float64_reference(model, aa):
    inps, g = _inputs(3000, 96, 64, 0, 1)
    _compare([_settings(inps[0], 0, model, aa)], [_model_kw(inps[0], model)[1]], g, _points(g, 2001), aa=aa, tag=(model, aa))


def test_one_call_mixing_all_four_models_with_a_device_fov():
    inps, g = _inputs(3000, 80, 72, 0, 4)
    views = [_settings(inps[v], 0, m) for v, m in enumerate(MODELS)]
    refviews = [_model_kw(inps[v], m)[1] for v, m in enumerate(MODELS)]
    tf = torch.tensor([[float(s.tanfovx), float(s.tanfovy)] for s in views], device="cuda")
    _compare(views, refviews, g, _points(g, 1500, seed=1), tan_fov=tf, tag="mixed+fov")


# --------------------------------------------------------------------------- 2. against the render
@pytest.mark.parametrize("model", ["pinhole", "fisheye"])
def test_cloud_gradients_of_T_at_pixel_centres_match_the_alpha_plane_backward(model):
    from manigaussian_b200 import gaussian_renderer as GR
    W, H = 64, 48
    inps, g = _inputs(3000, W, H, 0, 1, seed=7)
    views = [_settings(inps[0], 0, model)]
    view = _model_kw(inps[0], model)[1]
    st = _states(views, g)[0]
    z = float(st["depths"][np.isfinite(st["depths"])].max()) * 1.05 + 0.1
    pts, target = _pixel_rays(view, W, H, z)
    # fp32 Newton on the kernel's own uv, so that most points land exactly on their pixel centre
    p32 = pts.astype(np.float32)
    for _ in range(3):
        uv = GR.point_visibility(views, _t(p32), *(_t(g[k]) for k in ("means3D", "rotations", "scales", "opacities")))["uv"][0]
        uv = uv.double().cpu().numpy()
        miss = np.any(uv != target, 1)
        base, _, _ = VG.V64.project(p32.astype(np.float64), view)
        Jw = np.stack([(VG.V64.project(p32.astype(np.float64) + 1e-4 * np.eye(3)[k], view)[0] - base) / 1e-4 for k in range(3)], 2)
        corr = np.einsum("qij,qj->qi", np.linalg.pinv(Jw), target - uv)
        p32 = np.where(miss[:, None], (p32.astype(np.float64) + corr).astype(np.float32), p32)
    p32 = _t(p32)
    leaves = [_t(g[k]).requires_grad_() for k in ("means3D", "rotations", "scales", "opacities")]
    out = GR.point_visibility(views, p32, *leaves, differentiable=True)
    T = out["transmittance"][0]
    uv = out["uv"][0].detach().double().cpu().numpy()
    exact = torch.tensor(np.all(uv == target, 1), device="cuda") & out["in_view"][0]
    assert bool((T[exact] == _t(st["final_T"].ravel())[exact]).all())
    c = torch.randn(H * W, device="cuda") * exact
    ours = torch.autograd.grad((c * T).sum(), leaves)
    rl = [_t(g[k]).requires_grad_() for k in ("means3D", "rotations", "scales", "opacities")]
    ren = GR.render_views(views, rl[0], rl[1], rl[2], rl[3], pts_rgb=torch.zeros(rl[0].shape[0], 3, device="cuda"),
                          return_alpha=True)
    theirs = torch.autograd.grad(-(c.view(H, W) * ren["alpha"][0]).sum(), rl)
    errs = [_rel(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(ours, theirs)]
    print(f"[{model}] {int(exact.sum())} exact pixel centres, rel-L2 means/rotations/scales/opacities {errs}")
    assert max(errs) <= TOL, errs


# --------------------------------------------------------------------------- 3. behaviour and edges
def test_default_unchanged_and_differentiable_forward_bitwise_equal():
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(3000, 96, 64, 0, 2)
    views = [_settings(inps[0], 0), _settings(inps[1], 0, "fisheye")]
    pts = _t(_points(g, 1000))
    cloud = [_t(g[k]).requires_grad_() for k in ("means3D", "rotations", "scales", "opacities")]
    a = GR.point_visibility(views, pts.requires_grad_(), *cloud)
    b = GR.point_visibility(views, pts, *cloud, differentiable=True)
    for k in a:
        assert a[k].grad_fn is None and not a[k].requires_grad
        assert torch.equal(torch.nan_to_num(a[k].float(), 7.0), torch.nan_to_num(b[k].float(), 7.0)), k
    assert b["transmittance"].grad_fn is not None and b["in_view"].dtype == torch.bool and not b["in_view"].requires_grad


def test_only_requested_gradients_are_computed():
    inps, g = _inputs(3000, 96, 64, 0, 1)
    views = [_settings(inps[0], 0)]
    pts = _points(g, 800)
    (uv, d, inv, T), _ = _gpu(views, g, pts, (None, None, None), camera=False, want_cloud=False)
    cot = _cotangents(uv, inv.astype(bool), np.zeros_like(inv, bool), 5)
    _, full = _gpu(views, g, pts, cot)
    _, pts_only = _gpu(views, g, pts, cot, want_cloud=False, camera=False)
    _, cloud_only = _gpu(views, g, pts, cot, want_points=False, camera=False)
    _, cam_only = _gpu(views, g, pts, cot, want_points=False, want_cloud=False)
    assert pts_only[1:5] == (None,) * 4 and pts_only[5] is None and torch.equal(pts_only[0], full[0])
    assert cloud_only[0] is None and cloud_only[5] is None
    for a, b in zip(cloud_only[1:5], full[1:5]):
        assert _rel(a.cpu().numpy(), b.cpu().numpy()) <= 1e-6
    assert cam_only[0] is None and cam_only[1:5] == (None,) * 4
    for a, b in zip(cam_only[5][:3], full[5][:3]):
        assert _rel(a.cpu().numpy(), b.cpu().numpy()) <= 1e-5



@pytest.mark.parametrize("need", ["points", "means", "opacity", "scales_rotations", "camera", "all"])
def test_the_autograd_node_asks_only_for_the_gradients_autograd_needs(need, monkeypatch):
    """the node passes exactly the inputs that require grad to the backward call, and returns None for the others; the values
    it returns equal those of a call that asks for everything"""
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import camera_batch
    from test_camera_grad_gpu import _intr, _scene, _w2c
    sc = _scene(3000, sh=False, seed=2)
    pts0 = sc["pts_xyz"][:700].detach() + 0.02 * torch.randn(700, 3, device="cuda")
    seen = []
    real = GR.visibility_views_backward_raw

    def spy(*args, **kw):
        seen.append((kw["want_points"], tuple(bool(x) for x in kw["want_cloud"]), bool(kw["camera_grads"])))
        return real(*args, **kw)

    def run(which):
        w2c = _w2c(2, seed=2).requires_grad_("camera" in which)
        cams = camera_batch(w2c, _intr(2, 96, 80), 96, 80)
        p = pts0.clone().requires_grad_("points" in which)
        cl = {k: sc[k].detach().clone().requires_grad_(k in which) for k in ("pts_xyz", "rotations", "scales", "opacity")}
        out = GR.point_visibility(cams, p, cl["pts_xyz"], cl["rotations"], cl["scales"], cl["opacity"], differentiable=True)
        loss = (out["transmittance"] * torch.arange(out["transmittance"].numel(), device="cuda").view_as(out["transmittance"])
                .remainder(7)).sum() + torch.nan_to_num(out["uv"]).sum() * 1e-2 + torch.nan_to_num(out["depth"]).sum()
        named = dict(points=p, camera=w2c, **cl)
        keys = [k for k in named if k in which]
        return dict(zip(keys, torch.autograd.grad(loss, [named[k] for k in keys])))

    every = ("points", "camera", "pts_xyz", "rotations", "scales", "opacity")
    which = dict(points=("points",), means=("pts_xyz",), opacity=("opacity",), scales_rotations=("scales", "rotations"),
                 camera=("camera",), all=every)[need]
    full = run(every)
    monkeypatch.setattr(GR, "visibility_views_backward_raw", spy)
    got = run(which)
    # want_cloud in the raw call's order: means, opacity, scales, rotations
    want = ("points" in which, tuple(k in which for k in ("pts_xyz", "opacity", "scales", "rotations")), "camera" in which)
    assert seen == [want], (seen, want)
    for k, v in got.items():
        assert torch.isfinite(v).all() and float(v.abs().sum()) > 0, k
        assert _rel(v, full[k]) <= 1e-5, k


def test_edges_zero_points_far_points_an_empty_view_and_ragged_q():
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(3000, 96, 64, 0, 2)
    views = [_settings(inps[0], 0), _settings(inps[1], 0)]
    cloud = [_t(g[k]).requires_grad_() for k in ("means3D", "rotations", "scales", "opacities")]
    empty = torch.zeros(0, 3, device="cuda", requires_grad=True)
    out = GR.point_visibility(views, empty, *cloud, differentiable=True)
    grads = torch.autograd.grad(out["transmittance"].sum() + out["uv"].sum(), [empty] + cloud, allow_unused=True)
    assert all(x is None or (x == 0).all() for x in grads)
    # behind the camera and outside every view: zero, finite gradients (uv and depth NaN where the cull fails)
    far = torch.tensor([[0, 0, -100], [100, 100, 100], [-1e3, 0, 0]], dtype=torch.float32, device="cuda").repeat(40, 1)
    far.requires_grad_()
    out = GR.point_visibility(views, far, *cloud, differentiable=True)
    assert not out["in_view"].any()
    loss = out["transmittance"].sum() + torch.nan_to_num(out["uv"], 0.0).sum() + torch.nan_to_num(out["depth"], 0.0).sum()
    grads = torch.autograd.grad(loss, [far] + cloud)
    assert all(torch.isfinite(x).all() for x in grads)
    assert all(float(x.abs().sum()) == 0 for x in grads[1:])
    # a view no Gaussian reaches: T == 1, and the cloud receives nothing through it
    moved = dict(g, means3D=(np.asarray(g["means3D"]) * 0.01 + np.array([0, 0, -50], np.float32)).astype(np.float32))
    (uv, d, inv, T), (dp, dm, dop, ds, dr, cam) = _gpu(views, moved, _points(g, 500), (np.ones((2, 500), np.float32), None, None))
    assert (T == 1).all() and float(dm.abs().sum()) == 0 and float(dop.abs().sum()) == 0
    # ragged Q against the reference
    for Q in (1, 33, 4099):
        pts = _points(g, max(Q, 8), seed=Q)[-Q:]
        (uv, d, inv, T), _ = _gpu(views[:1], g, pts, (None, None, None), camera=False, want_cloud=False)
        if inv.sum() >= 1:
            _compare(views[:1], [_model_kw(inps[0], "pinhole")[1]], g, pts, tag=("Q", Q))


def test_voxel_centres_at_c3_size_match_the_reference_on_a_subsample():
    import bench
    from manigaussian_b200 import GaussianRasterizationSettings, gaussian_renderer as GR, rasterizer as R, scenes
    wl = bench.WORKLOADS["c3"]
    P, W, H = wl["P"], wl["W"], wl["H"]
    g = scenes.make_gaussians(P, F=0, sh_degree=bench.SH_DEGREE, seed=1234)
    c = scenes.make_camera(W, H, 0, wl["views"])
    bg = torch.zeros(3, device="cuda")
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, _t(c["viewmatrix"]), _t(c["projmatrix"]),
                                           bench.SH_DEGREE, _t(c["campos"]), False, False, False)]
    view = dict(viewmatrix=np.asarray(c["viewmatrix"], np.float64).reshape(-1),
                projmatrix=np.asarray(c["projmatrix"], np.float64).reshape(-1), W=W, H=H, tanfovx=float(c["tanfovx"]),
                tanfovy=float(c["tanfovy"]))
    pts, _ = GR.voxel_centres(scenes.SCENE_BOUNDS, 100, "cuda")
    p = pts.cpu().numpy()
    m, o, s, r = (_t(g[k]) for k in ("means3D", "opacities", "scales", "rotations"))
    uv, d, inv, T, state = R.visibility_views_raw(views, m, o, s, r, 1.0, None, pts, keep_state=True)
    uv, d, inv = uv.cpu().numpy(), d.cpu().numpy(), inv.cpu().numpy().astype(bool)
    st = _states(views, g)[0]
    sub = np.random.default_rng(2).choice(len(p), 300, replace=False)
    acc, border = VG.decisions(st, uv[0, sub].astype(np.float64), d[0, sub].astype(np.float64), inv[0, sub])
    # cotangents on the subsample only, so that every gradient is comparable
    cs = _cotangents(uv[:, sub], inv[:, sub], border[None], 9)
    cot = [np.zeros((1, len(p)) + x.shape[2:], np.float32) for x in cs]
    for full, x in zip(cot, cs):
        full[:, sub] = x
    dp, dm, dop, ds, dr, cam = R.visibility_views_backward_raw(state, pts, m, o, s, r, 1.0, None, T, *(_t(x) for x in cot),
                                                               camera_grads=True)
    ref = _reference([view], g, p[sub], [acc], cs)
    errs = [_rel(dp.cpu().numpy()[sub], ref[0]), _rel(dm.cpu().numpy(), ref[1]), _rel(ds.cpu().numpy(), ref[2]),
            _rel(dr.cpu().numpy(), ref[3]), _rel(dop.cpu().numpy(), ref[4]), _rel(cam[0].cpu().numpy(), ref[5][None]),
            _rel(cam[1].cpu().numpy(), ref[6][None])]
    print(f"[c3 voxels] {int(inv.sum())} in view, rel-L2 {errs}")
    assert max(errs) <= TOL, errs


# --------------------------------------------------------------------------- 4. graph capture, other device
def test_cuda_graph_capture_of_forward_and_backward_replays_on_new_values():
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(3000, 96, 64, 0, 2)
    views = [_settings(inps[0], 0, "pinhole"), _settings(inps[1], 0, "distorted")]
    cloud = [_t(g[k]).requires_grad_() for k in ("means3D", "rotations", "scales", "opacities")]
    pts = _t(_points(g, 1500)).requires_grad_()
    w = torch.randn(2, 1500, device="cuda")

    def step():
        out = GR.point_visibility(views, pts, *cloud, differentiable=True)
        return torch.autograd.grad((w * out["transmittance"]).sum() + torch.nan_to_num(out["depth"]).sum() * 1e-3, [pts] + cloud)

    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        step()
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = step()
    with torch.no_grad():
        pts.copy_(pts.flip(0))
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    for a, b in zip(cap, eager):
        assert _rel(a.cpu().numpy(), b.cpu().numpy()) <= 1e-5


def test_a_call_on_a_non_current_device_gives_the_same_gradients():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(3000, 96, 64, 0, 1)
    views = [_settings(inps[0], 0)]
    pts = _points(g, 1000)

    def run(dev, vs):
        cloud = [_t(g[k]).to(dev).requires_grad_() for k in ("means3D", "rotations", "scales", "opacities")]
        p = _t(pts).to(dev).requires_grad_()
        out = GR.point_visibility(vs, p, *cloud, differentiable=True)
        return [x.cpu() for x in torch.autograd.grad(out["transmittance"].sum(), [p] + cloud)]

    ref = run(torch.device("cuda:0"), views)
    d1 = torch.device("cuda:1")
    mv = lambda x: x.to(d1)  # noqa: E731
    s1 = views[0]._replace(bg=mv(views[0].bg), viewmatrix=mv(views[0].viewmatrix), projmatrix=mv(views[0].projmatrix),
                           campos=mv(views[0].campos))
    with torch.cuda.device(0):
        got = run(d1, [s1])
    for a, b in zip(got, ref):
        assert _rel(a.numpy(), b.numpy()) <= 1e-5
