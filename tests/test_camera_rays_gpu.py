"""Camera rays on the GPU (rays.cu, mgs_camera_rays, gaussian_renderer.camera_rays).

1. Against the float64 reference (tests/rays_ref64.py), per camera model and in one call mixing all four with a device field
   of view: equal valid masks, and origin and direction within 1e-4 (1 + |ref|) per element.  The pinhole and orthographic
   rays are an fp32 3x3 solve whose matrices have condition numbers of order 10 to 100; the lens rays are fp32 Newton solves
   whose residual bound is 1e-6 (1 + |xd|) in normalised units: either loses at most a few hundred ulps, ~1e-5 relative.
2. The round trip through the renderer's own map: point_visibility(origin + z direction) gives uv equal to the pixel within
   1e-3 px and depth == z (to fp32 rounding), on the grid at several depths and at random continuous pixels, including
   pixels just inside the theta_max and r_max borders (and none just outside them is valid).
3. The rendered-depth round trip: depth / alpha of a scene, unprojected at pixel centres, projects back to those centres at
   that depth.
4. Gradients to the pixels, the view and projection matrices, tan_fov and a camera_batch's learnable pose against the
   reference's autograd at rel-L2 <= 1e-4, bit for bit repeatable.
5. Q = 0, invalid pixels (NaN outputs, cotangents ignored), CUDA-graph capture with replay on new camera values, and a
   non-current device.
"""
import numpy as np
import pytest
import torch

import rays_ref64 as R
import util  # noqa: F401  (sys.path)
from test_planar_depth_gpu import MODELS, _inputs, _model_kw, _settings, _t

pytestmark = pytest.mark.gpu
D64 = torch.float64
TOL = 1e-4


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as RS
    RS.reset_capacity_estimates()
    yield
    RS.reset_capacity_estimates()


def _rel(got, ref):
    got, ref = (np.asarray(x.detach().cpu().numpy() if torch.is_tensor(x) else x, np.float64).ravel() for x in (got, ref))
    return float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))


def _lens(s, **kw):
    """settings s with its camera-model keywords replaced (_replace keeps only the tuple's fields)"""
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    lens = dict(orthographic=s.orthographic, fisheye=s.fisheye, distortion=s.distortion)
    lens.update(kw)
    return GaussianRasterizationSettings(*s, **lens)


def _grid(W, H):
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    return np.stack([u.ravel(), v.ravel()], -1)


def _random_pixels(W, H, n, seed):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(-0.5, W - 0.5, n), rng.uniform(-0.5, H - 0.5, n)], -1)


def _check_against_reference(o, d, ok, pix, view, tag):
    ro, rd, rok = R.rays(torch.tensor(pix, dtype=D64), view)
    ok = ok.cpu().numpy().astype(bool)
    assert (ok == rok.numpy()).all(), tag
    o, d = o.cpu().numpy().astype(np.float64), d.cpu().numpy().astype(np.float64)
    assert np.isnan(o[~ok]).all() and np.isnan(d[~ok]).all(), tag
    for got, ref in ((o[ok], ro.numpy()[ok]), (d[ok], rd.numpy()[ok])):
        err = np.abs(got - ref) / (1 + np.abs(ref))
        assert err.max() <= TOL, (tag, err.max())


# --------------------------------------------------------------------------- 1. reference
@pytest.mark.parametrize("model", MODELS)
def test_grid_rays_match_the_float64_reference(model):
    from manigaussian_b200 import gaussian_renderer as GR
    inps, _ = _inputs(64, 96, 64, 0, 2)
    views = [_settings(inp, 0, model) for inp in inps]
    out = GR.camera_rays(views)
    assert out["origin"].shape == (2, 64, 96, 3) and out["valid"].shape == (2, 64, 96) and out["valid"].dtype == torch.bool
    for v, inp in enumerate(inps):
        _check_against_reference(out["origin"][v].reshape(-1, 3), out["direction"][v].reshape(-1, 3), out["valid"][v].reshape(-1),
                                 _grid(96, 64), _model_kw(inp, model)[1], f"{model} view {v}")


def test_one_call_mixing_all_four_models_with_a_device_fov():
    from manigaussian_b200 import rasterizer as RS
    inps, _ = _inputs(64, 80, 60, 0, 4)
    views = [_settings(inp, 0, m) for inp, m in zip(inps, MODELS)]
    tf = torch.tensor([[float(s.tanfovx) * 1.05, float(s.tanfovy) * 0.97] for s in views], device="cuda")
    pix = np.stack([_random_pixels(80, 60, 500, seed=v) for v in range(4)])
    o, d, ok = RS.camera_rays_raw(views, _t(pix), tan_fov=tf)
    for v, (inp, m) in enumerate(zip(inps, MODELS)):
        view = dict(_model_kw(inp, m)[1], tanfovx=float(tf[v, 0]), tanfovy=float(tf[v, 1]))
        _check_against_reference(o[v], d[v], ok[v], pix[v], view, m)


# --------------------------------------------------------------------------- 2. round trip through the renderer's map
def _visibility(views, g, pts):
    from manigaussian_b200 import gaussian_renderer as GR
    return GR.point_visibility(views, pts, _t(g["means3D"]), _t(g["rotations"]), _t(g["scales"]), _t(g["opacities"]))


@pytest.mark.parametrize("model", MODELS)
def test_rays_project_back_to_their_pixels_at_every_depth(model):
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(2000, 96, 64, 0, 1)
    s = _settings(inps[0], 0, model)
    fe_or_dc = _model_kw(inps[0], model)[1]  # the reference's view
    grid = torch.tensor(_grid(96, 64), dtype=torch.float32, device="cuda")
    rnd = torch.tensor(_random_pixels(96, 64, 3000, seed=7), dtype=torch.float32, device="cuda")
    pix = [grid, rnd]
    if model == "fisheye":
        # just inside theta_max rho(theta_max), in every direction (outside the image: rays exist for any pixel)
        fe = fe_or_dc["fisheye"]
        k, tmax = [float(x) for x in fe[2:6]], float(fe[6])
        fx, fy = (float(x) for x in R._focal(fe_or_dc))
        ang = np.linspace(0, 2 * np.pi, 64, endpoint=False)
        r = tmax * R._rho(tmax, k)
        for scale, want in ((0.999, True), (1.001, False)):
            b = torch.tensor(np.stack([fe[0] + fx * scale * r * np.cos(ang), fe[1] + fy * scale * r * np.sin(ang)], -1),
                             dtype=torch.float32, device="cuda")
            assert bool((GR.camera_rays([s], b[None])["valid"] == want).all()), scale
            if want:
                pix.append(b)
    for p in pix:
        out = GR.camera_rays([s], p[None])
        ok = out["valid"][0]
        assert bool(ok.all()), model
        for z in (0.5, 1.7, 6.0):
            pts = out["origin"][0] + z * out["direction"][0]
            vis = _visibility([s], g, pts)
            err = (vis["uv"][0] - p).abs().max()
            assert float(err) <= 1e-3, (model, z, float(err))
            assert float(((vis["depth"][0] - z).abs() / z).max()) <= 1e-5


def test_distorted_rays_at_the_r_max_border():
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(2000, 96, 64, 0, 1)
    kw, view = _model_kw(inps[0], "distorted")
    dc = tuple(view["distortion"][:10]) + (0.4,)
    s = _lens(_settings(inps[0], 0, "distorted"), distortion=dc)
    view = dict(view, distortion=dc)
    fx, fy = (float(x) for x in R._focal(view))
    ang = np.linspace(0, 2 * np.pi, 64, endpoint=False)
    # the pixels of normalised radius r = 0.4 (1 -+ 1e-3) along every direction, through the float64 forward map
    for scale, want in ((0.999, True), (1.001, False)):
        t = torch.tensor(np.stack([0.4 * scale * np.cos(ang), 0.4 * scale * np.sin(ang), np.ones_like(ang)], -1), dtype=D64)
        pix = R.P64._map(t, view).float().cuda()
        out = GR.camera_rays([s], pix[None])
        assert bool((out["valid"][0] == want).all()), scale
        if want:
            vis = _visibility([s], g, out["origin"][0] + 2.0 * out["direction"][0])
            assert float((vis["uv"][0] - pix).abs().max()) <= 1e-3


# --------------------------------------------------------------------------- 3. rendered depth
@pytest.mark.parametrize("model", MODELS)
def test_rendered_depth_over_alpha_unprojects_to_its_pixel_centres(model):
    from manigaussian_b200 import gaussian_renderer as GR
    inps, g = _inputs(3000, 96, 64, 0, 1)
    s = _settings(inps[0], 0, model)
    cl = [_t(g[k]) for k in ("means3D", "rotations", "scales", "opacities")]
    ren = GR.render_views([s], cl[0], cl[1], cl[2], cl[3], pts_rgb=torch.zeros(cl[0].shape[0], 3, device="cuda"),
                          return_depth=True, return_alpha=True)
    depth, alpha = ren["depth"].reshape(64, 96), ren["alpha"].reshape(64, 96)
    z = (depth / alpha).detach()
    rays = GR.camera_rays([s])
    keep = (alpha > 0.5) & (z > 0.3) & rays["valid"][0]
    assert int(keep.sum()) > 500
    pts = (rays["origin"][0] + z[..., None] * rays["direction"][0])[keep]
    vis = _visibility([s], g, pts)
    centres = torch.tensor(_grid(96, 64), dtype=torch.float32, device="cuda").reshape(64, 96, 2)[keep]
    assert float((vis["uv"][0] - centres).abs().max()) <= 1e-3
    assert float(((vis["depth"][0] - z[keep]).abs() / z[keep]).max()) <= 1e-5


# --------------------------------------------------------------------------- 4. gradients
def _raw_grads(views, pix, go, gd, tf):
    from manigaussian_b200 import rasterizer as RS
    dpix, cam = RS.camera_rays_backward_raw(views, pix, go, gd, tan_fov=tf, camera_grads=True)
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (dpix, cam[0], cam[1], cam[3])]


def _ref_grads(view, pix, go, gd, ok):
    p = torch.tensor(pix, dtype=D64, requires_grad=True)
    vm = torch.tensor(np.asarray(view["viewmatrix"], np.float64), requires_grad=True)
    pm = torch.tensor(np.asarray(view["projmatrix"], np.float64), requires_grad=True)
    tf = torch.tensor([view["tanfovx"], view["tanfovy"]], dtype=D64, requires_grad=True)
    o, d, _ = R.rays(p, dict(view, viewmatrix=vm, projmatrix=pm, tanfovx=tf[0], tanfovy=tf[1]))
    m = torch.as_tensor(ok)[:, None]
    loss = (torch.where(m, o, 0) * torch.tensor(go, dtype=D64)).sum() + (torch.where(m, d, 0) * torch.tensor(gd, dtype=D64)).sum()
    leaves = [p, vm, pm, tf]
    grads = torch.autograd.grad(loss, leaves, allow_unused=True)  # tan_fov enters no pinhole or orthographic ray
    return [(g if g is not None else torch.zeros_like(x)).detach().numpy() for g, x in zip(grads, leaves)]


@pytest.mark.parametrize("model", MODELS)
def test_gradients_match_the_float64_reference_and_repeat_bit_for_bit(model):
    from manigaussian_b200 import rasterizer as RS
    inps, _ = _inputs(64, 96, 64, 0, 2)
    views = [_settings(inp, 0, model) for inp in inps]
    tf = torch.tensor([[float(s.tanfovx), float(s.tanfovy)] for s in views], device="cuda")
    rng = np.random.default_rng(11)
    pix = np.stack([_random_pixels(96, 64, 4000, seed=20 + v) for v in range(2)])
    go, gd = rng.standard_normal((2, 4000, 3)), rng.standard_normal((2, 4000, 3))
    _, _, ok = RS.camera_rays_raw(views, _t(pix), tan_fov=tf)
    ok = ok.cpu().numpy().astype(bool)
    got = _raw_grads(views, _t(pix), _t(go), _t(gd), tf)
    again = _raw_grads(views, _t(pix), _t(go), _t(gd), tf)
    for a, b in zip(got, again):
        assert np.array_equal(a, b)
    for v, inp in enumerate(inps):
        ref = _ref_grads(_model_kw(inp, model)[1], pix[v], go[v], gd[v], ok[v])
        names = ("pixels", "viewmatrix", "projmatrix", "tan_fov")
        for name, a, b in zip(names, (got[0][v], got[1][v], got[2][v], got[3][v]), ref):
            if not np.any(b):
                assert not np.any(a), (model, name)
                continue
            assert _rel(a, b) <= TOL, (model, v, name, _rel(a, b))


def test_camera_batch_pose_gradients_through_the_autograd_node():
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import camera_batch
    from test_camera_grad_gpu import _intr, _w2c
    w2c64 = torch.as_tensor(_w2c(2, seed=4)).detach().cpu().to(D64)
    w2c = w2c64.float().cuda().requires_grad_(True)
    cams = camera_batch(w2c, _intr(2, 96, 80), 96, 80)
    pix = torch.tensor(np.stack([_random_pixels(96, 80, 1000, seed=v) for v in range(2)]), dtype=torch.float32,
                       device="cuda", requires_grad=True)
    out = GR.camera_rays(cams, pix)
    assert out["origin"].grad_fn is not None and out["origin"].grad_fn is out["direction"].grad_fn
    rng = np.random.default_rng(5)
    go, gd = (torch.tensor(rng.standard_normal((2, 1000, 3)), dtype=torch.float32, device="cuda") for _ in range(2))
    loss = (out["origin"] * go).sum() + (out["direction"] * gd).sum()
    g_w2c, g_pix = torch.autograd.grad(loss, [w2c, pix])
    # the reference: the same camera_batch in float64, through rays_ref64
    w = w2c64.clone().requires_grad_(True)
    c64 = camera_batch(w, _intr(2, 96, 80), 96, 80)
    p64 = pix.detach().cpu().double().requires_grad_(True)
    ref_loss = 0
    for v in range(2):
        view = dict(viewmatrix=c64.world_view_transform[v].reshape(-1), projmatrix=c64.full_proj_transform[v].reshape(-1),
                    W=96, H=80, tanfovx=float(cams.tanfovx[v]), tanfovy=float(cams.tanfovy[v]))
        o, d, ok = R.rays(p64[v], view)
        assert bool(ok.all())
        ref_loss = ref_loss + (o * go[v].cpu().double()).sum() + (d * gd[v].cpu().double()).sum()
    r_w2c, r_pix = torch.autograd.grad(ref_loss, [w, p64])
    assert _rel(g_w2c, r_w2c) <= TOL and _rel(g_pix, r_pix) <= TOL
    # no input requires grad: no node
    plain = GR.camera_rays(camera_batch(w2c.detach(), _intr(2, 96, 80), 96, 80), pix.detach())
    assert plain["origin"].grad_fn is None and torch.equal(plain["origin"], out["origin"].detach())


# --------------------------------------------------------------------------- 5. edges, graphs, devices
def test_zero_pixels_invalid_pixels_and_ignored_cotangents():
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200 import rasterizer as RS
    inps, _ = _inputs(64, 96, 64, 0, 1)
    s = _settings(inps[0], 0, "fisheye")
    empty = GR.camera_rays([s], torch.zeros(1, 0, 2, device="cuda", requires_grad=True))
    assert empty["origin"].shape == (1, 0, 3)
    tf = torch.tensor([[float(s.tanfovx), float(s.tanfovy)]], device="cuda")
    dpix, cam = RS.camera_rays_backward_raw([s], torch.zeros(1, 0, 2, device="cuda"), None, None, tan_fov=tf, camera_grads=True)
    assert not any(bool(c.any()) for c in cam if c is not None)
    # a pixel far past theta_max and a NaN pixel beside a valid one
    pix = torch.tensor([[[48.0, 30.0], [1e5, 30.0], [float("nan"), 3.0]]], device="cuda")
    o, d, ok = RS.camera_rays_raw([s], pix)
    assert ok.tolist() == [[1, 0, 0]] and torch.isnan(o[0, 1:]).all() and torch.isnan(d[0, 1:]).all()
    go = torch.ones(1, 3, 3, device="cuda")
    base = RS.camera_rays_backward_raw([s], pix, go, go, tan_fov=tf, camera_grads=True)
    noisy = RS.camera_rays_backward_raw([s], pix, go.index_fill(1, torch.tensor([1, 2], device="cuda"), float("nan")),
                                        go.index_fill(1, torch.tensor([1, 2], device="cuda"), 1e9), tan_fov=tf, camera_grads=True)
    assert torch.equal(base[0], noisy[0]) and (base[0][0, 1:] == 0).all()
    for a, b in zip(base[1], noisy[1]):
        assert a is None or torch.equal(a, b)


def test_fisheye_axis_pixel_has_finite_rays_and_derivatives():
    from manigaussian_b200 import rasterizer as RS
    inps, _ = _inputs(64, 96, 64, 0, 1)
    s = _settings(inps[0], 0, "fisheye")
    cx, cy = s.fisheye[:2]
    pix = torch.tensor([[[cx, cy], [cx + 1e-3, cy + 1e-3]]], device="cuda")
    o, d, ok = RS.camera_rays_raw([s], pix)
    assert bool(ok.all()) and torch.isfinite(d).all()
    go = torch.randn(1, 2, 3, device="cuda")
    dpix, cam = RS.camera_rays_backward_raw([s], pix, None, go[:, [0, 0]], camera_grads=True)
    assert torch.isfinite(dpix).all() and all(torch.isfinite(c).all() for c in cam if c is not None)
    assert _rel(dpix[0, 0], dpix[0, 1]) <= 1e-3


def test_cuda_graph_capture_replays_on_new_camera_values():
    from manigaussian_b200 import cameras as C
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    from test_camera_grad_gpu import _intr, _w2c
    w2c = torch.as_tensor(_w2c(2, seed=6)).detach().float().cuda().requires_grad_(True)
    pix = torch.tensor(np.stack([_random_pixels(96, 80, 700, seed=v) for v in range(2)]), dtype=torch.float32,
                       device="cuda", requires_grad=True)
    w = torch.randn(2, 700, 3, device="cuda")
    K = _intr(2, 96, 80)
    # the projection is uploaded once: a capture may not copy from pageable host memory
    projT = torch.tensor(np.swapaxes(C.projection_from_intrinsics(0.1, 4.0, K, 80, 96), -1, -2).copy(), dtype=torch.float32,
                         device="cuda")
    tan = [(96 / (2 * K[v, 0, 0]), 80 / (2 * K[v, 1, 1])) for v in range(2)]
    bg = torch.zeros(3, device="cuda")

    def step():
        views = [GaussianRasterizationSettings(80, 96, tan[v][0], tan[v][1], bg, 1.0, w2c[v].T, w2c[v].T @ projT[v], 0, bg, False,
                                               False, False) for v in range(2)]
        out = GR.camera_rays(views, pix)
        loss = (w * out["origin"]).sum() + (w * out["direction"]).sum()
        return (out["direction"],) + torch.autograd.grad(loss, [w2c, pix])

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
        w2c.copy_(torch.as_tensor(_w2c(2, seed=9)).float())
        pix.add_(0.25)
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    for a, b in zip(cap, eager):
        assert torch.equal(a, b)


def test_a_call_on_a_non_current_device_gives_the_same_rays_and_gradients():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manigaussian_b200 import rasterizer as RS
    inps, _ = _inputs(64, 96, 64, 0, 1)
    s = _settings(inps[0], 0, "distorted")
    pix = torch.tensor(_random_pixels(96, 64, 500, seed=3)[None], dtype=torch.float32)
    go = torch.randn(1, 500, 3)

    def run(dev, sv):
        o, d, ok = RS.camera_rays_raw([sv], pix.to(dev))
        dp, cam = RS.camera_rays_backward_raw([sv], pix.to(dev), go.to(dev), go.to(dev), camera_grads=True)
        return [x.cpu() for x in (o, d, ok, dp, cam[0])]

    ref = run(torch.device("cuda:0"), s)
    d1 = torch.device("cuda:1")
    mv = lambda x: x.to(d1)  # noqa: E731
    s1 = _lens(s._replace(bg=mv(s.bg), viewmatrix=mv(s.viewmatrix), projmatrix=mv(s.projmatrix), campos=mv(s.campos)),
               distortion=s.distortion)
    with torch.cuda.device(0):
        got = run(d1, s1)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
