"""Planar depth on the GPU (include/mgs_rasterizer.h, mgs_render_options.planar_depth).

* Per-Gaussian quad: {a, b, e} read back from the geometry state equals the float64 reference (tests/planar_ref64.py) for
  pinhole, orthographic, fisheye and distorted views.
* Blend, against the existing feature path as oracle: the same cloud rendered with planar depth and, per view, without it but
  with that view's quads as three more feature channels.  The planar depth plane is the oracle's depth + px Fa + py Fb + Fe;
  with the depth cotangent g entering those channels as (g px, g py, g), the gradients of opacities, SHs and features agree,
  and those of means3D, scales and rotations differ from the oracle's by the float64 chain of the oracle's dL/d(a, b, e)
  through the quad (torch autograd of the reference).  Also with AA, F = 0 / 32 / 64 (channel groups) and 2 views.
* The median depth is its contributor's z + a px + b py + e; colour, features, alpha and radii are bit-identical with
  planar depth on and off.
* A tilted plane of flat Gaussians: the depth RMSE against the analytic plane is lower with planar depth.
* Contract errors, the public paths and a CUDA-graph replay.
"""
import numpy as np
import pytest

import util
import planar_ref64 as R64

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _t(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


MODELS = ("pinhole", "ortho", "fisheye", "distorted")


def _inputs(P, W, H, F, V, seed=5):
    inps = [util.make_inputs(P=P, W=W, H=H, F=F, seed=seed, view=v, num_views=max(V, 4), bg=(0.3, 0.6, 0.9)) for v in range(V)]
    return inps, inps[0]["g"]


def _model_kw(inp, model):
    """settings keywords and the reference's view dict for one camera model on util's camera"""
    W, H, cam = inp["W"], inp["H"], inp["cam"]
    view = dict(viewmatrix=np.asarray(cam["viewmatrix"], np.float64).reshape(-1), projmatrix=np.asarray(cam["projmatrix"], np.float64).reshape(-1),
                W=W, H=H, tanfovx=float(cam["tanfovx"]), tanfovy=float(cam["tanfovy"]))
    kw = {}
    cx, cy = (W - 1) / 2.0, (H - 1) / 2.0
    if model == "ortho":
        from manigaussian_b200 import cameras as C
        hw, hh = float(cam["tanfovx"]) * 2.0, float(cam["tanfovy"]) * 2.0  # half extents of a view volume around the cloud
        pm = np.asarray(C.projection_orthographic(0.01, 100.0, hw, hh), np.float64)
        vm = np.asarray(cam["viewmatrix"], np.float64).reshape(4, 4)
        full = (vm @ pm.T).reshape(-1)
        view.update(ortho=True, tanfovx=hw, tanfovy=hh, projmatrix=full)
        kw = dict(orthographic=True, tanfovx=hw, tanfovy=hh, projmatrix=full)
    elif model == "fisheye":
        fe = (cx, cy, 0.02, -0.01, 0.003, -0.001, 1.4)
        view.update(fisheye=fe)
        kw = dict(fisheye=fe)
    elif model == "distorted":
        dc = (cx, cy, -0.05, 0.01, 0.001, -0.002, 0.0, 0.0, 0.0, 0.0, float("inf"))
        view.update(distortion=dc)
        kw = dict(distortion=dc)
    return kw, view


def _settings(inp, F, model="pinhole", aa=False, planar=False):
    from manigaussian_b200 import rasterizer as R
    cam = inp["cam"]
    kw, _ = _model_kw(inp, model)
    tx, ty = kw.pop("tanfovx", cam["tanfovx"]), kw.pop("tanfovy", cam["tanfovy"])
    pm = kw.pop("projmatrix", None)
    pm = cam["projmatrix"] if pm is None else pm
    return R.GaussianRasterizationSettings(inp["H"], inp["W"], tx, ty, _t(inp["bg"]), 1.0, _t(cam["viewmatrix"]), _t(pm),
                                           inp["g"]["sh_degree"], _t(cam["campos"]), False, False, F > 0, antialiasing=aa,
                                           planar_depth=planar, **kw)


def _ref_view(inp, model):
    return _model_kw(inp, model)[1]


def _cloud_args(g, feature):
    return (_t(g["means3D"]), None, feature, _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]), 1.0, None, _t(g["shs"]),
            g["sh_degree"], feature is not None)


def _quads(o, P):
    import torch
    from manigaussian_b200 import rasterizer as R
    torch.cuda.synchronize()
    geom = o[4]
    off = R.state_array("geometry", "nrm", geom, P) - geom.data_ptr()
    return geom[off:off + 16 * P].view(torch.float32).reshape(P, 4).clone()


def _cots(V, F, H, W, seed=11):
    rng = np.random.default_rng(seed)
    mk = lambda *s: _t(rng.standard_normal(s))  # noqa: E731
    return dict(color=mk(V, 3, H, W), feature=mk(V, F, H, W) if F else None, depth=mk(V, H, W), alpha=mk(V, H, W))


def _run(views, g, F, aa, ct=None, median=False, planar=None):
    import torch
    from manigaussian_b200 import rasterizer as R
    args = _cloud_args(g, _t(g["feature"]) if F else None)
    outs, streams = R.rasterize_views_raw(views, *args, return_depth=True, return_alpha=True, antialiasing=aa, return_median=median,
                                          planar_depth=planar)
    assert not any(o.overflowed() for o in outs)
    if ct is None:
        torch.cuda.synchronize()
        return outs, None
    grads = R.rasterize_views_backward_raw(
        views, outs, streams, ct["color"], ct["feature"] if F else None, args[0], None, args[2], args[4], args[5], 1.0, None,
        args[8], g["sh_degree"], F > 0, grads_depth=ct["depth"], grads_alpha=ct["alpha"], antialiasing=aa, planar_depth=planar)
    torch.cuda.synchronize()
    return outs, grads


def _pix(H, W):
    import torch
    py, px = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float32), torch.arange(W, device="cuda", dtype=torch.float32),
                            indexing="ij")
    return px, py


def _oracle(inps, g, F, quads, aa, ct, model):
    """one call per view, planar depth off, with [feature | a, b, e] as F + 3 channels and the depth cotangent entering them as
    (g px, g py, g): the planar planes, the summed gradients and the blend-stage dL/d(a, b, e) per view"""
    import torch
    from manigaussian_b200 import rasterizer as R
    planes, dq, total = [], [], None
    for v, inp in enumerate(inps):
        H, W = inp["H"], inp["W"]
        s = _settings(inp, F + 3, model, aa)
        feat = torch.cat([_t(g["feature"]), quads[v][:, :3]], 1).contiguous() if F else quads[v][:, :3].contiguous()
        args = _cloud_args(g, feat)
        outs, streams = R.rasterize_views_raw([s], *args, return_depth=True, return_alpha=True, antialiasing=aa)
        px, py = _pix(H, W)
        gd = ct["depth"][v]
        gq = torch.stack([gd * px, gd * py, gd], 0)
        gf = torch.cat([ct["feature"][v], gq], 0).contiguous() if F else gq.contiguous()
        gr = R.rasterize_views_backward_raw([s], outs, streams, [ct["color"][v]], [gf], args[0], None, feat, args[4], args[5], 1.0,
                                            None, args[8], g["sh_degree"], True, grads_depth=[gd], grads_alpha=[ct["alpha"][v]],
                                            antialiasing=aa)
        torch.cuda.synchronize()
        fq = outs[0][2][F:F + 3]
        planes.append((outs[0][7] + px * fq[0] + py * fq[1] + fq[2]).clone())
        dq.append(gr[2][:, F:F + 3].double().cpu().numpy())
        keep = dict(feature=gr[2][:, :F], opacity=gr[3], means3D=gr[4], sh=gr[6], scales=gr[7], rot=gr[8])
        total = keep if total is None else {k: total[k] + keep[k] for k in keep}
    return planes, total, dq


def _rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b)) / max(float(np.linalg.norm(b)), 1e-30)


@pytest.mark.parametrize("model", MODELS)
def test_per_gaussian_quad_matches_the_float64_reference(model):
    import torch
    P = 3000
    inps, g = _inputs(P, 96, 64, 0, 1)
    outs, _ = _run([_settings(inps[0], 0, model, planar=True)], g, 0, False)
    got = _quads(outs[0], P).double().cpu().numpy()
    live = outs[0][3].cpu().numpy() > 0
    assert live.sum() > P // 4
    assert (got[~live] == 0).all() and (got[:, 3] == 0).all()
    m, s, r = (torch.as_tensor(g[k], dtype=torch.float64) for k in ("means3D", "scales", "rotations"))
    ref, _ = R64.quads(m, s, r, _ref_view(inps[0], model))
    ref = ref.detach().numpy()
    # a and b in depth units per pixel; e is mu-scaled: compare it as the depth offset it adds at the mean
    for c in range(2):
        assert _rel(got[live, c], ref[live, c]) < 1e-4, (model, c)
    assert _rel(got[live, 2], ref[live, 2]) < 1e-4, model


CASES = [("pinhole", 0, 1, False), ("pinhole", 32, 2, True), ("pinhole", 64, 1, False), ("ortho", 0, 1, True), ("ortho", 32, 1, False),
         ("fisheye", 0, 1, False), ("fisheye", 64, 2, True), ("distorted", 0, 1, True), ("distorted", 32, 1, False)]


@pytest.mark.parametrize("model,F,V,aa", CASES)
def test_plane_and_gradients_against_the_feature_path(model, F, V, aa):
    import torch
    P, W, H = 2000, 120, 80
    inps, g = _inputs(P, W, H, F, V, seed=7 + F)
    ct = _cots(V, F, H, W)
    views = [_settings(i, F, model, aa, planar=True) for i in inps]
    outs, grads = _run(views, g, F, aa, ct=ct)
    quads = [_quads(o, P) for o in outs]
    planes, og, dq = _oracle(inps, g, F, quads, aa, ct, model)
    for v in range(V):
        scale = float(planes[v].abs().max())
        assert scale > 0.1
        assert float((outs[v][7] - planes[v]).abs().max()) <= 2e-5 * scale, v
    for k, i in dict(opacity=3, sh=6).items() | ({"feature": 2} if F else {}).items():
        assert _rel(grads[i].double().cpu().numpy(), og[k].double().cpu().numpy()) < 2e-5, k
    # means3D, scales, rotations: the oracle's plus the float64 chain of its dL/d(a, b, e) through the quad
    chain = [np.zeros((P, 3)), np.zeros((P, 3)), np.zeros((P, 4))]
    for v in range(V):
        live = outs[v][3].cpu().numpy() > 0
        cm, cs, cr = R64.quad_chain(g["means3D"], g["scales"], g["rotations"], _ref_view(inps[v], model), dq[v], live)
        chain = [chain[0] + cm, chain[1] + cs, chain[2] + cr]
    for (k, i), c in zip(dict(means3D=4, scales=7, rot=8).items(), chain):
        want = og[k].double().cpu().numpy() + c
        got = grads[i].double().cpu().numpy()
        assert np.abs(c).max() > 0, k
        assert _rel(got, want) < 1e-3, (k, _rel(got, want))
        # the planar share on its own: a wrong factor in the chain shows here even where it is a small part of the total
        assert _rel(got - og[k].double().cpu().numpy(), c) < 2e-2, (k, _rel(got - og[k].double().cpu().numpy(), c))


def test_median_depth_and_nothing_else_moves():
    import torch
    P, W, H, F = 2500, 96, 64, 8
    inps, g = _inputs(P, W, H, F, 1, seed=3)
    off, _ = _run([_settings(inps[0], F)], g, F, False, median=True)
    on, _ = _run([_settings(inps[0], F, planar=True)], g, F, False, median=True)
    for i in (1, 2, 3):  # colour, features, radii; alpha and the median id below
        assert torch.equal(off[0][i], on[0][i]), i
    alpha_off, alpha_on = off[0][8], on[0][8]
    assert torch.equal(alpha_off, alpha_on)
    mid_off, mid_on = off[0][-1], on[0][-1]
    assert torch.equal(mid_off, mid_on)
    q = _quads(on[0], P)
    px, py = _pix(H, W)
    ids = mid_on.long()
    has = ids >= 0
    z = torch.zeros_like(px)
    # the contributor's depth from the colour-blind depth plane of the off render is not per Gaussian: read z from the record
    geom = on[0][4]
    from manigaussian_b200 import rasterizer as R
    offs = R.state_array("geometry", "rgbd", geom, P) - geom.data_ptr()
    rgbd = geom[offs:offs + 16 * P].view(torch.float32).reshape(P, 4)
    z[has] = rgbd[ids[has], 3]
    want = z + q[ids.clamp(min=0), 0] * px + q[ids.clamp(min=0), 1] * py + q[ids.clamp(min=0), 2]
    want[~has] = 0
    med = on[0][-2]
    assert float((med - want).abs().max()) < 1e-4 * float(want.abs().max())
    assert not torch.equal(off[0][7], on[0][7])  # the depth plane does move


def test_tilted_plane_depth_rmse_is_lower_with_planar_depth():
    """flat Gaussians tiling the plane z = z0 + 0.5 x (view space) seen by util's first camera: RMSE against the analytic
    ray-plane depth over the covered pixels"""
    import torch
    from manigaussian_b200 import rasterizer as R
    inp = util.make_inputs(P=4, W=160, H=120, F=0, seed=1, view=0, num_views=4)
    cam = inp["cam"]
    vm = np.asarray(cam["viewmatrix"], np.float64).reshape(4, 4)  # column-major storage: t = vm[:3,:3]^T p + vm[3,:3]
    Rv, tv = vm[:3, :3].T, vm[3, :3]
    W, H = inp["W"], inp["H"]
    fx, fy = W / (2 * cam["tanfovx"]), H / (2 * cam["tanfovy"])
    z0, slope = 3.0, 0.5
    n = np.array([-slope, 0.0, 1.0]) / np.sqrt(1 + slope * slope)  # plane normal in view space
    u = np.array([1.0, 0.0, slope]) / np.sqrt(1 + slope * slope)
    w = np.array([0.0, 1.0, 0.0])
    grid = np.stack(np.meshgrid(np.linspace(-1.2, 1.2, 60), np.linspace(-0.9, 0.9, 45)), -1).reshape(-1, 2)
    tview = np.array([0.0, 0.0, z0]) + grid[:, :1] * u + grid[:, 1:] * w
    means = (tview - tv) @ Rv  # world = Rv^T (t - tv)
    Rw = Rv.T @ np.stack([u, w, n], 1)  # columns: the Gaussian's axes in world space
    qw = np.sqrt(max(1e-12, 1 + Rw[0, 0] + Rw[1, 1] + Rw[2, 2])) / 2
    q = np.array([qw, (Rw[2, 1] - Rw[1, 2]) / (4 * qw), (Rw[0, 2] - Rw[2, 0]) / (4 * qw), (Rw[1, 0] - Rw[0, 1]) / (4 * qw)])
    P = means.shape[0]
    scales = np.tile([0.05, 0.05, 1e-4], (P, 1))
    s = R.GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], _t([0, 0, 0]), 1.0, _t(cam["viewmatrix"]),
                                        _t(cam["projmatrix"]), 0, _t(cam["campos"]), False, False, False)
    args = (_t(means), _t(np.full((P, 3), 0.5)), None, _t(np.full((P, 1), 0.9)), _t(scales), _t(np.tile(q, (P, 1))), 1.0, None, None, 0, False)
    err = {}
    for planar in (False, True):
        outs, _ = R.rasterize_views_raw([s], *args, return_depth=True, return_alpha=True, planar_depth=planar)
        torch.cuda.synchronize()
        d, a = outs[0][7].double().cpu().numpy(), outs[0][8].double().cpu().numpy()
        px, py = np.meshgrid(np.arange(W), np.arange(H))
        rx, ry = (px - (W - 1) / 2) / fx, (py - (H - 1) / 2) / fy
        # ray t = s (rx, ry, 1): n . (t - (0, 0, z0)) = 0
        depth = z0 * n[2] / (n[0] * rx + n[1] * ry + n[2])
        m = a > 0.99
        assert m.sum() > 1000
        err[planar] = float(np.sqrt(np.mean((d[m] / a[m] - depth[m]) ** 2)))
    print(f"tilted plane depth RMSE: centre depth {err[False]:.5f}, planar depth {err[True]:.5f}")
    assert err[True] < 0.5 * err[False]


def test_contract_errors():
    import torch
    from manigaussian_b200 import rasterizer as R
    P = 500
    inps, g = _inputs(P, 64, 48, 0, 1)
    s = _settings(inps[0], 0, planar=True)
    with pytest.raises(ValueError):
        R.rasterize_views_raw([s], *_cloud_args(g, None), return_normal=True)
    with pytest.raises(ValueError):
        R.rasterize_views_raw([s, _settings(inps[0], 0)], *_cloud_args(g, None))


def test_public_paths_agree_and_capture():
    import torch
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import render_views, render_clouds
    P, W, H = 1500, 64, 48
    inps, g = _inputs(P, W, H, 0, 2, seed=9)
    views = [_settings(i, 0) for i in inps]
    leaves = lambda: [torch.tensor(g[k], device="cuda", requires_grad=True) for k in ("means3D", "rotations", "scales", "opacities", "shs")]  # noqa: E731
    res = []
    for path in ("rasterizer", "views", "clouds"):
        m, r, s, o, sh = leaves()
        if path == "rasterizer":
            out = GaussianRasterizer(views[0]._replace(planar_depth=True), return_depth=True)(
                means3D=m, means2D=torch.zeros_like(m), opacities=o, shs=sh, scales=s, rotations=r)
            depth = out[3]
        elif path == "views":
            depth = render_views(views[:1], m, r, s, o, features_color=sh, return_depth=True, planar_depth=True)["depth"][0]
        else:
            depth = render_clouds([dict(cameras=views[:1], pts_xyz=m, rotations=r, scales=s, opacity=o, features_color=sh)],
                                  return_depth=True, planar_depth=True)[0]["depth"][0]
        depth.square().sum().backward()
        res.append((depth.detach(), m.grad, s.grad, r.grad))
    for other in res[1:]:
        for a, b in zip(res[0], other):
            assert _rel(a.double().cpu().numpy(), b.double().cpu().numpy()) < 1e-5
    # a CUDA-graph capture of a render_views step
    m, r, s, o, sh = leaves()
    step = lambda: render_views(views, m, r, s, o, features_color=sh, return_depth=True, planar_depth=True)["depth"].sum()  # noqa: E731
    step().backward()
    torch.cuda.synchronize()
    ref = m.grad.clone()
    graph = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m.grad = None
        step().backward()
    torch.cuda.current_stream().wait_stream(st)
    with torch.cuda.graph(graph):
        m.grad = None
        step().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert _rel(m.grad.double().cpu().numpy(), ref.double().cpu().numpy()) < 1e-5


def _cov6(g):
    """the packed world covariance of util's cloud (scale modifier 1), float32 [P,6]"""
    import torch
    S = R64.covariance(torch.as_tensor(g["scales"], dtype=torch.float64), torch.as_tensor(g["rotations"], dtype=torch.float64)).numpy()
    return np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).astype(np.float32)


def _camera_pass(views, g, tf, ct, aa, cov=None, feat=None, planar=None, grads_depth=True):
    """forward + backward of `views` with the device field of view tf [V,2] and camera gradients; cov: packed cov3D_precomp in
    place of scales and rotations.  Returns (outs, grads)"""
    import torch
    from manigaussian_b200 import rasterizer as R
    F = 0 if feat is None else feat.shape[1]
    sc, rot = (None, None) if cov is not None else (_t(g["scales"]), _t(g["rotations"]))
    cv = None if cov is None else _t(cov)
    args = (_t(g["means3D"]), None, feat, _t(g["opacities"]), sc, rot, 1.0, cv, _t(g["shs"]), g["sh_degree"], F > 0)
    outs, streams = R.rasterize_views_raw(views, *args, return_depth=True, return_alpha=True, antialiasing=aa, tan_fov=tf,
                                          planar_depth=planar)
    V = len(views)
    gf = ct.get("feature_planes")
    grads = R.rasterize_views_backward_raw(
        views, outs, streams, ct["color"][:V], gf, args[0], None, feat, sc, rot, 1.0, cv, args[8], g["sh_degree"], F > 0,
        grads_depth=ct["depth"][:V], grads_alpha=ct["alpha"][:V], antialiasing=aa, camera_grads=True, tan_fov=tf, planar_depth=planar)
    torch.cuda.synchronize()
    return outs, grads


CAM_CASES = [(m, aa) for m in MODELS for aa in (False, True)]


@pytest.mark.parametrize("model,aa", CAM_CASES)
@pytest.mark.parametrize("cov", [False, True], ids=["scale_rot", "cov3D"])
def test_camera_tan_fov_and_cov3D_gradients(model, aa, cov):
    """camera gradients, the learnable field of view and cov3D_precomp: the planar render's against the feature-path oracle
    plus the float64 chain of the oracle's dL/d(a, b, e) through the quad w.r.t. viewmatrix, projmatrix, tan_fov and
    means3D / scales / rotations or the packed covariance"""
    import torch
    P, W, H, V = 1500, 96, 64, 2
    inps, g = _inputs(P, W, H, 0, V, seed=21)
    ct = _cots(V, 0, H, W, seed=5)
    c6 = _cov6(g) if cov else None
    views = [_settings(i, 0, model, aa, planar=True) for i in inps]
    tf = _t([[float(v.tanfovx), float(v.tanfovy)] for v in views])
    outs, grads = _camera_pass(views, g, tf, ct, aa, cov=c6)
    cam = grads[9]
    names = ["means3D", "cov3D"] if cov else ["means3D", "scales", "rot"]
    gi = dict(means3D=4, cov3D=5, scales=7, rot=8)
    got = {k: grads[gi[k]].double().cpu().numpy() for k in names}
    got.update(vm=cam[0].double().cpu().numpy(), pm=cam[1].double().cpu().numpy(), tf=cam[3].double().cpu().numpy())
    og = {k: np.zeros_like(v) for k, v in got.items()}
    chain = {k: np.zeros_like(v) for k, v in got.items()}
    for v, inp in enumerate(inps):
        q = _quads(outs[v], P)
        s = _settings(inp, 3, model, aa)
        c1 = {"color": ct["color"][v:v + 1], "depth": ct["depth"][v:v + 1], "alpha": ct["alpha"][v:v + 1]}
        px, py = _pix(H, W)
        gd = ct["depth"][v]
        c1["feature_planes"] = [torch.stack([gd * px, gd * py, gd], 0).contiguous()]
        o1, g1 = _camera_pass([s], g, tf[v:v + 1].contiguous(), c1, aa, cov=c6, feat=q[:, :3].contiguous())
        scale = float(o1[0][7].abs().max())
        fq = o1[0][2]
        assert float((outs[v][7] - (o1[0][7] + px * fq[0] + py * fq[1] + fq[2])).abs().max()) <= 2e-5 * scale
        for k in names:
            og[k] += g1[gi[k]].double().cpu().numpy()
        og["vm"][v] = g1[9][0][0].double().cpu().numpy()
        og["pm"][v] = g1[9][1][0].double().cpu().numpy()
        og["tf"][v] = g1[9][3][0].double().cpu().numpy()
        live = outs[v][3].cpu().numpy() > 0
        dq = g1[2][:, :3].double().cpu().numpy()
        ref = _ref_view(inp, model)
        res = R64.full_chain(g["means3D"], g["scales"], g["rotations"], ref, dq, live, cov3D=c6,
                             tan_fov=tf[v].double().cpu().numpy())
        for k, r in zip(names + ["vm", "pm", "tf"], res):
            if r is None:
                continue
            if k in ("vm", "pm", "tf"):
                chain[k][v] += r.reshape(chain[k][v].shape)
            else:
                chain[k] += r
    for k in got:
        want = og[k] + chain[k]
        if not np.abs(want).max() > 0:
            assert np.abs(got[k]).max() == 0, k  # projmatrix of a fisheye or distorted view
            continue
        assert _rel(got[k], want) < 1e-3, (k, _rel(got[k], want))
        if np.abs(chain[k]).max() > 0:
            assert _rel(got[k] - og[k], chain[k]) < 2e-2, (k, _rel(got[k] - og[k], chain[k]))
    assert np.abs(chain["tf"]).max() > 0 and np.abs(chain["vm"]).max() > 0


@pytest.mark.parametrize("model,aa", [("pinhole", False), ("ortho", True), ("fisheye", False), ("distorted", True)])
def test_median_depth_gradient(model, aa):
    """only a median-depth cotangent: the planar render's gradients are the centre-depth render's (the cotangent on z) plus the
    float64 chain of g (px, py, 1), summed over each Gaussian's median pixels through median_id, through the quad"""
    import torch
    from manigaussian_b200 import rasterizer as R
    P, W, H = 2000, 96, 64
    inps, g = _inputs(P, W, H, 0, 1, seed=13)
    gm = _t(np.random.default_rng(4).standard_normal((H, W)))
    res = {}
    for planar in (False, True):
        s = _settings(inps[0], 0, model, aa, planar=planar)
        args = _cloud_args(g, None)
        outs, streams = R.rasterize_views_raw([s], *args, return_depth=True, return_alpha=True, antialiasing=aa, return_median=True)
        z = torch.zeros(3, H, W, device="cuda")
        gr = R.rasterize_views_backward_raw([s], outs, streams, [z], None, args[0], None, None, args[4], args[5], 1.0, None, args[8],
                                            g["sh_degree"], False, antialiasing=aa, grads_median=[gm], median_ids=[outs[0][-1]])
        torch.cuda.synchronize()
        res[planar] = (outs, gr)
    outs, gr = res[True]
    ids = outs[0][-1].cpu().numpy().ravel()
    assert np.array_equal(ids, res[False][0][0][-1].cpu().numpy().ravel())
    py, px = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    gmn = gm.double().cpu().numpy().ravel()
    has = ids >= 0
    dq = np.zeros((P, 3))
    for c, w in enumerate((px.ravel(), py.ravel(), np.ones(H * W))):
        np.add.at(dq[:, c], ids[has], (gmn * w)[has])
    live = outs[0][3].cpu().numpy() > 0
    cm, cs, cr = R64.quad_chain(g["means3D"], g["scales"], g["rotations"], _ref_view(inps[0], model), dq, live)
    for (i, c) in ((4, cm), (7, cs), (8, cr)):
        got, og = gr[i].double().cpu().numpy(), res[False][1][i].double().cpu().numpy()
        assert _rel(got, og + c) < 1e-3, (i, _rel(got, og + c))
        assert _rel(got - og, c) < 2e-2, (i, _rel(got - og, c))


@pytest.mark.parametrize("model,aa", [("pinhole", False), ("pinhole", True), ("fisheye", True), ("distorted", False), ("ortho", False)])
def test_depth_and_mask_heads_on_the_planar_depth(model, aa):
    """targets {"rgb", "depth", "mask"} with planar depth: the heads' losses and gradients equal those of a torch restatement of
    the heads (INTEGRATION.md section 4) applied to the planar depth and alpha planes of the same render"""
    import torch
    import torch.nn.functional as Fn
    from manigaussian_b200.gaussian_renderer import render_views
    P, W, H, V = 2000, 96, 64, 2
    inps, g = _inputs(P, W, H, 0, V, seed=17)
    views = [_settings(i, 0, model, aa, planar=True) for i in inps]
    rng = np.random.default_rng(8)
    gd = _t(rng.uniform(2.0, 8.0, (V, H, W)) * (rng.uniform(0, 1, (V, H, W)) > 0.2))
    gmask = _t(rng.uniform(0, 1, (V, H, W)) > 0.5)
    leaves = lambda: [torch.tensor(g[k], device="cuda", requires_grad=True) for k in ("means3D", "rotations", "scales", "opacities", "shs")]  # noqa: E731
    m1, r1, s1, o1, sh1 = leaves()
    out = render_views(views, m1, r1, s1, o1, features_color=sh1, targets={"rgb": torch.zeros(V, 3, H, W, device="cuda"), "depth": gd,
                                                                             "mask": gmask}, antialiasing=aa)
    (out["loss_depth"].sum() + out["loss_mask"].sum()).backward()
    m2, r2, s2, o2, sh2 = leaves()
    ref = render_views(views, m2, r2, s2, o2, features_color=sh2, return_depth=True, return_alpha=True, antialiasing=aa)
    D, A = ref["depth"], ref["alpha"]
    valid = ((gd > 0) & (A > 0.5)).detach()
    d = torch.where(valid, D / torch.where(valid, A, torch.ones_like(A)), torch.zeros_like(D))
    err = torch.where(valid, (d - gd).abs(), torch.zeros_like(D))
    loss_depth = err.flatten(1).sum(1) / valid.flatten(1).sum(1).clamp(min=1)
    loss_mask = torch.stack([Fn.binary_cross_entropy(A[v].clamp(1e-4, 1 - 1e-4), gmask[v]) for v in range(V)])
    (loss_depth.sum() + loss_mask.sum()).backward()
    assert _rel(out["loss_depth"].detach().double().cpu().numpy(), loss_depth.detach().double().cpu().numpy()) < 1e-5
    assert _rel(out["loss_mask"].detach().double().cpu().numpy(), loss_mask.detach().double().cpu().numpy()) < 1e-5
    for a, b in ((m1, m2), (r1, r2), (s1, s2), (o1, o2)):
        assert float(b.grad.abs().max()) > 0
        assert _rel(a.grad.double().cpu().numpy(), b.grad.double().cpu().numpy()) < 1e-4


def test_render_clouds_with_two_clouds_matches_render_views():
    """two clouds of different sizes in one render_clouds call: the planar depth planes and gradients of each equal
    render_views of that cloud alone (the per-cloud view offsets of the planar per-Gaussian backward)"""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views, render_clouds
    W, H = 64, 48
    specs = [(1500, 2, 31, "pinhole"), (1100, 3, 32, "fisheye")]
    data = []
    for P, V, seed, model in specs:
        inps, g = _inputs(P, W, H, 0, V, seed=seed)
        data.append(([_settings(i, 0, model) for i in inps], g))
    mk = lambda g: [torch.tensor(g[k], device="cuda", requires_grad=True) for k in ("means3D", "rotations", "scales", "opacities", "shs")]  # noqa: E731
    L = [mk(g) for _, g in data]
    res = render_clouds([dict(cameras=vs, pts_xyz=l[0], rotations=l[1], scales=l[2], opacity=l[3], features_color=l[4])
                         for (vs, _), l in zip(data, L)], return_depth=True, planar_depth=True)
    sum(r["depth"].square().sum() for r in res).backward()
    for (vs, g), l, r in zip(data, L, res):
        l2 = mk(g)
        one = render_views(vs, l2[0], l2[1], l2[2], l2[3], features_color=l2[4], return_depth=True, planar_depth=True)
        one["depth"].square().sum().backward()
        assert _rel(r["depth"].detach().double().cpu().numpy(), one["depth"].detach().double().cpu().numpy()) < 1e-6
        for a, b in zip(l, l2):
            assert _rel(a.grad.double().cpu().numpy(), b.grad.double().cpu().numpy()) < 1e-5
