"""The flow plane on the GPU (include/mgs_rasterizer.h, flow plane).

* Per-Gaussian quads {dx, dy, 0, 0} read back from the geometry state equal the float64 reference (tests/flow_ref64.py) for
  all four camera models, and are exactly 0 when the next means are the current ones.
* Blend, against the existing feature path as oracle: each view rendered alone without flow but with its displacements as
  two more feature channels.  The planes agree, the gradients of opacities, scales, rotations, SHs and features agree, the
  means3D gradient differs by exactly the float64 m-chain of the oracle's dL/dfeature on the two channels, and
  dL/dflow_means3D is the float64 m'-chain of the same.  Camera and field-of-view gradients likewise, with and without a
  next-frame pose.  All four models, AA on and off, F = 0, 32 and 64.
* Next means that fail the cull (behind the near plane, past a fisheye view's theta_max) give delta = 0 and receive nothing
  through either end.
* Nothing else moves with flow on, and a zero flow cotangent changes no gradient.
* One call mixing the four models, a moved next-frame pose through render_views, the dyna pair through render_clouds (the
  shared tensor receives the sum of its two uses), GaussianRasterizer / render_views at V = 1, CUDA-graph capture and replay,
  the argument errors and steady device memory.
"""
import numpy as np
import pytest

import flow_ref64 as F64
import util
from test_planar_depth_gpu import MODELS, _cloud_args, _inputs, _model_kw, _quads, _rel, _settings, _t

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _next(g, scale=0.03, seed=3):
    rng = np.random.default_rng(seed)
    return (np.asarray(g["means3D"], np.float64) + scale * rng.standard_normal(np.shape(g["means3D"]))).astype(np.float32)


def _ref_view(inp, model):
    return _model_kw(inp, model)[1]


def _moved_pose(view, model, dx=0.02):
    """the view dict and (viewmatrix, projmatrix) float32 tensors of the same camera translated by dx along its x axis"""
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).copy()
    pm = np.asarray(view["projmatrix"], np.float64).reshape(4, 4)
    T = np.eye(4)
    T[3, 0] = -dx  # column-major: translation in the last row, view-space x shifts by -dx
    vm2 = vm @ T
    pm2 = np.linalg.inv(vm) @ pm  # the projection part, then re-compose with the moved pose
    pm2 = vm2 @ pm2
    nv = dict(view, viewmatrix=vm2.reshape(-1), projmatrix=pm2.reshape(-1))
    return nv, (_t(vm2), _t(pm2))


def _run(views, g, F, aa, nxt, poses=None, gflow=None, ct=None, camera=False, tf=None):
    import torch
    from manigaussian_b200 import rasterizer as R
    args = _cloud_args(g, _t(g["feature"]) if F else None)
    fm = _t(nxt)
    outs, streams = R.rasterize_views_raw(views, *args, return_depth=True, return_alpha=True, antialiasing=aa, tan_fov=tf,
                                          flow_means3D=fm, flow_poses=poses)
    assert not any(o.overflowed() for o in outs)
    if ct is None:
        torch.cuda.synchronize()
        return outs, None
    grads = R.rasterize_views_backward_raw(
        views, outs, streams, ct["color"], ct["feature"] if F else None, args[0], None, args[2], args[4], args[5], 1.0, None,
        args[8], g["sh_degree"], F > 0, grads_depth=ct["depth"], grads_alpha=ct["alpha"], antialiasing=aa, tan_fov=tf,
        camera_grads=True if camera else None, flow_means3D=fm, flow_poses=poses, grads_flow=gflow, flows=[o[-1] for o in outs])
    torch.cuda.synchronize()
    return outs, grads


def _cots(V, F, H, W, seed=11):
    rng = np.random.default_rng(seed)
    mk = lambda *s: _t(rng.standard_normal(s))  # noqa: E731
    return dict(color=mk(V, 3, H, W), feature=mk(V, F, H, W) if F else None, depth=mk(V, H, W), alpha=mk(V, H, W),
                flow=mk(V, 2, H, W))


def _oracle(inps, g, F, quads, aa, ct, model, camera=False, tf=None):
    """one call per view without flow, with [feature | dx, dy] as F + 2 channels: the planes, the summed gradients, the
    blend-stage dL/d(dx, dy) per view and the camera gradients per view"""
    import torch
    from manigaussian_b200 import rasterizer as R
    planes, dq, cams, total = [], [], [], None
    for v, inp in enumerate(inps):
        s = _settings(inp, F + 2, model, aa)
        feat = torch.cat([_t(g["feature"]), quads[v][:, :2]], 1).contiguous() if F else quads[v][:, :2].contiguous()
        args = _cloud_args(g, feat)
        tv = tf[v:v + 1] if tf is not None else None
        outs, streams = R.rasterize_views_raw([s], *args, return_depth=True, return_alpha=True, antialiasing=aa, tan_fov=tv)
        gf = torch.cat([ct["feature"][v], ct["flow"][v]], 0).contiguous() if F else ct["flow"][v].contiguous()
        gr = R.rasterize_views_backward_raw([s], outs, streams, [ct["color"][v]], [gf], args[0], None, feat, args[4], args[5], 1.0,
                                            None, args[8], g["sh_degree"], True, grads_depth=[ct["depth"][v]],
                                            grads_alpha=[ct["alpha"][v]], antialiasing=aa, tan_fov=tv,
                                            camera_grads=True if camera else None)
        torch.cuda.synchronize()
        planes.append(outs[0][2][F:F + 2].clone())
        dq.append(gr[2][:, F:F + 2].double().cpu())
        if camera:
            cams.append(tuple(t.double().cpu().clone() for t in gr[9]))
        keep = dict(feature=gr[2][:, :F], opacity=gr[3], means3D=gr[4], sh=gr[6], scales=gr[7], rot=gr[8])
        total = keep if total is None else {k: total[k] + keep[k] for k in keep}
    return planes, total, dq, cams


def _chains(means, nxt, view, nview, dq, live, wrt_camera=False):
    """float64 vector-Jacobian products of the oracle's dL/d(dx, dy) [P,2]: through -m (at means, the view's camera) and +m'
    (at nxt, nview, where valid).  Returns (dL/dmeans, dL/dnext) and, with wrt_camera, the view-matrix, projection-matrix
    and tan_fov gradients of each end ((m, m'), each a triple)"""
    import torch
    D = torch.float64
    mu = torch.tensor(np.asarray(means, np.float64), dtype=D, requires_grad=True)
    q = torch.tensor(np.asarray(nxt, np.float64), dtype=D, requires_grad=True)
    w = dq.clone() * torch.as_tensor(live, dtype=D).unsqueeze(-1)

    def tens(v):
        vm = torch.tensor(np.asarray(v["viewmatrix"], np.float64), dtype=D, requires_grad=True)
        pm = torch.tensor(np.asarray(v["projmatrix"], np.float64), dtype=D, requires_grad=True)
        tf = torch.tensor([v["tanfovx"], v["tanfovy"]], dtype=D, requires_grad=True)
        return dict(v, viewmatrix=vm, projmatrix=pm, tanfovx=tf[0], tanfovy=tf[1]), (vm, pm, tf)

    v0, c0 = tens(view)
    v1, c1 = tens(nview)
    m = F64.screen_mean(mu, v0)
    ok = F64.valid(q, v1)
    w = w * ok.to(D).unsqueeze(-1)  # an invalid pair's delta is 0: neither end receives anything
    mn = F64.screen_mean(q, v1)
    mn = torch.where(ok.unsqueeze(-1), mn, torch.zeros_like(mn))
    (-(m * w).sum()).backward()
    (torch.nan_to_num(mn) * w).sum().backward()
    out = (mu.grad.numpy(), q.grad.numpy())
    if wrt_camera:
        grab = lambda c: tuple(t.grad.clone() if t.grad is not None else torch.zeros_like(t) for t in c)  # noqa: E731
        out += (grab(c0), grab(c1))
    return out


def _distortion_edge(t, dc, tol=1e-5):
    """next means within fp32 error of the distorted view's culls: r2 at r_max^2, or det Dd at 0"""
    import torch
    r2, det = (x.numpy() for x in F64.distortion_r2_det(torch.tensor(t, dtype=torch.float64), dc))
    r_max = float(dc[10])
    near_rmax = np.abs(r2 - r_max * r_max) < tol * np.maximum(1.0, r2) if np.isfinite(r_max) else np.zeros_like(r2, bool)
    return near_rmax | (np.abs(det) < tol)


def _invalid_next(g, view, model, frac=0.15, seed=4):
    """next means of which a fraction fails the cull: behind the near plane, and for fisheye views past theta_max"""
    nxt = _next(g, seed=seed).astype(np.float64)
    rng = np.random.default_rng(seed)
    P = nxt.shape[0]
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4)  # row r of Rv is column r of this storage
    Rv, tv = vm[:3, :3].T, vm[3, :3]
    t = nxt @ Rv.T + tv
    bad = rng.random(P) < frac
    behind = bad & (rng.random(P) < 0.5 if model == "fisheye" else np.ones(P, bool))
    t[behind, 2] = 0.1  # view-space z below NEAR_Z = 0.2
    wide = bad & ~behind
    t[wide, 0] = 8.0 * t[wide, 2]  # theta = atan(8) = 1.45 > theta_max = 1.4
    nxt = (t - tv) @ Rv
    return nxt.astype(np.float32), bad


@pytest.mark.parametrize("model", MODELS)
def test_per_gaussian_quad_matches_the_float64_reference(model):
    import torch
    P = 3000
    inps, g = _inputs(P, 96, 64, 0, 1)
    nxt = _next(g)
    view = _ref_view(inps[0], model)
    for moved in (False, True):
        nview, pose = _moved_pose(view, model) if moved else (view, None)
        outs, _ = _run([_settings(inps[0], 0, model)], g, 0, False, nxt, poses=[pose] if moved else None)
        got = _quads(outs[0], P).double().cpu().numpy()
        live = outs[0][3].cpu().numpy() > 0
        assert live.sum() > P // 4
        assert (got[~live] == 0).all() and (got[:, 2:] == 0).all()
        mu = torch.tensor(np.asarray(g["means3D"], np.float64))
        q = torch.tensor(np.asarray(nxt, np.float64))
        ref, ok = F64.delta(mu, q, view, nview)
        m, mn = F64.screen_mean(mu, view), F64.screen_mean(q, nview)
        # Bound.  Each end is a chain of at most ~16 dependent fp32 roundings (u = 2^-24): a 4-term dot product per row,
        # 1 / (w + 1e-7), the product and ndc2pix (whose + W/2 puts the error on the scale |m| + W/2), or for the lens maps
        # x / z, atan2f / sqrtf (a few ulp each) and a degree-9 polynomial in Horner form.  Each rounding is relative to a
        # value of at most the end's scale S = max(|m|, |m'|) + W/2 times the cancellation of the 4-term products, which is
        # below 2 for these clouds (all points in front, |t| ~ |p|).  So each end is within 16 * 2 u S, and delta within
        # 64 u S.
        scale = torch.maximum(m.abs(), torch.nan_to_num(mn).abs()).max(-1).values.numpy() + 0.5 * max(inps[0]["W"], inps[0]["H"])
        bound = 64 * 2.0 ** -24 * scale
        # a next mean within its fp32 error of a cull threshold may go either way: near plane, theta_max, r_max, det Dd = 0
        t = F64.view_space(q, nview).numpy()
        edge = np.abs(t[:, 2] - F64.NEAR_Z) < 1e-5
        if nview.get("fisheye") is not None:
            th = np.arctan2(np.hypot(t[:, 0], t[:, 1]), t[:, 2])
            edge |= np.abs(th - nview["fisheye"][6]) < 1e-5
        if nview.get("distortion") is not None:
            edge |= _distortion_edge(t, nview["distortion"])
        err = np.abs(got[:, :2] - ref.numpy()).max(-1)
        chk = live & ~edge
        assert (err[chk] <= bound[chk]).all(), (model, moved, float((err[chk] / bound[chk]).max()))
    # the same means under the view's own camera: exactly 0, for the tensor itself and for a clone
    for same in (g["means3D"], np.array(g["means3D"], copy=True)):
        outs, _ = _run([_settings(inps[0], 0, model)], g, 0, False, same)
        assert float(_quads(outs[0], P)[:, :2].abs().max()) == 0.0


CASES = [("pinhole", 0, 1, False), ("pinhole", 32, 2, True), ("pinhole", 64, 1, False), ("ortho", 0, 1, True), ("ortho", 32, 1, False),
         ("fisheye", 0, 1, False), ("fisheye", 64, 2, True), ("distorted", 0, 1, True), ("distorted", 32, 1, False)]


@pytest.mark.parametrize("model,F,V,aa", CASES)
def test_plane_and_gradients_against_the_feature_path(model, F, V, aa):
    P, W, H = 2000, 120, 80
    inps, g = _inputs(P, W, H, F, V, seed=7 + F)
    nxt = _next(g, seed=F + V)
    ct = _cots(V, F, H, W)
    views = [_settings(i, F, model, aa) for i in inps]
    outs, grads = _run(views, g, F, aa, nxt, gflow=list(ct["flow"]), ct=ct)
    quads = [_quads(o, P) for o in outs]
    planes, og, dq, _ = _oracle(inps, g, F, quads, aa, ct, model)
    for v in range(V):
        assert float(outs[v][-1][2].abs().max()) == 0.0
        assert _rel(outs[v][-1][:2].cpu().numpy(), planes[v].cpu().numpy()) < 1e-5, v
    for k, i in dict(opacity=3, sh=6, scales=7, rot=8).items() | ({"feature": 2} if F else {}).items():
        assert _rel(grads[i].double().cpu().numpy(), og[k].double().cpu().numpy()) < 1e-4, k
    cm, cn = np.zeros((P, 3)), np.zeros((P, 3))
    for v in range(V):
        live = outs[v][3].cpu().numpy() > 0
        a, b = _chains(g["means3D"], nxt, _ref_view(inps[v], model), _ref_view(inps[v], model), dq[v], live)
        cm, cn = cm + a, cn + b
    assert np.abs(cm).max() > 0 and np.abs(cn).max() > 0
    want = og["means3D"].double().cpu().numpy() + cm
    assert _rel(grads[4].double().cpu().numpy(), want) < 1e-4, _rel(grads[4].double().cpu().numpy(), want)
    assert _rel(grads[-1].double().cpu().numpy(), cn) < 1e-4, _rel(grads[-1].double().cpu().numpy(), cn)


@pytest.mark.parametrize("model,aa", [("pinhole", False), ("fisheye", True), ("distorted", False)])
def test_invalid_pairs_receive_nothing(model, aa):
    import torch
    P, W, H, F = 2000, 120, 80, 0
    inps, g = _inputs(P, W, H, F, 1, seed=17)
    nxt, bad = _invalid_next(g, _ref_view(inps[0], model), model)
    ok = F64.valid(torch.tensor(nxt, dtype=torch.float64), _ref_view(inps[0], model)).numpy()
    assert (~ok).sum() > P // 20 and not (ok & bad).any()
    ct = _cots(1, F, H, W)
    views = [_settings(inps[0], F, model, aa)]
    outs, grads = _run(views, g, F, aa, nxt, gflow=list(ct["flow"]), ct=ct, camera=True)
    quads = [_quads(o, P) for o in outs]
    assert float(quads[0][torch.as_tensor(~ok, device="cuda")].abs().max()) == 0.0
    planes, og, dq, cams = _oracle(inps, g, F, quads, aa, ct, model, camera=True)
    live = outs[0][3].cpu().numpy() > 0
    assert (live & ~ok).sum() > 0
    cm, cn, c_m, c_n = _chains(g["means3D"], nxt, _ref_view(inps[0], model), _ref_view(inps[0], model), dq[0], live, True)
    # nothing reaches an invalid pair's next mean, and its current mean gets only the blend-weight terms of the oracle
    assert float(grads[-1][torch.as_tensor(~ok, device="cuda")].abs().max()) == 0.0
    got = grads[4].double().cpu().numpy()
    want = og["means3D"].double().cpu().numpy() + cm
    assert _rel(got, want) < 1e-4, _rel(got, want)
    assert _rel(got[live & ~ok], og["means3D"].double().cpu().numpy()[live & ~ok]) < 1e-4
    assert _rel(grads[-1].double().cpu().numpy(), cn) < 1e-4
    for got_c, o, a, b in zip((grads[9][0][0], grads[9][1][0]), (cams[0][0][0], cams[0][1][0]), c_m, c_n):
        want_c = (o + a + b).numpy()
        assert _rel(got_c.double().cpu().numpy(), want_c) < 1e-3


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("moved", [False, True])
def test_camera_and_tan_fov_gradients(model, moved):
    import torch
    P, W, H, V = 2000, 120, 80, 2
    inps, g = _inputs(P, W, H, 0, V, seed=21)
    nxt = _next(g, seed=5)
    ct = _cots(V, 0, H, W)
    views = [_settings(i, 0, model, False) for i in inps]
    refs = [_ref_view(i, model) for i in inps]
    moves = [_moved_pose(r, model) for r in refs] if moved else [(r, None) for r in refs]
    tf = torch.tensor([[r["tanfovx"], r["tanfovy"]] for r in refs], dtype=torch.float32, device="cuda")
    outs, grads = _run(views, g, 0, False, nxt, poses=[m[1] for m in moves] if moved else None, gflow=list(ct["flow"]), ct=ct,
                       camera=True, tf=tf)
    quads = [_quads(o, P) for o in outs]
    _, _, dq, cams = _oracle(inps, g, 0, quads, False, ct, model, camera=True, tf=tf)
    dvm, dpm, dtf = (t.double().cpu() for t in (grads[9][0], grads[9][1], grads[9][3]))
    for v in range(V):
        live = outs[v][3].cpu().numpy() > 0
        _, _, c_m, c_n = _chains(g["means3D"], nxt, refs[v], moves[v][0], dq[v], live, wrt_camera=True)
        want = [cams[v][0][0] + c_m[0], cams[v][1][0] + c_m[1], cams[v][3][0] + c_m[2]]
        if not moved:  # the view's own camera also takes the m' terms; a next pose is a constant
            want = [want[0] + c_n[0], want[1] + c_n[1], want[2] + c_n[2]]
        for got, w, name in zip((dvm[v], dpm[v], dtf[v]), want, ("viewmatrix", "projmatrix", "tan_fov")):
            # every entry: those the forward never reads (the projection matrix's z row, the view matrix's fourth row) are 0 on
            # both sides
            assert _rel(got.numpy(), w.numpy()) < 1e-3, (model, moved, name, _rel(got.numpy(), w.numpy()))


def test_nothing_else_moves_and_a_zero_cotangent_changes_no_gradient():
    import torch
    from manigaussian_b200 import rasterizer as R
    P, W, H, F = 2000, 120, 80, 32
    inps, g = _inputs(P, W, H, F, 2, seed=9)
    views = [_settings(i, F, "pinhole", True) for i in inps]
    args = _cloud_args(g, _t(g["feature"]))
    ct = _cots(2, F, H, W)
    base, st0 = R.rasterize_views_raw(views, *args, return_depth=True, return_alpha=True, antialiasing=True, return_median=True)
    g0 = R.rasterize_views_backward_raw(views, base, st0, ct["color"], ct["feature"], args[0], None, args[2], args[4], args[5], 1.0,
                                        None, args[8], g["sh_degree"], True, grads_depth=ct["depth"], grads_alpha=ct["alpha"],
                                        antialiasing=True)
    fm = _t(_next(g))
    outs, st1 = R.rasterize_views_raw(views, *args, return_depth=True, return_alpha=True, antialiasing=True, return_median=True,
                                      flow_means3D=fm)
    zero = [torch.zeros((3, H, W), device="cuda") for _ in range(2)]
    g1 = R.rasterize_views_backward_raw(views, outs, st1, ct["color"], ct["feature"], args[0], None, args[2], args[4], args[5], 1.0,
                                        None, args[8], g["sh_degree"], True, grads_depth=ct["depth"], grads_alpha=ct["alpha"],
                                        antialiasing=True, flow_means3D=fm, grads_flow=zero, flows=[o[-1] for o in outs])
    torch.cuda.synchronize()
    for v in range(2):
        for i in (1, 2, 3, 7, 8, 9, 10):  # colour, features, radii, depth, alpha, median depth, median id
            assert torch.equal(base[v][i], outs[v][i]), (v, i)
    for i in (0, 2, 3, 4, 6, 7, 8):
        assert _rel(g1[i].double().cpu().numpy(), g0[i].double().cpu().numpy()) < 1e-6, i
    assert float(g1[-1].abs().max()) == 0.0


def test_one_call_mixing_the_four_models():
    import torch
    P = 3000
    inps, g = _inputs(P, 96, 64, 0, 4, seed=23)
    nxt = _next(g)
    views = [_settings(inps[v], 0, m) for v, m in enumerate(MODELS)]
    outs, _ = _run(views, g, 0, False, nxt)
    q = torch.tensor(np.asarray(nxt, np.float64))
    mu = torch.tensor(np.asarray(g["means3D"], np.float64))
    for v, m in enumerate(MODELS):
        view = _ref_view(inps[v], m)
        ref, ok = F64.delta(mu, q, view)
        live = outs[v][3].cpu().numpy() > 0
        got = _quads(outs[v], P).double().cpu().numpy()[:, :2]
        t = F64.view_space(q, view).numpy()
        chk = live & ~(np.abs(t[:, 2] - F64.NEAR_Z) < 1e-5)
        assert np.abs(got[chk] - ref.numpy()[chk]).max() < 1e-3, m


def _leaves(g):
    import torch
    return [torch.tensor(np.asarray(g[k], np.float32), device="cuda", requires_grad=True)
            for k in ("means3D", "rotations", "scales", "opacities", "shs")]


def test_public_paths_moved_pose_and_dyna_pair():
    import torch
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    P, W, H = 2000, 96, 64
    inps, g = _inputs(P, W, H, 0, 2, seed=13)
    views = [_settings(i, 0) for i in inps]
    nxt_np = _next(g)
    gf = torch.randn((2, 2, H, W), device="cuda")
    gc = torch.randn((2, 3, H, W), device="cuda")
    # GaussianRasterizer, render_views at V = 1 (its fast path) and V = 2 against the raw call
    raw, _ = _run(views, g, 0, False, nxt_np)
    m, r, s_, o, sh = _leaves(g)
    nxt = _t(nxt_np).requires_grad_(True)
    out = GaussianRasterizer(views[0])(means3D=m, means2D=torch.zeros_like(m), opacities=o.reshape(-1, 1), shs=sh, scales=s_,
                                       rotations=r, flow_means3D=nxt)
    assert torch.equal(out[-1], raw[0][-1][:2])
    (out[-1] * gf[0]).sum().backward()
    g_rast = (m.grad.clone(), nxt.grad.clone())
    for V in (1, 2):
        m.grad = nxt.grad = None
        res = render_views(views[:V], m, r, s_, o.reshape(-1, 1), features_color=sh, flow_xyz=nxt)
        for v in range(V):
            assert torch.equal(res["flow"][v], raw[v][-1][:2])
        (res["flow"] * gf[:V]).sum().backward()
        if V == 1:
            assert _rel(m.grad.cpu().numpy(), g_rast[0].cpu().numpy()) < 1e-6
            assert _rel(nxt.grad.cpu().numpy(), g_rast[1].cpu().numpy()) < 1e-6
    # a moved next-frame pose through render_views equals the raw call with that pose
    nv, pose = _moved_pose(_ref_view(inps[0], "pinhole"), "pinhole")
    moved = views[0]._replace(viewmatrix=pose[0], projmatrix=pose[1])
    res = render_views(views[:1], m, r, s_, o.reshape(-1, 1), features_color=sh, flow_xyz=nxt, flow_cameras=[moved])
    raw_m, _ = _run(views[:1], g, 0, False, nxt_np, poses=[pose])
    assert torch.equal(res["flow"][0], raw_m[0][-1][:2])
    with pytest.raises(ValueError):
        render_views(views[:1], m, r, s_, o.reshape(-1, 1), features_color=sh, flow_xyz=nxt,
                     flow_cameras=[moved._replace(tanfovx=float(views[0].tanfovx) * 1.1)])
    with pytest.raises(ValueError):
        render_views(views, m, r, s_, o.reshape(-1, 1), features_color=sh, flow_xyz=nxt[:10])
    with pytest.raises(ValueError):
        render_views(views, m, r, s_, o.reshape(-1, 1), features_color=sh, flow_xyz=nxt, return_normal=True)
    # the dyna pair: [current cloud with flow_xyz = the next cloud's means, next cloud] in one render_clouds call, against
    # render_views of each cloud; the shared tensor receives the sum of its two uses
    sums = []
    for path in ("clouds", "views"):
        m, r, s_, o, sh = _leaves(g)
        nxt = _t(nxt_np).requires_grad_(True)
        cur = dict(cameras=views, pts_xyz=m, rotations=r, scales=s_, opacity=o.reshape(-1, 1), features_color=sh, flow_xyz=nxt)
        nxc = dict(cameras=views, pts_xyz=nxt, rotations=r, scales=s_, opacity=o.reshape(-1, 1), features_color=sh)
        if path == "clouds":
            a, b = render_clouds([cur, nxc])
        else:
            a = render_views(views, m, r, s_, o.reshape(-1, 1), features_color=sh, flow_xyz=nxt)
            b = render_views(views, nxt, r, s_, o.reshape(-1, 1), features_color=sh)
        assert "flow" not in b
        ((a["flow"] * gf).sum() + (b["render"] * gc).sum()).backward()
        sums.append((a["flow"].detach(), b["render"].detach(), m.grad, nxt.grad, o.grad))
    for x, y in zip(*sums):
        assert _rel(x.double().cpu().numpy(), y.double().cpu().numpy()) < 1e-5


def test_capture_replay_and_memory():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, W, H = 2000, 96, 64
    inps, g = _inputs(P, W, H, 0, 2, seed=19)
    views = [_settings(i, 0) for i in inps]
    m, r, s_, o, sh = _leaves(g)
    nxt = _t(_next(g)).requires_grad_(True)
    gf = torch.randn((2, 2, H, W), device="cuda")
    step = lambda: (render_views(views, m, r, s_, o.reshape(-1, 1), features_color=sh, flow_xyz=nxt)["flow"] * gf).sum()  # noqa: E731
    step().backward()
    torch.cuda.synchronize()
    ref = (m.grad.clone(), nxt.grad.clone())
    # no device-memory growth over repeated eager steps
    for k in range(6):
        m.grad = nxt.grad = None
        step().backward()
        torch.cuda.synchronize()
        if k == 2:
            m2 = torch.cuda.memory_allocated()
    assert torch.cuda.memory_allocated() <= m2
    graph = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m.grad = nxt.grad = None
        step().backward()
    torch.cuda.current_stream().wait_stream(st)
    with torch.cuda.graph(graph):
        m.grad = nxt.grad = None
        step().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert _rel(m.grad.double().cpu().numpy(), ref[0].double().cpu().numpy()) < 1e-5
    assert _rel(nxt.grad.double().cpu().numpy(), ref[1].double().cpu().numpy()) < 1e-5
