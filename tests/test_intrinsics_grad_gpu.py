"""Learnable intrinsics on the GPU: the device field of view and dL/dtan_fov, through the raw calls and the renderers.

* Same values, same results: a device tan_fov equal to the host floats gives the host path's radii, sort keys, tile lists,
  tile ranges, images and instance counts bit for bit (AA on and off; the raw calls, render_views and render_clouds), and,
  on the same blend-stage records, the same per-Gaussian outputs and 27 camera entries bit for bit, with dL_dtan_fov asked
  for or not.  Through the renderers the per-Gaussian gradients agree within the blend stage's run-to-run spread (its
  float atomics rerun with every backward).
* Bound: dL/dtan_fov of every view of every CAM instantiation against intrinsics_ref64 fed blend_ref64's cotangents, and
  on the projection edge scenes of test_project_ref64_gpu (live Gaussians past the frustum clamp on both sides of each
  axis, AA needles on both sides of the 2.5e-5 clamp).
* Gauge identity, with no oracle: scaling fx by s and row 0 of w2c by 1 / s leaves every render unchanged (projection,
  Jacobian, clamp decision and radii are invariant), so through camera_batch with a learnable intr
  fx dL/dK[0,0] = sum_c w2c[0,c] dL/dw2c[0,c], and likewise fy with row 1.  Precomputed colours (campos moves with w2c).
  Tolerance: relative to the sum of the magnitudes of the identity's terms, 4x the worst measured ratio (1.2e-6, H100 80GB
  HBM3): 5e-6.
* accumulate and NULL outputs; a CUDA graph replayed after a new K is written into the captured intr equals an eager step
  at the new K; a 20 % focal change between two steps renders as the host path at the new focal length.
"""
import math

import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
from test_camera_grad_gpu import _intr, _loss, _scene, _targets, _w2c

pytestmark = pytest.mark.gpu
GAUGE_TOL = 5e-6


@pytest.fixture(autouse=True, scope="module")
def _own_capacity_history():
    """The binning-capacity history is process-wide and keyed by (device, P, W, H, view slot): this module starts from an
    empty one and leaves an empty one, so its scenes never size the binning state of another module's first render."""
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _views(V, seed=3, W=96, H=80, device_fov=False, K=None):
    """settings of V cameras of camera_batch; device_fov: tanfovx / tanfovy as 0-dim CUDA tensors of the same floats"""
    from manigaussian_b200.cameras import camera_batch
    cams = camera_batch(_w2c(V, seed), _intr(V, W, H) if K is None else K, W, H)
    vs = [cams.settings(i, torch.zeros(3, device="cuda"), 1, False) for i in range(V)]
    if device_fov:
        vs = [s._replace(tanfovx=torch.tensor(float(np.float32(s.tanfovx)), device="cuda"),
                         tanfovy=torch.tensor(float(np.float32(s.tanfovy)), device="cuda")) for s in vs]
    else:
        vs = [s._replace(tanfovx=float(np.float32(s.tanfovx)), tanfovy=float(np.float32(s.tanfovy))) for s in vs]
    return vs


def _fov(views):
    return torch.tensor([[float(s.tanfovx), float(s.tanfovy)] for s in views], dtype=torch.float32, device="cuda")


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("kind", ["views", "clouds"])
def test_device_fov_equal_to_the_host_floats_renders_bit_for_bit(kind, aa):
    from manigaussian_b200 import rasterizer as R
    V = 5
    sc = _scene(4000, sh=True, seed=21)
    views = _views(V)
    args = (sc["pts_xyz"], None, None, sc["opacity"], sc["scales"], sc["rotations"], 1.0, None, sc["features_color"], 1, False)
    caps = [1 << 17] * V

    def run(tf):
        if kind == "views":
            outs, _ = R.rasterize_views_raw(views, *args, return_depth=True, antialiasing=aa, capacities=caps, tan_fov=tf)
        else:
            c = dict(views=views, means3D=sc["pts_xyz"], sh=sc["features_color"], opacity=sc["opacity"], scales=sc["scales"],
                     rotations=sc["rotations"], capacities=caps)
            if tf is not None:
                c["tan_fov"] = tf
            outs = R.rasterize_clouds_raw([c, dict(c, opacity=sc["opacity"] * 0.7)], 1, False, return_depth=True,
                                          antialiasing=aa)[0]
            outs = outs[0] + outs[1]
        torch.cuda.synchronize()
        res = []
        for o in outs:
            n, cap = int(o.status[0]), int(o[0])
            T = ((96 + 15) // 16) * ((80 + 15) // 16)
            keys = S._arr(R, "binning", "tile_ids", o[5], cap, 0, torch.int32, n)
            plist = S._arr(R, "binning", "point_list", o[5], cap, 0, torch.int32, n)
            ranges = S._arr(R, "image", "ranges", o[6], 96, 80, torch.int32, 2 * T)
            depth_keys = S._arr(R, "geometry", "depths", o[4], 4000, 0, torch.int32, 4000)
            res.append((n, [o[1].clone(), o[3].clone(), o[7].clone()], [keys, plist, ranges, depth_keys]))
        return res

    import test_project_ref64_gpu as S
    host, dev = run(None), run(_fov(views))
    for (n0, t0, a0), (n1, t1, a1) in zip(host, dev):
        assert n0 == n1 and n0 > 0
        assert all(torch.equal(x, y) for x, y in zip(t0, t1))
        assert all(np.array_equal(x, y) for x, y in zip(a0, a1))


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("kind", ["views", "clouds"])
def test_device_fov_through_the_renderers(kind, aa):
    """render_views / render_clouds with the field of view as CUDA tensors equal to the host floats: images and radii bit
    for bit, the per-Gaussian gradients within the blend stage's run-to-run spread"""
    from manigaussian_b200 import gaussian_renderer as GR
    V = 4
    sc = _scene(4000, sh=True, seed=23)

    def run(dev_fov):
        views = _views(V, device_fov=dev_fov)
        p = sc["pts_xyz"].clone().requires_grad_()
        o_ = sc["opacity"].clone().requires_grad_()
        common = dict(pts_xyz=p, rotations=sc["rotations"], scales=sc["scales"], opacity=o_, features_color=sc["features_color"],
                      antialiasing=aa)
        if kind == "views":
            outs = [GR.render_views(views, **common)]
        else:
            c1 = dict(common, opacity=o_ * 0.8)
            c1.pop("antialiasing")
            c0 = dict(common)
            c0.pop("antialiasing")
            outs = GR.render_clouds([dict(cameras=views, **c0), dict(cameras=views, **c1)], antialiasing=aa)
        loss = sum(_loss(o, 41 + i) for i, o in enumerate(outs))
        gp, go = torch.autograd.grad(loss, [p, o_])
        torch.cuda.synchronize()
        return [(o["render"].detach().clone(), o["radii"].clone()) for o in outs], (gp, go)

    (host, gh), (dev, gd) = run(False), run(True)
    for (c0, r0), (c1, r1) in zip(host, dev):
        assert torch.equal(c0, c1) and torch.equal(r0, r1)
    for x, y in zip(gh, gd):
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-6 * float(x.abs().max())), float((x - y).abs().max())


@pytest.mark.parametrize("aa", [False, True])
def test_same_records_give_the_same_outputs_with_and_without_the_intrinsics_option(aa):
    """Stage 2 four times on one set of blend-stage records: {host, device} field of view x {without, with} dL_dtan_fov.
    Every per-Gaussian output and the 27 camera entries are bit-identical; dL_dtan_fov is bit-identical with the host or
    the device field of view."""
    from manigaussian_b200 import _binding as B
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200.parallel import PackedGradients
    V = 17
    sc = _scene(5000, sh=True, seed=3)
    views = _views(V)
    tf = _fov(views)
    outs, streams = R.rasterize_views_raw(views, sc["pts_xyz"], None, None, sc["opacity"], sc["scales"], sc["rotations"], 1.0, None,
                                          sc["features_color"], 1, False, antialiasing=aa, tan_fov=tf)
    g = torch.Generator(device="cuda").manual_seed(5)
    gc = [torch.randn((3, 80, 96), generator=g, device="cuda") for _ in range(V)]
    P = sc["pts_xyz"].shape[0]
    pk = PackedGradients(P, 0, 4, sc["pts_xyz"].device, colors=False, zero=False)
    m2d = torch.empty((V, P, 3), device="cuda")
    cam = (torch.empty((V, 16), device="cuda"), torch.empty((V, 16), device="cuda"), torch.empty((V, 3), device="cuda"),
           torch.empty((V, 2), device="cuda"))
    snaps = []
    real = B.lib()

    class Proxy:
        def __getattr__(self, name):
            return getattr(real, name)

        def mgs_backward_views(self, *args):
            if args[-3] != 2:
                return real.mgs_backward_views(*args)
            iarr = args[2].intrinsics
            for dev_fov, want in ((False, False), (True, False), (True, True), (False, True)):
                a = list(args)
                ia = (B.ViewIntrinsics * V)()
                for v in range(V):
                    ia[v].tan_fov = iarr[v].tan_fov if dev_fov else None
                    ia[v].dL_dtan_fov = iarr[v].dL_dtan_fov if want else None
                a[2] = B.RenderOptions.from_buffer_copy(args[2])
                a[2].intrinsics = ia
                cam[3].fill_(float("nan"))
                rc = real.mgs_backward_views(*a)
                if rc < 0:
                    return rc
                torch.cuda.synchronize()
                snaps.append(([t.clone() for t in pk.views.values()] + [m2d.clone()], [t.clone() for t in cam[:3]],
                              cam[3].clone() if want else None))
            return 0

    orig = R._b.lib
    R._b.lib = lambda: Proxy()
    try:
        R.rasterize_views_backward_raw(views, outs, streams, gc, None, sc["pts_xyz"], None, None, sc["scales"], sc["rotations"],
                                       1.0, None, sc["features_color"], 1, False, antialiasing=aa, camera_grads=cam,
                                       after_blend=lambda: None, accumulate_into=pk.views, means2D_per_view=m2d, tan_fov=tf)
    finally:
        R._b.lib = orig
    assert len(snaps) == 4
    for s in snaps[1:]:
        for x, y in zip(snaps[0][0] + snaps[0][1], s[0] + s[1]):
            assert torch.equal(x, y)
    assert torch.equal(snaps[2][2], snaps[3][2])
    assert bool(torch.isfinite(snaps[2][2]).all()) and float(snaps[2][2].abs().max()) > 0


def test_accumulate_and_null_outputs():
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200.parallel import PackedGradients
    V = 5
    sc = _scene(5000, sh=True, seed=8)
    views = _views(V, device_fov=True)
    outs, streams = R.rasterize_views_raw(views, sc["pts_xyz"], None, None, sc["opacity"], sc["scales"], sc["rotations"], 1.0, None,
                                          sc["features_color"], 1, False)
    g = torch.Generator(device="cuda").manual_seed(9)
    gc = [torch.randn((3, 80, 96), generator=g, device="cuda") for _ in range(V)]
    P = sc["pts_xyz"].shape[0]

    def bwd(cam, acc=False):
        pk = PackedGradients(P, 0, 4, sc["pts_xyz"].device, colors=False, zero=True)
        r = R.rasterize_views_backward_raw(views, outs, streams, gc, None, sc["pts_xyz"], None, None, sc["scales"], sc["rotations"],
                                           1.0, None, sc["features_color"], 1, False, camera_grads=cam, accumulate_into=pk.views,
                                           accumulate=acc)
        torch.cuda.synchronize()
        return r[9] if cam is not None else None

    full = bwd(True)
    assert len(full) == 4 and float(full[3].abs().max()) > 0
    seed = torch.randn((V, 2), device="cuda")
    got = bwd((None, None, None, seed.clone()), acc=True)
    assert got[0] is None and got[1] is None and got[2] is None
    assert torch.allclose(got[3], seed + full[3], rtol=1e-4, atol=1e-5 * float(full[3].abs().max()))
    # the other outputs with dL_dtan_fov NULL
    got = bwd((torch.empty((V, 16), device="cuda"), None, None, None))
    assert got[3] is None and torch.allclose(got[0], full[0], rtol=1e-4, atol=1e-5 * float(full[0].abs().max()))
    # nothing asked for: the device field of view alone
    assert bwd(None) is None


# --------------------------------------------------------------------------- every view against the float64 bound
CAM_CASES = [("views", 1, False, [4]), ("views", 2, False, [17]), ("views", 3, False, [4]), ("views", 1, True, [33]),
             ("views", 2, True, [4]), ("views", 3, True, [17]), ("clouds", 1, False, [2] * 20), ("clouds", 2, False, [3, 2]),
             ("clouds", 3, False, [17]), ("clouds", 1, True, [2, 2]), ("clouds", 2, True, [2, 3]), ("clouds", 3, True, [3])]


@pytest.mark.parametrize("kind,deg,aa,nv", CAM_CASES, ids=[f"{k}-deg{d}-{'aa' if a else 'noaa'}-{'x'.join(map(str, n))}"
                                                          for k, d, a, n in CAM_CASES])
def test_every_tan_fov_gradient_is_within_the_float64_bound(kind, deg, aa, nv):
    import intrinsics_ref64 as I64
    import test_project_ref64_gpu as S
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200 import scenes
    W, H = 32, 24
    clouds, gs, camss = [], [], []
    for b, n in enumerate(nv):
        g = S._cloud_g(150 + 7 * b, deg, 400 + 10 * deg + b)
        cams = [scenes.make_camera(W, H, v + b, n + b) for v in range(n)]
        a = S.g_args(g)
        views = [S.settings(c, deg, aa) for c in cams]
        clouds.append(dict(views=views, means3D=a["means3D"], sh=a["sh"], colors=a["colors"], opacity=a["opacity"],
                           scales=a["scales"], rotations=a["rotations"], cov3D_precomp=a["cov3D_precomp"], tan_fov=_fov(views)))
        gs.append(g)
        camss.append(cams)
    rng = np.random.default_rng(deg + 7 * len(nv))
    gc = [[rng.normal(0, 1, (3, H, W)).astype(np.float32) for _ in cams] for cams in camss]
    gd = [[rng.normal(0, 1, (H, W)).astype(np.float32) for _ in cams] for cams in camss]
    if kind == "views":
        c = clouds[0]
        outs, streams = R.rasterize_views_raw(c["views"], c["means3D"], c["colors"], None, c["opacity"], c["scales"], c["rotations"],
                                              1.0, None, c["sh"], deg, False, return_depth=True, antialiasing=aa, tan_fov=c["tan_fov"])
        outs = [outs]
    else:
        outs, streams = R.rasterize_clouds_raw(clouds, deg, False, return_depth=True, antialiasing=aa)
    torch.cuda.synchronize()
    per = [[S.view_cotangents(R, outs[b][v], len(gs[b]["means3D"]), cam, gc[b][v], gd[b][v]) for v, cam in enumerate(camss[b])]
           for b in range(len(nv))]
    if kind == "views":
        c = clouds[0]
        r = R.rasterize_views_backward_raw(c["views"], outs[0], streams, [S._t(x) for x in gc[0]], None, c["means3D"], c["colors"],
                                           None, c["scales"], c["rotations"], 1.0, None, c["sh"], deg, False,
                                           grads_depth=[S._t(x) for x in gd[0]], antialiasing=aa, camera_grads=True,
                                           tan_fov=c["tan_fov"])
        got = [r[9][3]]
    else:
        for b, c in enumerate(clouds):
            c["grad_color"], c["grad_depth"] = S._t(np.stack(gc[b])), S._t(np.stack(gd[b]))
        got = [d["dL_dtan_fov"] for d in R.rasterize_clouds_backward_raw(clouds, outs, streams, deg, False, antialiasing=aa,
                                                                         camera_grads=True)]
    torch.cuda.synchronize()
    worst, problems = 0.0, []
    for b in range(len(nv)):
        recs, cots = [r_[0] for r_ in per[b]], [r_[1] for r_ in per[b]]
        ref = I64.tan_fov_grads(gs[b], camss[b], cots, live=[k["radii"] > 0 for k in recs], antialias=aa)
        for v in range(len(camss[b])):
            x = got[b][v].cpu().numpy()
            r_ = I64.ratio(x, ref[v])
            worst = max(worst, float(r_.max()))
            if r_.max() > I64.KAPPA_INTR:
                problems.append((b, v, float(r_.max()), x.tolist(), ref[v][0].tolist()))
    print(f"{kind} deg{deg} aa={aa}: worst ratio {worst:.3g}")
    assert not problems, problems[:3]


EDGE_SCENES = [("clamp_x", False), ("clamp_y", False), ("aa1", True), ("aa3", True)]


@pytest.mark.parametrize("scene,aa", EDGE_SCENES, ids=[s for s, _ in EDGE_SCENES])
def test_tan_fov_gradient_on_the_projection_edge_scenes(scene, aa):
    """The edge scenes of test_project_ref64_gpu through the views call with the device field of view: dL/dtan_fov within
    the float64 bound.  The clamp scenes hold live Gaussians past the frustum clamp on both sides of their axis, whose clamp
    term therefore runs on the GPU with both signs."""
    import intrinsics_ref64 as I64
    import project_ref64 as P64
    import test_project_ref64_gpu as S
    from manigaussian_b200 import rasterizer as R
    sc = S.SCENES[scene]()
    g, cam = sc["g"], sc["cam"]
    deg = int(g["sh_degree"]) if g.get("shs") is not None else 0
    W, H = cam["W"], cam["H"]
    views = [S.settings(cam, deg, aa)]
    tf = _fov(views)
    a = S.g_args(g)
    outs, streams = R.rasterize_views_raw(views, a["means3D"], a["colors"], None, a["opacity"], a["scales"], a["rotations"], 1.0,
                                          a["cov3D_precomp"], a["sh"], deg, False, return_depth=True, antialiasing=aa, tan_fov=tf)
    torch.cuda.synchronize()
    rng = np.random.default_rng(11)
    gc, gd = rng.normal(0, 1, (3, H, W)).astype(np.float32), rng.normal(0, 1, (H, W)).astype(np.float32)
    P = len(g["means3D"])
    rec, cot = S.view_cotangents(R, outs[0], P, cam, gc, gd)
    r = R.rasterize_views_backward_raw(views, outs, streams, [S._t(gc)], None, a["means3D"], a["colors"], None, a["scales"],
                                       a["rotations"], 1.0, a["cov3D_precomp"], a["sh"], deg, False, grads_depth=[S._t(gd)],
                                       antialiasing=aa, camera_grads=True, tan_fov=tf)
    torch.cuda.synchronize()
    live = rec["radii"] > 0
    if scene.startswith("clamp"):
        ax = 0 if scene == "clamp_x" else 1
        G = P64._geometry(P64._cols(g["means3D"]), P64.cov3d(g)[0], P64.view_of(cam))
        u = (G["t"][ax] / G["tz"]).v
        out = ~(G["inx"] if ax == 0 else G["iny"]) & live
        assert (out & (u > 0)).any() and (out & (u < 0)).any()
    ref = I64.tan_fov_grads(g, [cam], [cot], live=[live], antialias=aa)[0]
    x = r[9][3][0].cpu().numpy()
    ratio = I64.ratio(x, ref)
    print(f"{scene}: dL/dtan_fov {x.tolist()} ref {ref[0].tolist()} ratio {float(ratio.max()):.3g}")
    assert np.abs(ref[0]).max() > 0
    assert float(ratio.max()) <= I64.KAPPA_INTR, (x.tolist(), ref[0].tolist())


# --------------------------------------------------------------------------- gauge identity through camera_batch
def _K(V, W=96, H=80):
    return torch.tensor(_intr(V, W, H), dtype=torch.float32, device="cuda")


GAUGE = [("views", 4, dict()), ("views", 1, dict()), ("views", 4, dict(antialiasing=True)),
         ("views", 4, dict(return_depth=True, return_alpha=True)), ("views", 4, dict(F=40)),
         ("views", 4, dict(targets=True, ssim=True, F=8)), ("views", 33, dict()), ("views", 4, dict(sync_gradients=True)),
         ("clouds", 3, dict()), ("clouds", 3, dict(antialiasing=True)), ("rasterizer", 1, dict()),
         ("rasterizer", 1, dict(antialiasing=True)), ("rasterizer", 1, dict(F=3))]


@pytest.mark.parametrize("kind,V,kw", GAUGE, ids=[f"{k}-V{V}-{'-'.join(kw) or 'plain'}" for k, V, kw in GAUGE])
def test_focal_scale_gauge_identity(kind, V, kw):
    from test_camera_grad_gpu import _render
    from manigaussian_b200.cameras import camera_batch
    kw = dict(kw)
    F = kw.pop("F", 0)
    sc = _scene(3000, F=F, sh=False, seed=17)
    if kw.pop("targets", False):
        kw["targets"] = _targets(V, F)
    w2c = _w2c(V).requires_grad_()
    K = _K(V).requires_grad_()
    cams = camera_batch(w2c, K, 96, 80)
    outs = _render(kind, cams, sc, V, **kw)
    loss = sum(_loss(o, 31 + i) for i, o in enumerate(outs))
    gw, gK = torch.autograd.grad(loss, [w2c, K])
    worst = 0.0
    for ax in (0, 1):
        lhs = (K[:, ax, ax] * gK[:, ax, ax]).double()
        terms = (w2c[:, ax, :] * gw[:, ax, :]).double()
        rhs = terms.sum(1)
        scale = lhs.abs() + terms.abs().sum(1)
        r = float(((lhs - rhs).abs() / scale).max())
        worst = max(worst, r)
        assert float(lhs.abs().max()) > 0
    print(f"{kind} V={V} {sorted(kw)}: worst ratio {worst:.3g}")
    assert worst <= GAUGE_TOL, worst


def test_focal_gradient_reaches_the_jacobian_path():
    """Without the kernel's dL/dtan_fov the gauge identity fails: the projection-matrix path alone is not the gradient."""
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import camera_batch
    V = 4
    sc = _scene(3000, sh=False, seed=17)
    w2c = _w2c(V).requires_grad_()
    K = _K(V).requires_grad_()
    cams = camera_batch(w2c, K, 96, 80)
    o = GR.render_views(cams, pts_xyz=sc["pts_xyz"], rotations=sc["rotations"], scales=sc["scales"], opacity=sc["opacity"],
                        pts_rgb=sc["pts_rgb"])
    loss = _loss(o, 5)
    g_tf, g_pm, gw, gK = torch.autograd.grad(loss, [cams.tan_fov, cams.full_proj_transform, w2c, K])
    assert float(g_tf.abs().max()) > 0
    lhs = (K[:, 0, 0] * gK[:, 0, 0]).double()
    only_pm = lhs - (K[:, 0, 0] * g_tf[:, 0] * (-cams.tan_fov[:, 0] / K[:, 0, 0])).double()
    rhs = (w2c[:, 0, :] * gw[:, 0, :]).double().sum(1)
    assert float(((only_pm - rhs).abs() / (lhs.abs() + rhs.abs())).max()) > 100 * GAUGE_TOL


# --------------------------------------------------------------------------- graph replay, focal change
def test_graph_replay_reads_the_new_intrinsics():
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import camera_batch
    V = 4
    sc = _scene(3000, sh=True, seed=12)
    w2c = _w2c(V).requires_grad_()
    K = _K(V).requires_grad_()
    tgt = _targets(V, 0)

    def step():
        cams = camera_batch(w2c, K, 96, 80)
        o = GR.render_views(cams, pts_xyz=sc["pts_xyz"], rotations=sc["rotations"], scales=sc["scales"],
                            opacity=sc["opacity"], features_color=sc["features_color"], targets=tgt)
        loss = o["loss_rgb"].sum()
        loss.backward()
        return loss.detach()

    def eager():
        w2c.grad = K.grad = None
        loss = step()
        torch.cuda.synchronize()
        return loss.clone(), w2c.grad.clone(), K.grad.clone()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            w2c.grad = K.grad = None
            step()
    torch.cuda.current_stream().wait_stream(s)
    old = eager()
    graph = torch.cuda.CUDAGraph()
    w2c.grad = K.grad = None
    with torch.cuda.graph(graph):
        g_loss = step()
    K2 = K.detach() * torch.tensor([[1.05, 1, 1], [1, 0.95, 1], [1, 1, 1]], device="cuda")
    with torch.no_grad():
        K.copy_(K2)
    graph.replay()
    torch.cuda.synchronize()
    rep = (g_loss.clone(), w2c.grad.clone(), K.grad.clone())
    new = eager()
    for x, y in zip(rep, new):
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-5 * float(y.abs().max())), float((x - y).abs().max())
    assert not torch.allclose(rep[0], old[0], rtol=1e-4)   # not the capture-time K


def test_twenty_percent_focal_change_between_steps():
    """The radii and instance counts change with the focal length; the device path at the new K renders as the host path
    at the new K, bit for bit (the capacity slack, warning and raise cover the new counts)."""
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import build_cameras, camera_batch
    V = 3
    sc = _scene(4000, sh=True, seed=14)
    w2c = _w2c(V)
    K = _K(V).requires_grad_()
    common = dict(pts_xyz=sc["pts_xyz"], rotations=sc["rotations"], scales=sc["scales"], opacity=sc["opacity"],
                  features_color=sc["features_color"])
    r0 = GR.render_views(camera_batch(w2c, K, 96, 80), **common)
    with torch.no_grad():
        K.mul_(torch.tensor([[1.2, 1, 1], [1, 1.2, 1], [1, 1, 1]], device="cuda"))
    cams = camera_batch(w2c, K, 96, 80)
    r1 = GR.render_views(cams, **common)
    torch.cuda.synchronize()
    assert not torch.equal(r0["radii"], r1["radii"])
    # the host path with the same float32 tan_fov values and the same matrices
    host = build_cameras(K.detach(), torch.linalg.inv(w2c.double()), 96, 80)
    tf = cams.tan_fov.detach().float().cpu()
    views = [host.settings(i, torch.zeros(3, device="cuda"), 1, False)._replace(
        tanfovx=float(tf[i, 0]), tanfovy=float(tf[i, 1]), viewmatrix=cams.world_view_transform[i].detach(),
        projmatrix=cams.full_proj_transform[i].detach(), campos=cams.camera_center[i].detach()) for i in range(V)]
    r2 = GR.render_views(views, **common)
    torch.cuda.synchronize()
    assert torch.equal(r1["radii"], r2["radii"]) and torch.equal(r1["render"], r2["render"])
    assert math.isfinite(float(r1["render"].sum()))
