"""Camera gradients on the GPU, through the public paths.

Gauge identity.  Translating the whole world by `a` (means p + a, cameras w2c T(-a)) leaves every render unchanged, so the
gradient reaching `a` through the cameras equals -sum_i dL/dmeans3D_i.  Rotating the world by exp([w]) (means R p, cameras
w2c R^T, quaternions composed, precomputed colours) likewise gives: camera-path gradient = -(Gaussian-path gradient).  Both
sides come from different kernels' sums (the camera rows against the per-Gaussian chain), so the identity checks every
camera term that reaches a rigid motion: dL/dvm through t and through J, dL/dpm, and dL/dcampos through the SH direction.
Tolerance: relative to sum_i |per-Gaussian term|, set at 4x the worst measured ratio (translation 6.7e-9, rotation
1.2e-8, on an H100 80GB HBM3): 5e-8.

Also: the per-Gaussian gradients are unchanged by asking for camera gradients; accumulate = 1 adds onto seeded buffers;
each output may be NULL; V crosses 16 views per launch; many clouds match render_views; a CUDA graph replays equal to
eager.
"""
import math

import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)

pytestmark = pytest.mark.gpu
TOL = 5e-8


def _scene(P, F=0, sh=True, seed=0, dev="cuda"):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)  # noqa: E731
    q = torch.randn(P, 4, generator=g, dtype=torch.float64)
    d = dict(pts_xyz=(r(P, 3) - 0.5) * 0.8, rotations=q / q.norm(dim=1, keepdim=True), scales=0.004 + 0.03 * r(P, 3),
             opacity=0.2 + 0.7 * r(P, 1))
    if sh:
        d["features_color"] = 0.3 * torch.randn(P, 4, 3, generator=g, dtype=torch.float64)
    else:
        d["pts_rgb"] = r(P, 3)
    if F:
        d["features_language"] = torch.randn(P, F, generator=g, dtype=torch.float64)
    return {k: v.float().to(dev) for k, v in d.items()}


def _w2c(V, seed=1):
    """V world->camera transforms looking at the origin from about 2 units away"""
    g = np.random.default_rng(seed)
    out = []
    for v in range(V):
        th, ph = 0.5 * g.standard_normal(), 0.3 * g.standard_normal()
        eye = 2.0 * np.array([math.sin(th) * math.cos(ph), math.sin(ph), -math.cos(th) * math.cos(ph)])
        f = -eye / np.linalg.norm(eye)
        rgt = np.cross(np.array([0.0, 1.0, 0.0]), f)
        rgt /= np.linalg.norm(rgt)
        up = np.cross(f, rgt)
        R = np.stack([rgt, up, f])
        M = np.eye(4)
        M[:3, :3], M[:3, 3] = R, -R @ eye
        out.append(M)
    return torch.tensor(np.stack(out), dtype=torch.float32, device="cuda")


def _intr(V, W=96, H=80):
    K = np.array([[90.0, 0, W / 2 + 3], [0, 95.0, H / 2 - 2], [0, 0, 1]])
    return np.broadcast_to(K, (V, 3, 3)).copy()


def _skew(w):
    z = torch.zeros_like(w[0])
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def _rot(w):
    return torch.linalg.matrix_exp(_skew(w))


def _loss(out, seed, depth=False, alpha=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    L = 0.0
    for k in ("render", "render_embed", "depth", "alpha"):
        x = out.get(k)
        if x is None:
            continue
        L = L + (x * torch.randn(x.shape, generator=g, device="cuda")).sum()
    for k in ("loss_rgb", "loss_embed", "loss_l1", "ssim"):
        if k in out:
            L = L + out[k].sum() * (1.0 + 0.25 * len(k))
    return L


def _render(kind, cams, sc, V, **kw):
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.rasterizer import GaussianRasterizer
    common = dict(pts_xyz=sc["pts_xyz"], rotations=sc["rotations"], scales=sc["scales"], opacity=sc["opacity"],
                  pts_rgb=sc.get("pts_rgb"), features_color=sc.get("features_color"), features_language=sc.get("features_language"))
    if kind == "views":
        return [GR.render_views(cams, **common, **kw)]
    if kind == "clouds":   # the dyna pair: two clouds sharing the camera tensors
        sc2 = {k: v for k, v in common.items()}
        sc2["opacity"] = common["opacity"] * 0.8
        return GR.render_clouds([dict(cameras=cams, **common), dict(cameras=cams, **sc2)], **kw)
    # GaussianRasterizer of view 0
    st = cams.settings(0, torch.zeros(3, device="cuda"), 1 if sc.get("features_color") is not None else 3,
                       sc.get("features_language") is not None)
    if kw.get("antialiasing"):
        st = st._replace(antialiasing=True)
    m2 = torch.zeros_like(sc["pts_xyz"], requires_grad=True)
    out = GaussianRasterizer(st)(means3D=common["pts_xyz"], means2D=m2, opacities=common["opacity"],
                                 shs=common["features_color"], colors_precomp=common["pts_rgb"] if common["features_color"] is None else None,
                                 language_feature_precomp=common["features_language"], scales=common["scales"],
                                 rotations=common["rotations"])
    return [{"render": out[0], "render_embed": out[1] if out[1].numel() else None}]


GAUGE = [
    ("views", 1, dict(), dict(sh=True)),
    ("views", 4, dict(), dict(sh=True)),
    ("views", 4, dict(antialiasing=True), dict(sh=True)),
    ("views", 4, dict(return_depth=True, return_alpha=True), dict(sh=True)),
    ("views", 4, dict(), dict(sh=False, F=3)),
    ("views", 4, dict(), dict(sh=True, F=40)),
    ("views", 4, dict(targets=True, ssim=True), dict(sh=True, F=32)),
    ("clouds", 2, dict(), dict(sh=True)),
    ("rasterizer", 1, dict(), dict(sh=True)),
    ("rasterizer", 1, dict(antialiasing=True), dict(sh=False)),
]


def _targets(V, F, seed=4):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = {"rgb": torch.rand((V, 3, 80, 96), generator=g, device="cuda")}
    if F:
        t["embed"] = torch.randn((V, F, 80, 96), generator=g, device="cuda")
    return t


@pytest.mark.parametrize("kind,V,kw,sk", GAUGE, ids=[f"{k}-V{V}-{'-'.join(kw) or 'plain'}-{'sh' if s['sh'] else 'rgb'}-F{s.get('F', 0)}"
                                                    for k, V, kw, s in GAUGE])
@pytest.mark.parametrize("motion", ["translate", "rotate"])
def test_rigid_motion_of_the_world_moves_no_gradient(kind, V, kw, sk, motion):
    from manigaussian_b200.cameras import camera_batch
    if motion == "rotate" and sk["sh"]:
        sk = dict(sk, sh=False)   # the rotation identity holds for view-independent colours (SH would need rotating)
    sc = _scene(3000, F=sk.get("F", 0), sh=sk["sh"], seed=7)
    kw = dict(kw)
    if kw.pop("targets", False):
        kw["targets"] = _targets(V, sk.get("F", 0))
    w2c0 = _w2c(V)
    a = torch.zeros(3, device="cuda", requires_grad=True)
    p = sc["pts_xyz"].clone().requires_grad_()
    rq = sc["rotations"].clone().requires_grad_()
    # camera path: the cameras follow the inverse motion, the Gaussians stay
    if motion == "translate":
        T = torch.eye(4, device="cuda").repeat(V, 1, 1)
        T = torch.cat([torch.cat([T[:, :3, :3], -a.expand(V, 3)[..., None]], 2), T[:, 3:]], 1)
        w2c = w2c0 @ T
    else:
        R4 = torch.nn.functional.pad(_rot(a).T, (0, 1, 0, 1)) + torch.nn.functional.pad(torch.ones(1, 1, device="cuda"), (3, 0, 3, 0))
        w2c = w2c0 @ R4
    sc2 = dict(sc, pts_xyz=p, rotations=rq)
    cams = camera_batch(w2c, _intr(V), 96, 80)
    outs = _render(kind, cams, sc2, V, **kw)
    loss = sum(_loss(o, 11 + i) for i, o in enumerate(outs))
    cam_side = torch.autograd.grad(loss, [a], retain_graph=True)[0].double()
    # the same gradient through the Gaussians only: the cameras held fixed
    a2 = torch.zeros(3, device="cuda", requires_grad=True)
    if motion == "translate":
        sc3 = dict(sc, pts_xyz=p + a2, rotations=rq)
    else:
        # the quaternion of exp([a2]) to first order, (1, a2 / 2), composed with rq: the gradient at a2 = 0 is what is checked
        Rw2 = _rot(a2)
        h2 = 0.5 * a2
        r1, v1 = rq[:, :1], rq[:, 1:]
        rot2 = torch.cat([r1 - (v1 @ h2)[:, None], v1 + r1 * h2 + torch.cross(h2.expand_as(v1), v1, dim=1)], 1)
        sc3 = dict(sc, pts_xyz=p @ Rw2.T, rotations=rot2)
    cams0 = camera_batch(w2c0, _intr(V), 96, 80)
    outs0 = _render(kind, cams0, sc3, V, **kw)
    loss0 = sum(_loss(o, 11 + i) for i, o in enumerate(outs0))
    gp, gq = torch.autograd.grad(loss0, [p, rq], retain_graph=True)
    gaus_side = torch.autograd.grad(loss0, [a2])[0].double()
    # scale: sum over Gaussians of the per-Gaussian magnitudes of that path
    if motion == "translate":
        scale = gp.double().abs().sum()
    else:
        scale = torch.cross(p.detach().double(), gp.double(), dim=1).abs().sum() + gq.double().abs().sum()
    ratio = float((cam_side + gaus_side).abs().max() / scale)
    print(f"{kind} V={V} {motion}: ratio {ratio:.3g}, cam {cam_side.tolist()}, gaussians {gaus_side.tolist()}")
    assert float(cam_side.abs().max()) > 0
    assert ratio <= TOL, (ratio, cam_side.tolist(), gaus_side.tolist())


# --------------------------------------------------------------------------- the raw calls
def _raw_setup(V, aa=False, seed=3, P=5000):
    from manigaussian_b200.cameras import camera_batch
    from manigaussian_b200.rasterizer import rasterize_views_raw
    sc = _scene(P, sh=True, seed=seed)
    cams = camera_batch(_w2c(V, seed), _intr(V), 96, 80)
    views = [cams.settings(i, torch.zeros(3, device="cuda"), 1, False) for i in range(V)]
    outs, streams = rasterize_views_raw(views, sc["pts_xyz"], None, None, sc["opacity"], sc["scales"], sc["rotations"], 1.0, None,
                                        sc["features_color"], 1, False, antialiasing=aa)
    torch.cuda.synchronize()
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    gc = [torch.randn((3, 80, 96), generator=g, device="cuda") for _ in range(V)]
    return sc, views, outs, streams, gc


def _raw_bwd(sc, views, outs, streams, gc, aa, camera_grads=None, after_blend=None, accumulate_into=None, accumulate=False):
    from manigaussian_b200.rasterizer import rasterize_views_backward_raw
    return rasterize_views_backward_raw(views, outs, streams, gc, None, sc["pts_xyz"], None, None, sc["scales"], sc["rotations"],
                                        1.0, None, sc["features_color"], 1, False, antialiasing=aa, camera_grads=camera_grads,
                                        after_blend=after_blend, accumulate_into=accumulate_into, accumulate=accumulate)


@pytest.mark.parametrize("V", [1, 4, 17, 33])
@pytest.mark.parametrize("aa", [False, True])
def test_camera_gradients_leave_the_per_gaussian_outputs_unchanged(V, aa):
    """V crosses 16 views per launch; the blend stage reruns with its float atomics on every call, so the per-Gaussian
    sums and the camera gradients of two calls agree within that stage's spread"""
    from manigaussian_b200.parallel import PackedGradients
    sc, views, outs, streams, gc = _raw_setup(V, aa)
    P = sc["pts_xyz"].shape[0]
    def run(cam):
        pk = PackedGradients(P, 0, 4, sc["pts_xyz"].device, colors=False, zero=False)
        r = _raw_bwd(sc, views, outs, streams, gc, aa, camera_grads=cam, accumulate_into=pk.views)
        torch.cuda.synchronize()
        return [t.clone() for t in pk.views.values()], (r[9] if cam else None)

    base, _ = run(None)
    on1, c1 = run(True)
    on2, c2 = run(True)
    # the blend stage reruns each time with float atomics; the per-Gaussian sums then see the records of their own run, so
    # the comparison is per field within the spread of the blend stage
    for x, y in zip(base, on1):
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-6 * float(x.abs().max() + 1e-30))
    for x, y in zip(c1, c2):
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-6 * float(x.abs().max() + 1e-30))
    assert all(bool(torch.isfinite(t).all()) for t in c1)
    # constant entries are exactly zero
    vm, pm = c1[0].view(V, 4, 4), c1[1].view(V, 4, 4)
    assert bool((vm[:, :, 3] == 0).all()) and bool((pm[:, :, 2] == 0).all())


@pytest.mark.parametrize("which", [0, 1, 2])
def test_accumulate_and_null_outputs(which):
    V = 5
    sc, views, outs, streams, gc = _raw_setup(V, False)
    full = _raw_bwd(sc, views, outs, streams, gc, False, camera_grads=True)[9]
    torch.cuda.synchronize()
    from manigaussian_b200 import _binding as B
    assert B.lib().mgs_camera_grad_scratch_bytes(sc["pts_xyz"].shape[0]) == math.ceil(sc["pts_xyz"].shape[0] / 128) * 27 * 4
    seeds = [torch.randn((V, 16), device="cuda"), torch.randn((V, 16), device="cuda"), torch.randn((V, 3), device="cuda")]
    bufs = [s.clone() for s in seeds]
    bufs[which] = None
    P = sc["pts_xyz"].shape[0]
    from manigaussian_b200.parallel import PackedGradients
    pk = PackedGradients(P, 0, 4, sc["pts_xyz"].device, colors=False, zero=True)
    got = _raw_bwd(sc, views, outs, streams, gc, False, camera_grads=tuple(bufs), accumulate_into=pk.views, accumulate=True)[9]
    torch.cuda.synchronize()
    for i in range(3):
        if i == which:
            assert got[i] is None
            continue
        want = seeds[i] + full[i]
        assert torch.allclose(got[i], want, rtol=1e-4, atol=1e-5 * float(full[i].abs().max() + 1e-30)), i


def test_clouds_of_many_views_and_many_clouds_match_render_views():
    """20 clouds x 2 views and one cloud of 17 views: each cloud's camera gradients equal render_views' on that cloud"""
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import camera_batch
    for B_, V in ((20, 2), (1, 17)):
        scs = [_scene(800, sh=True, seed=30 + b) for b in range(B_)]
        w2cs = [_w2c(V, 40 + b).requires_grad_() for b in range(B_)]
        cams = [camera_batch(w, _intr(V), 96, 80) for w in w2cs]
        common = lambda s: dict(pts_xyz=s["pts_xyz"], rotations=s["rotations"], scales=s["scales"], opacity=s["opacity"],  # noqa: E731
                                features_color=s["features_color"])
        outs = GR.render_clouds([dict(cameras=c, **common(s)) for c, s in zip(cams, scs)])
        sum(_loss(o, 70 + b) for b, o in enumerate(outs)).backward()
        got = [w.grad.clone() for w in w2cs]
        for b in range(B_):
            w = w2cs[b].detach().clone().requires_grad_()
            o = GR.render_views(camera_batch(w, _intr(V), 96, 80), **common(scs[b]))
            _loss(o, 70 + b).backward()
            scale = float(w.grad.abs().max())
            assert torch.allclose(got[b], w.grad, rtol=0, atol=1e-4 * scale), (b, float((got[b] - w.grad).abs().max()), scale)


def test_graph_replay_equals_eager():
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import CameraBatch, camera_batch
    V = 4
    sc = _scene(3000, sh=True, seed=12)
    w2c = _w2c(V).requires_grad_()
    p = sc["pts_xyz"].clone().requires_grad_()

    base = camera_batch(w2c.detach(), _intr(V), 96, 80)
    projT = torch.linalg.solve(base.world_view_transform, base.full_proj_transform)   # on the device, outside the capture
    tgt = _targets(V, 0)

    def step():
        # camera_batch's expressions of w2c, with the projection already on the device (its host->device copy cannot be
        # captured)
        wvt = w2c.transpose(-1, -2)
        cams = CameraBatch(*tuple(base)[:6], wvt, wvt @ projT, -(w2c[:, :3, :3].transpose(-1, -2) @ w2c[:, :3, 3:])[..., 0])
        o = GR.render_views(cams, pts_xyz=p, rotations=sc["rotations"], scales=sc["scales"],
                            opacity=sc["opacity"], features_color=sc["features_color"], targets=tgt)
        return o["loss_rgb"].sum()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            w2c.grad = None
            step().backward()
    torch.cuda.current_stream().wait_stream(s)
    eager = w2c.grad.clone()
    graph = torch.cuda.CUDAGraph()
    w2c.grad = None
    with torch.cuda.graph(graph):
        step().backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.allclose(w2c.grad, eager, rtol=1e-4, atol=1e-5 * float(eager.abs().max())), float((w2c.grad - eager).abs().max())


# --------------------------------------------------------------------------- every entry against the float64 bound
# (kernel, SH degree, AA, views): one case per CAM instantiation; the launchers dispatch on the degree (<= 1, 2, 3) and AA
CAM_CASES = [("views", 1, False, [4]), ("views", 2, False, [17]), ("views", 3, False, [4]), ("views", 1, True, [33]),
             ("views", 2, True, [4]), ("views", 3, True, [17]), ("clouds", 1, False, [2] * 20), ("clouds", 2, False, [3, 2]),
             ("clouds", 3, False, [17]), ("clouds", 1, True, [2, 2]), ("clouds", 2, True, [2, 3]), ("clouds", 3, True, [3])]
MEASURED = {}


@pytest.mark.parametrize("kind,deg,aa,nv", CAM_CASES, ids=[f"{k}-deg{d}-{'aa' if a else 'noaa'}-{'x'.join(map(str, n))}"
                                                          for k, d, a, n in CAM_CASES])
def test_every_camera_entry_is_within_the_float64_bound(kind, deg, aa, nv):
    """Each of the 12 CAM instantiations (checked on the launch) against camera_ref64 fed blend_ref64's cotangents of our
    records (test_project_ref64_gpu's builders and view_cotangents), depth cotangents on."""
    import camera_ref64 as C64
    import test_project_ref64_gpu as S
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200 import scenes
    W, H = 32, 24
    clouds, gs, camss = [], [], []
    for b, n in enumerate(nv):
        g = S._cloud_g(150 + 7 * b, deg, 400 + 10 * deg + b)
        cams = [scenes.make_camera(W, H, v + b, n + b) for v in range(n)]
        a = S.g_args(g)
        clouds.append(dict(views=[S.settings(c, deg, aa) for c in cams], means3D=a["means3D"], sh=a["sh"], colors=a["colors"],
                           opacity=a["opacity"], scales=a["scales"], rotations=a["rotations"], cov3D_precomp=a["cov3D_precomp"]))
        gs.append(g)
        camss.append(cams)
    rng = np.random.default_rng(deg + 7 * len(nv))
    gc = [[rng.normal(0, 1, (3, H, W)).astype(np.float32) for _ in cams] for cams in camss]
    gd = [[rng.normal(0, 1, (H, W)).astype(np.float32) for _ in cams] for cams in camss]
    if kind == "views":
        c = clouds[0]
        outs, streams = R.rasterize_views_raw(c["views"], c["means3D"], c["colors"], None, c["opacity"], c["scales"], c["rotations"],
                                              1.0, None, c["sh"], deg, False, return_depth=True, antialiasing=aa)
        outs = [outs]
    else:
        outs, streams = R.rasterize_clouds_raw(clouds, deg, False, return_depth=True, antialiasing=aa)
    torch.cuda.synchronize()
    per = [[S.view_cotangents(R, outs[b][v], len(gs[b]["means3D"]), cam, gc[b][v], gd[b][v]) for v, cam in enumerate(camss[b])]
           for b in range(len(nv))]

    def backward():
        if kind == "views":
            c = clouds[0]
            r = R.rasterize_views_backward_raw(c["views"], outs[0], streams, [S._t(x) for x in gc[0]], None, c["means3D"], c["colors"],
                                               None, c["scales"], c["rotations"], 1.0, None, c["sh"], deg, False,
                                               grads_depth=[S._t(x) for x in gd[0]], antialiasing=aa, camera_grads=True)
            return [dict(zip(("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos"), r[9]))]
        for b, c in enumerate(clouds):
            c["grad_color"], c["grad_depth"] = S._t(np.stack(gc[b])), S._t(np.stack(gd[b]))
        return R.rasterize_clouds_backward_raw(clouds, outs, streams, deg, False, antialiasing=aa, camera_grads=True)

    names = S._launched(lambda: backward())
    nsh = {1: 12, 2: 27, 3: 48}[deg]
    assert any(f"project_bwd_{kind}_kernel<{nsh}," in n and n.endswith(f"true, {'true' if aa else 'false'}>(mgs::ProjectBwd"
                                                                         f"{'Views' if kind == 'views' else 'Clouds'}Args)")
               for n in names), names
    got = backward()
    torch.cuda.synchronize()
    worst, problems = 0.0, []
    for b in range(len(nv)):
        recs, cots = [r[0] for r in per[b]], [r[1] for r in per[b]]
        ref = C64.camera_grads(gs[b], camss[b], cots, live=[k["radii"] > 0 for k in recs],
                               clamped=[S._bits(k["clamped"]) for k in recs], antialias=aa)
        for v in range(len(camss[b])):
            for q in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos"):
                x = got[b][q][v].reshape(-1).cpu().numpy()
                r = C64.ratio(x, ref[v][q])
                worst = max(worst, float(r.max()))
                if r.max() > C64.KAPPA_CAM:
                    problems.append((b, v, q, float(r.max()), x.tolist(), ref[v][q][0].tolist()))
    MEASURED[(kind, deg, aa)] = worst
    print(f"{kind} deg{deg} aa={aa}: worst ratio {worst:.3g}")
    assert not problems, problems[:3]


def test_stage_two_with_and_without_the_camera_option_on_the_same_records():
    """Stage 1 (the blend backward) once, then stage 2 (the per-Gaussian kernel) without cam, with cam, and with cam again on
    the same blend-stage records: the two CAM runs are bit-identical in every output, camera gradients included; without
    cam the per-Gaussian outputs agree to the last bits (a separately compiled instantiation)."""
    from manigaussian_b200 import _binding as B
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200.parallel import PackedGradients
    for V, aa in ((17, False), (4, True)):
        sc, views, outs, streams, gc = _raw_setup(V, aa)
        P = sc["pts_xyz"].shape[0]
        pk = PackedGradients(P, 0, 4, sc["pts_xyz"].device, colors=False, zero=False)
        m2d = torch.empty((V, P, 3), device="cuda")
        cam = (torch.empty((V, 16), device="cuda"), torch.empty((V, 16), device="cuda"), torch.empty((V, 3), device="cuda"))
        snaps = []
        real = B.lib()

        class Proxy:
            def __getattr__(self, name):
                return getattr(real, name)

            def mgs_backward_views(self, *args):
                stages = args[-3]
                if stages != 2:
                    return real.mgs_backward_views(*args)
                for with_cam in (False, True, True):
                    a = list(args)
                    if not with_cam:
                        a[2] = B.RenderOptions.from_buffer_copy(args[2])
                        a[2].camera_grad = None
                    rc = real.mgs_backward_views(*a)
                    if rc < 0:
                        return rc
                    torch.cuda.synchronize()
                    snaps.append(([t.clone() for t in pk.views.values()] + [m2d.clone()],
                                  [t.clone() for t in cam] if with_cam else None))
                return 0

        orig = R._b.lib
        R._b.lib = lambda: Proxy()
        try:
            R.rasterize_views_backward_raw(views, outs, streams, gc, None, sc["pts_xyz"], None, None, sc["scales"], sc["rotations"],
                                           1.0, None, sc["features_color"], 1, False, antialiasing=aa, camera_grads=cam,
                                           after_blend=lambda: None, accumulate_into=pk.views, means2D_per_view=m2d)
        finally:
            R._b.lib = orig
        assert len(snaps) == 3
        for x, y, z in zip(snaps[0][0], snaps[1][0], snaps[2][0]):
            assert torch.equal(y, z)   # two CAM runs: bit for bit
            # the CAM instantiation is compiled separately: where its extra uses of shared products change the compiler's
            # FMA contraction, a per-Gaussian output may move in its last bits, never more
            rel = float((x - y).abs().max() / (x.abs().max() + 1e-30))
            print(f"V={V} aa={aa}: per-Gaussian max |no cam - cam| / max |x| = {rel:.3g}")
            assert rel <= 4 * 2.0 ** -24, rel
        for x, y in zip(snaps[1][1], snaps[2][1]):
            assert torch.equal(x, y)
        assert float(snaps[1][1][0].abs().max()) > 0
