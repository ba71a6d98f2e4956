"""Fisheye views on the GPU (include/mgs_rasterizer.h, "Fisheye views").

* Forward records: every record of project_fwd<AA, FOV, MODEL_FISHEYE> (means2D, conic, radius, depth, tiles, o_eff)
  against tests/fisheye_ref64.py within KAPPA u e, on edge scenes: means on the optical axis and inside the series band,
  both sides of theta_max and of the near cull, theta near 80 degrees, a Kannala-Brandt (KB4) calibration; host and device
  focal lengths, AA on and off.  Gaussians with a borderline decision are left out.
* Backward: the 12 FISHEYE instantiations of project_bwd (views / clouds x AA x NSH in {12, 27, 48}), fed blend_ref64's
  cotangents of our own records: every per-Gaussian sum within KAPPA_FISHEYE u e + d, the 35 camera outputs within
  KAPPA_FISHEYE_CAM (u e + d) and dL/dtan_fov within KAPPA_FISHEYE_INTR (u e + d), over 1 to 33 views, SH degrees 0-3,
  precomputed colours and covariances, and 20 clouds.  Each instantiation is launched.
* Mixed pinhole + orthographic + fisheye batches: images, radii, sort keys and instance counts bit-identical to each view
  rendered alone, gradients the sum over the views within 1e-5 relative L2.  All-zero fisheye entries match a NULL fisheye
  array bit for bit (gradients within 1e-5: the float atomics' order).
* Public paths: render_views with every option, render_clouds, lift_views, GaussianRasterizer, a CUDA-graph replay and no
  device memory growth.

KAPPA: 4x the worst ratio measured over these cases on an H100 80GB HBM3 (700 W); the measured values are beside them and in
DESIGN.md §4.
"""
import json
import os

import numpy as np
import pytest
import torch

import camera_ref64 as C64
import fisheye_ref64 as F64
import intrinsics_ref64 as I64
import project_ref64 as P64
import test_ortho_gpu as TO
import test_project_ref64_gpu as TP
import util
from manigaussian_b200 import scenes

pytestmark = pytest.mark.gpu

UMI_K = (-0.0318, 0.0019, -0.0015, 0.0002)
# per-Gaussian quantities: within bound when max(|x - val| - d, 0) <= KAPPA u e (project_ref64's convention)
# Worst ratios measured over the cases below on an H100 80GB HBM3 (700 W): means2D 0.67, conic 0.19, opacity 0.31, rgb 0.63,
# depth 0; dL_dsh 0.0053; the other per-Gaussian sums 0 (the blend cotangents' inherited bound d covers the whole
# difference); they keep 1, as project_ref64's KAPPA does for quantities that measured 0.
KAPPA_FISHEYE = dict(means2D=2.7, conic=0.78, depth=1.0, opacity=1.25, rgb=2.53, dL_dmeans3D=1.0, dL_dcov3D=1.0, dL_dscales=1.0,
                     dL_drotations=1.0, dL_dsh=0.021, dL_dopacity=1.0, dL_dcolors=1.0, dL_dmeans2D=1.0)
# camera outputs: |x - val| <= KAPPA (u e + d), camera_ref64's convention; measured dL_dcampos 0.0020, dL_dviewmatrix 0.00080,
# dL_dprojmatrix exactly 0
KAPPA_FISHEYE_CAM = 0.008
# dL/dtan_fov, intrinsics_ref64's convention; measured 0.00089
KAPPA_FISHEYE_INTR = 0.0036
_RATIOS = {}


def _note(key, r):
    _RATIOS[key] = max(_RATIOS.get(key, 0.0), float(r))


@pytest.fixture(autouse=True, scope="module")
def _own_capacity_history():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()
    out = os.environ.get("MGS_RATIO_LOG")
    if out:
        with open(out, "w") as fh:
            json.dump(_RATIOS, fh, indent=1, sort_keys=True)


def fcam(v, n, W=32, H=24, k=(0.0, 0.0, 0.0, 0.0), dist=1.1, theta_max=None):
    """fisheye camera v of n around the scene centre, close enough that the cloud spans a wide angle"""
    az = 2.0 * np.pi * v / max(n, 1) + 0.3
    eye = scenes.SCENE_CENTER + np.array([dist * np.cos(az), dist * np.sin(az), 0.5 + 0.05 * v])
    f = W / 3.0
    return F64.fisheye_cam(W, H, f, f * 1.03, (W - 1) / 2 + 0.4, (H - 1) / 2 - 0.3, k, TO._look(eye), theta_max)


def fsettings(cam, deg, aa=False, device_fov=False):
    s = TP.settings(cam, deg, aa)._replace(fisheye=cam["fisheye"])
    if device_fov:
        s = s._replace(tanfovx=torch.tensor(float(cam["tanfovx"]), device="cuda"),
                       tanfovy=torch.tensor(float(cam["tanfovy"]), device="cuda"))
    return s


# --------------------------------------------------------------------------- forward records
def _edge_scene(kind, seed=0):
    """(g, cam): Gaussians placed by view-space angle for a camera at the origin looking along +z (t = p exactly)"""
    rng = np.random.default_rng(seed)
    W, H = 64, 48
    k = UMI_K if kind == "kb4" else (0.0, 0.0, 0.0, 0.0)
    tm = 1.2 if kind == "axis" else None
    cam = F64.fisheye_cam(W, H, W / 3.6, W / 3.5, (W - 1) / 2 + 0.25, (H - 1) / 2 - 0.4, k, np.eye(4), tm)
    if kind == "axis":
        # on the axis, in the series band (r / z from 1e-7 to just past 1/8), both sides of theta_max = 1.2 and of the near cull
        e = np.concatenate([np.zeros(4), 10.0 ** rng.uniform(-7, -1, 40), rng.uniform(0.11, 0.14, 16)])
        th = np.concatenate([np.arctan(e), rng.uniform(1.15, 1.25, 24)])
        z = np.concatenate([rng.uniform(0.5, 3.0, len(th) - 16), rng.uniform(0.15, 0.25, 16)])
    else:
        th = rng.uniform(0.0, 1.45 if kind == "wide" else 1.3, 96)   # up to 83 degrees
        z = rng.uniform(0.4, 2.5, len(th))
    phi = rng.uniform(0, 2 * np.pi, len(th))
    r = np.tan(th) * z
    t = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)
    n = len(t)
    g = scenes.make_gaussians(n, sh_degree=1, seed=seed)
    g["means3D"] = t.astype(np.float32)
    g["scales"] = (np.exp(rng.normal(np.log(0.01), 0.5, (n, 3))) * z[:, None]).astype(np.float32)
    g["cov3D_precomp"] = None
    return g, cam


FWD = [("axis", False, False), ("axis", True, True), ("wide", False, True), ("wide", True, False), ("kb4", False, False),
       ("kb4", True, True)]


@pytest.mark.parametrize("kind,aa,dev", FWD, ids=[f"{k}-{'aa' if a else 'noaa'}-{'device' if d else 'host'}" for k, a, d in FWD])
def test_forward_records_against_float64(kind, aa, dev):
    from manigaussian_b200 import rasterizer as R
    g, cam = _edge_scene(kind)
    a = TP.g_args(g)
    outs, _ = R.rasterize_views_raw([fsettings(cam, 1, aa, dev)], a["means3D"], a["colors"], None, a["opacity"], a["scales"],
                                    a["rotations"], 1.0, None, a["sh"], 1, False, antialiasing=aa)
    torch.cuda.synchronize()
    P = len(g["means3D"])
    k = TP.records(R, outs[0][4], P)
    radii = outs[0][3].cpu().numpy()
    ref = F64.forward(g, cam, 1.0, antialias=aa)
    keep = ~ref["border"]
    assert keep.sum() > 0.7 * P and (~ref["culled"] & keep).sum() > 0.3 * P
    np.testing.assert_array_equal(radii[keep], ref["radius"][keep])
    np.testing.assert_array_equal(k["tiles_touched"][keep], ref["tiles_touched"][keep])
    vis = keep & ~ref["culled"]
    if kind == "axis":   # the scene reaches what it is for: the axis, the band, both culls
        assert (ref["theta"][vis] == 0).any() and (ref["theta"] > 1.2).any() and (ref["culled"] & (g["means3D"][:, 2] > 0.2)).any()
    if kind == "wide":
        assert ref["theta"][vis].max() > np.radians(80)
    got = dict(means2D=k["means2D"], conic=k["conic_opacity"][:, :3], depth=k["depths"], opacity=k["conic_opacity"][:, 3],
               rgb=k["rgb"])
    for q in ("means2D", "conic", "depth", "opacity", "rgb"):
        r = np.abs(got[q][vis] - ref[q][vis]) / (P64.U * ref[q + "_B"][vis] + 1e-30)
        _note(f"fwd {q}", r.max())
        assert float(r.max()) <= KAPPA_FISHEYE[q], (q, float(r.max()))


# --------------------------------------------------------------------------- backward against float64
def _run(g, cams, aa, camera=False, dev=False, shared=True):
    from manigaussian_b200 import rasterizer as R
    deg = int(g["sh_degree"])
    views = [fsettings(c, deg, aa, dev) for c in cams]
    a = TP.g_args(g)
    outs, streams = R.rasterize_views_raw(views, a["means3D"], a["colors"], None, a["opacity"], a["scales"], a["rotations"], 1.0,
                                          a["cov3D_precomp"], a["sh"], deg, False, return_depth=True, antialiasing=aa)
    torch.cuda.synchronize()
    P = len(g["means3D"])
    rng = np.random.default_rng(len(cams) + deg)
    gc = [rng.normal(0, 1, (3, c["H"], c["W"])).astype(np.float32) for c in cams]
    gd = [rng.normal(0, 1, (c["H"], c["W"])).astype(np.float32) for c in cams]
    rc = [TP.view_cotangents(R, outs[v], P, c, gc[v], gd[v]) for v, c in enumerate(cams)]
    grads = R.rasterize_views_backward_raw(views, outs, streams, [TP._t(x) for x in gc], None, a["means3D"], a["colors"], None,
                                           a["scales"], a["rotations"], 1.0, a["cov3D_precomp"], a["sh"], deg, False,
                                           grads_depth=[TP._t(x) for x in gd], antialiasing=aa,
                                           camera_grads=True if camera else None)
    torch.cuda.synchronize()
    return outs, rc, grads


def _check(g, cams, rc, grads, aa, camera, shared=True):
    recs, cots = [r[0] for r in rc], [r[1] for r in rc]
    rb = F64.backward(g, cams, cots, 1.0, antialias=aa, live=[k["radii"] > 0 for k in recs],
                      clamped=[k["clamped"].astype(np.int64) for k in recs], shared_mean2D=shared)
    keep = ~rb["border"]
    for k in recs:
        assert (k["radii"] > 0).sum() > 10
    names = ("dL_dmeans2D", "dL_dcolors", "dL_dfeature", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
             "dL_drotations")
    got = {n: (None if t is None else t.cpu().numpy()) for n, t in zip(names, grads[:9])}
    got.pop("dL_dfeature")
    m2 = got.pop("dL_dmeans2D")
    got["dL_dopacity"] = got["dL_dopacity"][:, 0]
    if g.get("shs") is None:
        got.pop("dL_dsh")
    if g.get("scales") is None:
        got.pop("dL_dscales"), got.pop("dL_drotations")
    else:
        got.pop("dL_dcov3D")
    if g.get("colors_precomp") is None:
        got.pop("dL_dcolors")
    got["dL_dmeans2D"] = (m2[None] if shared else m2)[..., :2]
    problems = []
    for q, x in got.items():
        v, e, d = rb[q]
        if q == "dL_dmeans2D":
            v, e, d = (np.broadcast_to(np.asarray(z), x.shape)[:, keep] for z in (v, e, d))
            x = x[:, keep]
        else:
            v, e, d = (np.broadcast_to(np.asarray(z), x.shape)[keep] for z in (v, e, d))
            x = x[keep]
        r = np.maximum(np.abs(x - v) - d, 0.0) / (P64.U * e + 1e-30)
        w = float(r.max()) if r.size else 0.0
        _note(q, w)
        if w > KAPPA_FISHEYE[q]:
            problems.append(f"{q}: worst {w:.3g}")
    if camera:
        cg = grads[9]
        for vi in range(len(cams)):
            for j, nm in enumerate(("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos")):
                rr = C64.ratio(cg[j][vi].cpu().numpy(), rb["camera"][vi][nm])
                _note(nm, rr.max())
                if rr.max() > KAPPA_FISHEYE_CAM:
                    problems.append(f"view {vi} {nm}: {rr.max():.3g} of the bound")
            assert float(cg[1][vi].abs().max()) == 0   # projmatrix is not read
            if len(cg) > 3:
                rr = I64.ratio(cg[3][vi].cpu().numpy(), rb["tan_fov"][vi])
                _note("dL_dtan_fov", rr.max())
                if rr.max() > KAPPA_FISHEYE_INTR:
                    problems.append(f"view {vi} dL_dtan_fov: {rr.max():.3g} of the bound")
                assert np.abs(rb["tan_fov"][vi][0]).max() > 0
    return problems


VIEWS = [(1, 0, False, False, "sh"), (4, 1, True, True, "sh"), (17, 2, False, True, "sh"), (33, 3, True, True, "sh"),
         (4, 2, True, True, "sh"), (3, 3, False, True, "sh"), (2, 1, False, True, "rgb"), (2, 1, False, True, "cov"),
         (3, 1, False, True, "kb4")]


@pytest.mark.parametrize("V,deg,aa,camera,kind", VIEWS,
                         ids=[f"V{v}-deg{d}-{'aa' if a else 'noaa'}-{'cam' if c else 'nocam'}-{k}" for v, d, a, c, k in VIEWS])
def test_views_backward_against_float64(V, deg, aa, camera, kind):
    g = TP._cloud_g(160, deg, 40 + V + deg, precomp=(kind == "rgb"))
    if kind == "cov":
        S = P64.cov3d(g)[0]
        g["cov3D_precomp"] = np.stack([S[0][0].v, S[0][1].v, S[0][2].v, S[1][1].v, S[1][2].v, S[2][2].v], 1).astype(np.float32)
        g["scales"] = g["rotations"] = None
    cams = [fcam(v, V, k=UMI_K if kind == "kb4" else (0.02 * (v % 3), 0.0, 0.0, 0.0)) for v in range(V)]
    _, rc, grads = _run(g, cams, aa, camera, dev=camera)
    problems = _check(g, cams, rc, grads, aa, camera)
    assert not problems, "\n".join(problems)


CLOUDS = [("20x1", [1] * 20, 1, False), ("2x3-aa", [3, 2], 1, True), ("deg2", [2, 2], 2, False), ("deg2-aa", [2], 2, True),
          ("deg3", [2, 1], 3, False), ("deg3-aa", [1, 2], 3, True)]


@pytest.mark.parametrize("name,nv,deg,aa", CLOUDS, ids=[c[0] for c in CLOUDS])
def test_clouds_backward_against_float64(name, nv, deg, aa):
    from manigaussian_b200 import rasterizer as R
    clouds, gs, camss = [], [], []
    for b, n in enumerate(nv):
        g = TP._cloud_g(100 + 9 * b, deg, 500 + b)
        cams = [fcam(v + b, n + b) for v in range(n)]
        a = TP.g_args(g)
        clouds.append(dict(views=[fsettings(c, deg, aa) for c in cams], means3D=a["means3D"], sh=a["sh"], colors=a["colors"],
                           opacity=a["opacity"], scales=a["scales"], rotations=a["rotations"], cov3D_precomp=None))
        gs.append(g)
        camss.append(cams)
    outs, streams = R.rasterize_clouds_raw(clouds, deg, False, return_depth=True, antialiasing=aa)
    torch.cuda.synchronize()
    rng = np.random.default_rng(len(nv))
    per = []
    for b, c in enumerate(clouds):
        P = len(gs[b]["means3D"])
        gc = [rng.normal(0, 1, (3, 24, 32)).astype(np.float32) for _ in camss[b]]
        gd = [rng.normal(0, 1, (24, 32)).astype(np.float32) for _ in camss[b]]
        per.append([TP.view_cotangents(R, outs[b][v], P, cam, gc[v], gd[v]) for v, cam in enumerate(camss[b])])
        c["grad_color"], c["grad_depth"] = TP._t(np.stack(gc)), TP._t(np.stack(gd))
    grads = R.rasterize_clouds_backward_raw(clouds, outs, streams, deg, False, antialiasing=aa, camera_grads=True)
    torch.cuda.synchronize()
    problems = []
    for b, gr in enumerate(grads):
        tup = tuple(gr[k] for k in ("dL_dmeans2D", "dL_dcolors", "dL_dfeature", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D",
                                    "dL_dsh", "dL_dscales", "dL_drotations"))
        cam = (gr["dL_dviewmatrix"], gr["dL_dprojmatrix"], gr["dL_dcampos"])
        problems += [f"cloud {b}: {p}" for p in _check(gs[b], camss[b], per[b], tup + (cam,), aa, True, shared=False)]
    assert not problems, "\n".join(problems)


def test_every_fisheye_project_bwd_instantiation_is_run():
    """The 12 FISHEYE instantiations (views / clouds x NSH x AA) are launched by configurations of the cases above."""
    names = set()
    for deg in (1, 2, 3):
        for aa in (False, True):
            g = TP._cloud_g(64, deg, 7)
            cams = [fcam(v, 2) for v in range(2)]

            def views():
                _run(g, cams, aa)

            def clouds():
                from manigaussian_b200 import rasterizer as R
                a = TP.g_args(g)
                cl = [dict(views=[fsettings(c, deg, aa) for c in cams], means3D=a["means3D"], sh=a["sh"], colors=a["colors"],
                           opacity=a["opacity"], scales=a["scales"], rotations=a["rotations"], cov3D_precomp=None,
                           grad_color=torch.ones((2, 3, 24, 32), device="cuda"))]
                outs, streams = R.rasterize_clouds_raw(cl, deg, False, antialiasing=aa)
                R.rasterize_clouds_backward_raw(cl, outs, streams, deg, False, antialiasing=aa)

            names |= TP._launched(views) | TP._launched(clouds)
    want = {(k, n, aa) for k in ("views", "clouds") for n in (12, 27, 48) for aa in (False, True)}
    seen = set()
    for n in names:
        for kind, nsh, aa in want:
            if f"project_bwd_{kind}_kernel<{nsh}, " in n and f", true, true, true, {'true' if aa else 'false'}>" in n:
                seen.add((kind, nsh, aa))
    assert seen == want, (sorted(want - seen), sorted(names))


# --------------------------------------------------------------------------- mixed batches, NULL and all-zero entries
def _render_raw(views, g, camera=False, seed=3, fisheye=None, ortho=None):
    from manigaussian_b200 import rasterizer as R
    deg = int(g["sh_degree"])
    a = TP.g_args(g)
    P = len(g["means3D"])
    outs, streams = R.rasterize_views_raw(views, a["means3D"], a["colors"], None, a["opacity"], a["scales"], a["rotations"], 1.0,
                                          None, a["sh"], deg, False, return_depth=True, capacities=TO._caps(views, P),
                                          fisheye=fisheye, ortho=ortho)
    torch.cuda.synchronize()
    assert not any(o.overflowed() for o in outs)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    gc = [torch.randn((3, s.image_height, s.image_width), generator=gen, device="cuda") for s in views]
    gd = [torch.randn((s.image_height, s.image_width), generator=gen, device="cuda") for s in views]
    grads = R.rasterize_views_backward_raw(views, outs, streams, gc, None, a["means3D"], a["colors"], None, a["scales"],
                                           a["rotations"], 1.0, None, a["sh"], deg, False, grads_depth=gd,
                                           camera_grads=True if camera else None, fisheye=fisheye, ortho=ortho)
    torch.cuda.synchronize()
    return outs, grads, gc, gd


def _keys(R, o):
    n, cap = o.num_rendered(), int(o[0])
    return TP._arr(R, "binning", "tile_ids", o[5], cap, 0, torch.int32, n)


def test_small_angle_fisheye_matches_the_pinhole_render_and_its_gradients():
    """End to end through a rendered loss: a k = 0 fisheye view of a distant cloud (theta below about 0.02) renders the image
    of the pinhole view of the same K whose principal point is moved by half a pixel (projection_from_intrinsics places the
    axis at cx - 0.5), and the gradients of the same loss of the two images agree to theta^2 and fp32 noise.  The fisheye
    backward takes the blend's mean cotangent in the pinhole path's convention (w.r.t. ndc), so a wrong scale of it shows
    here as a gap of W / 2 in dL/dmeans3D."""
    from manigaussian_b200 import cameras
    g = TP._cloud_g(2000, 1, 21)
    W, H, D = 32, 24, 40.0   # 2 x 2 tiles: the explicit binning capacities of _render_raw hold every instance
    direction = np.array([1.5, -1.0, 1.3]) / np.linalg.norm([1.5, -1.0, 1.3])
    c2w = TO._look(scenes.SCENE_CENTER + D * direction)
    f = 0.5 * W * D / 0.6
    cx, cy = (W - 1) / 2, (H - 1) / 2
    fc = F64.fisheye_cam(W, H, f, f, cx, cy, (0.0, 0.0, 0.0, 0.0), c2w)
    K = np.array([[f, 0.0, cx + 0.5], [0.0, f, cy + 0.5], [0.0, 0.0, 1.0]])
    proj = cameras.projection_from_intrinsics(0.1, 100.0, K, H, W)
    pc = {k: v for k, v in fc.items() if k != "fisheye"}
    pc["projmatrix"] = (np.linalg.inv(c2w).T @ proj.T).astype(np.float32)
    of, gf, _, _ = _render_raw([fsettings(fc, 1)], g, seed=5)
    op, gp, _, _ = _render_raw([TP.settings(pc, 1)], g, seed=5)
    assert int((of[0][3] > 0).sum()) > 1000 and int(((of[0][3] > 0) != (op[0][3] > 0)).sum()) <= 10
    assert util.rel_l2(of[0][1].cpu().numpy(), op[0][1].cpu().numpy()) < 2e-3
    for j, name in ((3, "dL_dopacity"), (4, "dL_dmeans3D"), (7, "dL_dscales"), (8, "dL_drotations")):
        err = util.rel_l2(gf[j].cpu().numpy(), gp[j].cpu().numpy())
        assert err < 1e-2, (name, err)


def test_mixed_batch_matches_each_view_alone():
    from manigaussian_b200 import rasterizer as R
    g = TP._cloud_g(3000, 1, 11)
    views = []
    for v in range(6):
        views.append(fsettings(fcam(v, 6, k=UMI_K), 1) if v % 3 == 0 else TO.osettings(TO.ocam(v, 6), 1) if v % 3 == 1
                     else TP.settings(TO._pcam(v, 6), 1))
    outs, grads, gc, gd = _render_raw(views, g, camera=True)
    total = {}
    for v, s in enumerate(views):
        a = TP.g_args(g)
        o1, st1 = R.rasterize_views_raw([s], a["means3D"], None, None, a["opacity"], a["scales"], a["rotations"], 1.0, None,
                                        a["sh"], 1, False, return_depth=True, capacities=TO._caps([s], 3000))
        torch.cuda.synchronize()
        assert not o1[0].overflowed()
        assert torch.equal(o1[0][1], outs[v][1]) and torch.equal(o1[0][3], outs[v][3]) and torch.equal(o1[0][7], outs[v][7])
        assert o1[0].num_rendered() == outs[v].num_rendered() and outs[v].num_rendered() > 1000
        np.testing.assert_array_equal(_keys(R, o1[0]), _keys(R, outs[v]))
        g1 = R.rasterize_views_backward_raw([s], o1, st1, [gc[v]], None, a["means3D"], None, None, a["scales"], a["rotations"], 1.0,
                                            None, a["sh"], 1, False, grads_depth=[gd[v]], camera_grads=True)
        torch.cuda.synchronize()
        for j in (0, 3, 4, 6, 7, 8):
            total[j] = total.get(j, 0) + g1[j].double()
        for j in range(3):
            assert util.rel_l2(grads[9][j][v].cpu().numpy(), g1[9][j][0].cpu().numpy()) < 1e-5, (v, j)
    for j, t in total.items():
        assert util.rel_l2(grads[j].cpu().numpy(), t.cpu().numpy()) < 1e-5, j


def test_mixed_views_of_one_cloud_in_render_clouds():
    from manigaussian_b200 import rasterizer as R
    g = TP._cloud_g(2000, 2, 12)
    a = TP.g_args(g)
    views = [TP.settings(TO._pcam(0, 2), 2), fsettings(fcam(1, 2), 2), TO.osettings(TO.ocam(0, 2), 2)]
    cl = [dict(views=views, means3D=a["means3D"], sh=a["sh"], colors=None, opacity=a["opacity"], scales=a["scales"],
               rotations=a["rotations"], cov3D_precomp=None, grad_color=torch.ones((3, 3, 24, 32), device="cuda"),
               capacities=TO._caps(views, 2000))]
    outs, streams = R.rasterize_clouds_raw(cl, 2, False)
    assert not any(o.overflowed() for o in outs[0])
    gr = R.rasterize_clouds_backward_raw(cl, outs, streams, 2, False)[0]
    o2, _, _, _ = _render_raw(views, g)
    for v in range(3):
        assert torch.equal(outs[0][v][1], o2[v][1]) and torch.equal(outs[0][v][3], o2[v][3])
    assert torch.isfinite(gr["dL_dmeans3D"]).all() and gr["dL_dmeans3D"].abs().max() > 0


def test_zero_entries_match_the_ortho_calls(monkeypatch):
    """All-zero fisheye entries give the results of a NULL fisheye array: the entries' other fields are ignored, and the launches run the ORTHO kernels."""
    from manigaussian_b200 import _binding as B
    from manigaussian_b200 import rasterizer as R
    g = TP._cloud_g(3000, 1, 13)
    views = [TP.settings(TO._pcam(0, 3), 1), TO.osettings(TO.ocam(1, 3), 1), TP.settings(TO._pcam(2, 3), 1)]
    o0, g0, _, _ = _render_raw(views, g)   # no fisheye array
    calls = []
    real = R._fisheye_array

    def zeros(vs, fisheye=None):
        assert real(vs, fisheye) is None
        calls.append(len(vs))
        arr = (B.ViewFisheye * len(vs))()
        for e in arr:   # fisheye = 0 with parameters that would be rejected: the entry is ignored
            e.cx, e.k1, e.theta_max = 1e3, 5.0, -1.0
        return arr
    monkeypatch.setattr(R, "_fisheye_array", zeros)
    o1, g1, _, _ = _render_raw(views, g)
    assert calls
    for a, b in zip(o0, o1):
        assert torch.equal(a[1], b[1]) and torch.equal(a[3], b[3]) and torch.equal(a[7], b[7])
        assert a.num_rendered() == b.num_rendered()
        np.testing.assert_array_equal(_keys(R, a), _keys(R, b))
    for j in (0, 3, 4, 7, 8):
        assert util.rel_l2(g1[j].cpu().numpy(), g0[j].cpu().numpy()) < 1e-5, j


# --------------------------------------------------------------------------- public paths
def _fcams(V, learn=False, W=64, H=48, k=UMI_K):
    from manigaussian_b200.cameras import build_fisheye_cameras, fisheye_camera_batch
    c2w = np.stack([TO._look(scenes.SCENE_CENTER + np.array([1.2 * np.cos(a), 1.2 * np.sin(a), 0.6])) for a in np.linspace(0, 3, V)])
    f, c = W / 3.2, ((W - 1) / 2, (H - 1) / 2)
    if not learn:
        K = np.array([[f, 0, c[0]], [0, f, c[1]], [0, 0, 1.0]])
        return build_fisheye_cameras(np.repeat(K[None], V, 0), np.array([k] * V), c2w, W, H, device="cuda")
    w2c = torch.tensor(np.linalg.inv(c2w), dtype=torch.float32, device="cuda").requires_grad_()
    foc = torch.tensor([[f, f]] * V, device="cuda").requires_grad_()
    return fisheye_camera_batch(w2c, foc, [c] * V, [k] * V, W, H), w2c, foc


OPTIONS = [dict(), dict(antialiasing=True), dict(return_alpha=True, return_depth=True), dict(return_median_depth=True),
           dict(return_normal=True), dict(targets="depth_mask"), dict(targets="ssim"), dict(camera=True), dict(learn=True),
           dict(learn=True, antialiasing=True, return_normal=True), dict(F=40), dict(sync_gradients=True)]


@pytest.mark.parametrize("opt", OPTIONS, ids=["-".join(o) or "plain" for o in OPTIONS])
def test_render_views_with_every_option(opt):
    from manigaussian_b200 import gaussian_renderer as GR
    opt = dict(opt)
    V, W, H = 4, 64, 48
    sc = TO._gauss(F=opt.pop("F", 0))
    w2c = foc = None
    if opt.pop("learn", False):
        cams, w2c, foc = _fcams(V, learn=True)
    elif opt.pop("camera", False):
        from manigaussian_b200.cameras import fisheye_camera_batch
        c2w = np.stack([TO._look(scenes.SCENE_CENTER + np.array([1.2 * np.cos(a), 1.2 * np.sin(a), 0.6])) for a in np.linspace(0, 3, V)])
        w2c = torch.tensor(np.linalg.inv(c2w), dtype=torch.float32, device="cuda").requires_grad_()
        cams = fisheye_camera_batch(w2c, [[20.0, 20.0]] * V, [[31.5, 23.5]] * V, [UMI_K] * V, W, H)
    else:
        cams = _fcams(V)
    t = opt.pop("targets", None)
    if t is not None:
        gen = torch.Generator(device="cuda").manual_seed(2)
        opt["targets"] = {"rgb": torch.rand((V, 3, H, W), generator=gen, device="cuda")}
        if t == "depth_mask":
            opt["targets"]["depth"] = 1.0 + torch.rand((V, H, W), generator=gen, device="cuda")
            opt["targets"]["mask"] = (torch.rand((V, H, W), generator=gen, device="cuda") > 0.5).float()
        else:
            opt["ssim"] = True
    for k in ("pts_xyz", "scales", "opacity", "features_color"):
        sc[k].requires_grad_()
    out = GR.render_views(cams, pts_xyz=sc["pts_xyz"], rotations=sc["rotations"], scales=sc["scales"], opacity=sc["opacity"],
                          features_color=sc["features_color"], features_language=sc.get("features_language"), **opt)
    loss = 0.0
    for k in ("render", "render_embed", "depth", "alpha", "median_depth", "normal"):
        if out.get(k) is not None and out[k].requires_grad:
            loss = loss + (out[k] * torch.linspace(-1, 1, out[k].numel(), device="cuda").reshape(out[k].shape)).sum()
    for k in ("loss_rgb", "loss_embed", "loss_depth", "loss_mask", "loss_l1", "ssim"):
        if k in out:
            loss = loss + out[k].sum()
    loss.backward()
    torch.cuda.synchronize()
    assert float(out["render"].abs().max()) > 0 and int((out["radii"] > 0).sum()) > 1000
    for k in ("pts_xyz", "scales", "opacity", "features_color"):
        assert torch.isfinite(sc[k].grad).all() and float(sc[k].grad.abs().max()) > 0, k
    for leaf in (w2c, foc):
        if leaf is not None:
            assert torch.isfinite(leaf.grad).all() and float(leaf.grad.abs().max()) > 0


def test_render_clouds_lift_and_rasterizer():
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.rasterizer import GaussianRasterizer
    V = 3
    sc = TO._gauss(seed=4)
    cams = _fcams(V)
    with pytest.raises(ValueError):
        cams.as_novel_view()
    common = dict(pts_xyz=sc["pts_xyz"], rotations=sc["rotations"], scales=sc["scales"], opacity=sc["opacity"],
                  features_color=sc["features_color"])
    ref = GR.render_views(cams, **common, return_depth=True)
    outs = GR.render_clouds([dict(cameras=cams, **common), dict(cameras=cams, **common)], return_depth=True)
    for o in outs:
        assert torch.equal(o["render"], ref["render"]) and torch.equal(o["depth"], ref["depth"])
    lf = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], ref["render"].detach())
    assert float(lf["weight"].sum()) > 0 and torch.isfinite(lf["lifted"]).all()
    w = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], None)["weight"]
    assert torch.allclose(w, lf["weight"], rtol=1e-4, atol=1e-6)
    vis = (ref["radii"] > 0).any(0)
    assert bool((w[~vis] == 0).all()) and float(w[vis].max()) > 0
    st = cams.settings(0, torch.zeros(3, device="cuda"), 1, False)
    m2 = torch.zeros_like(sc["pts_xyz"], requires_grad=True)
    out = GaussianRasterizer(st)(means3D=sc["pts_xyz"], means2D=m2, opacities=sc["opacity"], shs=sc["features_color"],
                                 scales=sc["scales"], rotations=sc["rotations"])
    assert torch.equal(out[0], ref["render"][0])
    xyz = sc["pts_xyz"].clone().requires_grad_()
    out2 = GaussianRasterizer(st)(means3D=xyz, means2D=m2, opacities=sc["opacity"], shs=sc["features_color"],
                                  cov3D_precomp=TO._cov6(sc["scales"], sc["rotations"] / sc["rotations"].norm(dim=1, keepdim=True)))
    assert torch.allclose(out2[0], out[0], atol=1e-4)
    out2[0].sum().backward()
    assert float(xyz.grad.abs().max()) > 0


def test_cuda_graph_replay_and_memory():
    from manigaussian_b200 import gaussian_renderer as GR
    V = 3
    sc = TO._gauss(seed=6)
    _, w2c, foc = _fcams(V, learn=True)
    xyz = sc["pts_xyz"].clone().requires_grad_()
    gen = torch.Generator(device="cuda").manual_seed(9)
    tgt = {"rgb": torch.rand((V, 3, 48, 64), generator=gen, device="cuda")}

    def step():
        from manigaussian_b200.cameras import fisheye_camera_batch
        c = fisheye_camera_batch(w2c, foc, [(31.5, 23.5)] * V, [UMI_K] * V, 64, 48)
        o = GR.render_views(c, pts_xyz=xyz, rotations=sc["rotations"], scales=sc["scales"], opacity=sc["opacity"],
                            features_color=sc["features_color"], targets=tgt)
        loss = o["loss_rgb"].sum()
        loss.backward()
        return loss.detach()

    def eager():
        xyz.grad = w2c.grad = foc.grad = None
        loss = step()
        torch.cuda.synchronize()
        return loss.clone(), xyz.grad.clone(), w2c.grad.clone(), foc.grad.clone()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            xyz.grad = w2c.grad = foc.grad = None
            step()
    torch.cuda.current_stream().wait_stream(s)
    eager()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    for _ in range(5):
        eager()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= m0 + (1 << 20)
    graph = torch.cuda.CUDAGraph()
    xyz.grad = w2c.grad = foc.grad = None
    with torch.cuda.graph(graph):
        g_loss = step()
    with torch.no_grad():
        foc.mul_(1.05)
    graph.replay()
    torch.cuda.synchronize()
    rep = (g_loss.clone(), xyz.grad.clone(), w2c.grad.clone(), foc.grad.clone())
    new = eager()
    for x, y in zip(rep, new):
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-5 * float(y.abs().max())), float((x - y).abs().max())
    assert float(new[3].abs().max()) > 0
