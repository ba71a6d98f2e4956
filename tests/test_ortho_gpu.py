"""Orthographic views on the GPU (include/mgs_rasterizer.h, "Orthographic views").

* Forward records: every record of project_fwd<AA, FOV, ORTHO = true> (means2D, conic, radius, depth, tiles, o_eff) against
  tests/ortho_ref64.py within KAPPA u e (project_ref64's KAPPA convention), with means near the extent edges, needles and
  AA across the 2.5e-5 clamp, host and device half extents.  Gaussians with a borderline decision are left out.
* Backward: the 12 ORTHO instantiations of project_bwd (views / clouds x AA x NSH in {12, 27, 48}), fed blend_ref64's
  cotangents of our own records (as test_project_ref64_gpu does): every per-Gaussian sum within its bound, the 35 camera
  outputs within KAPPA_ORTHO_CAM (below) and dL/dtan_fov within intrinsics_ref64.KAPPA_INTR, over 1 to 33 views (spanning
  launches), SH degrees 0-3, precomputed colours and covariances, and 20 clouds.  Each instantiation is launched.
* Images: the blend of the orthographic records against blend_ref64.
* Mixed batches: each view's image, radii and instance count are bit-identical to the view rendered alone, and the
  gradients are the sum over the views within float-atomic order.
* An all-zero ortho array: bit-identical images, radii, sort keys and counts to a NULL one, gradients within 1e-5 relative L2 (the float atomics' order).  The renders compared bit for bit take explicit
  binning capacities and are checked not to overflow.
* Public paths: render_views / render_clouds / lift_views / GaussianRasterizer with every option, a CUDA-graph replay, and
  no device memory growth over steps.
"""
import numpy as np
import pytest
import torch

import blend_ref64 as B64
import camera_ref64 as C64
import intrinsics_ref64 as I64
import ortho_ref64 as O64
import project_ref64 as P64
import test_project_ref64_cpu as CPU
import test_project_ref64_gpu as TP
import util
from manigaussian_b200 import scenes

pytestmark = pytest.mark.gpu

# camera outputs: within bound when |x - val| <= KAPPA_ORTHO_CAM (u e + d), camera_ref64's convention.  Over the cases below
# the orthographic dL/dviewmatrix reached 0.035 of u e + d on an H100 80GB HBM3 (700 W), above the 0.0016 camera_ref64
# measured for pinhole views (its KAPPA_CAM = 0.0064); the other camera outputs stayed within KAPPA_CAM.  The entries near
# their bound are the depth row, vm[2], vm[6], vm[10] and vm[14] (dL/dRv[2][c] and dL/dtv.z).  For an orthographic view
# they are sum_i dL/ddepth_i p_i alone: dt.z is the depth cotangent, with no chain through J(t).  Their deviation is the
# blend's own error in dL/ddepth carried through that sum: 2-3 % of its inherited bound d, and below u e.  Their e holds
# only the product and the summation tree.  For a pinhole view the same entries also carry dt.z's chain through
# J(t) (fx dJ00 / tz^2 and the rest), whose rounding bound widens u e + d while the kernel's deviation stays the inherited
# one; so the same deviation is a smaller share of the bound there.  KAPPA_ORTHO_CAM is about 4x the worst ratio, still
# far inside the first-order bound (ratio 1).
KAPPA_ORTHO_CAM = 0.15


@pytest.fixture(autouse=True, scope="module")
def _own_capacity_history():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _look(eye, target=scenes.SCENE_CENTER):
    fwd = np.asarray(target, np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    if np.linalg.norm(right) < 1e-6:
        right = np.array([1.0, 0.0, 0.0])
    right /= np.linalg.norm(right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, np.cross(fwd, right), fwd, eye
    return c2w


def ocam(v, n, W=32, H=24, half=(0.75, 0.6)):
    """orthographic camera v of n around the scene centre, 2.5 units out"""
    az = 2.0 * np.pi * v / max(n, 1) + 0.3
    eye = scenes.SCENE_CENTER + np.array([2.0 * np.cos(az), 2.0 * np.sin(az), 1.2 + 0.1 * v])
    return O64.ortho_cam(W, H, half[0], half[1], _look(eye))


def osettings(cam, deg, aa=False, device_fov=False):
    s = TP.settings(cam, deg, aa)._replace(orthographic=True)
    if device_fov:
        s = s._replace(tanfovx=torch.tensor(float(cam["tanfovx"]), device="cuda"),
                       tanfovy=torch.tensor(float(cam["tanfovy"]), device="cuda"))
    return s


# --------------------------------------------------------------------------- forward records
def _edge_scene(kind, cam, seed=0):
    """Gaussians placed in pixel space: across the extent edges, needles (AA on both sides of the clamp), random."""
    rng = np.random.default_rng(seed)
    W, H = cam["W"], cam["H"]
    n = 96
    px = np.concatenate([rng.uniform(-6, 2, n // 4), rng.uniform(W - 2, W + 6, n // 4), rng.uniform(0, W, n // 2)])
    py = np.concatenate([rng.uniform(0, H, n // 2), rng.uniform(-6, 2, n // 4), rng.uniform(H - 2, H + 6, n // 4)])
    z = rng.uniform(0.8, 3.0, n)
    vm = np.asarray(cam["viewmatrix"], np.float64).T      # world -> view rows
    fx, fy = W / (2 * cam["tanfovx"]), H / (2 * cam["tanfovy"])
    t = np.stack([(px + 0.5 - W / 2) / fx, (py + 0.5 - H / 2) / fy, z], 1)
    means = (t - vm[:3, 3]) @ np.linalg.inv(vm[:3, :3]).T
    deg = 1
    g = scenes.make_gaussians(n, sh_degree=deg, seed=seed)
    g["means3D"] = means.astype(np.float32)
    g["scales"] = np.exp(rng.normal(np.log(0.02), 0.6, (n, 3))).astype(np.float32)
    if kind == "needles":   # lines: det0 / det below the 2.5e-5 clamp for the even ones, above it for the odd ones
        thin = np.where(np.arange(n) % 2 == 0, 1e-5, 3e-3).astype(np.float32)
        g["scales"][:, 0], g["scales"][:, 1], g["scales"][:, 2] = 0.05, thin, thin
    g["cov3D_precomp"] = None
    return g


FWD = [("edges", False, False), ("edges", False, True), ("needles", True, False), ("needles", True, True),
       ("random", False, False)]


@pytest.mark.parametrize("kind,aa,dev", FWD, ids=[f"{k}-{'aa' if a else 'noaa'}-{'device' if d else 'host'}" for k, a, d in FWD])
def test_forward_records_against_float64(kind, aa, dev):
    from manigaussian_b200 import rasterizer as R
    cam = ocam(1, 3, W=48, H=40)
    g = _edge_scene(kind, cam) if kind != "random" else TP._cloud_g(300, 2, 5)
    deg = int(g["sh_degree"])
    a = TP.g_args(g)
    outs, _ = R.rasterize_views_raw([osettings(cam, deg, aa, dev)], a["means3D"], a["colors"], None, a["opacity"], a["scales"],
                                    a["rotations"], 1.0, a["cov3D_precomp"], a["sh"], deg, False, antialiasing=aa)
    torch.cuda.synchronize()
    P = len(g["means3D"])
    k = TP.records(R, outs[0][4], P)
    radii = outs[0][3].cpu().numpy()
    ref = O64.forward(g, cam, 1.0, antialias=aa)
    keep = ~ref["border"]
    assert keep.sum() > 0.7 * P and (~ref["culled"] & keep).sum() > 0.3 * P
    np.testing.assert_array_equal(radii[keep], ref["radius"][keep])
    np.testing.assert_array_equal(k["tiles_touched"][keep], ref["tiles_touched"][keep])
    vis = keep & ~ref["culled"]
    got = dict(means2D=k["means2D"], conic=k["conic_opacity"][:, :3], depth=k["depths"], opacity=k["conic_opacity"][:, 3],
               rgb=k["rgb"])
    for q, qk in (("means2D", "means2D"), ("conic", "conic"), ("depth", "depth"), ("opacity", "opacity"), ("rgb", "rgb")):
        r = P64.ratio(got[q][vis], (ref[q][vis], ref[q + "_B"][vis]), qk)
        print(f"{kind} aa={aa}: {q} worst {float(r.max()):.3g} of KAPPA")
        assert float(r.max()) <= 1.0, (q, float(r.max()))
    if kind == "needles" and aa:
        S = P64.cov3d(g)[0]
        G = O64._geometry(P64._cols(g["means3D"]), S, P64.view_of(cam))
        rr = ((G["a0"] * G["c0"] - G["b"] * G["b"]) / G["det"]).v[vis]
        assert (rr < P64.AA_CLAMP).any() and (rr > P64.AA_CLAMP).any()


# --------------------------------------------------------------------------- backward against float64
def _run(g, cams, aa, camera=False, dev=False, shared=True):
    from manigaussian_b200 import rasterizer as R
    deg = int(g["sh_degree"])
    views = [osettings(c, deg, aa, dev) for c in cams]
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
                                           camera_grads=True if camera else None,
                                           means2D_per_view=None if shared else torch.empty((len(cams), P, 3), device="cuda"))
    torch.cuda.synchronize()
    return outs, rc, grads


def _check(g, cams, rc, grads, aa, camera, shared=True):
    recs, cots = [r[0] for r in rc], [r[1] for r in rc]
    rb = O64.backward(g, cams, cots, 1.0, antialias=aa, live=[k["radii"] > 0 for k in recs],
                      clamped=[k["clamped"].astype(np.int64) for k in recs], shared_mean2D=shared)
    keep = ~rb["border"]
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
    rows = {}
    problems = CPU.compare_backward(rb, got, keep, rows, "ortho", names=tuple(got))
    v, e, d = rb["dL_dmeans2D"]
    x = (m2[None] if shared else m2)[..., :2]
    r = np.maximum(np.abs(x - v) - d, 0.0)[:, keep] / (P64.U * e[:, keep] + 1e-30)
    if r.size and r.max() > P64.KAPPA["dL_dmeans2D"]:
        problems.append(f"dL_dmeans2D worst {r.max():.3g}")
    if camera:
        cg = grads[9]
        for vi in range(len(cams)):
            for j, nm in enumerate(("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos")):
                rr = C64.ratio(cg[j][vi].cpu().numpy(), rb["camera"][vi][nm])
                if rr.max() > KAPPA_ORTHO_CAM:
                    problems.append(f"view {vi} {nm}: {rr.max():.3g} of the bound")
            if len(cg) > 3:
                rr = I64.ratio(cg[3][vi].cpu().numpy(), rb["tan_fov"][vi])
                if rr.max() > I64.KAPPA_INTR:
                    problems.append(f"view {vi} dL_dtan_fov: {rr.max():.3g} of the bound")
                assert np.abs(rb["tan_fov"][vi][0]).max() > 0
    return problems


VIEWS = [(1, 0, False, False, "sh"), (4, 1, True, True, "sh"), (17, 2, False, True, "sh"), (33, 3, True, True, "sh"),
         (4, 2, True, True, "sh"), (3, 3, False, True, "sh"), (2, 1, False, True, "rgb"), (2, 1, False, True, "cov")]


@pytest.mark.parametrize("V,deg,aa,camera,kind", VIEWS,
                         ids=[f"V{v}-deg{d}-{'aa' if a else 'noaa'}-{'cam' if c else 'nocam'}-{k}" for v, d, a, c, k in VIEWS])
def test_views_backward_against_float64(V, deg, aa, camera, kind):
    g = TP._cloud_g(160, deg, 40 + V + deg, precomp=(kind == "rgb"))
    if kind == "cov":
        S = P64.cov3d(g)[0]
        g["cov3D_precomp"] = np.stack([S[0][0].v, S[0][1].v, S[0][2].v, S[1][1].v, S[1][2].v, S[2][2].v], 1).astype(np.float32)
        g["scales"] = g["rotations"] = None
    cams = [ocam(v, V) for v in range(V)]
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
        cams = [ocam(v + b, n + b) for v in range(n)]
        a = TP.g_args(g)
        clouds.append(dict(views=[osettings(c, deg, aa) for c in cams], means3D=a["means3D"], sh=a["sh"], colors=a["colors"],
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


def test_every_ortho_project_bwd_instantiation_is_run():
    """The 12 ORTHO instantiations (views / clouds x NSH x AA) are launched by configurations of the cases above."""
    names = set()
    for deg in (1, 2, 3):
        for aa in (False, True):
            g = TP._cloud_g(64, deg, 7)
            cams = [ocam(v, 2) for v in range(2)]

            def views():
                _run(g, cams, aa)

            def clouds():
                from manigaussian_b200 import rasterizer as R
                a = TP.g_args(g)
                cl = [dict(views=[osettings(c, deg, aa) for c in cams], means3D=a["means3D"], sh=a["sh"], colors=a["colors"],
                           opacity=a["opacity"], scales=a["scales"], rotations=a["rotations"], cov3D_precomp=None,
                           grad_color=torch.ones((2, 3, 24, 32), device="cuda"))]
                outs, streams = R.rasterize_clouds_raw(cl, deg, False, antialiasing=aa)
                R.rasterize_clouds_backward_raw(cl, outs, streams, deg, False, antialiasing=aa)

            names |= TP._launched(views) | TP._launched(clouds)
    want = {(k, n, aa) for k in ("views", "clouds") for n in (12, 27, 48) for aa in (False, True)}
    seen = set()
    for n in names:
        for kind, nsh, aa in want:
            if f"project_bwd_{kind}_kernel<{nsh}, " in n and f", true, true, {'true' if aa else 'false'}>" in n:
                seen.add((kind, nsh, aa))
    assert seen == want, (sorted(want - seen), sorted(names))


# --------------------------------------------------------------------------- images
def test_blend_of_orthographic_records_against_float64():
    from manigaussian_b200 import rasterizer as R
    cam = ocam(0, 1, W=48, H=40)
    g = TP._cloud_g(400, 1, 77)
    a = TP.g_args(g)
    outs, _ = R.rasterize_views_raw([osettings(cam, 1)], a["means3D"], a["colors"], None, a["opacity"], a["scales"], a["rotations"],
                                    1.0, None, a["sh"], 1, False, return_depth=True)
    torch.cuda.synchronize()
    o = outs[0]
    P, W, H = 400, 48, 40
    T = ((W + 15) // 16) * ((H + 15) // 16)
    cap, Rn = int(o[0]), o.num_rendered()
    S = (cap + 11) & ~3
    k = TP.records(R, o[4], P)
    st = dict(W=W, H=H, ranges=TP._arr(R, "image", "ranges", o[6], W, H, torch.int32, 2 * T).view(np.uint32).reshape(T, 2),
              point_list=TP._arr(R, "binning", "point_list", o[5], cap, 0, torch.int32, Rn).view(np.uint32),
              means2D=k["means2D"], conic_opacity=k["conic_opacity"], colors=k["rgbd"][:, :3], depth=k["rgbd"][:, 3],
              feature=None, bg=np.zeros(3, np.float32), g_color=np.zeros((3, H, W), np.float32), g_feature=None,
              g_depth=np.zeros((H, W), np.float32), g_alpha=None)
    bl = TP._arr(R, "binning", "block_lists", o[5], cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    pmk = TP._arr(R, "binning", "pixel_masks", o[5], cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    nw = TP._arr(R, "image", "block_nwalk", o[6], W, H, torch.int32, 8 * T).view(np.uint32).reshape(T, 8)
    ref = B64.blend(st, B64.masks_from_blocks(st, bl, pmk, nw))
    color = o[1].cpu().numpy()
    assert Rn > 1000 and np.abs(ref["color"]).max() > 0.1
    bound = B64.KAPPA["color"] * B64.U * ref["color_B"] if "color" in B64.KAPPA else 4 * B64.U * ref["color_B"]
    assert np.all(np.abs(color - ref["color"]) <= bound + 1e-30), float((np.abs(color - ref["color"]) - bound).max())
    depth = o[7].cpu().numpy()
    bd = B64.KAPPA["depth"] * B64.U * ref["depth_B"] if "depth" in B64.KAPPA else 4 * B64.U * ref["depth_B"]
    assert np.all(np.abs(depth - ref["depth"]) <= bd + 1e-30)


# --------------------------------------------------------------------------- mixed batches and all-zero flags
def _pcam(v, n, W=32, H=24):
    return scenes.make_camera(W, H, v, n)


# The renders compared bit for bit below take explicit binning capacities: the capacity history is keyed by (cloud size,
# image size, view slot), which views of other scenes and models share, and a render that overflows its capacity drops
# instances.  A 32x24 image has 2x2 tiles, so no Gaussian emits more than 4 instances.
def _caps(views, P):
    return [4 * P + 4096] * len(views)


def _render_raw(views, g, ortho=None, camera=False, seed=3):
    from manigaussian_b200 import rasterizer as R
    deg = int(g["sh_degree"])
    a = TP.g_args(g)
    P = len(g["means3D"])
    outs, streams = R.rasterize_views_raw(views, a["means3D"], a["colors"], None, a["opacity"], a["scales"], a["rotations"], 1.0,
                                          None, a["sh"], deg, False, return_depth=True, ortho=ortho, capacities=_caps(views, P))
    torch.cuda.synchronize()
    assert not any(o.overflowed() for o in outs)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    gc = [torch.randn((3, s.image_height, s.image_width), generator=gen, device="cuda") for s in views]
    gd = [torch.randn((s.image_height, s.image_width), generator=gen, device="cuda") for s in views]
    grads = R.rasterize_views_backward_raw(views, outs, streams, gc, None, a["means3D"], a["colors"], None, a["scales"],
                                           a["rotations"], 1.0, None, a["sh"], deg, False, grads_depth=gd, ortho=ortho,
                                           camera_grads=True if camera else None)
    torch.cuda.synchronize()
    return outs, grads, gc, gd


def test_mixed_batch_matches_each_view_alone():
    from manigaussian_b200 import rasterizer as R
    g = TP._cloud_g(3000, 1, 11)
    views = []
    for v in range(6):
        views.append(osettings(ocam(v, 6), 1) if v % 2 else TP.settings(_pcam(v, 6), 1))
    outs, grads, gc, gd = _render_raw(views, g, camera=True)
    total = {}
    for v, s in enumerate(views):
        a = TP.g_args(g)
        o1, st1 = R.rasterize_views_raw([s], a["means3D"], None, None, a["opacity"], a["scales"], a["rotations"], 1.0, None,
                                        a["sh"], 1, False, return_depth=True, capacities=_caps([s], 3000))
        torch.cuda.synchronize()
        assert not o1[0].overflowed()
        assert torch.equal(o1[0][1], outs[v][1]) and torch.equal(o1[0][3], outs[v][3]) and torch.equal(o1[0][7], outs[v][7])
        assert o1[0].num_rendered() == outs[v].num_rendered() and outs[v].num_rendered() > 1000
        g1 = R.rasterize_views_backward_raw([s], o1, st1, [gc[v]], None, a["means3D"], None, None, a["scales"], a["rotations"], 1.0,
                                            None, a["sh"], 1, False, grads_depth=[gd[v]], camera_grads=True)
        torch.cuda.synchronize()
        for j in (0, 3, 4, 6, 7, 8):
            total[j] = total.get(j, 0) + g1[j].double()
        for j in range(3):   # this view's camera gradients: those of the view alone
            assert util.rel_l2(grads[9][j][v].cpu().numpy(), g1[9][j][0].cpu().numpy()) < 1e-5, (v, j)
    for j, t in total.items():
        assert util.rel_l2(grads[j].cpu().numpy(), t.cpu().numpy()) < 1e-5, j


def test_mixed_views_of_one_cloud_in_render_clouds():
    from manigaussian_b200 import rasterizer as R
    g = TP._cloud_g(2000, 2, 12)
    a = TP.g_args(g)
    views = [TP.settings(_pcam(0, 2), 2), osettings(ocam(1, 2), 2), osettings(ocam(0, 2), 2)]
    cl = [dict(views=views, means3D=a["means3D"], sh=a["sh"], colors=None, opacity=a["opacity"], scales=a["scales"],
               rotations=a["rotations"], cov3D_precomp=None, grad_color=torch.ones((3, 3, 24, 32), device="cuda"),
               capacities=_caps(views, 2000))]
    outs, streams = R.rasterize_clouds_raw(cl, 2, False)
    assert not any(o.overflowed() for o in outs[0])
    gr = R.rasterize_clouds_backward_raw(cl, outs, streams, 2, False)[0]
    o2, g2, _, _ = _render_raw(views, g)
    for v in range(3):
        assert torch.equal(outs[0][v][1], o2[v][1]) and torch.equal(outs[0][v][3], o2[v][3])
    assert torch.isfinite(gr["dL_dmeans3D"]).all() and gr["dL_dmeans3D"].abs().max() > 0


def test_all_zero_flags_match_the_calls_without_them(monkeypatch):
    import ctypes
    from manigaussian_b200 import rasterizer as R
    g = TP._cloud_g(3000, 1, 13)
    views = [TP.settings(_pcam(v, 3), 1) for v in range(3)]
    o0, g0, _, _ = _render_raw(views, g)
    calls = []
    real = R._ortho_flags

    def zeros(vs, ortho=None):
        assert real(vs, ortho) is None
        calls.append(len(vs))
        return (ctypes.c_int * len(vs))(*([0] * len(vs)))
    monkeypatch.setattr(R, "_ortho_flags", zeros)
    o1, g1, _, _ = _render_raw(views, g)
    assert calls   # the all-zero flag arrays reached the calls
    for a, b in zip(o0, o1):
        assert torch.equal(a[1], b[1]) and torch.equal(a[3], b[3]) and torch.equal(a[7], b[7])
        assert a.num_rendered() == b.num_rendered()
        n, cap = a.num_rendered(), int(a[0])
        ka = TP._arr(R, "binning", "tile_ids", a[5], cap, 0, torch.int32, n)
        kb = TP._arr(R, "binning", "tile_ids", b[5], int(b[0]), 0, torch.int32, n)
        np.testing.assert_array_equal(ka, kb)
    # the same kernels: the gradients differ only by the float atomics' order in the blend backward
    for j in (0, 3, 4, 7, 8):
        assert util.rel_l2(g1[j].cpu().numpy(), g0[j].cpu().numpy()) < 1e-5, j


# --------------------------------------------------------------------------- public paths
def _gauss(P=3000, F=0, seed=0):
    from test_camera_grad_gpu import _scene
    sc = _scene(P, F=F, sh=True, seed=seed)
    sc["pts_xyz"] = sc["pts_xyz"] + torch.tensor(scenes.SCENE_CENTER, device="cuda")
    return sc


def _ocams(V, learn=False, W=64, H=48):
    from manigaussian_b200.cameras import build_ortho_cameras, ortho_camera_batch
    c2w = np.stack([_look(scenes.SCENE_CENTER + np.array([2.0 * np.cos(a), 2.0 * np.sin(a), 1.5])) for a in np.linspace(0, 3, V)])
    if not learn:
        return build_ortho_cameras(c2w, (0.8, 0.6), W, H, device="cuda")
    w2c = torch.tensor(np.linalg.inv(c2w), dtype=torch.float32, device="cuda").requires_grad_()
    h = torch.tensor([[0.8, 0.6]] * V, device="cuda").requires_grad_()
    return ortho_camera_batch(w2c, h, W, H), w2c, h


OPTIONS = [dict(), dict(antialiasing=True), dict(return_alpha=True, return_depth=True), dict(return_median_depth=True),
           dict(return_normal=True), dict(targets="depth_mask"), dict(targets="ssim"), dict(camera=True), dict(learn=True),
           dict(learn=True, antialiasing=True, return_normal=True), dict(F=40), dict(sync_gradients=True)]


@pytest.mark.parametrize("opt", OPTIONS, ids=["-".join(o) or "plain" for o in OPTIONS])
def test_render_views_with_every_option(opt):
    from manigaussian_b200 import gaussian_renderer as GR
    opt = dict(opt)
    V, W, H = 4, 64, 48
    sc = _gauss(F=opt.pop("F", 0))
    w2c = h = None
    if opt.pop("learn", False):
        cams, w2c, h = _ocams(V, learn=True)
    elif opt.pop("camera", False):
        from manigaussian_b200.cameras import ortho_camera_batch
        c2w = np.stack([_look(scenes.SCENE_CENTER + np.array([2.0 * np.cos(a), 2.0 * np.sin(a), 1.5])) for a in np.linspace(0, 3, V)])
        w2c = torch.tensor(np.linalg.inv(c2w), dtype=torch.float32, device="cuda").requires_grad_()
        cams = ortho_camera_batch(w2c, 0.7, W, H)
    else:
        cams = _ocams(V)
    t = opt.pop("targets", None)
    if t is not None:
        gen = torch.Generator(device="cuda").manual_seed(2)
        opt["targets"] = {"rgb": torch.rand((V, 3, H, W), generator=gen, device="cuda")}
        if t == "depth_mask":
            opt["targets"]["depth"] = 2.0 + torch.rand((V, H, W), generator=gen, device="cuda")
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
    for leaf in (w2c, h):
        if leaf is not None:
            assert torch.isfinite(leaf.grad).all() and float(leaf.grad.abs().max()) > 0


def test_render_clouds_lift_and_rasterizer():
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.rasterizer import GaussianRasterizer
    V = 3
    sc = _gauss(seed=4)
    cams = _ocams(V)
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
    # the visible Gaussians of the orthographic renders are the lifted ones
    vis = (ref["radii"] > 0).any(0)
    assert bool((w[~vis] == 0).all()) and float(w[vis].max()) > 0
    # GaussianRasterizer takes the orthographic settings down the multi-view path, with cov3D_precomp too
    st = cams.settings(0, torch.zeros(3, device="cuda"), 1, False)
    m2 = torch.zeros_like(sc["pts_xyz"], requires_grad=True)
    out = GaussianRasterizer(st)(means3D=sc["pts_xyz"], means2D=m2, opacities=sc["opacity"], shs=sc["features_color"],
                                 scales=sc["scales"], rotations=sc["rotations"])
    assert torch.equal(out[0], ref["render"][0])
    q = sc["rotations"] / sc["rotations"].norm(dim=1, keepdim=True)
    cov = _cov6(sc["scales"], q)
    xyz = sc["pts_xyz"].clone().requires_grad_()
    out2 = GaussianRasterizer(st)(means3D=xyz, means2D=m2, opacities=sc["opacity"], shs=sc["features_color"], cov3D_precomp=cov)
    assert torch.allclose(out2[0], out[0], atol=1e-4)
    out2[0].sum().backward()
    assert float(xyz.grad.abs().max()) > 0


def _cov6(s, q):
    r, x, y, z = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z), 1 - 2 * (x * x + z * z),
                     2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    S = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).contiguous()


def test_top_down_heightmap():
    """A flat layer of Gaussians at height z renders a top-down depth of (camera height - z) where it covers the image."""
    from manigaussian_b200 import gaussian_renderer as GR
    from manigaussian_b200.cameras import top_down_camera
    b = scenes.SCENE_BOUNDS.astype(np.float64)
    cam = top_down_camera(b, 64, 64, device="cuda")
    n = 60
    gx, gy = np.meshgrid(np.linspace(b[0], b[3], n), np.linspace(b[1], b[4], n))
    z = 1.1
    xyz = torch.tensor(np.stack([gx.ravel(), gy.ravel(), np.full(n * n, z)], 1), dtype=torch.float32, device="cuda")
    P = n * n
    rot = torch.tensor([[1.0, 0, 0, 0]], device="cuda").repeat(P, 1)
    sc = torch.full((P, 3), 0.02, device="cuda")
    op = torch.full((P, 1), 0.99, device="cuda")
    out = GR.render_views(cam, xyz, rot, sc, op, pts_rgb=torch.rand((P, 3), device="cuda"), return_depth=True, return_alpha=True)
    depth, alpha = out["depth"][0], out["alpha"][0]
    inner = alpha[8:-8, 8:-8] > 0.99
    assert bool(inner.all())
    height = (b[5] + 0.5) - (depth[8:-8, 8:-8] / alpha[8:-8, 8:-8])
    assert torch.allclose(height, torch.full_like(height, z), atol=1e-3)


def test_cuda_graph_replay_and_memory():
    from manigaussian_b200 import gaussian_renderer as GR
    V = 3
    sc = _gauss(seed=6)
    # only the leaves: a batch built here would keep their AccumulateGrad nodes alive on the default stream, which the
    # capture on a side stream must not depend on
    _, w2c, h = _ocams(V, learn=True)
    xyz = sc["pts_xyz"].clone().requires_grad_()
    gen = torch.Generator(device="cuda").manual_seed(9)
    tgt = {"rgb": torch.rand((V, 3, 48, 64), generator=gen, device="cuda")}

    def step():
        from manigaussian_b200.cameras import ortho_camera_batch
        c = ortho_camera_batch(w2c, h, 64, 48)
        o = GR.render_views(c, pts_xyz=xyz, rotations=sc["rotations"], scales=sc["scales"], opacity=sc["opacity"],
                            features_color=sc["features_color"], targets=tgt)
        loss = o["loss_rgb"].sum()
        loss.backward()
        return loss.detach()

    def eager():
        xyz.grad = w2c.grad = h.grad = None
        loss = step()
        torch.cuda.synchronize()
        return loss.clone(), xyz.grad.clone(), w2c.grad.clone(), h.grad.clone()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            xyz.grad = w2c.grad = h.grad = None
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
    xyz.grad = w2c.grad = h.grad = None
    with torch.cuda.graph(graph):
        g_loss = step()
    with torch.no_grad():
        h.mul_(1.1)
    graph.replay()
    torch.cuda.synchronize()
    rep = (g_loss.clone(), xyz.grad.clone(), w2c.grad.clone(), h.grad.clone())
    new = eager()
    for x, y in zip(rep, new):
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-5 * float(y.abs().max())), float((x - y).abs().max())
    assert float(new[3].abs().max()) > 0
