"""Point visibility on the GPU element by element against the bounded float64 reference (visibility_ref64.bounded): every
in-view point's T, every point's dL/duv through T (the backward scratch's duv) and every Gaussian's blend-stage row (its
gb), within KAPPA u B + D, through visibility_views_raw / visibility_views_backward_raw(return_scratch=True) with each
view's projected and sorted state read from the call itself.  The tile and the depth cut are replayed in fp32 from the
kernel's own uv and depth, so no point is excluded: each scene asserts that every in-view point is checked.  Pairs whose
alpha, power or running product lies in its rounding band are kept, with their either-side share in D; the run prints how
many pairs carried one.

* Every camera model, AA on and off, one call mixing the four models with a device field of view, and V = 17 (two launches
  of each backward chain).
* Tiles holding exactly 1, 31, 32, 33, 64, 65 and 15,360 points (hot rows: about 480 warp items reduce into each of the
  hot tile's Gaussians), asserted from the kernel's own uv.  In the longest other tile list every pixel sits on its ray at
  a depth midway between two list entries, so the cuts 0, 1, 7, 8, 9, 31, 32, 33, 64, 65 and 200 are placed and asserted,
  and each warp item mixes lanes of cut 0 and 200.  g_T = 0 on every third point, beside live lanes with g_T != 0.
* Points within 1e-5 px of the tile seams, of u = -0.5 and of W - 0.5; points at Gaussian centres, whose depth ties the
  Gaussian's fp32 depth; runs of ten Gaussians with one mean and so one fp32 depth.
* Opaque clouds whose stacks reach T_STOP in the second chunk, mid k-step and on a chunk's last record (asserted), with
  Gaussians under the 0.99 clamp, and opacities at 1/255 and a few ulps above.
* Every requested-gradient subset (points only, cloud only, camera only, all); grad_T, grad_uv and grad_depth each absent
  and each zero (grad_uv and grad_depth feed only the point chain: duv and gb must not move).
* The c3-size 100^3 voxel grid x 4 views, T and duv on a seeded subsample, g_T zero elsewhere so that gb sums exactly the
  sampled points and is checked whole.

Not checked here, per element: uv and depth (test_visibility_gpu.py checks them against visibility_ref64.project to 1e-3
px) and the final gradients after the per-Gaussian and point chains (test_visibility_grad_gpu.py checks them by relative
L2 against visibility_grad_ref64's autograd).  Those chains are shared with the render's backward and the flow plane;
chaining their bounded references from the kernel's gb and duv is left to a later change.

Measured worst (|x - v| - D) / (u B) per quantity over every case, on an NVIDIA H100 80GB HBM3 at a 700 W power limit
(printed at the end of a `-s` run); visibility_ref64.KAPPA is 4x these:

    T 0.301   duv 0.309   gb 0.403

About 25 of 5e7 walked pairs were either-side.  The file runs in about 80 s on that GPU, 43 s of it the c3 voxel case.
"""
import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
import visibility_ref64 as V64
from test_planar_depth_gpu import MODELS, _inputs, _model_kw, _settings, _t
from test_visibility_gpu import _pixel_rays, _points

pytestmark = pytest.mark.gpu
QUANTITIES = ("T", "duv", "gb")
WORST = {}
EITHER = [0, 0]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nvisibility_ref64 worst (|x - v| - D) / (u B): " + ", ".join(f"{q}={WORST.get(q, 0.0):.4g}" for q in QUANTITIES) +
          f"; {EITHER[0]} of {EITHER[1]} pairs either-side")


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _view_state(state, v, W, H):
    """the view's projected and sorted state as the visibility call left it"""
    from manigaussian_b200 import rasterizer as R
    P = state["P"]
    geom, img, binb = state["keep"][1 + 7 * v: 4 + 7 * v]
    cap = int(state["arr"][v].binning_capacity)
    nt = ((W + 15) // 16) * ((H + 15) // 16)

    def arr(which, name, buf, a0, a1, dtype, count):
        off = R.state_array(which, name, buf, a0, a1) - buf.data_ptr()
        n = count * torch.empty((), dtype=dtype).element_size()
        return buf[off:off + n].view(dtype).cpu().numpy()

    ranges = arr("image", "ranges", img, W, H, torch.int32, 2 * nt).view(np.uint32).reshape(nt, 2)
    return dict(W=W, H=H, ranges=ranges,
                means2D=arr("geometry", "means2D", geom, P, 0, torch.float32, 2 * P).reshape(P, 2),
                conic_opacity=arr("geometry", "conic_opacity", geom, P, 0, torch.float32, 4 * P).reshape(P, 4),
                depths=arr("geometry", "depths", geom, P, 0, torch.float32, P),
                point_list=arr("binning", "point_list", binb, cap, 0, torch.int32, int(ranges[:, 1].max())).view(np.uint32))


def _scratch(scratch, v, P, Q, name, n):
    from manigaussian_b200 import rasterizer as R
    buf = scratch[v]
    off = R.state_array("visibility_backward", name, buf, P, Q) - buf.data_ptr()
    return buf[off:off + 4 * n].view(torch.float32).cpu().numpy().astype(np.float64)


def _within(name, got, ref, sel=None):
    v, B, D = ref
    if sel is not None:
        got, v, B, D = got[sel], v[sel], B[sel], D[sel]
    raw = V64.ratio(got, (v, B, D))
    WORST[name] = max(WORST.get(name, 0.0), float(raw.max()) if raw.size else 0.0)
    r = V64.ratio(got, (v, B, D), name)
    worst = float(r.max()) if r.size else 0.0
    assert worst <= 1.0, (name, worst, np.unravel_index(int(r.argmax()), r.shape) if r.size else None)


def _cot(V, Q, seed, every=3):
    rng = np.random.default_rng(seed)
    gT = rng.standard_normal((V, Q)).astype(np.float32)
    gT[:, ::every] = 0.0
    return gT


def _check(views, g, pts, gT="random", aa=False, tan_fov=None, want_points=True, want_cloud=True, camera=True, sel=None,
           seed=0, tag="", guv="random", gd="random"):
    """forward and backward against the reference, view by view; returns the checked in-view count and each view's
    reference.  grad_uv and grad_depth ("random", "zero" or None) feed only the point chain: duv and gb must not move."""
    from manigaussian_b200 import rasterizer as R
    m, o, s, r = (_t(g[k]) for k in ("means3D", "opacities", "scales", "rotations"))
    p = pts if torch.is_tensor(pts) else _t(pts)
    uv, d, inv, T, state = R.visibility_views_raw(views, m, o, s, r, 1.0, None, p, antialiasing=aa, tan_fov=tan_fov,
                                                  keep_state=True)
    V, Q, P = len(views), p.shape[0], m.shape[0]
    if isinstance(gT, str):
        gT = _cot(V, Q, seed)
        if sel is not None:
            keep = np.zeros(Q, bool)
            keep[sel] = True
            gT = gT * keep
    rng = np.random.default_rng(seed + 1)
    cot = {"random": lambda *sh: _t(rng.standard_normal(sh)), "zero": lambda *sh: _t(np.zeros(sh)), None: lambda *sh: None}
    out = R.visibility_views_backward_raw(state, p, m, o, s, r, 1.0, None, T, None if gT is None else _t(gT), cot[guv](V, Q, 2),
                                          cot[gd](V, Q),
                                          want_points=want_points, want_cloud=want_cloud, camera_grads=camera,
                                          return_scratch=True)
    torch.cuda.synchronize()
    scratch = out[-1]
    uv, d, inv, T = (x.cpu().numpy() for x in (uv, d, inv, T))
    chain = want_points or camera
    gauss = bool(np.any(want_cloud)) or camera
    checked, refs = 0, []
    for v, view in enumerate(views):
        W, H = int(view.image_width), int(view.image_height)
        st = _view_state(state, v, W, H)
        iv = inv[v].astype(bool)
        ref = V64.bounded(st, uv[v], d[v], iv, None if gT is None else gT[v], T_out=T[v], sel=sel)
        refs.append(ref)
        EITHER[0] += ref["either"]
        EITHER[1] += ref["pairs"]
        ev = np.zeros(Q, bool)
        ev[np.nonzero(iv)[0] if sel is None else np.asarray(sel)[iv[sel]]] = True
        assert ref["checked"] == int(ev.sum()), tag
        checked += ref["checked"]
        assert (T[v][~iv] == 1.0).all(), tag
        _within("T", T[v], ref["T"], ev)
        if gT is None:
            if gauss:
                assert (_scratch(scratch, v, P, Q, "gb", 12 * P) == 0).all(), tag
            continue
        if chain:
            duv = _scratch(scratch, v, P, Q, "duv", 2 * Q).reshape(Q, 2)
            _within("duv", duv, ref["duv"])
        if gauss:
            gb = _scratch(scratch, v, P, Q, "gb", 12 * P).reshape(P, 12)
            _within("gb", gb[:, :6], ref["gb"])
            assert (gb[:, 6:] == 0).all(), tag
    print(f"[{tag}] {checked} in-view points checked")
    return checked, refs


# ---------------------------------------------------------------------------------------------------- camera models
@pytest.mark.parametrize("model,aa", [(m, False) for m in MODELS] + [("pinhole", True), ("fisheye", True)])
def test_every_camera_model_within_bound(model, aa):
    inps, g = _inputs(4000, 96, 64, 0, 1)
    n, _ = _check([_settings(inps[0], 0, model, aa)], g, _points(g, 3001), aa=aa, tag=(model, aa))
    assert n > 1000


def test_one_call_mixing_all_four_models_with_a_device_fov():
    inps, g = _inputs(3000, 80, 72, 0, 4)
    views = [_settings(inps[v], 0, m) for v, m in enumerate(MODELS)]
    tf = torch.tensor([[float(s.tanfovx), float(s.tanfovy)] for s in views], device="cuda")
    _check(views, g, _points(g, 1500, seed=1), tan_fov=tf, tag="mixed+fov")


def test_seventeen_views_take_two_launches_of_each_chain():
    inps, g = _inputs(2000, 64, 48, 0, 17)
    views = [_settings(inps[v], 0, MODELS[v % 4]) for v in range(17)]
    _check(views, g, _points(g, 700, seed=2), tag="V=17")


# ---------------------------------------------------------------------------------------------------- items, cuts, stops
COUNTS = [1, 31, 32, 33, 64, 65, 15360]     # points in tiles 0 .. 6
CUTS = [0, 1, 7, 8, 9, 31, 32, 33, 64, 65, 200]


def _rays(view, target, z):
    """float64 world points at view-space depth z [n] whose float64 projection is target [n,2] (Newton on the reference,
    as _pixel_rays)"""
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).T
    c2w = np.linalg.inv(vm)
    W, H = view["W"], view["H"]
    fx, fy = W / (2 * view["tanfovx"]), H / (2 * view["tanfovy"])
    t = np.stack([(target[:, 0] - (W - 1) / 2) / fx * z, (target[:, 1] - (H - 1) / 2) / fy * z, z], 1)
    world = lambda tt: tt @ c2w[:3, :3].T + c2w[:3, 3]  # noqa: E731
    for _ in range(8):
        uv, _, _ = V64.project(world(t), view)
        J = np.empty((len(t), 2, 2))
        for k in range(2):
            dt = t.copy()
            dt[:, k] += 1e-6 * z
            J[:, :, k] = (V64.project(world(dt), view)[0] - uv) / (1e-6 * z)[:, None]
        t[:, :2] += np.linalg.solve(J, (target - uv)[:, :, None])[:, :, 0]
    return world(t)


def _tile_pixels(t, W, H):
    gx = (W + 15) // 16
    x0, y0 = 16 * (t % gx), 16 * (t // gx)
    yy, xx = np.meshgrid(np.arange(y0, min(y0 + 16, H)), np.arange(x0, min(x0 + 16, W)), indexing="ij")
    return np.stack([xx.ravel(), yy.ravel()], 1).astype(np.float64)


def _edge_scene(opaque):
    """A 96 x 64 pinhole view and points built for the query's edges: COUNTS points in tiles 0 .. 6 at depths through the
    scene (tile 6 is hot); in the longest other tile list, every pixel on its ray at a depth between two list entries
    that gives cut CUTS[k % 11] (so each warp item mixes cuts 0 and 200); points within 1e-5 px of the tile seams, of -0.5
    and of W - 0.5; and points at Gaussian centres (depth ties) outside those tiles.  Five runs of ten Gaussians share a
    mean, so their fp32 depths are equal.  `opaque`: opacities in [0.9, 1] (stacks reach T_STOP, 200 under the 0.99 clamp)
    and six at 1/255 and a few ulps above."""
    from manigaussian_b200 import rasterizer as R
    W, H = 96, 64
    inps, g = _inputs(4000, W, H, 0, 1, seed=9)
    g = dict(g)
    rng = np.random.default_rng(11)
    m = np.array(g["means3D"], np.float32)
    for j in range(5):
        m[300 + 10 * j: 310 + 10 * j] = m[300 + 10 * j]
    g["means3D"] = m
    if opaque:
        o = rng.uniform(0.9, 1.0, (4000, 1)).astype(np.float32)
        o[:200] = 1.0
        a255 = np.float32(1) / np.float32(255)
        o[200:206, 0] = [a255, np.nextafter(a255, np.float32(1)), a255 * np.float32(1.0000003), a255, 0.995, 0.9999]
        g["opacities"] = o
    view = _model_kw(inps[0], "pinhole")[1]
    settings = [_settings(inps[0], 0)]
    *_, state = R.visibility_views_raw(settings, *(_t(g[k]) for k in ("means3D", "opacities", "scales", "rotations")), 1.0,
                                       None, _t(np.zeros((1, 3))), keep_state=True)
    st = _view_state(state, 0, W, H)
    pts = []
    zs = np.linspace(0.5, 12.0, 60)
    for t, n in enumerate(COUNTS):
        px = _tile_pixels(t, W, H)
        k = np.arange(n)
        z = zs[k // len(px) % len(zs)] if n > len(px) else rng.choice(zs, n)
        pts.append(_rays(view, px[k % len(px)], z))
    # the cut tile: every cut of CUTS, a depth midway between list entries c - 1 and c
    lens = (st["ranges"][:, 1].astype(np.int64) - st["ranges"][:, 0])
    ct = 7 + int(np.argmax(lens[7:]))
    r0, r1 = (int(x) for x in st["ranges"][ct])
    dl = st["depths"][st["point_list"][r0:r1]].astype(np.float64)
    assert r1 - r0 > 200 and np.isfinite(dl).all()
    want = []
    for c in CUTS:
        while 0 < c < len(dl) and dl[c] - dl[c - 1] < 2e-5 * dl[c]:
            c += 1                                            # a depth tie: the next gap
        want.append(c)
    zc = np.array([dl[0] * (1 - 1e-3) if c == 0 else 0.5 * (dl[c - 1] + dl[c]) for c in want])
    px = _tile_pixels(ct, W, H)
    k = np.arange(len(px))
    pts.append(_rays(view, px, zc[k % len(want)]))
    # the seams: u + 0.5 at a multiple of 16 (rows 2 and 3), v + 0.5 at 32 and 48 (columns 1 .. 5), and the image edges
    n = 40
    off = np.array([0.0, 1e-5, -1e-5, 3e-6, -3e-6])
    us = np.array([15.5, 31.5, 47.5, 63.5, 79.5, -0.5 + 1e-5, W - 0.5 - 1e-5])
    tu = np.stack([rng.choice(us, n) + rng.choice(off, n), rng.uniform(32, H - 1, n)], 1)
    tv = np.stack([rng.uniform(16, W - 1, n), rng.choice([31.5, 47.5], n) + rng.choice(off, n)], 1)
    seam = np.concatenate([tu, tv])
    pts.append(_rays(view, seam, rng.uniform(0.5, 12.0, 2 * n)))
    # Gaussian centres outside tiles 0 .. 6 and the cut tile
    cuv, _, cok = V64.project(m.astype(np.float64), view)
    cin = V64.in_view(cuv, cok, W, H)
    cen = np.nonzero(cin)[0]
    ctile = V64.tile_of(cuv[cen], W, H)
    far = (ctile > 6) & (ctile != ct) & (np.abs(((cuv[cen] + 0.5) % 16) - 8) < 7).all(1)
    pts.append(m[rng.choice(cen[far], 500, replace=False)].astype(np.float64))
    pts = np.concatenate(pts).astype(np.float32)
    return settings, g, pts, ct, want, len(pts) - 500 - 2 * n - len(px)


@pytest.mark.parametrize("opaque", [False, True])
def test_tile_item_sizes_cuts_seams_and_stops(opaque):
    settings, g, pts, ct, want, c0 = _edge_scene(opaque)
    n, (ref,) = _check(settings, g, pts, tag=("edges", opaque))
    tile = ref["tile"]
    assert np.bincount(tile[tile >= 0], minlength=7)[:7].tolist() == COUNTS
    cut = ref["cut"][c0:c0 + 256]
    assert (tile[c0:c0 + 256] == ct).all()
    assert cut.tolist() == [want[k % len(want)] for k in range(256)], (want, cut[:11])
    assert want[0] == 0 and want[-1] >= 200
    print(f"cuts placed: {want}")
    # every in-view point is checked, including those within 1e-5 px of a seam
    assert n == int((tile >= 0).sum()) and n > 15000
    if opaque:
        stop = ref["stop"][ref["stop"] >= 0]
        print(f"{len(stop)} walks stop; at list index >= 32: {(stop >= 32).sum()}, on a chunk's last record: "
              f"{(stop % 32 == 31).sum()}, mid k-step: {(stop % 8 != 7).sum()}")
        assert (stop >= 32).any() and (stop % 32 == 31).any() and (stop % 8 != 7).any()
        assert (ref["T"][0][tile >= 0] >= V64.R64.T_STOP).all()  # T_out stops before the pair that crosses T_STOP


# ---------------------------------------------------------------------------------------------------- requested gradients
@pytest.mark.parametrize("subset", ["points", "cloud", "camera", "all"])
def test_every_requested_gradient_subset(subset):
    inps, g = _inputs(3000, 96, 64, 0, 2)
    views = [_settings(inps[0], 0), _settings(inps[1], 0, "fisheye")]
    kw = dict(points=dict(want_cloud=False, camera=False), cloud=dict(want_points=False, camera=False),
              camera=dict(want_points=False, want_cloud=False), all={})[subset]
    _check(views, g, _points(g, 1200, seed=3), tag=subset, **kw)


@pytest.mark.parametrize("cot", ["T_absent", "T_zero", "uv_absent", "uv_zero", "depth_absent", "depth_zero"])
def test_absent_and_zero_cotangents(cot):
    inps, g = _inputs(3000, 96, 64, 0, 1)
    pts = _points(g, 1200, seed=4)
    which, how = cot.split("_")
    if which == "T":
        kw = dict(gT=None if how == "absent" else np.zeros((1, 1200), np.float32))
    else:
        kw = {"guv" if which == "uv" else "gd": None if how == "absent" else "zero"}
    _check([_settings(inps[0], 0)], g, pts, tag=cot, **kw)


# ---------------------------------------------------------------------------------------------------- scale
def test_voxel_centres_at_c3_size_on_a_subsample():
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
    sub = np.sort(np.random.default_rng(2).choice(pts.shape[0], 2000, replace=False))
    n, _ = _check(views, g, pts, sel=sub, tag="c3 voxels")
    assert n > 2000
