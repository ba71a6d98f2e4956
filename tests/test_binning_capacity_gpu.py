"""A binning state too small for its view's instances, checked against tests/binning_ref.py and the float64 blend.

A multi-view, multi-cloud, lift or visibility call sizes each view's binning state from a capacity (the history in
rasterizer._CAPACITY, or `capacities=`) instead of reading the instance count back.  When a view emits more instances than
that, binning.cu keeps the first `capacity` it emits (the nearest Gaussians: emission is in depth order, a Gaussian may
keep part of its tile rectangle), raises status[1], and the image and its backward are those of the kept lists.

1. Lists: status, point_list, tile_ids and ranges equal binning_ref exactly, and the block lists keep the invariants of
   test_block_lists_gpu.py, at capacities 0, 1, 17, one = 15 (mod 16), a Gaussian boundary, inside the first and a later
   row of a splat spanning >= 3 x 3 tiles, R - 1, R, R + 1 and R + 4097.
2. Float64: on the same renders, checks (a) to (d) of test_blend_pairs_gpu.check_blend with its KAPPA, and the blend's
   float64 cotangents carried through project_ref64's chain to the per-Gaussian gradients.  Capacity 0 renders the
   background with final_T = 1, n_contrib = 0 and every gradient exactly 0.
3. Several views and clouds: one undersized view leaves the others' images bit for bit and their gradients unchanged,
   and the sums equal the single-view backwards at the same capacities.
4. The history path (render_views): a step whose count outgrows the learned capacity renders and backpropagates exactly
   what the raw call at that capacity does; the next call warns, does not overflow, and renders the full lists.
5. A CUDA-graph replay whose scales grew past the captured capacity reads {R', 1} and equals the eager call.
6. The capacity _calibrate learns for orthographic, fisheye and distorted views through its one-slot lift.
7. Tile counts either side of the tile sort's bit boundaries (T = 1, 2, 256, 257, 512, 513) and tiny images rendered into
   the middle slice of a batch tensor.

Measured on an NVIDIA H100 80GB HBM3 (700 W limit): worst raw ratio |x - ref64| / (u B) per scene over its eleven
capacities (the bound is KAPPA of blend_ref64 times u B):

| scene | colour | depth | final_T | alpha | features | dmeans2D | dopacity | dcolors | dfeature | gb dconic | gb ddepth |
|---|---|---|---|---|---|---|---|---|---|---|---|
| ragged F 3 | 2.89 | 2.12 | 0.24 | 0.48 | 2.82 | 0.014 | 0.054 | 0.105 | 0.137 | 0.0070 | 0.119 |
| ragged F 40 | 2.89 | 2.12 | 0.24 | 0.48 | 3.65 | 0.015 | 0.052 | 0.097 | 0.257 | 0.0050 | 0.080 |
| sh3_big F 8 | 1.48 | 4.07 | 0.21 | 0.22 | 2.44 | 0.011 | 0.020 | - | 0.175 | 0.0062 | 0.149 |
| big F 3 | 1.33 | 3.13 | 0.36 | 0.37 | 3.41 | 0.019 | 0.056 | 0.326 | 0.261 | 0.0084 | 0.220 |
| tile widths (7.) | 2.55 | 3.82 | 0.46 | 0.45 | 4.31 | 0.058 | 0.200 | 0.716 | 0.503 | 0.0187 | 0.355 |

No cull violation; borderline pixels at most 0.013 %.  The tile-width scenes (up to 1500 splats over up to 513 tiles) put
the blend-stage record's dL_dconic and dL_ddepth at 0.0187 and 0.355, past blend_ref64's KAPPA of 0.012 and 0.26 (4x the
worst of the smaller scenes it was measured on), though far below one u B: rounding of fp32 sums, not a wrong list.  Those
scenes check every other quantity of (a) to (d), and the conic and depth cotangents through the per-Gaussian chain, at
the existing KAPPA.  All cases take about 40 s.
"""
import numpy as np
import pytest

import binning_ref as BR
import blend_ref64 as R64
import util
from manigaussian_b200 import scenes
from test_blend_pairs_gpu import _scene, check_blend, iso, run_kernels, scene_ragged, state_of, _random
from test_block_lists_gpu import check_block_lists

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _own_capacity_history():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


# --------------------------------------------------------------------------- scenes and capacities
def scene_big(F=3):
    """Splats of 5 to 14 px standard deviation on a 6 x 5-tile image (each rectangle spans >= 3 x 3 tiles), with small
    ones between them, at distinct depths."""
    rng = np.random.default_rng(21)
    n, m = 14, 60
    parts = [dict(px=rng.uniform(10, 86, n), py=rng.uniform(8, 72, n), z=1.0 + rng.random(n),
                  cov2d=iso(n, 1.0) * rng.uniform(25, 200, (n, 1, 1)), opac=rng.uniform(0.2, 0.7, n)),
             dict(px=rng.uniform(0, 96, m), py=rng.uniform(0, 80, m), z=0.9 + rng.random(m), cov2d=iso(m, 1.0) *
                  rng.uniform(0.5, 10, (m, 1, 1)), opac=rng.uniform(0.1, 0.9, m))]
    return _scene(96, 80, parts, F, 22)


SCENES = {
    "ragged": scene_ragged,
    "sh3_big": lambda F: _random(dict(P=1500, W=128, H=96, F=F, seed=5, sh_degree=3, scale0=0.04, bg=(1.0, 1.0, 1.0))),
    "big": scene_big,
}
SCENE_CASES = [("ragged", 3), ("ragged", 40), ("sh3_big", 8), ("big", 3)]
CAPS = ("0", "1", "17", "15mod16", "boundary", "first_row", "later_row", "R-1", "R", "R+1", "R+4097")
_PROJ = {}


def _projection(scene, F):
    """(inp, the reference's full emission, with the projection's radii and means) of a scene: the projection is the same at
    every capacity."""
    key = (scene, F)
    if key not in _PROJ:
        inp = SCENES[scene](F)
        k = run_kernels(inp)
        ref = BR.reference(k["radii"], k["means2D"], k["depths"], k["W"], k["H"], k["R"])
        assert ref["status"][0] == k["R"]
        ref.update(radii=k["radii"], means2D=k["means2D"])
        _PROJ[key] = (inp, ref)
    return _PROJ[key]


def capacity(name, ref, W, H):
    """The capacity `name` of CAPS for the emission `ref` (binning_ref.reference)."""
    R, off, cnt = ref["R"], ref["offset"], ref["count"]
    if name.startswith("R"):
        return R + int(name[1:] or 0)
    if name == "15mod16":
        return 16 * (R // 32) + 15
    if name in ("0", "1", "17"):
        return int(name)
    if name == "boundary":   # the start of the emitted Gaussian nearest the middle of the emission
        starts = off[cnt > 0]
        return int(starts[np.argmin(np.abs(starts - R // 2))])
    # a splat whose rectangle is at least 3 x 3 tiles, nearest the middle of the emission: its widths from the reference
    x0, y0, x1, y1 = BR.tile_rect(ref["means2D"], ref["radii"], (W + 15) // 16, (H + 15) // 16)
    w, h = x1 - x0, y1 - y0
    big = np.nonzero((ref["radii"] > 0) & (w >= 3) & (h >= 3))[0]
    assert len(big), "the scene has no splat spanning 3 x 3 tiles"
    g = big[np.argmin(np.abs(off[big] - R // 2))]
    return int(off[g] + 1) if name == "first_row" else int(off[g] + w[g] + 1)


MEASURED = {}


def _record(scene, report):
    row = MEASURED.setdefault(scene, {})
    for q, v in report.items():
        if q.endswith(" raw") or q in ("cull_violations", "borderline_pixel_share"):
            row[q] = max(row.get(q, 0.0), v)


def check_lists(k, cap):
    """1: the kernels' lists against binning_ref, and the block-list invariants."""
    want = BR.reference(k["radii"], k["means2D"], k["depths"], k["W"], k["H"], cap)
    got = dict(status=k["status"], point_list=k["point_list"], tile_ids=k["tile_ids"], ranges=k["ranges"])
    bad = BR.compare(got, want)
    assert not bad, f"capacity {cap} (R = {want['R']}): " + "; ".join(bad)
    check_block_lists(k["W"], k["H"], k["ranges"], k["block_bits"], k["block_lists"], k["pixel_masks"], k["block_count"],
                      k["block_nwalk"], k["n_contrib"])
    return want


def chain_problems(name, inp, k, ref):
    """2: the blend's float64 cotangents (blend_ref64 on our masks) through project_ref64's chain, against the kernels'
    per-Gaussian gradients (test_project_ref64_gpu.check_sums)."""
    import test_project_ref64_gpu as TP
    kb = lambda q: R64.KAPPA[q] * R64.U * ref[q + "_B"]  # noqa: E731
    cot = dict(dL_dmean2D=ref["dL_dmeans2D"], dL_dmean2D_B=kb("dL_dmeans2D"), dL_dconic=ref["dL_dconic"],
               dL_dconic_B=kb("dL_dconic"), dL_dopacity=ref["dL_dopacity"], dL_dopacity_B=kb("dL_dopacity"),
               dL_dcolor=ref["dL_dcolors"], dL_dcolor_B=kb("dL_dcolors"), dL_ddepth=ref["dL_ddepth"],
               dL_ddepth_B=kb("dL_ddepth"))
    cam = dict(inp["cam"], W=k["W"], H=k["H"])
    rec = dict(radii=k["radii"], clamped=k["clamped"])
    got = dict(k["grads"])
    got.pop("dL_dfeature")
    return TP.check_sums(name, inp["g"], [cam], [rec], [cot], got, False, True)


def _check_render(name, inp, k, cap, records=True):
    want = check_lists(k, cap)
    st = state_of(inp, k)
    _, ref, problems, report = check_blend(k, st, inp, records=records)
    problems = [p for p in problems if p]
    problems += chain_problems(name, inp, k, ref)
    _record(name.split(" ")[0], report)
    print(f"[{name} cap={cap} R={want['R']}] " + " ".join(f"{a}={b:.3g}" for a, b in report.items() if a.endswith("raw")))
    assert not problems, "\n".join(problems)
    return want


@pytest.mark.parametrize("cap_name", CAPS)
@pytest.mark.parametrize("scene,F", SCENE_CASES, ids=[f"{s}-F{f}" for s, f in SCENE_CASES])
def test_overflowed_state_against_float64(scene, F, cap_name):
    inp, full = _projection(scene, F)
    cap = capacity(cap_name, full, inp["W"], inp["H"])
    k = run_kernels(inp, capacity=cap)
    assert k["R"] == full["R"]
    assert (cap < full["R"]) == bool(k["status"][1])
    if cap_name in ("first_row", "later_row"):
        # the cut falls strictly inside one Gaussian's rectangle
        assert not np.any(full["offset"][full["count"] > 0] == cap)
    _check_render(f"{scene}-F{F}", inp, k, cap)
    if cap == 0:
        bg = inp["bg"].reshape(3, 1, 1)
        assert np.array_equal(k["color"], np.broadcast_to(bg, k["color"].shape))
        assert np.all(k["final_T"] == 1) and np.all(k["n_contrib"] == 0) and np.all(k["alpha"] == 0)
        for q, v in k["grads"].items():
            assert v is None or not np.any(v), q
        assert not np.any(k["gb"])



# --------------------------------------------------------------------------- several views and clouds
def _tensors(g):
    t = util._t
    return dict(means3D=t(g["means3D"]), opacity=t(g["opacities"]), scales=t(g["scales"]), rotations=t(g["rotations"]),
                sh=t(g["shs"]), feature=t(g["feature"]) if g["feature"] is not None else None)


def _settings(cams, deg, include):
    from manigaussian_b200 import rasterizer as R
    t = util._t
    bg = np.array([0.1, 0.2, 0.3], np.float32)
    return [R.GaussianRasterizationSettings(c["H"], c["W"], c["tanfovx"], c["tanfovy"], t(bg), 1.0, t(c["viewmatrix"]),
                                            t(c["projmatrix"]), deg, t(c["campos"]), False, False, include) for c in cams]


def _views_step(a, views, caps, cots, deg):
    """Forward and backward of `views` through rasterize_views_raw at `caps`, per-view dL_dmeans2D kept apart."""
    import torch
    from manigaussian_b200 import rasterizer as R
    from test_blend_pairs_gpu import GRAD_NAMES
    F = a["feature"].shape[1] if a["feature"] is not None else 0
    outs, streams = R.rasterize_views_raw(views, a["means3D"], None, a["feature"], a["opacity"], a["scales"], a["rotations"], 1.0,
                                          None, a["sh"], deg, F > 0, return_depth=True, capacities=caps)
    m2 = torch.full((len(views), a["means3D"].shape[0], 3), float("nan"), device="cuda")
    grads = R.rasterize_views_backward_raw(views, outs, streams, [c[0] for c in cots], [c[1] for c in cots] if F else None,
                                           a["means3D"], None, a["feature"], a["scales"], a["rotations"], 1.0, None, a["sh"], deg,
                                           F > 0, grads_depth=[c[2] for c in cots], means2D_per_view=m2)
    torch.cuda.synchronize()
    return dict(img=[(o[1], o[2], o[7]) for o in outs], status=[(o.num_rendered(), o.overflowed()) for o in outs],
                m2=m2.cpu().numpy(), grads={n: g.cpu().numpy() for n, g in zip(GRAD_NAMES, grads) if g is not None and n != "dL_dmeans2D"})


def _cotangents(cams, F, seed):
    t = util._t
    rng = np.random.default_rng(seed)
    return [(t(rng.normal(0, 1, (3, c["H"], c["W"])).astype(np.float32)),
             t(rng.normal(0, 1, (F, c["H"], c["W"])).astype(np.float32)) if F else None,
             t(rng.normal(0, 1, (c["H"], c["W"])).astype(np.float32))) for c in cams]


def _same_image(x, y):
    import torch
    return all(torch.equal(a, b) for a, b in zip(x, y) if a.numel() or b.numel())


def test_one_undersized_view_of_four():
    """View 2's capacity is below its count: views 0, 1, 3 render bit for bit what ample capacities give and keep their
    dL_dmeans2D; the sums equal the four single-view backwards (view 2 at the same capacity)."""
    P, W, H, V, F, deg = 4000, 96, 72, 4, 3, 1
    g = util.make_inputs(P=P, W=W, H=H, F=F, seed=31)["g"]
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    a, views, cots = _tensors(g), _settings(cams, deg, True), _cotangents(cams, F, 31)
    counts = [r for r, _ in _views_step(a, views, [1 << 20] * V, cots, deg)["status"]]
    ample = [c + 64 for c in counts]
    small = list(ample)
    small[2] = counts[2] * 2 // 3
    A, B = _views_step(a, views, ample, cots, deg), _views_step(a, views, small, cots, deg)
    assert [o for _, o in B["status"]] == [False, False, True, False] and [r for r, _ in B["status"]] == counts
    for v in (0, 1, 3):
        assert _same_image(B["img"][v], A["img"][v]), v
        assert util.rel_l2(B["m2"][v], A["m2"][v]) < 1e-5, v
    assert not _same_image(B["img"][2], A["img"][2])
    want = {}
    for v in range(V):
        one = _views_step(a, views[v:v + 1], small[v:v + 1], cots[v:v + 1], deg)
        assert one["status"][0] == B["status"][v] and _same_image(one["img"][0], B["img"][v]), v
        assert util.rel_l2(one["m2"][0], B["m2"][v]) < 1e-5, v
        for n, x in one["grads"].items():
            want[n] = want.get(n, 0) + x.astype(np.float64)
    for n, x in B["grads"].items():
        assert util.rel_l2(x, want[n]) < 1e-5, n


def test_one_undersized_view_of_two_clouds():
    """rasterize_clouds_raw / rasterize_clouds_backward_raw: cloud 1's view 0 overflows; cloud 0's images and gradients and
    cloud 1's other view are unchanged."""
    import copy
    import torch
    from manigaussian_b200.rasterizer import rasterize_clouds_backward_raw, rasterize_clouds_raw
    from test_clouds_gpu import _leaves, _raw_clouds
    from test_render_gpu import _cams
    cams = _cams(2, 64, 64)
    hosts = [_leaves(3000, 32, 80 + b, "sh") for b in range(2)]
    rng = np.random.default_rng(5)
    cot = [(util._t(rng.normal(0, 1, (2, 3, 64, 64)).astype(np.float32)), util._t(rng.normal(0, 1, (2, 32, 64, 64)).astype(np.float32)))
           for _ in hosts]

    def run(caps):
        clouds = _raw_clouds(cams, hosts, caps)
        outs, streams = rasterize_clouds_raw(clouds, 1, True)
        for c, (gc, gf) in zip(clouds, cot):
            c["grad_color"], c["grad_feature"] = gc, gf
        grads = rasterize_clouds_backward_raw(clouds, outs, streams, 1, True)
        torch.cuda.synchronize()
        return outs, [{k: (None if v is None else v.cpu().numpy()) for k, v in gr.items()} for gr in grads]

    first, _ = run([[1 << 20] * 2] * 2)
    counts = [[o.num_rendered() for o in co] for co in first]
    ample = [[c + 64 for c in cc] for cc in counts]
    small = copy.deepcopy(ample)
    small[1][0] = counts[1][0] // 2
    oa, ga = run(ample)
    ob, gb = run(small)
    for b in range(2):
        for v in range(2):
            assert ob[b][v].num_rendered() == counts[b][v] and ob[b][v].overflowed() == ((b, v) == (1, 0)), (b, v)
            if (b, v) != (1, 0):
                assert all(torch.equal(ob[b][v][i], oa[b][v][i]) for i in (1, 2, 3)), (b, v)
    for k, x in gb[0].items():
        if x is not None:
            assert util.rel_l2(x, ga[0][k]) < 1e-5, k
    assert util.rel_l2(gb[1]["dL_dmeans2D"][1], ga[1]["dL_dmeans2D"][1]) < 1e-5


# --------------------------------------------------------------------------- the history path
def _leaf_tensors(g, scale=1.0, grad=True):
    t = util._t
    d = dict(xyz=t(g["means3D"]), rot=t(g["rotations"]), scale=t(g["scales"] * np.float32(scale)), opac=t(g["opacities"]),
             sh=t(g["shs"]))
    return {k: v.requires_grad_(grad) for k, v in d.items()}


def _raw_step(L, views, caps, cts):
    """The raw multi-view forward and backward at `caps`: (images [V,3,H,W], leaf gradients keyed like L, outs)."""
    import torch
    from manigaussian_b200 import rasterizer as R
    outs, streams = R.rasterize_views_raw(views, L["xyz"], None, None, L["opac"], L["scale"], L["rot"], 1.0, None, L["sh"], 1, False,
                                          capacities=caps)
    g = R.rasterize_views_backward_raw(views, outs, streams, list(cts), None, L["xyz"], None, None, L["scale"], L["rot"], 1.0, None,
                                       L["sh"], 1, False)
    torch.cuda.synchronize()
    grads = dict(xyz=g[4], rot=g[8], scale=g[7], opac=g[3], sh=g[6])
    return torch.stack([o[1] for o in outs]), {k: v.cpu().numpy() for k, v in grads.items()}, outs


def _counts(g, views, scale):
    with_grad = _leaf_tensors(g, scale, grad=False)
    cts = [util._t(np.zeros((3, s.image_height, s.image_width), np.float32)) for s in views]
    return [o.num_rendered() for o in _raw_step(with_grad, views, [1 << 21] * len(views), cts)[2]]


def _grow(g, views, caps):
    """The smallest listed factor on the scales that takes every view's instance count past its capacity, and the counts."""
    for s in (1.5, 2.0, 3.0, 4.0, 6.0):
        n = _counts(g, views, s)
        if all(c > cap for c, cap in zip(n, caps)):
            return s, n
    raise AssertionError(f"no scale factor takes the counts {n} past {caps}")


def test_history_path_step_past_the_learned_capacity():
    """render_views at fixed P: the first call calibrates; a step whose counts outgrow the learned capacities renders the
    truncated lists exactly as rasterize_views_raw(capacities=learned) does and backpropagates the same leaf gradients; the
    next call warns, does not overflow, and renders the full lists bit for bit."""
    import torch
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200.gaussian_renderer import render_views
    from test_render_gpu import _cams, _cloud
    R.reset_capacity_estimates()
    P, W, H, V = 16384, 96, 96, 2
    g = _cloud(P, 3, 41)
    cams = _cams(V, W, H)
    views = [cams.settings(v, torch.zeros(3, device="cuda"), 1, False) for v in range(V)]
    cts = torch.from_numpy(np.random.default_rng(41).normal(0, 1, (V, 3, H, W)).astype(np.float32)).cuda()

    def step(scale):
        L = _leaf_tensors(g, scale)
        out = render_views(cams, pts_xyz=L["xyz"], rotations=L["rot"], scales=L["scale"], opacity=L["opac"], features_color=L["sh"])
        (out["render"] * cts).sum().backward()
        torch.cuda.synchronize()
        return out["render"].detach(), {k: v.grad.cpu().numpy() for k, v in L.items()}

    step(1.0)
    keys = [(torch.cuda.current_device(), P, W, H, v) for v in range(V)]
    caps = [R._CAPACITY[k] for k in keys]
    s, counts = _grow(g, views, caps)
    img, grads = step(s)
    # the next call of any rasterize_views_raw route polls the finished forward's status: this one warns
    with pytest.warns(UserWarning, match="tile instances"):
        img2, _ = step(s)
    assert all(R._CAPACITY[k] > n for k, n in zip(keys, counts))
    assert len(R._PENDING_STATUS) == V
    assert all(int(st[1]) == 0 and int(st[0]) == n for (_, st, _, _), n in zip(R._PENDING_STATUS, counts))
    raw_img, raw_grads, _ = _raw_step(_leaf_tensors(g, s, grad=False), views, caps, cts)
    assert torch.equal(img, raw_img)
    for k in grads:
        assert util.rel_l2(grads[k], raw_grads[k]) < 1e-5, k
    full_img, _, _ = _raw_step(_leaf_tensors(g, s, grad=False), views, [n + 64 for n in counts], cts)
    assert torch.equal(img2, full_img) and not torch.equal(img, img2)


def test_captured_step_replays_past_its_capacity():
    """A raw forward and backward captured at the history's capacities; the scales grow in place past them and the graph
    replays: the pinned status reads {R', 1}, the image equals the eager call at the same capacities bit for bit and the
    gradients match it."""
    import torch
    from manigaussian_b200 import rasterizer as R
    from test_render_gpu import _cams, _cloud
    P, W, H, V = 8192, 64, 64, 2
    g = _cloud(P, 3, 43)
    cams = _cams(V, W, H)
    views = [cams.settings(v, torch.zeros(3, device="cuda"), 1, False) for v in range(V)]
    cts = [util._t(np.random.default_rng(43 + v).normal(0, 1, (3, H, W)).astype(np.float32)) for v in range(V)]
    L = _leaf_tensors(g, grad=False)

    def step(caps=None):
        outs, streams = R.rasterize_views_raw(views, L["xyz"], None, None, L["opac"], L["scale"], L["rot"], 1.0, None, L["sh"], 1,
                                              False, capacities=caps)
        return outs, R.rasterize_views_backward_raw(views, outs, streams, cts, None, L["xyz"], None, None, L["scale"], L["rot"],
                                                    1.0, None, L["sh"], 1, False)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    caps = [R._CAPACITY[(torch.cuda.current_device(), P, W, H, v)] for v in range(V)]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs, grads = step()
    s, counts = _grow(g, views, caps)
    with torch.no_grad():
        L["scale"].mul_(s)
    graph.replay()
    torch.cuda.synchronize()
    assert [(int(o.status[0]), int(o.status[1])) for o in outs] == [(n, 1) for n in counts]
    e_outs, e_grads = step(caps)
    torch.cuda.synchronize()
    for o, e in zip(outs, e_outs):
        assert torch.equal(o[1], e[1])
    for x, y in zip(grads, e_grads):
        if x is not None:
            assert util.rel_l2(x.cpu().numpy(), y.cpu().numpy()) < 1e-5


# --------------------------------------------------------------------------- calibration of non-pinhole views
def _camera(model, W, H):
    from manigaussian_b200 import cameras
    from test_render_gpu import GOLD
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("mk", os.path.join(GOLD, "make_camera_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    extr = mk.look_at([1.8, 0.0, 1.5], [0.2, 0, 1.1])[None].astype(np.float32)
    f = W / (2 * np.tan(np.deg2rad(20)))
    K = np.array([[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]]], np.float32)
    if model == "ortho":
        return cameras.build_ortho_cameras(extr, (0.8, 0.6), W, H, device="cuda")
    if model == "fisheye":
        return cameras.build_fisheye_cameras(K, np.array([[0.05, -0.01, 0.002, 0.0]]), extr, W, H, device="cuda")
    return cameras.build_distorted_cameras(K, np.array([[-0.1, 0.02, 0.001, -0.001, 0.0]]), extr, W, H, device="cuda")


@pytest.mark.parametrize("model", ["ortho", "fisheye", "distorted"])
def test_calibration_of_non_pinhole_views(model):
    """_calibrate counts these views with a one-slot lift (which overflows): the capacity it learns is
    _round_capacity(1.25 R + 4096), R the count of a render with ample capacity."""
    import torch
    from manigaussian_b200 import rasterizer as R
    from test_render_gpu import _cloud
    P, W, H = 6000 + ["ortho", "fisheye", "distorted"].index(model), 80, 64
    g = _cloud(P, 3, 47)
    cb = _camera(model, W, H)
    views = [cb.settings(0, torch.zeros(3, device="cuda"), 1, False)]
    key = (torch.cuda.current_device(), P, W, H, 0)
    R.reset_capacity_estimates()
    L = _leaf_tensors(g, grad=False)
    args = (L["xyz"], None, None, L["opac"], L["scale"], L["rot"], 1.0, None, L["sh"], 1, False)
    outs, _ = R.rasterize_views_raw(views, *args)
    learned = R._CAPACITY[key]
    ample, _ = R.rasterize_views_raw(views, *args, capacities=[1 << 20])
    n = ample[0].num_rendered()
    assert n > 1000 and learned == R._round_capacity(n * 1.25 + 4096), (n, learned)
    assert outs[0].num_rendered() == n and not outs[0].overflowed()
    assert torch.equal(outs[0][1], ample[0][1])


# --------------------------------------------------------------------------- tile-sort widths and tiny images
TILE_CASES = [(1, 1), (7, 3), (16, 16), (32, 16), (4096, 16), (4112, 16), (4096, 32), (432, 304)]  # T = 1 1 1 2 256 257 512 513


def scene_tiles(W, H, F=3):
    """Random splats over the whole image and a little past its edges."""
    rng = np.random.default_rng(W * 7 + H)
    n = int(min(1500, max(12, W * H // 48)))
    parts = [dict(px=rng.uniform(-4, W + 4, n), py=rng.uniform(-4, H + 4, n), z=0.8 + rng.random(n),
                  cov2d=iso(n, 1.0) * rng.uniform(0.5, 20, (n, 1, 1)), opac=1 / (1 + np.exp(-rng.normal(-1, 1.5, n))))]
    return _scene(W, H, parts, F, 23)


def _render_into_middle(inp, k):
    """The same forward through out_buffers into slice 1 of NaN-filled [3, ...] batch tensors: slice 1 holds what the
    ViewOut planes held, slices 0 and 2 stay NaN."""
    import torch
    from manigaussian_b200 import rasterizer as R
    t = util._t
    cam, g = inp["cam"], inp["g"]
    W, H, F = inp["W"], inp["H"], inp["F"]
    s = R.GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], t(inp["bg"]), 1.0, t(cam["viewmatrix"]),
                                        t(cam["projmatrix"]), 0, t(cam["campos"]), False, False, F > 0)
    nan = dict(dtype=torch.float32, device="cuda")
    bufs = (torch.full((3, 3, H, W), float("nan"), **nan), torch.full((3, F, H, W), float("nan"), **nan),
            torch.full((3, H, W), float("nan"), **nan), torch.full((3, H, W), float("nan"), **nan))
    R.rasterize_views_raw([s], t(g["means3D"]), t(g["colors_precomp"]), t(g["feature"]), t(g["opacities"]), None, None, 1.0,
                          t(g["cov3D_precomp"]), None, 0, F > 0, return_depth=True, return_alpha=True,
                          out_buffers=tuple(b[1:2] for b in bufs))
    torch.cuda.synchronize()
    for b, want in zip(bufs, (k["color"], k["feature"], k["depth"], k["alpha"])):
        x = b.cpu().numpy()
        assert np.isnan(x[0]).all() and np.isnan(x[2]).all()
        assert np.array_equal(x[1], want)


@pytest.mark.parametrize("W,H", TILE_CASES, ids=[f"{w}x{h}" for w, h in TILE_CASES])
def test_tile_sort_widths_and_tiny_images(W, H):
    inp = scene_tiles(W, H)
    k = run_kernels(inp)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    assert k["R"] > 0 and not k["status"][1]
    if T > 2:
        assert int(k["tile_ids"].max()) >= T - 2, "the instances must reach the last tiles"
    # the blend-stage records are checked through the chain only here (see the module docstring)
    _check_render(f"tiles {W}x{H}", inp, k, k["cap"], records=T <= 2)
    if W * H <= 256:
        _render_into_middle(inp, k)


def test_report():
    """Prints the worst raw ratio per scene over the cases above (run with -s after the others)."""
    for scene, row in MEASURED.items():
        print(f"[worst {scene}] " + " ".join(f"{q}={v:.3g}" for q, v in sorted(row.items())))
