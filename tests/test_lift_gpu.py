"""The lift (lift.cu, mgs_lift_views, gaussian_renderer.lift_views) on the GPU.

1. Per Gaussian against float64: on the screen-space scenes of test_blend_pairs_gpu, with the forward's pixel masks as the
   decisions, every element of lifted and weight is within KAPPA["dL_dfeature"] u B of blend_ref64's w^T map (its
   dL_dfeature with the map as the feature cotangent; a ones map for weight).
2. Equal to the autograd route (render_views of zero features with C + 1 channels, normalize_feature=False, then
   torch.autograd.grad with the maps and a ones channel) to 1e-5 rel-L2, over view counts, image shapes, widths, the
   anti-aliased mode, cov3D_precomp and device field-of-view cameras.
3. Identities against a render_views of the same scene: sum_g weight = sum_p alpha, sum_g lifted[:, c] = sum_p map[c] alpha,
   <lifted, f> = <map, render_embed(f)>.
4. Edges: a culled cloud, a view that sees nothing, unaligned maps and C % 4 != 0, no growth of device memory.
"""
import numpy as np
import pytest
import torch

import blend_ref64 as R64
import util  # noqa: F401  (sys.path)
from test_blend_pairs_gpu import SCENES, run_kernels, state_of
from test_camera_grad_gpu import _intr, _scene, _w2c

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _own_capacity_history():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))


# --------------------------------------------------------------------------- 1. per Gaussian against float64
PAIR_CASES = [("lists", 3), ("lists", 40), ("term32", 0), ("term64", 32), ("empty_run", 67), ("needles", 3),
              ("offscreen", 3), ("opacity", 32), ("ragged", 0), ("ragged", 67), ("ragged_f32", 32), ("sh3_big", 40),
              ("offscreen", 512)]


@pytest.mark.parametrize("scene,C", PAIR_CASES, ids=[f"{s}-C{c}" for s, c in PAIR_CASES])
def test_lift_per_gaussian_against_float64(scene, C):
    from manigaussian_b200 import rasterizer as R
    t = util._t
    inp = SCENES[scene](0)
    k = run_kernels(inp)
    st = state_of(inp, k)
    W, H, P = k["W"], k["H"], inp["P"]
    cam, g = inp["cam"], inp["g"]
    masks = R64.masks_from_blocks(st, k["block_lists"], k["pixel_masks"], k["block_nwalk"])
    rng = np.random.default_rng(11 + C)
    maps = rng.normal(0, 1, (C, H, W)).astype(np.float32)
    s = R.GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], t(inp["bg"]), 1.0, t(cam["viewmatrix"]),
                                        t(cam["projmatrix"]), g["sh_degree"], t(cam["campos"]), False, False, False)
    lifted, weight = R.lift_views_raw([s], t(g["means3D"]), t(g["opacities"]), t(g["scales"]), t(g["rotations"]), 1.0,
                                      t(g["cov3D_precomp"]), [t(maps)] if C else None)
    torch.cuda.synchronize()
    # the reference's dL_dfeature is w^T g_feature: features of any value, the map as their cotangent, plus a ones plane
    planes = np.concatenate([maps, np.ones((1, H, W), np.float32)], 0)
    ref = R64.blend(dict(st, feature=np.zeros((P, C + 1), np.float32), g_feature=planes), masks)
    got = np.concatenate([lifted.cpu().numpy().reshape(P, C), weight.cpu().numpy()[:, None]], 1)
    r = R64.ratio(got, ref["dL_dfeature"], ref["dL_dfeature_B"], "dL_dfeature")
    raw = float(r.max()) * R64.KAPPA["dL_dfeature"] if r.size else 0.0
    print(f"[{scene} C={C}] worst raw ratio {raw:.3g}")
    assert r.max() <= 1.0, (np.unravel_index(np.argmax(r), r.shape), raw)
    # the lift's decisions are the forward's: Gaussians that blended nowhere get exactly nothing
    seen = np.zeros(P, bool)
    for tile, m in enumerate(masks):
        r0, r1 = (int(v) for v in k["ranges"][tile])
        seen[k["point_list"][r0:r1][m.any(0)]] = True
    assert np.all(got[~seen] == 0.0)
    assert np.all(weight.cpu().numpy()[seen] > 0.0)


# --------------------------------------------------------------------------- 2. equal to the autograd route
def _cams(V, W, H, learnable=False):
    from manigaussian_b200.cameras import camera_batch
    K = torch.tensor(_intr(V, W, H), dtype=torch.float32, device="cuda")
    if learnable:
        K.requires_grad_()
    return camera_batch(_w2c(V, seed=V), K, W, H)


def _autograd_lift(cams, sc, maps, aa):
    from manigaussian_b200 import gaussian_renderer as GR
    V, C = len(maps), maps[0].shape[0]
    P = sc["pts_xyz"].shape[0]
    f = torch.zeros(P, C + 1, device="cuda", requires_grad=True)
    out = GR.render_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], pts_rgb=sc["pts_rgb"],
                          features_language=f, normalize_feature=False, antialiasing=aa)
    H, W = maps[0].shape[1:]
    cot = torch.stack([torch.cat([m, torch.ones(1, H, W, device="cuda")], 0) for m in maps])
    (g,) = torch.autograd.grad(out["render_embed"], [f], cot)
    return g[:, :C], g[:, C]


ROUTE_CASES = [  # (V, W, H, C, aa, learnable intr)
    (1, 96, 80, 0, False, False), (1, 96, 80, 3, True, False), (2, 96, 80, 8, False, False), (4, 96, 80, 32, False, False),
    (4, 96, 80, 40, True, False), (2, 61, 37, 67, False, False), (17, 64, 48, 3, False, False), (2, 96, 80, 128, False, False),
    (4, 61, 37, 32, True, True), (2, 96, 80, 0, False, True)]


@pytest.mark.parametrize("V,W,H,C,aa,learn", ROUTE_CASES, ids=[f"V{c[0]}-{c[1]}x{c[2]}-C{c[3]}{'-aa' if c[4] else ''}"
                                                               f"{'-intr' if c[5] else ''}" for c in ROUTE_CASES])
def test_lift_equals_the_autograd_route(V, W, H, C, aa, learn):
    from manigaussian_b200 import gaussian_renderer as GR
    sc = _scene(6000, sh=False, seed=40 + C)
    cams = _cams(V, W, H, learn)
    gen = torch.Generator(device="cuda").manual_seed(C + V)
    maps = torch.randn(V, C, H, W, device="cuda", generator=gen)
    out = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps if C else None, antialiasing=aa)
    assert out["lifted"].shape == (sc["pts_xyz"].shape[0], C) and out["weight"].shape == (sc["pts_xyz"].shape[0],)
    assert not out["lifted"].requires_grad and not out["weight"].requires_grad
    ref_l, ref_w = _autograd_lift(cams, sc, list(maps), aa)
    assert float(ref_w.sum()) > 0
    assert _rel_l2(out["weight"], ref_w) < 1e-5
    if C:
        assert _rel_l2(out["lifted"], ref_l) < 1e-5


def test_lift_with_cov3D_precomp_equals_the_raw_backward():
    from manigaussian_b200 import rasterizer as R
    inp = SCENES["ragged"](0)
    t = util._t
    cam, g = inp["cam"], inp["g"]
    W, H, P, C = inp["W"], inp["H"], inp["P"], 5
    s = R.GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], t(inp["bg"]), 1.0, t(cam["viewmatrix"]),
                                        t(cam["projmatrix"]), 0, t(cam["campos"]), False, False, True)
    maps = torch.randn(C, H, W, device="cuda")
    feat = torch.zeros(P, C + 1, device="cuda")
    args = (t(g["means3D"]), t(g["colors_precomp"]), feat, t(g["opacities"]), None, None, 1.0, t(g["cov3D_precomp"]), None, 0, True)
    outs, streams = R.rasterize_views_raw([s], *args)
    cot = torch.cat([maps, torch.ones(1, H, W, device="cuda")], 0)
    grads = R.rasterize_views_backward_raw([s], outs, streams, [torch.zeros(3, H, W, device="cuda")], [cot], args[0], args[1],
                                           args[2], None, None, 1.0, args[7], None, 0, True)
    lifted, weight = R.lift_views_raw([s], args[0], args[3], None, None, 1.0, args[7], [maps])
    assert _rel_l2(lifted, grads[2][:, :C]) < 1e-5 and _rel_l2(weight, grads[2][:, C]) < 1e-5


# --------------------------------------------------------------------------- 3. identities
@pytest.mark.parametrize("aa", [False, True])
def test_lift_identities_against_a_render(aa):
    from manigaussian_b200 import gaussian_renderer as GR
    V, W, H, C = 3, 96, 80, 6
    sc = _scene(5000, sh=False, seed=5)
    cams = _cams(V, W, H)
    maps = torch.rand(V, C, H, W, device="cuda")
    out = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps, antialiasing=aa)
    f = torch.randn(sc["pts_xyz"].shape[0], C, device="cuda")
    r = GR.render_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], pts_rgb=sc["pts_rgb"],
                        features_language=f, normalize_feature=False, return_alpha=True, antialiasing=aa)
    alpha = r["alpha"].double()
    w_sum, a_sum = float(out["weight"].double().sum()), float(alpha.sum())
    assert abs(w_sum - a_sum) <= 1e-5 * a_sum
    for c in range(C):
        want = float((maps[:, c].double() * alpha).sum())
        assert abs(float(out["lifted"][:, c].double().sum()) - want) <= 1e-5 * abs(want)
    lhs = float((out["lifted"].double() * f.double()).sum())
    rhs = float((maps.double() * r["render_embed"].double()).sum())
    scale = float((out["lifted"].double().abs() * f.double().abs()).sum())
    assert abs(lhs - rhs) <= 1e-5 * scale


# --------------------------------------------------------------------------- 4. edges
def test_culled_cloud_and_empty_view_give_zeros():
    from manigaussian_b200 import gaussian_renderer as GR
    sc = _scene(2000, sh=False, seed=9)
    cams = _cams(2, 64, 48)
    maps = torch.randn(2, 4, 48, 64, device="cuda")
    # the cameras sit near z = -2 looking along +z: a cloud at z = -50 is behind every one of them
    behind = dict(sc, pts_xyz=sc["pts_xyz"] * 0.01 + torch.tensor([0.0, 0.0, -50.0], device="cuda"))
    out = GR.lift_views(cams, behind["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps)
    assert torch.count_nonzero(out["lifted"]) == 0 and torch.count_nonzero(out["weight"]) == 0
    # the culled cloud taught the capacity table an empty binning for this (P, W, H): start the visible cloud afresh
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    # view 1 looks away from the cloud (camera turned around): it adds nothing to what view 0 gives alone
    w2c = _w2c(2, seed=2)
    flip = torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0], device="cuda"))
    w2c = torch.stack([w2c[0], flip @ w2c[0]])
    from manigaussian_b200.cameras import camera_batch
    cams2 = camera_batch(w2c, _intr(2, 64, 48), 64, 48)
    both = GR.lift_views(cams2, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps)
    one = GR.lift_views(cams2, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps[:1], view_ids=[0])
    only1 = GR.lift_views(cams2, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps[1:], view_ids=[1])
    assert torch.count_nonzero(only1["weight"]) == 0 and torch.count_nonzero(only1["lifted"]) == 0
    assert float(one["weight"].sum()) > 0
    assert _rel_l2(both["weight"], one["weight"]) < 1e-6 and _rel_l2(both["lifted"], one["lifted"]) < 1e-6


@pytest.mark.parametrize("C", [3, 5, 36, 67])
def test_unaligned_maps_and_odd_widths_match_the_aligned_case(C):
    from manigaussian_b200 import gaussian_renderer as GR
    V, W, H = 2, 61, 37
    sc = _scene(4000, sh=False, seed=C)
    cams = _cams(V, W, H)
    maps = torch.randn(V, C, H, W, device="cuda")
    ref = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps)
    n = C * H * W
    base = torch.empty(V, n + 1, device="cuda")
    base[:, 1:] = maps.reshape(V, n)
    shifted = [base[v, 1:].view(C, H, W) for v in range(V)]  # 4-byte offset: no 16-byte alignment
    assert all(m.data_ptr() % 16 for m in shifted)
    got = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], shifted)
    assert _rel_l2(got["lifted"], ref["lifted"]) < 1e-6 and _rel_l2(got["weight"], ref["weight"]) < 1e-6
    # C % 4 != 0 takes the padded path; the channels agree with lifting them one by one (the C = 1 .. 3 paths)
    if C < 8:
        for c in range(C):
            one = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps[:, c:c + 1])
            assert _rel_l2(one["lifted"][:, 0], ref["lifted"][:, c]) < 1e-6


def test_repeated_calls_do_not_accumulate_device_memory():
    from manigaussian_b200 import gaussian_renderer as GR
    sc = _scene(5000, sh=False, seed=3)
    cams = _cams(3, 96, 80)
    maps = torch.randn(3, 16, 80, 96, device="cuda")
    for _ in range(3):
        GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for _ in range(20):
        out = GR.lift_views(cams, sc["pts_xyz"], sc["rotations"], sc["scales"], sc["opacity"], maps)
        del out
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= before
