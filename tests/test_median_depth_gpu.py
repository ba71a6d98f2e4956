"""The median-depth plane and the per-pixel surface Gaussian on the GPU.

* The rule holds against the kernel's own decisions: the pixel masks, block lists, point_list and final_T are read back through
  mgs_state_array, T is recomputed in float64 for every pixel, and the chosen contributor is the last one whose incoming
  T > 0.5 (tests/median_ref64.py), either neighbour being accepted where an incoming T lies within the fp32 bound of 0.5.
  median_depth is bit for bit the depth of Gaussian median_id in the geometry state; -1 / 0 where nothing contributes.
* Nothing else moves: with the median on and off, the images, final_T, n_contrib, radii and instance counts are bit-identical
  and the colour / feature gradients agree within the float atomics' noise.
* Gradient: a median cotangent g alone gives dL/dmeans3D_i = (sum over the pixels of Gaussian i of g) R_v[2,:], exactly zero
  gradients everywhere else, and dL/dviewmatrix equal to float64 autograd of z = (V [p, 1]).z summed the same way; with a
  colour cotangent as well, the sum of the two runs.
* Public paths: GaussianRasterizer, render, render_views and render_clouds return the planes and backpropagate through them;
  targets with return_median_depth raise; a captured CUDA graph replays the step with the eager outputs.
"""
import numpy as np
import pytest

import util
import blend_ref64 as B
import median_ref64 as M

pytestmark = pytest.mark.gpu


def _t(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def _scene(kind, F):
    W, H = (200, 120) if kind != "small" else (61, 37)
    # the culled cloud has a size of its own: the binning capacity learnt from its empty lists must not size the others
    P = {"small": 800, "culled": 4000}.get(kind, 5000)
    inp = util.make_inputs(P=P, W=W, H=H, F=F, seed=3 + F, bg=(0.3, 0.6, 0.9))
    if kind == "culled":  # every Gaussian at the camera centre, in front of the near plane: empty tile lists
        inp["g"]["means3D"] = np.tile(np.asarray(inp["cam"]["campos"], np.float32).reshape(1, 3), (inp["P"], 1))
    return inp


def _settings(inp):
    from manigaussian_b200 import rasterizer as R
    cam, g = inp["cam"], inp["g"]
    return R.GaussianRasterizationSettings(inp["H"], inp["W"], cam["tanfovx"], cam["tanfovy"], _t(inp["bg"]), 1.0, _t(cam["viewmatrix"]),
                                           _t(cam["projmatrix"]), g["sh_degree"], _t(cam["campos"]), False, False, inp["F"] > 0)


def _args(inp):
    g, F = inp["g"], inp["F"]
    return (_t(g["means3D"]), None, _t(g["feature"]) if F else None, _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]), 1.0,
            None, _t(g["shs"]), g["sh_degree"], F > 0)


def _forward(inp, median, aa=False):
    from manigaussian_b200 import rasterizer as R
    s = _settings(inp)
    args = _args(inp)
    outs, streams = R.rasterize_views_raw([s], *args, return_depth=True, return_alpha=True, antialiasing=aa, return_median=median)
    assert not outs[0].overflowed()
    return s, args, outs, streams


def _state(inp, o):
    import torch
    from manigaussian_b200 import rasterizer as R
    torch.cuda.synchronize()
    P, W, H = inp["P"], inp["W"], inp["H"]
    cap, Rn = int(o[0]), o.num_rendered()
    T = ((W + 15) // 16) * ((H + 15) // 16)
    S = (cap + 11) & ~3

    def arr(which, name, state, a0, a1, dtype, count):
        off = R.state_array(which, name, state, a0, a1) - state.data_ptr()
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return state[off:off + nbytes].view(dtype).cpu().numpy()

    geomB, binB, imgB = o[4], o[5], o[6]
    k = dict(W=W, H=H, R=Rn)
    k["means2D"] = arr("geometry", "means2D", geomB, P, 0, torch.float32, 2 * P).reshape(P, 2)
    k["conic_opacity"] = arr("geometry", "conic_opacity", geomB, P, 0, torch.float32, 4 * P).reshape(P, 4)
    k["rgbd"] = arr("geometry", "rgbd", geomB, P, 0, torch.float32, 4 * P).reshape(P, 4)
    k["point_list"] = arr("binning", "point_list", binB, cap, 0, torch.int32, max(Rn, 1)).view(np.uint32)[:Rn]
    k["block_lists"] = arr("binning", "block_lists", binB, cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    k["pixel_masks"] = arr("binning", "pixel_masks", binB, cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    k["ranges"] = arr("image", "ranges", imgB, W, H, torch.int32, 2 * T).view(np.uint32).reshape(T, 2)
    k["block_nwalk"] = arr("image", "block_nwalk", imgB, W, H, torch.int32, 8 * T).view(np.uint32).reshape(T, 8)
    k["final_T"] = arr("image", "final_T", imgB, W, H, torch.float32, W * H).reshape(H, W)
    k["n_contrib"] = arr("image", "n_contrib", imgB, W, H, torch.int32, W * H).reshape(H, W)
    return k


CASES = [("small", 3, False), ("ragged", 3, False), ("ragged", 32, False), ("ragged", 64, False), ("ragged", 3, True),
         ("ragged", 32, True), ("culled", 3, False)]


@pytest.mark.parametrize("kind,F,aa", CASES)
def test_rule_holds_against_the_kernels_decisions(kind, F, aa):
    inp = _scene(kind, F)
    s, args, outs, _ = _forward(inp, True, aa)
    o = outs[0]
    k = _state(inp, o)
    med_depth, med_id = o[9].cpu().numpy(), o[10].cpu().numpy()
    W, H = inp["W"], inp["H"]
    assert med_id.shape == (H, W) and med_id.dtype == np.int32
    if kind == "culled":
        assert k["R"] == 0 and (med_id == -1).all() and (med_depth == 0).all() and not np.signbit(med_depth).any()
        return
    masks = B.masks_from_blocks(k, k["block_lists"], k["pixel_masks"], k["block_nwalk"])
    n_pix = n_band = n_cross = 0
    for tile in range(k["ranges"].shape[0]):
        px, py, inside = B.tile_pixels(W, H, tile)
        m = masks[tile]
        if m.shape[1] == 0:
            assert (med_id[py[inside], px[inside]] == -1).all()
            continue
        p = B._pairs(k, tile)
        lo, hi = M.median_band(p["alpha"], m, p["ea"])
        exact = M.median(p["alpha"], m)
        ids = p["ids"]
        for j in np.nonzero(inside)[0]:
            got = int(med_id[py[j], px[j]])
            n_pix += 1
            if not m[j].any():
                assert got == -1 and med_depth[py[j], px[j]] == 0, (tile, j)
                continue
            pos = np.nonzero(ids == got)[0]
            assert len(pos) == 1, (tile, j, got)
            q = int(pos[0])
            assert m[j, q], (tile, j, q)  # a contributor of the pixel
            assert lo[j] <= q <= hi[j], (tile, j, q, lo[j], hi[j], exact[j])
            n_band += lo[j] != hi[j]
            n_cross += q != m[j].nonzero()[0][-1]
            # bit for bit the depth the depth channel blends for that Gaussian
            assert med_depth[py[j], px[j]].view(np.uint32) == k["rgbd"][got, 3].view(np.uint32)
    assert n_pix == W * H
    assert n_cross > 0  # the crossing is exercised, not only "last contributor"
    assert n_band < 0.01 * n_pix


@pytest.mark.parametrize("F,aa", [(3, False), (32, False), (64, False), (32, True)])
def test_nothing_else_moves(F, aa):
    import torch
    from manigaussian_b200 import rasterizer as R
    inp = _scene("ragged", F)
    res = {}
    for median in (False, True):
        s, args, outs, streams = _forward(inp, median, aa)
        o = outs[0]
        k = _state(inp, o)
        ct = inp["ct"]
        grads = R.rasterize_views_backward_raw([s], outs, streams, [_t(ct["dL_dcolor"])], [_t(ct["dL_dfeature"])] if F else None,
                                               args[0], None, args[2], args[4], args[5], 1.0, None, args[8], args[9], F > 0,
                                               antialiasing=aa)
        torch.cuda.synchronize()
        res[median] = dict(planes=[o[i].cpu().numpy() for i in (1, 2, 3, 7, 8)], final_T=k["final_T"], n_contrib=k["n_contrib"],
                           R=k["R"], grads=[None if x is None else x.cpu().numpy() for x in grads])
    a, b = res[False], res[True]
    assert a["R"] == b["R"]
    for x, y in zip(a["planes"], b["planes"]):
        assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y)
    assert np.array_equal(a["final_T"].view(np.uint32), b["final_T"].view(np.uint32))
    assert np.array_equal(a["n_contrib"], b["n_contrib"])
    for x, y in zip(a["grads"], b["grads"]):
        if x is not None:
            assert util.rel_l2(y, x) < 1e-5


def _median_grads(inp, aa, color):
    """(median plane, median ids, gradients, camera gradients) of a backward with a random median cotangent and, when `color`,
    the inputs' colour cotangent (else zero colour and feature cotangents)"""
    import torch
    from manigaussian_b200 import rasterizer as R
    s, args, outs, streams = _forward(inp, True, aa)
    o = outs[0]
    F, H, W = inp["F"], inp["H"], inp["W"]
    g = np.random.default_rng(11).normal(0, 1, (H, W)).astype(np.float32)
    gc = _t(inp["ct"]["dL_dcolor"]) if color else torch.zeros((3, H, W), device="cuda")
    gf = [torch.zeros((F, H, W), device="cuda")] if F else None
    grads = R.rasterize_views_backward_raw([s], outs, streams, [gc], gf, args[0], None, args[2], args[4], args[5], 1.0, None, args[8],
                                           args[9], F > 0, antialiasing=aa, camera_grads=True, grads_median=[_t(g)],
                                           median_ids=[o[10]])
    torch.cuda.synchronize()
    return g, o[10].cpu().numpy(), [None if x is None else (x.cpu().numpy() if torch.is_tensor(x) else x) for x in grads[:9]], \
        [x.cpu().numpy() for x in grads[9][:3]]


@pytest.mark.parametrize("F,aa", [(3, False), (32, True)])
def test_median_gradient(F, aa):
    import torch
    inp = _scene("ragged", F)
    P = inp["P"]
    g, ids, grads, cam = _median_grads(inp, aa, False)
    valid = ids >= 0
    G = np.bincount(ids[valid], weights=g[valid].astype(np.float64), minlength=P)
    Gabs = np.bincount(ids[valid], weights=np.abs(g[valid]).astype(np.float64), minlength=P)
    vm = np.asarray(inp["cam"]["viewmatrix"], np.float64).reshape(4, 4)
    p = np.asarray(inp["g"]["means3D"], np.float64)
    ph = np.concatenate([p, np.ones((P, 1))], 1)
    # the view-space z of the layout: the depth the projection stores
    _, _, outs, _ = _forward(inp, False, aa)
    rgbd = _state(inp, outs[0])["rgbd"]
    vis = np.unique(ids[valid])
    assert np.allclose((ph @ vm[:, 2])[vis], rgbd[vis, 3], rtol=1e-5, atol=1e-6)
    exp = G[:, None] * vm[:3, 2][None, :]
    d3 = grads[4]
    assert np.all(np.abs(d3 - exp) <= 2e-5 * Gabs[:, None] * np.abs(vm[:3, 2])[None, :] + 1e-7)
    assert np.abs(exp).max() > 0
    # m2d colours feature opacity - cov3D sh scales rotations
    for i in (0, 1, 2, 3, 6, 7, 8):
        if grads[i] is not None:
            assert not grads[i].any(), i
    v64 = torch.tensor(vm, dtype=torch.float64, requires_grad=True)
    z = (torch.from_numpy(ph) @ v64)[:, 2]
    (torch.from_numpy(G) * z).sum().backward()
    ref = v64.grad.numpy()
    scale = (Gabs[:, None] * np.abs(ph)).sum(0).max()
    assert np.abs(cam[0].reshape(4, 4) - ref).max() <= 1e-5 * scale
    # together with a colour cotangent: the sum of the two runs
    _, _, both, cam_b = _median_grads(inp, aa, True)
    from manigaussian_b200 import rasterizer as R
    s, args, outs, streams = _forward(inp, False, aa)
    gf = [torch.zeros((F, inp["H"], inp["W"]), device="cuda")] if F else None
    col = R.rasterize_views_backward_raw([s], outs, streams, [_t(inp["ct"]["dL_dcolor"])], gf, args[0], None, args[2], args[4], args[5],
                                         1.0, None, args[8], args[9], F > 0, antialiasing=aa, camera_grads=True)
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(both, col[:9])):
        if x is not None:
            y = y.cpu().numpy()
            ref = y + (grads[i] if grads[i] is not None else 0)
            assert util.rel_l2(x, ref) < 1e-5, i
    assert util.rel_l2(cam_b[0], col[9][0].cpu().numpy() + cam[0]) < 1e-5


# --------------------------------------------------------------------------- public paths
def _cams(V, W, H):
    """V cameras on a circle around the scene, looking at its centre (a CameraBatch)"""
    import importlib.util
    import os
    from manigaussian_b200 import cameras
    spec = importlib.util.spec_from_file_location("mk", os.path.join(os.path.dirname(__file__), "golden", "make_camera_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    f = W / (2 * np.tan(np.deg2rad(20)))
    intr = np.tile(np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], np.float32), (V, 1, 1))
    extr = np.stack([mk.look_at([0.2 + 1.6 * np.cos(2 * np.pi * v / V), 1.6 * np.sin(2 * np.pi * v / V), 1.5], [0.2, 0, 1.1])
                     for v in range(V)]).astype(np.float32)
    return cameras.build_cameras(intr, extr, W, H, device="cuda")


def _leaves(P, F, seed):
    from manigaussian_b200 import scenes
    g = scenes.make_gaussians(P, F=F, sh_degree=1, seed=seed)
    return {k: _t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs", "feature")}


def _check_backward(L, med, ct):
    import torch
    for v in L.values():
        v.grad = None
    (med * ct).sum().backward()
    assert L["means3D"].grad.abs().max() > 0
    for k in ("opacities", "rotations", "scales", "shs", "feature"):
        assert L[k].grad is None or not L[k].grad.any(), k
    return L["means3D"].grad.clone()


def test_public_paths_return_and_differentiate_the_planes():
    import torch
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import render, render_clouds, render_views
    P, F, W, H, V = 6000, 32, 72, 56, 2
    L = _leaves(P, F, 5)
    cams = _cams(V, W, H)
    ct = torch.randn(V, H, W, device="cuda")
    kw = dict(features_color=L["shs"], features_language=L["feature"])
    o = render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], **kw, return_median_depth=True,
                     return_depth=True, return_alpha=True)
    assert o["median_depth"].shape == (V, H, W) and o["median_id"].dtype == torch.int32 and not o["median_id"].requires_grad
    assert (o["median_id"] >= 0).any() and (o["median_id"] < P).all()
    cover = o["median_id"] >= 0
    assert torch.equal(o["alpha"][~cover], torch.zeros_like(o["alpha"][~cover]))
    g_views = _check_backward(L, o["median_depth"], ct)
    # view by view through render() and GaussianRasterizer: the same planes, and gradients that sum to the multi-view one
    data = {"novel_view": cams.as_novel_view()}
    gsum = torch.zeros_like(g_views)
    for v in range(V):
        r = render(data, v, L["means3D"], L["rotations"], L["scales"], L["opacities"], [0, 0, 0], **kw, return_median_depth=True,
                   return_alpha=True)
        assert torch.equal(r["median_id"], o["median_id"][v]) and torch.equal(r["median_depth"], o["median_depth"][v].detach())
        assert torch.equal(r["alpha"], o["alpha"][v].detach())
        gsum += _check_backward(L, r["median_depth"], ct[v])
        rast = GaussianRasterizer(cams.settings(v, torch.zeros(3, device="cuda"), 1, True), return_median_depth=True)
        out = rast(means3D=L["means3D"], means2D=torch.zeros_like(L["means3D"]), opacities=L["opacities"], shs=L["shs"],
                   language_feature_precomp=L["feature"], scales=L["scales"], rotations=L["rotations"])
        assert len(out) == 5 and torch.equal(out[4], o["median_id"][v]) and torch.equal(out[3], o["median_depth"][v].detach())
    assert util.rel_l2(gsum.cpu().numpy(), g_views.cpu().numpy()) < 1e-5
    # both frames of the dyna step: each cloud's planes are its own render_views planes
    L2 = {k: v for k, v in L.items()}
    L2["means3D"] = (L["means3D"].detach() + 0.01).requires_grad_(True)
    clouds = [dict(cameras=cams, pts_xyz=X["means3D"], rotations=X["rotations"], scales=X["scales"], opacity=X["opacities"],
                   features_color=X["shs"], features_language=X["feature"]) for X in (L, L2)]
    oc = render_clouds(clouds, return_median_depth=True)
    o2 = render_views(cams, L2["means3D"], L2["rotations"], L2["scales"], L2["opacities"], features_color=L2["shs"],
                      features_language=L2["feature"], return_median_depth=True)
    assert torch.equal(oc[0]["median_id"], o["median_id"]) and torch.equal(oc[1]["median_id"], o2["median_id"])
    assert torch.equal(oc[1]["median_depth"], o2["median_depth"])
    for v in list(L.values()) + [L2["means3D"]]:
        v.grad = None
    ((oc[0]["median_depth"] * ct).sum() + (oc[1]["median_depth"] * ct).sum()).backward()
    assert util.rel_l2(L["means3D"].grad.cpu().numpy(), g_views.cpu().numpy()) < 1e-5
    assert L2["means3D"].grad.abs().max() > 0 and not L["opacities"].grad.any()
    # targets are not combined with the median planes
    tgt = {"rgb": torch.zeros(V, 3, H, W, device="cuda")}
    with pytest.raises(ValueError):
        render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], **kw, targets=tgt, return_median_depth=True)
    with pytest.raises(ValueError):
        render_clouds([dict(clouds[0], targets=tgt)], return_median_depth=True)


def test_cuda_graph_replays_the_median_step():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, F, W, H, V = 12000, 32, 80, 64, 3
    L = _leaves(P, F, 84)
    cams = _cams(V, W, H)
    cts = (torch.randn(V, 3, H, W, device="cuda"), torch.randn(V, F, H, W, device="cuda"), torch.randn(V, H, W, device="cuda"))
    keep = {}

    def fwd_bwd():
        o = render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L["feature"], return_median_depth=True)
        loss = (o["render"] * cts[0]).sum() + (o["render_embed"] * cts[1]).sum() + (o["median_depth"] * cts[2]).sum()
        loss.backward()
        keep["med"], keep["id"] = o["median_depth"].detach(), o["median_id"]
        return loss

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for v in L.values():
                v.grad = None
            fwd_bwd()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eager = {k: v.grad.clone() for k, v in L.items()}
    eager_med, eager_id = keep["med"].clone(), keep["id"].clone()
    for v in L.values():
        v.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fwd_bwd()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(keep["med"], eager_med) and torch.equal(keep["id"], eager_id)
    for k in L:
        assert util.rel_l2(L[k].grad.cpu().numpy(), eager[k].cpu().numpy()) < 1e-5, k
