"""The anti-aliased projection on the GPU: mode off is the existing path, mode on leaves every piece of projection geometry
bit for bit as it was and changes the opacity the blend sees only, the kernels match the anti-aliased oracle
(tests/aa_oracle.py: the C oracle with a float64 compensation) stage by stage, block culling stays sound where the
compensation is strongest, and every public path agrees with every other."""
import numpy as np
import pytest

import aa_oracle as AA
import blend_ref64 as R64
import util
from test_clouds_gpu import _leaves, _mk
from test_render_gpu import _cams, _cloud, _t

pytestmark = pytest.mark.gpu

GRAD_NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dfeature", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
              "dL_drotations")


def _arr(which, name, state, a0, a1, dtype, count):
    import torch
    from manigaussian_b200 import rasterizer as R
    off = R.state_array(which, name, state, a0, a1) - state.data_ptr()
    nbytes = count * torch.empty((), dtype=dtype).element_size()
    return state[off:off + nbytes].view(dtype).cpu().numpy()


def _run(inp, aa, scale_modifier=1.0, prefiltered=False, capacity=None, backward=True):
    """One view through rasterize_views_raw / rasterize_views_backward_raw; returns the images, the projection and binning
    state and the nine gradients as numpy."""
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings as S
    from manigaussian_b200 import rasterizer as R
    cam, g, ct = inp["cam"], inp["g"], inp["ct"]
    P, W, H, F = inp["P"], inp["W"], inp["H"], inp["F"]
    t = util._t
    view = S(H, W, cam["tanfovx"], cam["tanfovy"], t(inp["bg"]), scale_modifier, t(cam["viewmatrix"]), t(cam["projmatrix"]),
             g["sh_degree"], t(cam["campos"]), prefiltered, False, F > 0)
    args = (t(g["means3D"]), t(g["colors_precomp"]), t(g["feature"]) if F else None, t(g["opacities"]), t(g["scales"]), t(g["rotations"]),
            scale_modifier, t(g["cov3D_precomp"]), t(g["shs"]), g["sh_degree"], F > 0)
    if not capacity:
        R.reset_capacity_estimates()  # cases share (P, W, H) but not their instance counts (scale_modifier)
    outs, sts = R.rasterize_views_raw([view], *args, antialiasing=aa, capacities=[capacity] if capacity else None)
    o = outs[0]
    Rn = o.num_rendered()
    assert not o.overflowed()
    cap = int(o[0])
    T = ((W + 15) // 16) * ((H + 15) // 16)
    k = dict(R=Rn, cap=cap, color=o[1].cpu().numpy(), feature=o[2].cpu().numpy() if F else None, radii=o[3].cpu().numpy(), W=W, H=H)
    geomB, binB, imgB = o[4], o[5], o[6]
    for name, dt, cnt in (("depths", torch.float32, P), ("means2D", torch.float32, 2 * P), ("conic_opacity", torch.float32, 4 * P),
                          ("tiles_touched", torch.int32, P), ("extent", torch.float32, 2 * P), ("depth_order", torch.int32, P)):
        k[name] = _arr("geometry", name, geomB, P, 0, dt, cnt)
    k["means2D"] = k["means2D"].reshape(P, 2)
    k["conic_opacity"] = k["conic_opacity"].reshape(P, 4)
    for name, dt in (("point_list", torch.int32), ("tile_ids", torch.int32), ("block_bits", torch.uint8)):
        k[name] = _arr("binning", name, binB, cap, 0, dt, Rn)
    k["ranges"] = _arr("image", "ranges", imgB, W, H, torch.int32, 2 * T).reshape(T, 2)
    k["final_T"] = _arr("image", "final_T", imgB, W, H, torch.float32, W * H)
    if backward:
        gc = [t(ct["dL_dcolor"])]
        gf = [t(ct["dL_dfeature"])] if F else None
        m3, col, feat, op, sc, rot, smod, cov, sh, deg, inc = args
        grads = R.rasterize_views_backward_raw([view], outs, sts, gc, gf, m3, col, feat, sc, rot, smod, cov, sh, deg, inc, antialiasing=aa)
        torch.cuda.synchronize()
        k.update({n: (v.cpu().numpy() if v is not None else None) for n, v in zip(GRAD_NAMES, grads)})
    return k


def test_mode_off_through_the_aa_calls_is_the_existing_path(monkeypatch):
    """The _aa calls with 0 in place of mgs_forward_views / mgs_backward_views: images, radii and instance counts bit for bit,
    gradients within the run-to-run spread of the blend's float atomics."""
    from manigaussian_b200 import _binding
    inp = util.make_inputs(P=20000, W=128, H=96, F=32, seed=31, bg=(0.2, 0.3, 0.4))
    a = _run(inp, False)
    a2 = _run(inp, False, capacity=a["cap"])
    L = _binding.lib()
    monkeypatch.setattr(L, "mgs_forward_views", lambda V, arr, *rest: L.mgs_forward_views_aa(V, arr, None, None, 0, *rest), raising=False)
    monkeypatch.setattr(L, "mgs_backward_views", lambda V, arr, *rest: L.mgs_backward_views_aa(V, arr, None, None, 0, *rest), raising=False)
    b = _run(inp, False, capacity=a["cap"])
    for key in ("color", "feature", "radii", "R", "point_list", "final_T"):
        assert np.array_equal(a[key], b[key]), key
    # the projection writes conic_opacity for the Gaussians it keeps; a culled row is never read and holds whatever the
    # geometry buffer held before (the caching allocator's previous contents), so only kept rows are defined
    vis = a["radii"] > 0
    assert np.array_equal(a["conic_opacity"][vis], b["conic_opacity"][vis]), "conic_opacity"
    for key in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dsh", "dL_dscales", "dL_drotations", "dL_dfeature"):
        spread = util.rel_l2(a2[key], a[key])
        assert util.rel_l2(b[key], a[key]) <= max(4 * spread, 1e-6), key


@pytest.mark.parametrize("name", ["mg_real_f3", "subpixel"])
def test_mode_on_leaves_the_projection_geometry_alone(name):
    """Against mode off on the same inputs, bit for bit: radii, means2D, depths, conic xyz, tiles_touched, the instance count,
    the depth order, point_list, tile keys and ranges.  Each instance's block bits are a subset of its bits with the mode off
    (the compensated opacity shrinks the alpha >= 1/255 footprint), and conic_opacity.w only ever decreases."""
    kw = dict(P=16384, W=128, H=128, F=3, seed=2) if name == "mg_real_f3" else dict(P=20000, W=128, H=128, F=0, seed=32, scale0=0.003)
    inp = util.make_inputs(**kw)
    off = _run(inp, False, backward=False)
    on = _run(inp, True, capacity=off["cap"], backward=False)
    for key in ("radii", "depths", "tiles_touched", "R", "depth_order", "point_list", "tile_ids", "ranges"):
        assert np.array_equal(off[key], on[key]), key
    vis = off["radii"] > 0   # means2D and conic_opacity are written for the kept Gaussians only
    assert np.array_equal(off["means2D"][vis], on["means2D"][vis])
    assert np.array_equal(off["conic_opacity"][vis, :3], on["conic_opacity"][vis, :3])
    assert np.all(on["conic_opacity"][vis, 3] <= off["conic_opacity"][vis, 3])
    assert np.all((on["block_bits"] & ~off["block_bits"]) == 0)
    assert (on["block_bits"] != off["block_bits"]).any()  # the footprints do shrink
    assert not np.array_equal(on["color"], off["color"])


def _oracle_aa(inp, scale_modifier=1.0):
    g, cam, ct = inp["g"], inp["cam"], inp["ct"]
    kw = dict(scales=g["scales"], rotations=g["rotations"], cov3D_precomp=g["cov3D_precomp"], shs=g["shs"], sh_degree=g["sh_degree"],
              colors_precomp=g["colors_precomp"], feature=g["feature"], scale_modifier=scale_modifier, antialiasing=True)
    fw = AA.forward(g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], inp["W"], inp["H"], cam["tanfovx"],
                   cam["tanfovy"], inp["bg"], **kw)
    bw = AA.backward(fw, ct["dL_dcolor"], ct["dL_dfeature"], g["means3D"], cam["viewmatrix"], cam["projmatrix"], cam["campos"],
                    cam["tanfovx"], cam["tanfovy"], inp["bg"], **kw)
    return fw, bw


PARITY = {
    "f0_sh0": (dict(P=3000, W=64, H=64, F=0, seed=41, sh_degree=0), {}),
    "f3_sh1": (dict(P=16384, W=128, H=128, F=3, seed=42), {}),
    "f32_sh2": (dict(P=5000, W=200, H=120, F=32, seed=43, sh_degree=2, bg=(0.3, 0.6, 0.9)), {}),
    "f40_sh3": (dict(P=4000, W=96, H=80, F=40, seed=44, sh_degree=3), {}),
    "f67_sh1": (dict(P=3000, W=80, H=64, F=67, seed=45), {}),
    "rgb_precomp_cov": (dict(P=4000, W=96, H=96, F=0, seed=46, precomp_colors=True, precomp_cov=True), {}),
    "smod_0.7": (dict(P=5000, W=96, H=96, F=3, seed=47), dict(scale_modifier=0.7)),
    "smod_1.9_prefiltered": (dict(P=5000, W=96, H=96, F=3, seed=48), dict(scale_modifier=1.9, prefiltered=True)),
    "subpixel_f3": (dict(P=20000, W=128, H=128, F=3, seed=49, scale0=0.003), {}),
}


@pytest.mark.parametrize("name", list(PARITY))
def test_aa_parity_with_the_oracle(name):
    """Stage by stage against the oracle's anti-aliased mode at the bars of test_parity_gpu: projection <= 1e-5, images
    <= 3e-4, gradients <= 1e-3 (relative L2).  conic_opacity.w per Gaussian within 2e-6 (1 + kappa0 + kappa1): d0 cancels
    by kappa0 = (a0 c0 + b^2) / d0 and the two sides round the 2D covariance differently (nvcc contracts FMAs)."""
    kw, opt = PARITY[name]
    inp = util.make_inputs(**kw)
    smod = opt.get("scale_modifier", 1.0)
    k = _run(inp, True, scale_modifier=smod, prefiltered=opt.get("prefiltered", False))
    fw, bw = _oracle_aa(inp, smod)
    vis = (fw["radii"] > 0) & (k["radii"] > 0)
    assert np.mean(fw["radii"] == k["radii"]) > 0.999
    assert util.rel_l2(k["means2D"][vis], fw["means2D"][vis]) <= 1e-5
    assert util.rel_l2(k["depths"][vis], fw["depths"][vis]) <= 1e-5
    assert util.rel_l2(k["conic_opacity"][vis, :3], fw["conic_opacity"][vis, :3]) <= 1e-5
    co = fw["conic_opacity"][vis].astype(np.float64)
    det1 = 1.0 / (co[:, 0] * co[:, 2] - co[:, 1] ** 2)  # the dilated covariance from the conic
    a, b, c = co[:, 2] * det1, -co[:, 1] * det1, co[:, 0] * det1
    a0, c0 = a - 0.3, c - 0.3
    d0 = np.maximum(np.abs(a0 * c0 - b * b), 1e-30)
    k0, k1 = (np.abs(a0 * c0) + b * b) / d0, (a * c + b * b) / (a * c - b * b)
    ow, gw = k["conic_opacity"][vis, 3].astype(np.float64), co[:, 3]
    rel = np.abs(ow - gw) / np.maximum(gw, 1e-30)
    assert np.all(rel <= 2e-6 * (1.0 + k0 + k1) + 1e-6), float((rel / (2e-6 * (1 + k0 + k1) + 1e-6)).max())
    assert util.rel_l2(k["color"], fw["out_color"]) <= 3e-4
    if inp["F"]:
        assert util.rel_l2(k["feature"], fw["out_feature"]) <= 3e-4
    g = inp["g"]
    for key in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dsh", "dL_dscales", "dL_drotations", "dL_dfeature", "dL_dcolors",
                "dL_dcov3D"):
        if k.get(key) is None or (key == "dL_dfeature" and not inp["F"]) or (key == "dL_dsh" and g["shs"] is None):
            continue
        if key in ("dL_dscales", "dL_drotations") and g["scales"] is None:
            continue
        if key == "dL_dcolors" and g["colors_precomp"] is None:
            continue
        if key == "dL_dcov3D" and g["cov3D_precomp"] is None:
            continue
        err = util.rel_l2(k[key].reshape(bw[key].shape), bw[key])
        assert err <= 1e-3, (key, err)


def test_culling_stays_sound_on_subpixel_gaussians():
    """Sub-pixel splats (s down to ~0.1): no pair with alpha >= 1/255 in float64 (tests/blend_ref64.decide, outside the fp32
    band) is missing from its block list."""
    inp = util.make_inputs(P=30000, W=160, H=128, F=0, seed=51, scale0=0.002)
    k = _run(inp, True, backward=False)
    st = dict(W=k["W"], H=k["H"], ranges=k["ranges"].view(np.uint32), point_list=k["point_list"].view(np.uint32), means2D=k["means2D"],
              conic_opacity=k["conic_opacity"])
    vis = k["radii"] > 0
    s_min = float((k["conic_opacity"][vis, 3] / inp["g"]["opacities"].reshape(-1)[vis]).min())
    assert s_min < 0.3
    bad, pairs = 0, 0
    lx, ly = np.arange(256) % 16, np.arange(256) // 16
    blk, _ = R64.pixel_block_bit(lx, ly)
    for t in range(k["ranges"].shape[0]):
        r0, r1 = (int(v) for v in k["ranges"][t])
        if r1 == r0:
            continue
        d = R64.decide(st, t)
        bits = k["block_bits"][r0:r1].astype(np.int64)
        listed = ((bits[None, :] >> blk[:, None]) & 1).astype(bool)
        bad += int((d["foot_in"] & ~listed).sum())
        pairs += int(d["foot_in"].sum())
    assert pairs > 10000 and bad == 0, (bad, pairs)


# ------------------------------------------------------------------------------------------------------------ public paths
def _data(cams):
    return {"novel_view": cams.as_novel_view()}


def test_public_paths_agree():
    """GaussianRasterizer(antialiasing=True), also with debug=True, == render == render_views (one view); render_views (V = 4)
    == a loop of render; render_clouds == render_views per cloud; return_alpha with the mode on.  Images bit for bit,
    gradients within the spread of the atomics' order."""
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings as S
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import normalize_features, render, render_clouds, render_views
    P, F, W, H, V = 7000, 32, 72, 56, 4
    cams = _cams(V, W, H)
    host = _leaves(P, F, 91, "sh")
    cts = [(torch.randn(3, H, W, device="cuda"), torch.randn(F, H, W, device="cuda"), torch.randn(H, W, device="cuda")) for _ in range(V)]

    def obj(img, emb, alpha, v):
        return (img * cts[v][0]).sum() + (emb * cts[v][1]).sum() + (alpha * cts[v][2]).sum()

    A = _mk(host)
    ov = render_views(cams, A["xyz"], A["rot"], A["scale"], A["opac"], (0.1, 0.2, 0.3), features_color=A["col"], features_language=A["feat"],
                      return_alpha=True, antialiasing=True)
    sum(obj(ov["render"][v], ov["render_embed"][v], ov["alpha"][v], v) for v in range(V)).backward()
    plain = render_views(cams, A["xyz"], A["rot"], A["scale"], A["opac"], (0.1, 0.2, 0.3), features_color=A["col"],
                         features_language=A["feat"], return_alpha=True)
    # lower opacities leave more transmittance (per pixel only up to the T < 1e-4 stop, which the plain render can reach a
    # strong splat earlier)
    assert not torch.equal(plain["render"], ov["render"]) and float(ov["alpha"].mean()) < float(plain["alpha"].mean())
    B = _mk(host)
    data = _data(cams)
    for v in range(V):
        o = render(data, v, B["xyz"], B["rot"], B["scale"], B["opac"], [0.1, 0.2, 0.3], features_color=B["col"], features_language=B["feat"],
                   return_alpha=True, antialiasing=True)
        assert torch.equal(o["render"], ov["render"][v]) and torch.equal(o["alpha"], ov["alpha"][v]), v
        obj(o["render"], o["render_embed"], o["alpha"], v).backward()
    for k in A:
        assert util.rel_l2(A[k].grad.cpu().numpy(), B[k].grad.cpu().numpy()) < 1e-6, k

    for debug in (False, True):
        C = _mk(host)
        s0 = cams.settings(1, torch.tensor([0.1, 0.2, 0.3], device="cuda"), 1, True, debug=debug)
        s = S(*s0, antialiasing=True)
        m2 = torch.zeros_like(C["xyz"], requires_grad=True)
        img, emb, radii, alpha = GaussianRasterizer(s, return_alpha=True)(
            means3D=C["xyz"], means2D=m2, opacities=C["opac"], shs=C["col"], language_feature_precomp=normalize_features(C["feat"]),
            scales=C["scale"], rotations=C["rot"])
        assert torch.equal(img, ov["render"][1]) and torch.equal(alpha, ov["alpha"][1]), debug
        obj(img, emb, alpha, 1).backward()
        D = _mk(host)
        o = render_views(cams, D["xyz"], D["rot"], D["scale"], D["opac"], (0.1, 0.2, 0.3), features_color=D["col"],
                         features_language=D["feat"], view_ids=[1], return_alpha=True, antialiasing=True)
        obj(o["render"][0], o["render_embed"][0], o["alpha"][0], 1).backward()
        for k in C:
            assert util.rel_l2(C[k].grad.cpu().numpy(), D[k].grad.cpu().numpy()) < 1e-6, (debug, k)
        assert util.rel_l2(m2.grad.cpu().numpy(), o["viewspace_points"].grad[0].cpu().numpy()) < 1e-6, debug
        # without return_alpha, the module still takes the anti-aliased path
        E = _mk(host)
        img2, _, _ = GaussianRasterizer(s)(means3D=E["xyz"], means2D=torch.zeros_like(E["xyz"]), opacities=E["opac"], shs=E["col"],
                                          language_feature_precomp=normalize_features(E["feat"]), scales=E["scale"], rotations=E["rot"])
        assert torch.equal(img2, ov["render"][1]), debug

    spec = [(P, cams, host), (3000, _cams(2, 48, 40), _leaves(3000, F, 92, "sh"))]
    cts2 = [torch.randn(len(c), c.height, c.width, device="cuda") for _, c, _ in spec]
    E = [_mk(hh) for _, _, hh in spec]
    oc = render_clouds([dict(cameras=c, pts_xyz=L["xyz"], rotations=L["rot"], scales=L["scale"], opacity=L["opac"], features_color=L["col"],
                             features_language=L["feat"]) for L, (_, c, _) in zip(E, spec)], bg_color=(0.1, 0.2, 0.3), return_alpha=True,
                       return_depth=True, antialiasing=True)
    sum((o["alpha"] * t).sum() + o["render"].sum() + o["depth"].sum() for o, t in zip(oc, cts2)).backward()
    for b, (_, c, hh) in enumerate(spec):
        G = _mk(hh)
        r = render_views(c, G["xyz"], G["rot"], G["scale"], G["opac"], (0.1, 0.2, 0.3), features_color=G["col"], features_language=G["feat"],
                         return_alpha=True, return_depth=True, antialiasing=True)
        ((r["alpha"] * cts2[b]).sum() + r["render"].sum() + r["depth"].sum()).backward()
        assert torch.equal(oc[b]["render"], r["render"]) and torch.equal(oc[b]["alpha"], r["alpha"]), b
        for k in G:
            assert util.rel_l2(E[b][k].grad.cpu().numpy(), G[k].grad.cpu().numpy()) < 1e-6, (b, k)


def test_fused_heads_equal_the_unfused_recipe_on_aa_planes():
    """targets (rgb, embed, depth, mask) with the mode on: the fused losses and gradients == INTEGRATION.md §4's recipe
    (test_depth_heads_gpu._recipe) on the anti-aliased planes of render_views(return_depth, return_alpha)."""
    import torch
    import torch.nn.functional as Fn
    from test_depth_heads_gpu import _recipe
    from manigaussian_b200.gaussian_renderer import render_views
    P, F, W, H, V = 8000, 16, 64, 48, 2
    cams = _cams(V, W, H)
    host = _leaves(P, F, 93, "sh")
    tg = {"rgb": torch.rand(V, 3, H, W, device="cuda"), "embed": Fn.normalize(torch.randn(V, F, H, W, device="cuda"), dim=1),
          "depth": torch.where(torch.rand(V, H, W, device="cuda") > 0.3, torch.full((V, H, W), 1.6, device="cuda"), torch.zeros(V, H, W, device="cuda")),
          "mask": (torch.rand(V, H, W, device="cuda") > 0.5).float()}
    A = _mk(host)
    o = render_views(cams, A["xyz"], A["rot"], A["scale"], A["opac"], features_color=A["col"], features_language=A["feat"], targets=tg,
                     antialiasing=True)
    (o["loss_rgb"].sum() + o["loss_embed"].sum() + o["loss_depth"].sum() + o["loss_mask"].sum()).backward()
    B = _mk(host)
    r = render_views(cams, B["xyz"], B["rot"], B["scale"], B["opac"], features_color=B["col"], features_language=B["feat"], return_depth=True,
                     return_alpha=True, antialiasing=True)
    assert torch.equal(o["render"], r["render"].detach())
    ref = _recipe(r, tg)
    for key in ("loss_rgb", "loss_embed", "loss_depth", "loss_mask"):
        assert util.rel_l2(o[key].detach().cpu().numpy(), ref[key].detach().cpu().numpy()) < 1e-4, key
    sum(ref[key].sum() for key in ("loss_rgb", "loss_embed", "loss_depth", "loss_mask")).backward()
    for k in A:
        assert util.rel_l2(A[k].grad.cpu().numpy(), B[k].grad.cpu().numpy()) < 2e-4, k


def test_dyna_step_with_the_mode_on():
    """Both frames of the dyna step in one render_clouds call, mode on: the deformation offsets (delta mu, delta r) receive
    finite, non-zero gradients."""
    import torch
    from manigaussian_b200.gaussian_params import activate_gaussians
    from manigaussian_b200.gaussian_renderer import render_clouds
    P, F, W, H = 6000, 32, 64, 64
    cams = _cams(2, W, H)
    g = _cloud(P, F, 94)
    rng = np.random.default_rng(5)
    mk = lambda v, grad=True: _t(np.asarray(v, np.float32)).requires_grad_(grad)
    xyz, d_xyz = mk(g["means3D"], False), mk(rng.normal(0, 0.01, (P, 3)))
    rot, scale = mk(g["rotations"]), mk(np.log(g["scales"]))
    opac, feat = mk(np.log(g["opacities"] / (1 - g["opacities"]))), mk(g["feature"])
    d_mu, d_r = mk(rng.normal(0, 0.01, (P, 3))), mk(rng.normal(0, 0.05, (P, 4)))
    sh = mk(g["shs"])
    cur = activate_gaussians(xyz, rot, scale, opac, feat, d_means=d_xyz, normalize_feature=False)
    nxt = activate_gaussians(cur[0].detach(), cur[1].detach(), cur[2].detach(), cur[3].detach(), None, d_means=d_mu, d_rotations=d_r,
                             scale_activation=None, opacity_activation=None)
    oc = render_clouds([dict(cameras=cams, pts_xyz=cur[0], rotations=cur[1], scales=cur[2], opacity=cur[3], features_color=sh,
                             features_language=cur[4]),
                        dict(cameras=cams, pts_xyz=nxt[0], rotations=nxt[1], scales=nxt[2], opacity=nxt[3], features_color=sh.detach(),
                             features_language=cur[4].detach())], antialiasing=True)
    (oc[0]["render"].square().mean() + oc[1]["render"].square().mean() + oc[0]["render_embed"].square().mean()).backward()
    for name, t in (("delta_mu", d_mu), ("delta_r", d_r), ("scale", scale), ("opacity", opac)):
        assert t.grad is not None and torch.isfinite(t.grad).all() and t.grad.abs().sum() > 0, name


def test_cuda_graph_capture_with_the_mode_on():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, F, W, H, V = 12000, 32, 80, 64, 3
    g = _cloud(P, F, 95)
    cams = _cams(V, W, H)
    names = ("means3D", "rotations", "scales", "opacities", "shs", "feature")
    L = {k: _t(np.asarray(g[k], np.float32)).requires_grad_(True) for k in names}
    cts = (torch.randn(V, 3, H, W, device="cuda"), torch.randn(V, F, H, W, device="cuda"))
    keep = {}

    def fwd_bwd():
        o = render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L["feature"], antialiasing=True)
        loss = (o["render"] * cts[0]).sum() + (o["render_embed"] * cts[1]).sum()
        loss.backward()
        keep["img"] = o["render"].detach()
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
    eager_img = keep["img"].clone()
    for v in L.values():
        v.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fwd_bwd()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(keep["img"], eager_img)
    for k in names:
        assert util.rel_l2(L[k].grad.cpu().numpy(), eager[k].cpu().numpy()) < 1e-5, k


@pytest.mark.parametrize("path", ["module", "render_views", "render_clouds"])
def test_steps_with_the_mode_on_do_not_accumulate_device_memory(path):
    import gc
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings as S
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    P, F, W, H, V = 6000, 32, 64, 48, 2
    g = _cloud(P, F, 96)
    cams = _cams(V, W, H)
    host = {k: np.asarray(g[k], np.float32) for k in ("means3D", "rotations", "scales", "opacities", "shs", "feature")}

    def step():
        L = {k: _t(v).requires_grad_(True) for k, v in host.items()}
        if path == "module":
            s = S(*cams.settings(0, torch.zeros(3, device="cuda"), 1, True), antialiasing=True)
            img, _, _ = GaussianRasterizer(s)(means3D=L["means3D"], means2D=torch.zeros_like(L["means3D"]), opacities=L["opacities"],
                                               shs=L["shs"], language_feature_precomp=L["feature"], scales=L["scales"], rotations=L["rotations"])
            loss = img.sum()
        else:
            kw = dict(pts_xyz=L["means3D"], rotations=L["rotations"], scales=L["scales"], opacity=L["opacities"], features_color=L["shs"],
                      features_language=L["feature"])
            o = render_views(cams, antialiasing=True, **kw) if path == "render_views" else \
                render_clouds([dict(cameras=cams, **kw)], antialiasing=True)[0]
            loss = o["render"].sum()
        loss.backward()
        return float(loss)

    gc.disable()
    try:
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        for _ in range(4):
            step()
        torch.cuda.synchronize()
        grown = torch.cuda.memory_allocated() - base
    finally:
        gc.enable()
    assert grown == 0, f"{grown} bytes stayed allocated after 4 more steps"
