"""The surface-normal plane on the GPU (include/mgs_rasterizer.h, mgs_view_normal).

* Per-Gaussian quad: `nrm` read back from the geometry state equals the float64 reference (tests/normal_ref64.py) to 1e-6 for
  every Gaussian of every view, the sign being free only where |a . (campos - mean)| is within the fp32 bound of 0.
* Blend, against the existing feature path as oracle: the same cloud rendered once with return_normal and once per view with
  that view's quads appended as three feature channels.  The planes agree, the gradients of opacities, means3D, scales, SHs
  and features agree under random cotangents on every plane at once, and dL_drot differs from the oracle's by exactly the
  float64 chain applied to the oracle's dL_dfeature of those three channels (which is the blend stage's dL/dn).
* Nothing else moves with normals on; colour-only plus normal-only cotangents sum; accumulate adds.
* Contract errors, the four public paths, CUDA-graph replay, no memory growth.
"""
import numpy as np
import pytest

import util
import normal_ref64 as N

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh_capacities():
    # the binning capacity is learnt per (cloud size, image size): what another test learnt from a different cloud of the
    # same size (an empty one, say) must not size these renders
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def _t(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def _inputs(P, W, H, F, V, seed=5, culled=False):
    inps = [util.make_inputs(P=P, W=W, H=H, F=F, seed=seed, view=v, num_views=max(V, 4), bg=(0.3, 0.6, 0.9)) for v in range(V)]
    g = inps[0]["g"]
    if culled:  # every Gaussian at the first camera's centre, in front of the near plane: empty tile lists
        g["means3D"] = np.tile(np.asarray(inps[0]["cam"]["campos"], np.float32).reshape(1, 3), (P, 1))
    return inps, g


def _settings(inp, F):
    from manigaussian_b200 import rasterizer as R
    cam = inp["cam"]
    return R.GaussianRasterizationSettings(inp["H"], inp["W"], cam["tanfovx"], cam["tanfovy"], _t(inp["bg"]), 1.0, _t(cam["viewmatrix"]),
                                           _t(cam["projmatrix"]), inp["g"]["sh_degree"], _t(cam["campos"]), False, False, F > 0)


def _cloud_args(g, feature):
    return (_t(g["means3D"]), None, feature, _t(g["opacities"]), _t(g["scales"]), _t(g["rotations"]), 1.0, None, _t(g["shs"]),
            g["sh_degree"], feature is not None)


def _nrm(o, P):
    import torch
    from manigaussian_b200 import rasterizer as R
    torch.cuda.synchronize()
    geom = o[4]
    off = R.state_array("geometry", "nrm", geom, P) - geom.data_ptr()
    return geom[off:off + 16 * P].view(torch.float32).reshape(P, 4).clone()


def _cots(V, F, H, W, seed=11):
    rng = np.random.default_rng(seed)
    mk = lambda *s: _t(rng.standard_normal(s))  # noqa: E731
    return dict(color=mk(V, 3, H, W), feature=mk(V, F, H, W) if F else None, depth=mk(V, H, W), alpha=mk(V, H, W), normal=mk(V, 3, H, W))


def _run(inps, g, F, aa=False, normal=True, ct=None, normal_ct=True, color_ct=True, accumulate_into=None):
    """forward of all views in one call (+ backward with the cotangents ct): (outs, grads)"""
    import torch
    from manigaussian_b200 import rasterizer as R
    views = [_settings(i, F) for i in inps]
    args = _cloud_args(g, _t(g["feature"]) if F else None)
    outs, streams = R.rasterize_views_raw(views, *args, return_depth=True, return_alpha=True, antialiasing=aa, return_normal=normal)
    assert not any(o.overflowed() for o in outs)
    if ct is None:
        return outs, None
    V = len(views)
    zero = lambda x: torch.zeros_like(x)  # noqa: E731
    grads = R.rasterize_views_backward_raw(
        views, outs, streams, ct["color"] if color_ct else zero(ct["color"]),
        (ct["feature"] if color_ct else zero(ct["feature"])) if F else None, *args[:1], None, args[2], args[4], args[5], 1.0, None,
        args[8], g["sh_degree"], F > 0, grads_depth=ct["depth"] if color_ct else None, grads_alpha=ct["alpha"] if color_ct else None,
        antialiasing=aa, grads_normal=list(ct["normal"]) if (normal and normal_ct) else None,
        normals=[o[-1] for o in outs] if (normal and normal_ct) else None,
        accumulate_into=accumulate_into, accumulate=accumulate_into is not None)
    torch.cuda.synchronize()
    return outs, grads


def _oracle(inps, g, F, nrm, aa, ct):
    """one call per view with [feature | n_v] as F + 3 channels; returns the planes, the summed gradients and dL/dn per view"""
    import torch
    from manigaussian_b200 import rasterizer as R
    planes, dn, total = [], [], None
    for v, inp in enumerate(inps):
        s = _settings(inp, F + 3)
        feat = torch.cat([_t(g["feature"]), nrm[v][:, :3]], 1).contiguous() if F else nrm[v][:, :3].contiguous()
        args = _cloud_args(g, feat)
        outs, streams = R.rasterize_views_raw([s], *args, return_depth=True, return_alpha=True, antialiasing=aa)
        gf = torch.cat([ct["feature"][v], ct["normal"][v]], 0).contiguous() if F else ct["normal"][v]
        gr = R.rasterize_views_backward_raw([s], outs, streams, [ct["color"][v]], [gf], args[0], None, feat, args[4], args[5], 1.0,
                                            None, args[8], g["sh_degree"], True, grads_depth=[ct["depth"][v]],
                                            grads_alpha=[ct["alpha"][v]], antialiasing=aa)
        torch.cuda.synchronize()
        planes.append(outs[0][2][F:F + 3].clone())
        dn.append(gr[2][:, F:F + 3].double().cpu().numpy())
        keep = dict(feature=gr[2][:, :F], opacity=gr[3], means3D=gr[4], sh=gr[6], scales=gr[7], rot=gr[8])
        total = keep if total is None else {k: total[k] + keep[k] for k in keep}
    return planes, total, dn


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    d = float((a - b).norm())
    return d / max(float(b.norm()), 1e-30)


def test_per_gaussian_quad_matches_the_float64_reference():
    P, V = 3000, 3
    inps, g = _inputs(P, 96, 64, 0, V)
    g["rotations"] = (g["rotations"] * np.geomspace(0.05, 20, P)[:, None]).astype(np.float32)  # non-unit quaternions
    g["scales"][:50, 1] = g["scales"][:50, 0]                                                    # ties
    outs, _ = _run(inps, g, 0)
    for v in range(V):
        got = _nrm(outs[v], P).cpu().numpy().astype(np.float64)
        ref, d = N.normals(g["means3D"], g["scales"], g["rotations"], inps[v]["cam"]["campos"])
        assert (got[:, 3] == 0).all()
        sure = np.abs(d) > 1e-5
        assert sure.mean() > 0.99
        assert np.abs(got[sure, :3] - ref[sure]).max() < 1e-6
        assert np.abs(np.abs(got[~sure, :3]) - np.abs(ref[~sure])).max() < 1e-6 if (~sure).any() else True
    assert (N.normals(g["means3D"], g["scales"], g["rotations"], inps[0]["cam"]["campos"])[1] < 0).any()  # the flip is exercised


CASES = [(0, 200, 120, 1, False), (3, 61, 37, 4, False), (8, 200, 120, 1, True), (32, 200, 120, 4, False), (40, 61, 37, 1, False),
         (67, 61, 37, 2, True), (3, 61, 37, 17, False)]


@pytest.mark.parametrize("F,W,H,V,aa", CASES)
def test_blend_and_gradients_against_the_feature_path(F, W, H, V, aa):
    import torch
    P = 2500
    inps, g = _inputs(P, W, H, F, V, seed=7 + F)
    g["rotations"] = (g["rotations"] * np.random.default_rng(1).uniform(0.5, 2.0, (P, 1))).astype(np.float32)
    ct = _cots(V, F, H, W)
    outs, grads = _run(inps, g, F, aa, ct=ct)
    nrm = [_nrm(o, P) for o in outs]
    planes, og, dn = _oracle(inps, g, F, nrm, aa, ct)
    for v in range(V):
        assert outs[v][-1].shape == (3, H, W)
        scale = float(planes[v].abs().max())
        assert scale > 0.1
        assert float((outs[v][-1] - planes[v]).abs().max()) <= 1e-6 * max(scale, 1.0) + 1e-7, v
    names = dict(opacity=3, means3D=4, sh=6, scales=7) | ({"feature": 2} if F else {})
    for k, i in names.items():
        assert _rel(grads[i], og[k]) < 2e-5, k
    # rotation: the oracle's own rotation gradient (through the covariance) plus the float64 chain of the oracle's dL/dn
    chain = N.rotation_grad(g["means3D"], g["scales"], g["rotations"], [i["cam"]["campos"] for i in inps], dn)
    assert np.abs(chain).max() > 0
    want = og["rot"].double().cpu().numpy() + chain
    got = grads[8].double().cpu().numpy()
    assert np.linalg.norm(got - want) / np.linalg.norm(want) < 1e-4
    assert np.linalg.norm(got - og["rot"].double().cpu().numpy() - chain) / np.linalg.norm(chain) < 1e-3
    assert torch.isfinite(grads[8]).all()


def test_fully_culled_cloud_gives_zeros():
    import torch
    inps, g = _inputs(1500, 61, 37, 3, 1, culled=True)
    ct = _cots(1, 3, 37, 61)
    outs, grads = _run(inps, g, 3, ct=ct)
    assert outs[0].num_rendered() == 0
    assert (outs[0][-1] == 0).all()
    assert torch.isfinite(grads[8]).all() and (grads[8] == 0).all()


@pytest.mark.parametrize("F,aa", [(3, False), (32, False), (40, True)])
def test_nothing_else_moves(F, aa):
    import torch
    from manigaussian_b200 import rasterizer as R
    inps, g = _inputs(4000, 200, 120, F, 2, seed=3)
    ct = _cots(2, F, 120, 200)
    res = {}
    for normal in (False, True):
        outs, grads = _run(inps, g, F, aa, normal=normal, ct=ct, normal_ct=False)
        st = []
        for o, inp in zip(outs, inps):
            img, W, H = o[6], inp["W"], inp["H"]
            fin = []
            for name in ("final_T", "n_contrib"):
                off = R.state_array("image", name, img, W, H) - img.data_ptr()
                fin.append(img[off:off + 4 * W * H].clone())
            st.append(dict(color=o[1], feature=o[2], radii=o[3], depth=o[7], alpha=o[8], final_T=fin[0], n_contrib=fin[1],
                           count=o.num_rendered()))
        res[normal] = (st, grads)
    for a, b in zip(*[res[k][0] for k in (False, True)]):
        assert a["count"] == b["count"]
        for k in ("color", "feature", "radii", "depth", "alpha", "final_T", "n_contrib"):
            assert torch.equal(a[k], b[k]), k
    for i in (2, 3, 4, 6, 7, 8):
        if F == 0 and i == 2:
            continue
        assert _rel(res[True][1][i], res[False][1][i]) < 2e-5, i


def test_cotangents_sum_and_accumulate_adds():
    import torch
    F, V = 8, 2
    inps, g = _inputs(3000, 96, 64, F, V, seed=9)
    ct = _cots(V, F, 64, 96)
    _, both = _run(inps, g, F, ct=ct)
    _, only_n = _run(inps, g, F, ct=ct, color_ct=False)
    _, only_c = _run(inps, g, F, ct=ct, normal_ct=False)
    for i in (2, 3, 4, 6, 7, 8):
        assert _rel(both[i], only_n[i] + only_c[i]) < 2e-5, i
    P = 3000
    base = dict(dL_dmeans3D=torch.randn(P, 3), dL_dmeans2D=torch.randn(P, 3), dL_dopacity=torch.randn(P, 1), dL_dscales=torch.randn(P, 3),
                dL_drotations=torch.randn(P, 4), dL_dsh=torch.randn(P, g["shs"].shape[1], 3), dL_dfeature=torch.randn(P, F))
    acc = {k: v.cuda().contiguous() for k, v in base.items()}
    before = {k: v.clone() for k, v in acc.items()}
    _run(inps, g, F, ct=ct, accumulate_into=acc)
    assert _rel(acc["dL_drotations"] - before["dL_drotations"], both[8]) < 2e-5
    assert _rel(acc["dL_dscales"] - before["dL_dscales"], both[7]) < 2e-5


def test_contract_errors():
    import torch
    from manigaussian_b200 import rasterizer as R
    inps, g = _inputs(500, 61, 37, 0, 1)
    s = _settings(inps[0], 0)
    cov = torch.eye(3, device="cuda")[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].repeat(500, 1).contiguous() * 0.01
    with pytest.raises(Exception, match="scales and rotations"):
        R.rasterize_views_raw([s], _t(g["means3D"]), None, None, _t(g["opacities"]), None, None, 1.0, cov, _t(g["shs"]), g["sh_degree"],
                              False, return_normal=True)
    # a cotangent without the forward's plane
    args = _cloud_args(g, None)
    outs, streams = R.rasterize_views_raw([s], *args)
    with pytest.raises(ValueError, match="normal planes"):
        R.rasterize_views_backward_raw([s], outs, streams, [torch.zeros(3, 37, 61, device="cuda")], None, args[0], None, None, args[4],
                                       args[5], 1.0, None, args[8], g["sh_degree"], False,
                                       grads_normal=[torch.zeros(3, 37, 61, device="cuda")])
    # the _median entry point (normal == NULL) gives what the plain call gives
    o2, _ = R.rasterize_views_raw([s], *args, return_median=True)
    assert torch.equal(outs[0][1], o2[0][1])
    # each pointer NULL in turn: a forward plane without a cotangent in the backward is a plain backward
    o3, st3 = R.rasterize_views_raw([s], *args, return_normal=True)
    gz = R.rasterize_views_backward_raw([s], o3, st3, [torch.ones(3, 37, 61, device="cuda")], None, args[0], None, None, args[4], args[5],
                                        1.0, None, args[8], g["sh_degree"], False)
    gp = R.rasterize_views_backward_raw([s], outs, streams, [torch.ones(3, 37, 61, device="cuda")], None, args[0], None, None, args[4],
                                        args[5], 1.0, None, args[8], g["sh_degree"], False)
    assert _rel(gz[8], gp[8]) < 2e-5


def _leaves(g, F):
    import torch
    L = {k: _t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs")}
    if F:
        L["feature"] = _t(g["feature"]).requires_grad_(True)
    return L


def test_public_paths_return_the_plane_and_backpropagate():
    import torch
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    F, V, W, H = 8, 3, 96, 64
    inps, g = _inputs(2000, W, H, F, V)
    views = [_settings(i, F) for i in inps]
    L = _leaves(g, F)
    ct = _cots(V, F, H, W)
    # raw reference for the plane
    outs, _ = _run(inps, g, F)
    out = render_views(views, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                       features_language=L["feature"], normalize_feature=False, return_normal=True, return_median_depth=True,
                       return_alpha=True)
    assert out["normal"].shape == (V, 3, H, W) and out["median_id"].dtype == torch.int32
    for v in range(V):
        assert torch.equal(out["normal"][v], outs[v][-1])
    (out["normal"] * ct["normal"]).sum().backward()
    rot_views = L["rotations"].grad.clone()
    assert torch.isfinite(rot_views).all() and float(rot_views.abs().max()) > 0
    assert float(L["opacities"].grad.abs().max()) > 0
    # the single-view operator
    for x in L.values():
        x.grad = None
    r = R.GaussianRasterizer(views[0], return_depth=True, return_normal=True)
    o = r(means3D=L["means3D"], means2D=torch.zeros_like(L["means3D"], requires_grad=True), opacities=L["opacities"], shs=L["shs"],
          language_feature_precomp=L["feature"], scales=L["scales"], rotations=L["rotations"])
    assert len(o) == 5 and torch.equal(o[4], outs[0][-1])
    (o[4] * ct["normal"][0]).sum().backward()
    assert float(L["rotations"].grad.abs().max()) > 0
    one = render_views(views[:1], L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                       features_language=L["feature"], normalize_feature=False, return_normal=True)
    assert torch.equal(one["normal"][0], outs[0][-1])
    with pytest.raises(ValueError, match="return_normal"):
        render_views(views, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                     targets={"rgb": torch.zeros(V, 3, H, W, device="cuda")}, return_normal=True)
    # two clouds of different P
    inps2, g2 = _inputs(1200, 61, 37, F, 2, seed=8)
    L2 = _leaves(g2, F)
    for x in L.values():
        x.grad = None
    res = render_clouds([dict(cameras=views, pts_xyz=L["means3D"], rotations=L["rotations"], scales=L["scales"], opacity=L["opacities"],
                              features_color=L["shs"], features_language=L["feature"]),
                         dict(cameras=[_settings(i, F) for i in inps2], pts_xyz=L2["means3D"], rotations=L2["rotations"],
                              scales=L2["scales"], opacity=L2["opacities"], features_color=L2["shs"], features_language=L2["feature"])],
                        normalize_feature=False, return_normal=True)
    assert res[0]["normal"].shape == (V, 3, H, W) and res[1]["normal"].shape == (2, 3, 37, 61)
    for v in range(V):
        assert torch.equal(res[0]["normal"][v], outs[v][-1])
    ((res[0]["normal"] * ct["normal"]).sum() + res[1]["normal"].sum()).backward()
    assert _rel(L["rotations"].grad, rot_views) < 2e-5
    assert float(L2["rotations"].grad.abs().max()) > 0


def test_cuda_graph_replay_and_no_memory_growth():
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    F, V, W, H = 8, 2, 96, 64
    inps, g = _inputs(2000, W, H, F, V)
    views = [_settings(i, F) for i in inps]
    L = _leaves(g, F)
    ct = _cots(V, F, H, W)

    def step():
        for x in L.values():
            x.grad = None
        o = render_views(views, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L["feature"], normalize_feature=False, return_normal=True)
        ((o["render"] * ct["color"]).sum() + (o["normal"] * ct["normal"]).sum()).backward()
        return o["normal"]

    # every eager step on the side stream the capture uses: the leaves' AccumulateGrad nodes then belong to that stream
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            eager = step().detach().clone()
        rot = L["rotations"].grad.clone()
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated()
        for _ in range(20):
            step()
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() <= m0 + (1 << 20)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for x in L.values():
        x.grad = None
    keep = {}
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o = render_views(views, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L["feature"], normalize_feature=False, return_normal=True)
        ((o["render"] * ct["color"]).sum() + (o["normal"] * ct["normal"]).sum()).backward()
        keep["normal"] = o["normal"].detach()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(keep["normal"], eager)
    assert _rel(L["rotations"].grad, rot) < 2e-5
