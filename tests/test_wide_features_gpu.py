"""Feature widths above 32 channels (run with `-m gpu` on an H100): the blends run in channel groups of 32, every group
walking the same tile lists (blend_common.cuh, BlendArgs::groups).  Checked against the C oracle stage by stage, against
the F <= 32 blend itself (a group is the same blend on other channels), and through the multi-view, fused-loss-head and
CUDA-graph paths."""
import numpy as np
import pytest

import util
from test_parity_gpu import check_stagewise_vs_oracle
from test_render_gpu import _cams, _cloud, _t

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("F", [33, 40, 47, 64, 96, 128, 512])
def test_wide_feature_stagewise_vs_oracle(F):
    """Remainder groups of 1 (F = 33), 8 (40), 15 (47, padded row path: F % 4 != 0) and 4 channels... up to 16 groups.
    Ragged image: partial tiles and partial 8x4 blocks."""
    inp = util.make_inputs(P=700, W=41, H=27, F=F, seed=300 + F, bg=(0.2, 0.1, 0.7))
    check_stagewise_vs_oracle(inp, 1e-3)


def test_wide_feature_large_cloud_vs_oracle():
    inp = util.make_inputs(P=50000, W=256, H=256, F=64, seed=41, bg=(0.3, 0.6, 0.9))
    check_stagewise_vs_oracle(inp, 1e-3)


def _with_features(inp, feature, dL_dfeature):
    out = dict(inp, F=feature.shape[1])
    out["g"] = dict(inp["g"], feature=np.ascontiguousarray(feature, np.float32))
    out["ct"] = dict(inp["ct"], dL_dfeature=np.ascontiguousarray(dL_dfeature, np.float32))
    return out


def test_channel_groups_are_the_same_blend():
    """F = 64 with features [f | f] renders both halves bit-identical to the F = 32 render of f, with the same colour and
    per-pixel state; with feature cotangent [g | 0] every gradient equals the F = 32 run's (atomic order only) and the
    second half's feature gradient is exactly zero.  F = 40 with channels 32..39 a copy of 0..7: the remainder group (8
    channels, whole 4-channel pieces) matches the full group it copies."""
    base = util.make_inputs(P=3000, W=83, H=61, F=32, seed=51, bg=(0.1, 0.5, 0.2))
    f, g = base["g"]["feature"], base["ct"]["dL_dfeature"]
    fw32, bw32 = util.run_ours(base)
    fw64, bw64 = util.run_ours(_with_features(base, np.concatenate([f, f], 1), np.concatenate([g, np.zeros_like(g)], 0)))
    of = fw64["out_feature"]
    assert of.shape[0] == 64
    assert np.array_equal(of[:32].view(np.uint32), of[32:].view(np.uint32))
    assert np.array_equal(of[:32].view(np.uint32), fw32["out_feature"].view(np.uint32))
    for k in ("out_color", "final_T", "n_contrib", "radii", "point_list"):
        assert np.array_equal(fw64[k], fw32[k]), k
    assert np.all(bw64["dL_dfeature"][:, 32:] == 0)
    assert util.rel_l2(bw64["dL_dfeature"][:, :32], bw32["dL_dfeature"]) < 1e-6
    for k in bw32:
        if k != "dL_dfeature":
            assert util.rel_l2(bw64[k], bw32[k]) < 1e-6, k

    f40 = np.concatenate([f, f[:, :8]], 1)
    g40 = np.concatenate([g, g[:8]], 0)
    fw40, bw40 = util.run_ours(_with_features(base, f40, g40))
    assert np.array_equal(fw40["out_color"], fw32["out_color"])
    assert np.array_equal(fw40["out_feature"][:32], fw32["out_feature"])
    assert util.rel_l2(fw40["out_feature"][32:], fw40["out_feature"][:8]) < 1e-6
    assert util.rel_l2(bw40["dL_dfeature"][:, 32:], bw40["dL_dfeature"][:, :8]) < 1e-6


def test_wide_render_views_equals_a_loop_of_render():
    """mgs_forward_views / mgs_backward_views at F = 64: images bit-identical to one render() per view, summed gradients
    equal to the loop's (the bars of test_render_views_equals_a_loop_of_render)."""
    import torch
    from manigaussian_b200.gaussian_renderer import render, render_views
    P, F, W, H, V = 8000, 64, 80, 64, 3
    g = _cloud(P, F, 61)
    cams = _cams(V, W, H)
    data = {"novel_view": cams.as_novel_view()}
    mk = lambda: {k: _t(v).requires_grad_(True) for k, v in dict(xyz=g["means3D"], rot=g["rotations"], scale=g["scales"],
                                                                 opac=g["opacities"], sh=g["shs"], feat=g["feature"]).items()}
    a, b = mk(), mk()
    cts = [(torch.randn(3, H, W, device="cuda"), torch.randn(F, H, W, device="cuda"), torch.randn(H, W, device="cuda")) for _ in range(V)]
    outs = render_views(cams, a["xyz"], a["rot"], a["scale"], a["opac"], (0, 0, 0), features_color=a["sh"], features_language=a["feat"],
                        return_depth=True)
    assert outs["render_embed"].shape == (V, F, H, W)
    loss = sum((outs["render"][v] * cts[v][0]).sum() + (outs["render_embed"][v] * cts[v][1]).sum() + (outs["depth"][v] * cts[v][2]).sum()
               for v in range(V))
    loss.backward()
    vsp = []
    for v in range(V):
        o = render(data, v, b["xyz"], b["rot"], b["scale"], b["opac"], [0, 0, 0], features_color=b["sh"], features_language=b["feat"],
                   return_depth=True)
        assert torch.equal(o["render"], outs["render"][v]) and torch.equal(o["render_embed"], outs["render_embed"][v])
        assert torch.equal(o["depth"], outs["depth"][v]) and torch.equal(o["radii"], outs["radii"][v])
        ((o["render"] * cts[v][0]).sum() + (o["render_embed"] * cts[v][1]).sum() + (o["depth"] * cts[v][2]).sum()).backward()
        vsp.append(o["viewspace_points"].grad)
    for k in a:
        assert util.rel_l2(a[k].grad.cpu().numpy(), b[k].grad.cpu().numpy()) < 1e-5, k
    for v in range(V):
        assert util.rel_l2(outs["viewspace_points"].grad[v].cpu().numpy(), vsp[v].cpu().numpy()) < 1e-5


@pytest.mark.parametrize("F,lam", [(64, 0.01), (100, 1.0)])
def test_wide_loss_heads(F, lam):
    """render_views(targets=...) at F > 32: the colour head in group 0's blend epilogue, the embedding head in the
    features-only loss-heads pass behind the blend; against the reference's PyTorch expressions on the unfused render."""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, W, H, V = 9000, 72, 56, 3
    g = _cloud(P, F, 67)
    cams = _cams(V, W, H)
    names = ("means3D", "rotations", "scales", "opacities", "shs", "feature")
    tgt_rgb = torch.rand(V, 3, H, W, device="cuda")
    tgt_emb = torch.randn(V, F, H, W, device="cuda")
    leaves = lambda: {k: _t(np.asarray(g[k], np.float32)).requires_grad_(True) for k in names}

    a = leaves()
    o = render_views(cams, a["means3D"], a["rotations"], a["scales"], a["opacities"], features_color=a["shs"],
                     features_language=a["feature"], targets={"rgb": tgt_rgb, "embed": tgt_emb})
    loss_a = o["loss_rgb"].sum() + lam * o["loss_embed"].sum()
    loss_a.backward()

    b = leaves()
    r = render_views(cams, b["means3D"], b["rotations"], b["scales"], b["opacities"], features_color=b["shs"],
                     features_language=b["feature"])
    loss_rgb, loss_emb = [], []
    for v in range(V):
        loss_rgb.append(((r["render"][v] - tgt_rgb[v]) ** 2).mean())
        cs = torch.nn.functional.cosine_similarity(r["render_embed"][v].permute(1, 2, 0), tgt_emb[v].permute(1, 2, 0), dim=-1)
        loss_emb.append(1 - cs.mean())
    loss_b = sum(loss_rgb) + lam * sum(loss_emb)
    loss_b.backward()
    assert torch.equal(o["render"], r["render"].detach())
    for v in range(V):
        got_rgb, got_emb = float(o["loss_rgb"][v].detach()), float(o["loss_embed"][v].detach())
        want_rgb, want_emb = float(loss_rgb[v].detach()), float(loss_emb[v].detach())
        assert abs(got_rgb - want_rgb) <= 1e-5 * abs(want_rgb)
        assert abs(got_emb - want_emb) <= 1e-5 * abs(want_emb) + 1e-6
    assert abs(float(loss_a) - float(loss_b)) <= 1e-5 * abs(float(loss_b))
    for k in names:
        assert a[k].grad is not None, k
        assert util.rel_l2(a[k].grad.cpu().numpy(), b[k].grad.cpu().numpy()) < 2e-5, k
    assert util.rel_l2(o["viewspace_points"].grad.cpu().numpy(), r["viewspace_points"].grad.cpu().numpy()) < 2e-5


def test_wide_step_is_cuda_graph_capturable():
    """A multi-view step at F = 64, with the fused loss heads (so the features-only head pass is in the graph too),
    captured once and replayed: replays reproduce the eager gradients."""
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    P, F, W, H, V = 12000, 64, 80, 64, 3
    g = _cloud(P, F, 71)
    cams = _cams(V, W, H)
    names = ("means3D", "rotations", "scales", "opacities", "shs", "feature")
    L = {k: _t(np.asarray(g[k], np.float32)).requires_grad_(True) for k in names}
    tgt = (torch.rand(V, 3, H, W, device="cuda"), torch.randn(V, F, H, W, device="cuda"))

    def fwd_bwd():
        o = render_views(cams, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L["feature"], targets={"rgb": tgt[0], "embed": tgt[1]})
        loss = o["loss_rgb"].sum() + 0.5 * o["loss_embed"].sum()
        loss.backward()
        return loss

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for v in L.values():
                v.grad = None
            eager_loss = float(fwd_bwd())
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eager = {k: v.grad.clone() for k, v in L.items()}
    for v in L.values():
        v.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = fwd_bwd()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert abs(float(loss) - eager_loss) <= 1e-6 * abs(eager_loss)
    for k in names:
        assert util.rel_l2(L[k].grad.cpu().numpy(), eager[k].cpu().numpy()) < 1e-5, k
