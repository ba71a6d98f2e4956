"""render_clouds / mgs_forward_clouds / mgs_backward_clouds: several Gaussian clouds in one call must compute exactly what one
render_views call per cloud computes -- images, depth and radii bit for bit, gradients within the spread of atomic ordering."""
import numpy as np
import pytest

import util
from test_render_gpu import _cams, _cloud, _t

pytestmark = pytest.mark.gpu

NAMES = ("xyz", "rot", "scale", "opac", "col", "feat")


def _leaves(P, F, seed, colour):
    g = _cloud(P, max(F, 1), seed)
    col = g["shs"] if colour == "sh" else np.random.default_rng(seed).uniform(0, 1, (P, 3)).astype(np.float32)
    d = dict(xyz=g["means3D"], rot=g["rotations"], scale=g["scales"], opac=g["opacities"], col=col)
    if F:
        d["feat"] = g["feature"][:, :F] if g["feature"].shape[1] >= F else np.tile(g["feature"], (1, F))[:, :F]
    return d


def _mk(host):
    return {k: _t(np.ascontiguousarray(v, np.float32)).requires_grad_(True) for k, v in host.items()}


def _kw(L, colour):
    kw = dict(pts_xyz=L["xyz"], rotations=L["rot"], scales=L["scale"], opacity=L["opac"], features_language=L.get("feat"))
    kw["features_color" if colour == "sh" else "pts_rgb"] = L["col"]
    return kw


def _objective(o, ct, depth):
    import torch
    loss = (o["render"] * ct[0]).sum()
    if o["render_embed"] is not None:
        loss = loss + (o["render_embed"] * ct[1]).sum()
    if depth:
        loss = loss + (o["depth"] * ct[2]).sum()
    return loss if torch.is_tensor(loss) else torch.zeros(())


def _compare(clouds_spec, colour, F, depth=True, bg=(0.1, 0.2, 0.3)):
    """clouds_spec: [(P, cameras, seed)].  One render_clouds call against one render_views call per cloud."""
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    hosts = [_leaves(P, F, seed, colour) for P, _, seed in clouds_spec]
    cts = []
    for P, cams, _ in clouds_spec:
        V, H, W = len(cams), cams.height, cams.width
        cts.append((torch.randn(V, 3, H, W, device="cuda"), torch.randn(V, F, H, W, device="cuda"), torch.randn(V, H, W, device="cuda")))
    A = [_mk(h) for h in hosts]
    outs = render_clouds([dict(cameras=cams, **_kw(L, colour)) for L, (_, cams, _) in zip(A, clouds_spec)], bg_color=bg,
                         return_depth=depth)
    sum(_objective(o, ct, depth) for o, ct in zip(outs, cts)).backward()
    for b, (L, (P, cams, _)) in enumerate(zip(A, clouds_spec)):
        Bl = _mk(hosts[b])
        r = render_views(cams, bg_color=bg, return_depth=depth, **_kw(Bl, colour))
        _objective(r, cts[b], depth).backward()
        o = outs[b]
        assert set(o) == set(r), b
        for k in ("render", "render_embed", "radii") + (("depth",) if depth else ()):
            assert (o[k] is None) == (r[k] is None), (b, k)
            if o[k] is not None:
                assert o[k].shape == r[k].shape and torch.equal(o[k], r[k]), (b, k)
        for k in L:
            assert L[k].grad is not None, (b, k)
            assert util.rel_l2(L[k].grad.cpu().numpy(), Bl[k].grad.cpu().numpy()) < 1e-5, (b, k)
        for v in range(len(cams)):
            assert util.rel_l2(o["viewspace_points"].grad[v].cpu().numpy(), r["viewspace_points"].grad[v].cpu().numpy()) < 1e-5, (b, v)
    return outs


@pytest.mark.parametrize("colour", ["sh", "rgb"])
@pytest.mark.parametrize("F", [0, 3, 32, 64])
def test_render_clouds_equals_one_render_views_per_cloud(colour, F):
    """3 clouds (one of 50 Gaussians), 1 / 3 / 2 views, two image sizes, depth on."""
    spec = [(50, _cams(1, 64, 64), 51), (6000, _cams(3, 80, 48), 52), (3000, _cams(2, 64, 64), 53)]
    _compare(spec, colour, F)


def test_per_gaussian_launches_pack_and_split_clouds():
    """20 clouds x 2 views need three per-Gaussian launches of whole clouds; one cloud of 20 views spans two launches, the
    second adding to what the first wrote."""
    cams2 = _cams(2, 48, 48)
    _compare([(700 + 13 * b, cams2, 60 + b) for b in range(20)], "sh", 3, depth=False)
    _compare([(4000, _cams(20, 48, 48), 90), (300, cams2, 91)], "sh", 32, depth=False)


def test_dyna_step_in_one_call():
    """The dyna step of test_render_gpu.test_dyna_step_end_to_end_gradients with both frames in ONE render_clouds call.  The
    next frame renders the detached SH and features of the current one: its dL_dfeature is not computed (NULL), while its
    feature cotangents and its SH view-direction term still reach the next-frame offsets."""
    import torch
    from manigaussian_b200 import GaussianRasterizer
    from manigaussian_b200.gaussian_params import activate_gaussians
    from manigaussian_b200.gaussian_renderer import render_clouds
    P, F, W, H, V = 6000, 32, 64, 64, 2
    g = _cloud(P, F, 23)
    cams = _cams(V, W, H)
    rng = np.random.default_rng(4)
    raw = dict(xyz=g["means3D"], xyz_maps=rng.normal(0, 0.01, (P, 3)), rot_maps=g["rotations"] * rng.uniform(0.5, 2, (P, 1)),
               scale_maps=np.log(g["scales"]) + rng.normal(0, 0.05, (P, 3)), opacity_maps=np.log(g["opacities"] / (1 - g["opacities"])),
               sh=g["shs"], feature_maps=g["feature"] * rng.uniform(0.5, 2, (P, 1)), next_xyz=rng.normal(0, 0.01, (P, 3)),
               next_rot=rng.normal(0, 0.05, (P, 4)))
    mk = lambda: {k: _t(np.asarray(v, np.float32)).requires_grad_(k != "xyz") for k, v in raw.items()}
    cts = [[(torch.randn(3, H, W, device="cuda"), torch.randn(F, H, W, device="cuda")) for _ in range(V)] for _ in range(2)]

    a = mk()
    cur = activate_gaussians(a["xyz"], a["rot_maps"], a["scale_maps"], a["opacity_maps"], a["feature_maps"], d_means=a["xyz_maps"],
                             normalize_feature=False)
    nxt = activate_gaussians(cur[0].detach(), cur[1].detach(), cur[2].detach(), cur[3].detach(), None, d_means=a["next_xyz"],
                             d_rotations=a["next_rot"], scale_activation=None, opacity_activation=None)
    o_cur, o_nxt = render_clouds([
        dict(cameras=cams, pts_xyz=cur[0], rotations=cur[1], scales=cur[2], opacity=cur[3], features_color=a["sh"], features_language=cur[4]),
        dict(cameras=cams, pts_xyz=nxt[0], rotations=nxt[1], scales=nxt[2], opacity=nxt[3], features_color=a["sh"].detach(),
             features_language=cur[4].detach())])
    loss = sum((o["render"][v] * c[v][0]).sum() + (o["render_embed"][v] * c[v][1]).sum() for o, c in ((o_cur, cts[0]), (o_nxt, cts[1]))
               for v in range(V))
    loss.backward()

    b = mk()
    scales = torch.clamp_max(torch.exp(b["scale_maps"]), 0.05)
    means = b["xyz"] + b["xyz_maps"]
    rots = torch.nn.functional.normalize(b["rot_maps"], dim=-1)
    opac = torch.sigmoid(b["opacity_maps"])
    n_means = means.detach() + b["next_xyz"]
    n_rots = torch.nn.functional.normalize(rots.detach() + b["next_rot"], dim=-1)

    def ref_render(v, m, r, s, o, sh, f):
        f = f / (f.norm(dim=-1, keepdim=True) + 1e-12)
        st = cams.settings(v, torch.zeros(3, device="cuda"), 1, True)
        return GaussianRasterizer(st)(means3D=m, means2D=torch.zeros_like(m), opacities=o, shs=sh, language_feature_precomp=f, scales=s, rotations=r)
    loss_b = 0
    for v in range(V):
        img, emb, _ = ref_render(v, means, rots, scales, opac, b["sh"], b["feature_maps"])
        loss_b = loss_b + (img * cts[0][v][0]).sum() + (emb * cts[0][v][1]).sum()
        img, emb, _ = ref_render(v, n_means, n_rots, scales.detach(), opac.detach(), b["sh"].detach(), b["feature_maps"].detach())
        loss_b = loss_b + (img * cts[1][v][0]).sum() + (emb * cts[1][v][1]).sum()
    loss_b.backward()
    assert abs(float(loss) - float(loss_b)) <= 1e-4 * abs(float(loss_b)) + 1e-3
    for k in ("xyz_maps", "rot_maps", "scale_maps", "opacity_maps", "sh", "feature_maps", "next_xyz", "next_rot"):
        assert a[k].grad is not None, k
        assert util.rel_l2(a[k].grad.cpu().numpy(), b[k].grad.cpu().numpy()) < 2e-5, k


@pytest.mark.parametrize("F", [32, 0])
def test_loss_heads_match_render_views_per_cloud(F):
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    spec = [(7000, _cams(3, 72, 56), 37), (2500, _cams(2, 64, 64), 38)]
    hosts = [_leaves(P, F, seed, "sh") for P, _, seed in spec]
    tg = [{"rgb": torch.rand(len(c), 3, c.height, c.width, device="cuda"),
           "embed": torch.randn(len(c), F, c.height, c.width, device="cuda") if F else None} for _, c, _ in spec]
    A = [_mk(h) for h in hosts]
    outs = render_clouds([dict(cameras=c, targets=t, **_kw(L, "sh")) for L, (_, c, _), t in zip(A, spec, tg)])
    sum(o["loss_rgb"].sum() + 0.01 * o["loss_embed"].sum() for o in outs).backward()
    for b, (P, c, _) in enumerate(spec):
        Bl = _mk(hosts[b])
        r = render_views(c, targets=tg[b], **_kw(Bl, "sh"))
        (r["loss_rgb"].sum() + 0.01 * r["loss_embed"].sum()).backward()
        assert torch.equal(outs[b]["render"], r["render"])
        for k in ("loss_rgb", "loss_embed"):
            assert util.rel_l2(outs[b][k].detach().cpu().numpy(), r[k].detach().cpu().numpy()) < 1e-6, (b, k)
        for k in A[b]:
            assert util.rel_l2(A[b][k].grad.cpu().numpy(), Bl[k].grad.cpu().numpy()) < 1e-5, (b, k)
        assert util.rel_l2(outs[b]["viewspace_points"].grad.cpu().numpy(), r["viewspace_points"].grad.cpu().numpy()) < 1e-5


def _raw_clouds(cams, hosts, caps=None):
    import torch
    return [dict(views=[cams.settings(v, torch.zeros(3, device="cuda"), 1, True) for v in range(len(cams))],
                 means3D=_t(h["xyz"]), sh=_t(h["col"]), feature=_t(h["feat"]), opacity=_t(h["opac"]), scales=_t(h["scale"]),
                 rotations=_t(h["rot"]), capacities=None if caps is None else caps[b]) for b, h in enumerate(hosts)]


def test_overflow_of_one_view_leaves_every_other_view_untouched():
    import torch
    from manigaussian_b200.rasterizer import rasterize_clouds_raw
    cams = _cams(2, 64, 64)
    hosts = [_leaves(5000, 32, 70 + b, "sh") for b in range(3)]
    ok, _ = rasterize_clouds_raw(_raw_clouds(cams, hosts), 1, True)
    counts = [[o.num_rendered() for o in co] for co in ok]
    caps = [[c + 64 for c in cc] for cc in counts]
    caps[1][0] = counts[1][0] // 2
    small, _ = rasterize_clouds_raw(_raw_clouds(cams, hosts, caps), 1, True)
    torch.cuda.synchronize()
    for b in range(3):
        for v in range(2):
            assert small[b][v].num_rendered() == counts[b][v]
            if (b, v) == (1, 0):
                assert small[b][v].overflowed() and not torch.equal(small[b][v][1], ok[b][v][1])
            else:
                assert not small[b][v].overflowed(), (b, v)
                for i in (1, 2, 3):
                    assert torch.equal(small[b][v][i], ok[b][v][i]), (b, v, i)


def _two_cloud_step(A, cams, cts):
    from manigaussian_b200.gaussian_renderer import render_clouds
    outs = render_clouds([dict(cameras=cams, **_kw(L, "sh")) for L in A])
    loss = sum((o["render"] * ct[0]).sum() + (o["render_embed"] * ct[1]).sum() for o, ct in zip(outs, cts))
    loss.backward()
    return loss


def test_two_cloud_step_is_cuda_graph_capturable():
    import torch
    F, W, H, V = 32, 80, 64, 2
    cams = _cams(V, W, H)
    A = [_mk(_leaves(P, F, seed, "sh")) for P, seed in ((9000, 81), (4000, 82))]
    cts = [(torch.randn(V, 3, H, W, device="cuda"), torch.randn(V, F, H, W, device="cuda")) for _ in A]
    leaves = [x for L in A for x in L.values()]

    def clear():
        for x in leaves:
            x.grad = None

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            clear()
            _two_cloud_step(A, cams, cts)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eager = [x.grad.clone() for x in leaves]
    clear()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _two_cloud_step(A, cams, cts)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for x, e in zip(leaves, eager):
        assert util.rel_l2(x.grad.cpu().numpy(), e.cpu().numpy()) < 1e-5
    with torch.no_grad():
        A[1]["xyz"].add_(0.01)
    graph.replay()
    torch.cuda.synchronize()
    moved = [x.grad.clone() for x in leaves]
    clear()
    _two_cloud_step(A, cams, cts)
    torch.cuda.synchronize()
    for x, m in zip(leaves, moved):
        assert util.rel_l2(m.cpu().numpy(), x.grad.cpu().numpy()) < 1e-5


@pytest.mark.parametrize("targets", [False, True])
def test_cloud_steps_do_not_accumulate_device_memory(targets):
    import gc
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds
    F, W, H, V = 32, 64, 48, 2
    cams = _cams(V, W, H)
    hosts = [_leaves(P, F, seed, "sh") for P, seed in ((6000, 33), (3000, 34))]
    tgt = (torch.rand(V, 3, H, W, device="cuda"), torch.randn(V, F, H, W, device="cuda"))

    def step():
        A = [_mk(h) for h in hosts]  # fresh leaves every step, like a network's outputs
        if targets:
            outs = render_clouds([dict(cameras=cams, targets={"rgb": tgt[0], "embed": tgt[1]}, **_kw(L, "sh")) for L in A])
            loss = sum(o["loss_rgb"].sum() + 0.01 * o["loss_embed"].sum() for o in outs)
        else:
            outs = render_clouds([dict(cameras=cams, **_kw(L, "sh")) for L in A])
            loss = sum((o["render"] * tgt[0]).sum() + (o["render_embed"] * tgt[1]).sum() for o in outs)
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
