"""Cost of default density control (gaussian_renderer.densify_stats / densify_and_prune; mgs_densify_stats /
mgs_densify_count / mgs_densify_emit) against gsplat's DefaultStrategy ops in PyTorch, and what it does to a short fit:

    python tools/bench_densify.py [--sizes 1000000 3000000] [--views 4] [--steps 20] [--warmup 3] [--runs 3] [--fit-steps 1500]

  stats     one statistics call per training step on P Gaussians x V views: the kernel, and its P (16 V + 24) bytes
            (each view's 12-byte gradient row and radius read, the three statistics read and written) over its time
            against the H100 SXM's 3.35 TB/s; the PyTorch arm is gsplat's norm, boolean select, two index_add_ and the
            radius maximum.
  refine    one refinement of a cloud with SH degree 3 ([P,16,3]) and Adam moments (exp_avg, exp_avg_sq) of every
            parameter, with 10 % cloned, 10 % split and 5 % pruned: ours is one densify_and_prune call; the PyTorch arm is
            gsplat's duplicate, split and remove (nonzero, the index gathers, randn, the concatenations of every parameter
            and moment, with the host reads they imply).  Neither writes its input, so every call starts from the same cloud.
  fit       bench_mcmc.py's fit (the scenes.py cloud of 16,384 Gaussians at SH degree 1 rendered from 8 cameras at
            128 x 128, Adam on 0.8 L1 + 0.2 (1 - SSIM) for --fit-steps steps) from 2,000 of the target's own means with
            the same initial scales, opacities and random colours, with and without default density control (statistics
            every step, refinement every 100 steps from step 300 to 80 % of the steps); the final L1, SSIM and P.
Times are CUDA events over --steps calls after --warmup calls, in --runs runs (median and range).  Prints the card name
and power limit read in the same run, and one JSON line.
"""
import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_knn import card, time_calls  # noqa: E402


def torch_stats(state, grad, radii, size, scale):
    """gsplat's DefaultStrategy._update_state for packed=False, V views of one size"""
    import torch
    grads = grad[..., :2].norm(dim=-1) * scale
    sel = radii > 0
    gs_ids = torch.where(sel)[1]
    state["grad2d"].index_add_(0, gs_ids, grads[sel])
    state["count"].index_add_(0, gs_ids, torch.ones_like(gs_ids, dtype=torch.float32))
    state["radii"][gs_ids] = torch.maximum(state["radii"][gs_ids], radii[sel] / float(size))


def _rotmat(q):
    import torch
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


def torch_refine(params, moments, grads, scene_scale, grow_grad2d=2e-4, grow_scale3d=0.01, prune_opa=0.005):
    """gsplat's _grow_gs (duplicate, then split) and _prune_gs on dicts of tensors; moments: {name: [tensors]}"""
    import torch
    is_high = grads > grow_grad2d
    is_small = torch.exp(params["scales"]).max(dim=-1).values <= grow_scale3d * scene_scale
    is_dupli, is_split = is_high & is_small, is_high & ~is_small
    n_dupli = int(is_dupli.sum().item())
    if n_dupli:
        sel = torch.where(is_dupli)[0]
        params = {k: torch.cat([v, v[sel]]) for k, v in params.items()}
        moments = {k: [torch.cat([v, torch.zeros((n_dupli,) + v.shape[1:], device=v.device)]) for v in vs] for k, vs in moments.items()}
    is_split = torch.cat([is_split, torch.zeros(n_dupli, dtype=torch.bool, device=is_split.device)])
    if int(is_split.sum().item()):
        sel, rest = torch.where(is_split)[0], torch.where(~is_split)[0]
        scales = torch.exp(params["scales"][sel])
        R = _rotmat(torch.nn.functional.normalize(params["rotations"][sel], dim=-1))
        samples = torch.einsum("nij,nj,bnj->bni", R, scales, torch.randn(2, len(sel), 3, device=sel.device))
        new = {}
        for k, v in params.items():
            if k == "pts_xyz":
                s = (v[sel] + samples).reshape(-1, 3)
            elif k == "scales":
                s = torch.log(scales / 1.6).repeat(2, 1)
            else:
                s = v[sel].repeat([2] + [1] * (v.dim() - 1))
            new[k] = torch.cat([v[rest], s])
        params = new
        moments = {k: [torch.cat([v[rest], torch.zeros((2 * len(sel),) + v.shape[1:], device=v.device)]) for v in vs]
                   for k, vs in moments.items()}
    is_prune = torch.sigmoid(params["opacity"].flatten()) < prune_opa
    if int(is_prune.sum().item()):
        keep = ~is_prune
        params = {k: v[keep] for k, v in params.items()}
        moments = {k: [v[keep] for v in vs] for k, vs in moments.items()}
    return params, moments


def refine_cloud(P, seed, device):
    """a cloud whose statistics clone 10 %, split 10 % and prune 5 % of it (scene_scale 1: small means exp(L) <= 0.01)"""
    import torch
    g = torch.Generator(device=device).manual_seed(seed)
    u = torch.rand(P, generator=g, device=device)
    scales = torch.rand(P, 3, generator=g, device=device) * 2 - 8        # all below log(0.01) = -4.6
    scales[u >= 0.1, 0] = -3.0                                           # 90 % large
    opacity = torch.rand(P, 1, generator=g, device=device) * 4 - 1
    opacity[(u >= 0.5) & (u < 0.55)] = -8.0                             # 5 % transparent, neither cloned nor split
    grad2d = torch.where(u < 0.2, 1e-3, 1e-5).float()                   # the first 20 %: 10 % small (clone), 10 % large (split)
    params = {"pts_xyz": torch.randn(P, 3, generator=g, device=device),
              "rotations": torch.randn(P, 4, generator=g, device=device), "scales": scales, "opacity": opacity,
              "sh": torch.randn(P, 16, 3, generator=g, device=device)}
    stats = {"grad2d": grad2d, "count": torch.ones(P, dtype=torch.int32, device=device),
             "radius": torch.zeros(P, device=device)}
    return params, stats


class _Opt:
    """the two attributes of a torch optimizer densify_and_prune reads and swaps"""

    def __init__(self, params, moments):
        self.param_groups = [{"params": [p]} for p in params.values()]
        self.state = {params[k]: {"exp_avg": moments[k][0], "exp_avg_sq": moments[k][1]} for k in params}


def bench_kernels(P, args):
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    dev = torch.device("cuda")
    V, size = args.views, 640
    g = torch.Generator(device=dev).manual_seed(P)
    grad = torch.randn(V, P, 3, generator=g, device=dev) * 1e-3
    radii = torch.randint(-1, 40, (V, P), generator=g, device=dev, dtype=torch.int32)
    stats = GR.densify_state(P, dev)
    tstate = {"grad2d": torch.zeros(P, device=dev), "count": torch.zeros(P, device=dev), "radii": torch.zeros(P, device=dev)}
    res = {"P": P, "V": V}
    t = time_calls(lambda: GR.densify_stats(stats, grad, radii, size, float(V)), args.steps, args.warmup, args.runs)
    res["stats_ms"] = t
    res["stats_bytes"] = P * (16 * V + 24)
    res["stats_TBps"] = res["stats_bytes"] / (t[0] * 1e-3) / 1e12
    res["stats_share_of_3.35TBps"] = res["stats_TBps"] / 3.35
    res["stats_torch_ms"] = time_calls(lambda: torch_stats(tstate, grad, radii, size, float(V)), args.steps, args.warmup,
                                       args.runs)

    base, bstats = refine_cloud(P, 0, dev)
    moments = {k: [torch.rand_like(v), torch.rand_like(v)] for k, v in base.items()}
    rng = torch.tensor([1, 0], dtype=torch.int64, device=dev)
    probe = GR.densify_and_prune(dict(base), dict(bstats), _Opt(dict(base), moments), scene_scale=1.0, rng=rng)["counts"]
    res["counts"] = probe

    def ours():
        params = dict(base)
        GR.densify_and_prune(params, dict(bstats), _Opt(params, moments), scene_scale=1.0, rng=rng)

    def theirs():
        torch_refine(base, moments, bstats["grad2d"] / bstats["count"].clamp_min(1).float(), 1.0)

    res["refine_ms"] = time_calls(ours, args.steps, args.warmup, args.runs)
    res["refine_torch_ms"] = time_calls(theirs, args.steps, args.warmup, args.runs)
    return res


def fit(densify, steps, seed=0):
    import torch
    from manigaussian_b200 import gaussian_renderer as GR, scenes
    from manigaussian_b200.cameras import camera_batch
    dev = torch.device("cuda")
    V, W = 8, 128
    cams = [scenes.make_camera(W, W, v, V) for v in range(V)]
    w2c = torch.tensor(np.stack([c["viewmatrix"].T for c in cams]), device=dev)
    fx = W / (2.0 * cams[0]["tanfovx"])
    K = np.tile(np.array([[fx, 0, W / 2.0], [0, fx, W / 2.0], [0, 0, 1]], np.float32), (V, 1, 1))
    batch = camera_batch(w2c, K, W, W)
    g = scenes.make_gaussians(16384, sh_degree=1, seed=1)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    with torch.no_grad():
        target = GR.render_views(batch, t(g["means3D"]), t(g["rotations"]), t(g["scales"]), t(g["opacities"]),
                                 features_color=t(g["shs"]))["render"].detach()
    rs = np.random.default_rng(seed)
    P0 = 2000
    pick = rs.choice(g["means3D"].shape[0], P0, replace=False)
    params = {"pts_xyz": t(g["means3D"][pick].astype(np.float32)),
              "rotations": t(np.tile(np.array([1, 0, 0, 0], np.float32), (P0, 1))),
              "scales": t(np.full((P0, 3), math.log(0.02), np.float32)),
              "opacity": t(np.full((P0, 1), -2.0, np.float32)),
              "rgb": t(rs.uniform(-1, 1, (P0, 3)).astype(np.float32))}
    params = {k: torch.nn.Parameter(v) for k, v in params.items()}
    lr = {"pts_xyz": 1.6e-4, "rotations": 1e-3, "scales": 5e-3, "opacity": 5e-2, "rgb": 2.5e-3}
    opt = torch.optim.Adam([{"params": [params[k]], "lr": lr[k]} for k in params], eps=1e-15)
    rng = torch.tensor([seed + 5, 0], dtype=torch.int64, device=dev)
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    scene_scale = float(np.linalg.norm(hi - lo) / 2)
    stats = GR.densify_state(P0, dev)
    for step in range(steps):
        out = GR.render_views(batch, params["pts_xyz"], params["rotations"], torch.exp(params["scales"]),
                              torch.sigmoid(params["opacity"]), pts_rgb=torch.sigmoid(params["rgb"]), targets={"rgb": target},
                              ssim=True)
        loss = 0.8 * out["loss_l1"].mean() + 0.2 * (1 - out["ssim"].mean())
        opt.zero_grad(set_to_none=True)
        loss.backward()
        if densify:
            GR.densify_stats(stats, out["viewspace_points"].grad, out["radii"], batch, scale=float(V))
        opt.step()
        if densify and 300 <= step < int(0.8 * steps) and step % 100 == 0:
            GR.densify_and_prune(params, stats, opt, scene_scale=scene_scale, rng=rng)
    with torch.no_grad():
        out = GR.render_views(batch, params["pts_xyz"], params["rotations"], torch.exp(params["scales"]),
                              torch.sigmoid(params["opacity"]), pts_rgb=torch.sigmoid(params["rgb"]), targets={"rgb": target},
                              ssim=True)
    return {"densify": densify, "P": int(params["pts_xyz"].shape[0]), "l1": float(out["loss_l1"].mean()),
            "ssim": float(out["ssim"].mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--fit-steps", type=int, default=1500)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_densify.py measures on a CUDA device; none is available")
    result = {"card": card(), "kernels": [], "fit": []}
    print(result["card"], flush=True)
    for P in args.sizes:
        r = bench_kernels(P, args)
        print(r, flush=True)
        result["kernels"].append(r)
    for densify in (False, True):
        r = fit(densify, args.fit_steps)
        print(r, flush=True)
        result["fit"].append(r)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
