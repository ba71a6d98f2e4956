"""Cost of MCMC density control (gaussian_renderer.mcmc_relocate / mcmc_perturb; mgs_mcmc_relocate / mgs_mcmc_perturb)
against a device-side PyTorch restatement of gsplat's MCMCStrategy ops, and what it does to a short fit:

    python tools/bench_mcmc.py [--sizes 1000000 3000000] [--steps 20] [--warmup 3] [--runs 3] [--fit-steps 1500]

  perturb   one position-noise call per training step on P Gaussians: the kernel, and its 56 bytes a Gaussian (means,
            quats, log-scales and logit read, means written) over its time against the H100 SXM's 3.35 TB/s; the
            PyTorch arm is gsplat's randn, quaternion-to-covariance and einsum.
  refine    one refinement of a cloud with SH degree 3 ([P,16,3]) and Adam moments (exp_avg, exp_avg_sq) of every
            parameter, 10 % of it dead, growing by 5 %: ours is one mcmc_relocate call (the growth's concatenations
            included); the PyTorch arm is gsplat's relocate + sample_add (nonzero, multinomial, bincount, the relocation
            formula and the index copies, with the host reads they imply).  Every call starts from the same cloud.
  fit       the scenes.py cloud (16,384 Gaussians, SH degree 1) rendered from 8 cameras at 128 x 128 as targets, fitted
            from 2,000 random Gaussians with Adam on 0.8 L1 + 0.2 (1 - SSIM) for --fit-steps steps, with and without MCMC
            (relocation and growth every 100 steps from step 300 to 80 % of the steps, cap 8,000; position noise after
            every step; 0.01 opacity and scale L1 regularisers); the final L1, SSIM and P.
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

N_MAX = 51


def _binoms(device):
    import torch
    return torch.tensor([[float(math.comb(n, j)) for j in range(N_MAX + 1)] for n in range(N_MAX + 1)], device=device)


def torch_relocation(o, s, ratios, binoms):
    """gsplat's compute_relocation in float32: o' = 1 - (1 - o)^(1/n), s' = s o / sum_j C(n,j) (-1)^(j-1) o'^j / sqrt(j)"""
    import torch
    n = ratios.clamp(1, N_MAX)
    a = 1.0 - (1.0 - o) ** (1.0 / n.float())
    j = torch.arange(1, N_MAX + 1, device=o.device)
    sign = torch.where(j % 2 == 1, 1.0, -1.0)
    terms = binoms[n][:, 1:] * sign * a[:, None] ** j / j.float().sqrt()
    den = torch.where(j[None] <= n[:, None], terms, torch.zeros_like(terms)).sum(1)
    return a, s * (o / den)[:, None]


def torch_refine(params, moments, n_new, binoms, min_opacity=0.005):
    """gsplat's relocate (dead onto live) then sample_add (n_new more), on dicts of tensors; moments: {name: [tensors]}"""
    import torch
    eps = torch.finfo(torch.float32).eps

    def split(sampled):
        o = torch.sigmoid(params["opacity"])[sampled]
        a, s = torch_relocation(o, torch.exp(params["scales"])[sampled], torch.bincount(sampled)[sampled] + 1, binoms)
        a = a.clamp(min_opacity, 1.0 - eps)
        params["opacity"][sampled] = torch.logit(a)
        params["scales"][sampled] = torch.log(s)
        for vs in moments.values():
            for v in vs:
                v[sampled] = 0

    opac = torch.sigmoid(params["opacity"])
    dead = opac <= min_opacity
    dead_idx, alive_idx = dead.nonzero(as_tuple=True)[0], (~dead).nonzero(as_tuple=True)[0]
    if dead_idx.numel() and alive_idx.numel():
        sampled = alive_idx[torch.multinomial(opac[alive_idx], dead_idx.numel(), replacement=True)]
        split(sampled)
        for k in params:
            params[k][dead_idx] = params[k][sampled]
    opac = torch.sigmoid(params["opacity"])
    sampled = torch.multinomial(opac, n_new, replacement=True)
    split(sampled)
    for k in params:
        params[k] = torch.cat([params[k], params[k][sampled]])
        moments[k] = [torch.cat([v, torch.zeros((n_new,) + v.shape[1:], device=v.device)]) for v in moments[k]]
    return params, moments


def torch_perturb(means, quats, log_scales, opacity, scale):
    """gsplat's inject_noise_to_position"""
    import torch
    q = torch.nn.functional.normalize(quats, dim=-1)
    r, x, y, z = q.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    M = R * torch.exp(log_scales)[:, None, :]
    covars = M @ M.transpose(1, 2)
    o = torch.sigmoid(opacity)
    noise = torch.randn_like(means) * (1 / (1 + torch.exp(-100 * ((1 - o) - 0.995))))[:, None] * scale
    means.add_(torch.einsum("bij,bj->bi", covars, noise))


def cloud(P, seed, device):
    import torch
    g = torch.Generator(device=device).manual_seed(seed)
    opacity = torch.rand(P, generator=g, device=device) * 10 - 4
    dead = torch.randperm(P, generator=g, device=device)[: P // 10]
    opacity[dead] = -8.0
    return {"pts_xyz": torch.randn(P, 3, generator=g, device=device),
            "rotations": torch.randn(P, 4, generator=g, device=device),
            "scales": torch.rand(P, 3, generator=g, device=device) * 4 - 6,
            "opacity": opacity,
            "sh": torch.randn(P, 16, 3, generator=g, device=device)}


class _Opt:
    """the two attributes of a torch optimizer mcmc_relocate reads and swaps"""

    def __init__(self, params, moments):
        self.param_groups = [{"params": [p]} for p in params.values()]
        self.state = {params[k]: {"exp_avg": moments[k][0], "exp_avg_sq": moments[k][1]} for k in params}


def bench_kernels(P, args):
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    dev = torch.device("cuda")
    base = cloud(P, 0, dev)
    moments = {k: [torch.rand_like(v), torch.rand_like(v)] for k, v in base.items()}
    rng = torch.tensor([1, 0], dtype=torch.int64, device=dev)
    scale = torch.tensor([0.08], device=dev)
    binoms = _binoms(dev)
    means = base["pts_xyz"].clone()
    res = {"P": P}

    def ours_perturb():
        GR.mcmc_perturb(means, base["rotations"], base["scales"], base["opacity"], scale, rng)

    def torch_perturb_call():
        torch_perturb(means, base["rotations"], base["scales"], base["opacity"], scale)

    t = time_calls(ours_perturb, args.steps, args.warmup, args.runs)
    res["perturb_ms"] = t
    res["perturb_bytes"] = 56 * P
    res["perturb_TBps"] = 56 * P / (t[0] * 1e-3) / 1e12
    res["perturb_share_of_3.35TBps"] = res["perturb_TBps"] / 3.35
    res["perturb_torch_ms"] = time_calls(torch_perturb_call, args.steps, args.warmup, args.runs)

    n_new = P // 20

    def ours_refine():
        params = dict(base)
        GR.mcmc_relocate(params, optimizer=_Opt(params, moments), n=P + n_new, rng=rng)

    def torch_refine_call():
        torch_refine({k: v.clone() for k, v in base.items()}, {k: [m.clone() for m in v] for k, v in moments.items()}, n_new, binoms)

    # ours grows from `base` without writing it; the PyTorch arm writes in place, so it works on a copy, whose cost is
    # timed separately and subtracted
    def copies():
        ({k: v.clone() for k, v in base.items()}, {k: [m.clone() for m in v] for k, v in moments.items()})

    res["refine_ms"] = time_calls(ours_refine, args.steps, args.warmup, args.runs)
    tr = time_calls(torch_refine_call, args.steps, args.warmup, args.runs)
    tc = time_calls(copies, args.steps, args.warmup, args.runs)
    res["refine_torch_ms"] = tr
    res["refine_torch_copy_ms"] = tc
    res["refine_torch_minus_copy_ms"] = tr[0] - tc[0]
    return res


def fit(mcmc, steps, seed=0):
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
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    params = {"pts_xyz": t((lo + (hi - lo) * rs.random((P0, 3))).astype(np.float32)),
              "rotations": t(np.tile(np.array([1, 0, 0, 0], np.float32), (P0, 1))),
              "scales": t(np.full((P0, 3), math.log(0.02), np.float32)),
              "opacity": t(np.full((P0, 1), -2.0, np.float32)),
              "rgb": t(rs.uniform(-1, 1, (P0, 3)).astype(np.float32))}
    params = {k: torch.nn.Parameter(v) for k, v in params.items()}
    lr = {"pts_xyz": 1.6e-4, "rotations": 1e-3, "scales": 5e-3, "opacity": 5e-2, "rgb": 2.5e-3}
    opt = torch.optim.Adam([{"params": [params[k]], "lr": lr[k]} for k in params], eps=1e-15)
    rng = torch.tensor([seed + 5, 0], dtype=torch.int64, device=dev)
    noise = torch.tensor([lr["pts_xyz"] * 5e5], device=dev)
    cap = 8000
    for step in range(steps):
        out = GR.render_views(batch, params["pts_xyz"], params["rotations"], torch.exp(params["scales"]),
                              torch.sigmoid(params["opacity"]), pts_rgb=torch.sigmoid(params["rgb"]), targets={"rgb": target},
                              ssim=True)
        loss = 0.8 * out["loss_l1"].mean() + 0.2 * (1 - out["ssim"].mean())
        if mcmc:
            loss = loss + 0.01 * torch.sigmoid(params["opacity"]).mean() + 0.01 * torch.exp(params["scales"]).mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        if mcmc:
            if 300 <= step < int(0.8 * steps) and step % 100 == 0:
                P = params["pts_xyz"].shape[0]
                GR.mcmc_relocate(params, optimizer=opt, n=min(cap, int(1.05 * P)), rng=rng)
            GR.mcmc_perturb(params["pts_xyz"], params["rotations"], params["scales"], params["opacity"], noise, rng)
    with torch.no_grad():
        out = GR.render_views(batch, params["pts_xyz"], params["rotations"], torch.exp(params["scales"]),
                              torch.sigmoid(params["opacity"]), pts_rgb=torch.sigmoid(params["rgb"]), targets={"rgb": target},
                              ssim=True)
    return {"mcmc": mcmc, "P": int(params["pts_xyz"].shape[0]), "l1": float(out["loss_l1"].mean()),
            "ssim": float(out["ssim"].mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--fit-steps", type=int, default=1500)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mcmc.py measures on a CUDA device; none is available")
    result = {"card": card(), "kernels": [], "fit": []}
    print(result["card"], flush=True)
    for P in args.sizes:
        r = bench_kernels(P, args)
        print(r, flush=True)
        result["kernels"].append(r)
    for mcmc in (False, True):
        r = fit(mcmc, args.fit_steps)
        print(r, flush=True)
        result["fit"].append(r)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
