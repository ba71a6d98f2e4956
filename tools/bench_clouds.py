"""One render_clouds call against a loop of render_views calls (one per cloud) for ManiGaussian's dynamic-field step.

    python tools/bench_clouds.py [--steps 30] [--warmup 5] [--runs 3]

Workloads (DESIGN.md section 5):
  c4      -- bench.py's c4 step: 500k Gaussians, 4 current-frame + 4 next-frame views of 256x256, F = 32, SH degree 1;
  mg16k_B -- ManiGaussian's real call (SURVEY.md finding 6): 16k Gaussians, 128x128, F = 3, SH degree 1, one view per frame,
             B samples = 2 B clouds, B in {1, 2, 4}.
Each step is activations -> render -> loss -> backward, as bench.py's make_dyna_step.  Both arms are timed with CUDA events
over --steps steps after --warmup steps, in --runs alternated runs; the table gives the median and the range.  Before timing,
the losses and every gradient of the two arms are compared (rel-L2 <= 1e-5, the spread of atomic ordering).  Prints the card
name, power limit and SM clock, one line per workload and a JSON summary.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definitions and the synthetic dyna inputs)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def workload(P, W, H, F, V, B):
    """B samples: raw network outputs per sample (its own cloud), and per sample V current- and V next-frame cameras."""
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    samples = []
    for s in range(B):
        g = scenes.make_gaussians(P, F=F, sh_degree=bench.SH_DEGREE, seed=1234 + s)
        raw = {k: torch.from_numpy(v).cuda() for k, v in bench.dyna_host_inputs(g, seed=4321 + s).items()}
        bg = torch.zeros(3, device="cuda")
        frames = []
        for f in range(2):
            cams = [scenes.make_camera(W, H, (2 * s + f) * V + v, 2 * B * V) for v in range(V)]
            t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
            frames.append([GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                                         bench.SH_DEGREE, t(c["campos"]), False, False, True) for c in cams])
        rng = np.random.default_rng(77 + s)
        cts = [(torch.from_numpy(rng.standard_normal((V, 3, H, W)).astype(np.float32)).cuda(),
                torch.from_numpy(rng.standard_normal((V, F, H, W)).astype(np.float32)).cuda()) for _ in range(2)]
        samples.append((raw, frames, cts))
    return samples


def step(arm, samples):
    """One training step of every sample's dyna objective; arm "clouds" renders all 2 B clouds in one render_clouds call,
    arm "loop" calls render_views once per cloud."""
    from manigaussian_b200.gaussian_params import activate_gaussians
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    clouds, cts, leaves = [], [], []
    for raw, frames, ct in samples:
        L = {k: (v.detach().requires_grad_(True) if k != "xyz" else v) for k, v in raw.items()}
        cur = activate_gaussians(L["xyz"], L["rot_maps"], L["scale_maps"], L["opacity_maps"], L["feature_maps"], d_means=L["xyz_maps"])
        nxt = activate_gaussians(cur[0].detach(), cur[1].detach(), cur[2].detach(), cur[3].detach(), None, d_means=L["next_xyz"],
                                 d_rotations=L["next_rot"], d_scales=L["next_scale"], scale_activation=None, opacity_activation=None)
        clouds += [dict(cameras=frames[0], pts_xyz=cur[0], rotations=cur[1], scales=cur[2], opacity=cur[3], features_color=L["sh"],
                        features_language=cur[4]),
                   dict(cameras=frames[1], pts_xyz=nxt[0], rotations=nxt[1], scales=nxt[2], opacity=nxt[3],
                        features_color=L["sh"].detach(), features_language=cur[4].detach())]
        cts += ct
        leaves.append(L)
    if arm == "clouds":
        outs = render_clouds(clouds, normalize_feature=False)
    else:
        outs = [render_views(c["cameras"], **{k: v for k, v in c.items() if k != "cameras"}, normalize_feature=False) for c in clouds]
    loss = sum((o["render"] * c[0]).sum() + (o["render_embed"] * c[1]).sum() for o, c in zip(outs, cts))
    loss.backward()
    return loss, leaves


def agreement(samples):
    def grads(arm):
        loss, leaves = step(arm, samples)
        return float(loss), [(k, v.grad.detach().double().cpu().numpy()) for L in leaves for k, v in L.items() if v.requires_grad]
    la, ga = grads("loop")
    lb, gb = grads("clouds")
    worst = abs(la - lb) / abs(la)
    for (k, a), (_, b) in zip(ga, gb):
        worst = max(worst, float(np.linalg.norm(a - b) / max(np.linalg.norm(a), 1e-30)))
    return worst


def timed(arm, samples, steps, warmup):
    import torch
    for _ in range(warmup):
        step(arm, samples)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step(arm, samples)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", nargs="*", help="workload names to run (default: all)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clouds needs a CUDA device")
    c4 = bench.WORKLOADS["c4"]
    loads = {"c4": (c4["P"], c4["W"], c4["H"], c4["F"], c4["views"], 1)}
    for B in (1, 2, 4):
        loads[f"mg16k_B{B}"] = (16384, 128, 128, 3, 1, B)
    info = card()
    print("card:", info, flush=True)
    rows = {}
    for name, (P, W, H, F, V, B) in loads.items():
        if a.only and name not in a.only:
            continue
        samples = workload(P, W, H, F, V, B)
        err = agreement(samples)
        assert err <= 1e-5, f"{name}: the two arms disagree (rel-L2 {err:.2e})"
        ms = {"loop": [], "clouds": []}
        for _ in range(a.runs):
            for arm in ("loop", "clouds"):
                ms[arm].append(timed(arm, samples, a.steps, a.warmup))
        med = {k: float(np.median(v)) for k, v in ms.items()}
        rows[name] = dict(P=P, WxH=f"{W}x{H}", F=F, clouds=2 * B, views_per_cloud=V, max_rel_l2=err,
                          loop_ms=med["loop"], loop_range=[min(ms["loop"]), max(ms["loop"])],
                          clouds_ms=med["clouds"], clouds_range=[min(ms["clouds"]), max(ms["clouds"])],
                          speedup=med["loop"] / med["clouds"])
        r = rows[name]
        print(f"{name:10s} {2 * B} clouds x {V} views  loop {r['loop_ms']:.3f} ms [{r['loop_range'][0]:.3f}, {r['loop_range'][1]:.3f}]  "
              f"clouds {r['clouds_ms']:.3f} ms [{r['clouds_range'][0]:.3f}, {r['clouds_range'][1]:.3f}]  x{r['speedup']:.2f}  "
              f"max rel-L2 {err:.1e}", flush=True)
        del samples
        torch.cuda.empty_cache()
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "workloads": rows}))


if __name__ == "__main__":
    main()
