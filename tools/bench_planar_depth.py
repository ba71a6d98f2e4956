"""Cost of planar depth on a render_views training step, on bench.py's c3 shape (500k Gaussians, 4 views 256x256, SH degree 1)
with return_depth and the depth head.

    python tools/bench_planar_depth.py [--steps 30] [--warmup 5] [--runs 3] [--F 32]

Two arms, each one training step (render_views with targets {"rgb", "depth"} -> loss -> backward) timed with CUDA events over
--steps steps after --warmup steps, alternated over --runs runs in one process: planar depth off and on.  Prints the card's
name and power limit, the median and range of each arm's step time, the on / off ratio of the medians, the median of the
per-run (paired) ratios, the device time per step of the kernel groups the feature touches (torch.profiler, a pass of its
own) and a JSON summary.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definitions)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def main():
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    from manigaussian_b200.gaussian_renderer import render_views
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--F", type=int, default=32)
    a = ap.parse_args()
    wl = bench.WORKLOADS["c3"]
    P, V, W, H, F = wl["P"], wl["views"], wl["W"], wl["H"], a.F
    g = scenes.make_gaussians(P, F=F, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    L = {k: t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs") + (("feature",) if F else ())}
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           bench.SH_DEGREE, t(c["campos"]), False, False, F > 0) for c in cams]
    rng = np.random.default_rng(7)
    targets = {"rgb": t(rng.uniform(0, 1, (V, 3, H, W))), "depth": t(rng.uniform(2.0, 6.0, (V, H, W)))}
    if F:
        targets["embed"] = t(rng.standard_normal((V, F, H, W)))

    def step(planar):
        for x in L.values():
            x.grad = None
        r = render_views(views, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L.get("feature"), targets=targets, planar_depth=planar)
        (r["loss_rgb"].sum() + r["loss_depth"].sum() + (r["loss_embed"].sum() if F else 0.0)).backward()

    times = {False: [], True: []}
    for planar in (False, True):
        for _ in range(a.warmup):
            step(planar)
    for _ in range(a.runs):
        for planar in (False, True):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                step(planar)
            e1.record()
            torch.cuda.synchronize()
            times[planar].append(e0.elapsed_time(e1) / a.steps)
    info = card()
    off, on = float(np.median(times[False])), float(np.median(times[True]))
    # each run times the two arms back to back: the per-run ratio cancels the drift of the shared machine between runs
    ratios = [b / a_ for a_, b in zip(times[False], times[True])]
    print(info)
    print(f"paired on / off ratio: median {float(np.median(ratios)):.3f} ({min(ratios):.3f}-{max(ratios):.3f}) over {len(ratios)} runs")
    print(f"c3 F={F} depth head, fwd+bwd step: planar off {off:.3f} ms ({min(times[False]):.3f}-{max(times[False]):.3f}), "
          f"on {on:.3f} ms ({min(times[True]):.3f}-{max(times[True]):.3f}), ratio {on / off:.3f}")
    # device time per step by kernel group (torch.profiler, CUDA activities, in a pass of its own after the timed runs): the
    # kernels' own durations, which the host-side noise of the step timing does not reach
    from torch.profiler import ProfilerActivity, profile
    groups = ("planar_fwd", "blend_fwd", "blend_bwd", "project_bwd", "project_fwd", "median_depth")
    kern = {}
    for planar in (False, True):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                step(planar)
            torch.cuda.synchronize()
        per = {k: 0.0 for k in groups + ("all kernels",)}
        for ev in prof.key_averages():
            us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if us <= 0:
                continue
            per["all kernels"] += us
            for k in groups:
                if k in ev.key:
                    per[k] += us
        kern[planar] = {k: v / a.steps / 1000.0 for k, v in per.items()}
    print("device ms per step:  " + "  ".join(f"{k}: off {kern[False][k]:.4f} on {kern[True][k]:.4f}" for k in groups + ("all kernels",)))
    print(json.dumps(dict(card=info, F=F, off_ms=off, on_ms=on, ratio=on / off, paired_ratio=float(np.median(ratios)), runs=times,
                          device_ms_per_step={"off": kern[False], "on": kern[True]})))


if __name__ == "__main__":
    main()
