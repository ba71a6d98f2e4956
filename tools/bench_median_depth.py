"""Cost of the median-depth plane on a render_views training step, on two of bench.py's workloads:
c3 (500k Gaussians, 4 views 256x256, F = 32) and mg (16k Gaussians, 1 view 128x128, F = 3), SH degree 1.

    python tools/bench_median_depth.py [--steps 40] [--warmup 5] [--runs 3] [--workloads c3,mg]

Two arms per workload, each one training step (render -> loss -> backward) timed with CUDA events over --steps steps after
--warmup steps, in --runs alternated runs (the table gives the median and the range):
  off     -- render_views without the median, colour and feature cotangents;
  median  -- the same with return_median_depth=True and a random median-depth cotangent.
It also reports the blend_fwd / blend_bwd stage times per view (mgs_profile_*, CUDA events around each launch; one extra
profiled step per arm, not part of the step timing), and prints the card name, power limit and SM clock and a JSON summary.
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


def workload(name):
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    wl = bench.WORKLOADS[name]
    P, V, W, H, F = wl["P"], wl["views"], wl["W"], wl["H"], wl["F"]
    g = scenes.make_gaussians(P, F=F, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    L = {k: t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs", "feature")}
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           bench.SH_DEGREE, t(c["campos"]), False, False, True) for c in cams]
    rng = np.random.default_rng(77)
    cts = [t(rng.standard_normal(s)) for s in ((V, 3, H, W), (V, F, H, W), (V, H, W))]
    return dict(name=name, P=P, V=V, W=W, H=H, F=F, L=L, views=views, cts=cts)


def step(arm, w):
    from manigaussian_b200.gaussian_renderer import render_views
    L, cts = w["L"], w["cts"]
    for v in L.values():
        v.grad = None
    o = render_views(w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                     features_language=L["feature"], normalize_feature=False, return_median_depth=(arm == "median"))
    loss = (o["render"] * cts[0]).sum() + (o["render_embed"] * cts[1]).sum()
    if arm == "median":
        loss = loss + (o["median_depth"] * cts[2]).sum()
    loss.backward()
    return loss


def timed(arm, w, steps, warmup):
    import torch
    for _ in range(warmup):
        step(arm, w)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step(arm, w)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def blend_stages(arm, w):
    """blend_fwd / blend_bwd ms per launch (= per view) of one profiled step"""
    import torch
    from manigaussian_b200 import _binding
    torch.cuda.synchronize()
    _binding.profile_enable(True)
    _binding.profile_read()
    step(arm, w)
    torch.cuda.synchronize()
    prof = _binding.profile_read()
    _binding.profile_enable(False)
    return {k: prof[k][0] / max(prof[k][1], 1) for k in ("blend_fwd", "blend_bwd")}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default="c3,mg")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_median_depth needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    arms = ("off", "median")
    summary = {}
    for name in a.workloads.split(","):
        w = workload(name)
        ms = {k: [] for k in arms}
        for _ in range(a.runs):
            for arm in arms:
                ms[arm].append(timed(arm, w, a.steps, a.warmup))
        rows = {}
        for arm in arms:
            st = blend_stages(arm, w)
            rows[arm] = dict(step_ms=float(np.median(ms[arm])), step_range=[min(ms[arm]), max(ms[arm])],
                             blend_fwd_ms_per_view=st["blend_fwd"], blend_bwd_ms_per_view=st["blend_bwd"])
            r = rows[arm]
            print(f"{name} {arm:6s} step {r['step_ms']:.3f} ms [{r['step_range'][0]:.3f}, {r['step_range'][1]:.3f}]  "
                  f"blend_fwd {r['blend_fwd_ms_per_view']:.3f} ms/view  blend_bwd {r['blend_bwd_ms_per_view']:.3f} ms/view", flush=True)
        summary[name] = dict(P=w["P"], views=w["V"], WxH=f"{w['W']}x{w['H']}", F=w["F"], arms=rows)
        del w
        torch.cuda.empty_cache()
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "step": "render_views training step", "steps": a.steps, "warmup": a.warmup, "runs": a.runs,
                      "workloads": summary}))


if __name__ == "__main__":
    main()
