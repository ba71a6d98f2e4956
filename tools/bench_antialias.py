"""Cost of the anti-aliased projection (opacity compensation) on a render_views training step, at bench.py's c3 (500k Gaussians,
4 views 256x256, F = 32, SH degree 1) and mg (ManiGaussian's call: 16384 Gaussians, 1 view 128x128, F = 3) workloads.

    python tools/bench_antialias.py [--steps 40] [--warmup 5] [--runs 3] [--workloads c3,mg]

Two arms per workload, each one training step (render_views -> colour and feature cotangents -> backward) timed with CUDA
events over --steps steps after --warmup steps, in --runs alternated runs (the table gives the median and the range):
  off -- render_views(antialiasing=False), the default;
  aa  -- render_views(antialiasing=True).
It also reports project_fwd, project_bwd, blend_fwd and blend_bwd per launch (mgs_profile_*, CUDA events around each launch; one
extra profiled step per arm, not part of the step timing), and prints the card name, power limit and SM clock before and after,
and a JSON summary.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (workload definitions)
from bench_alpha import card  # noqa: E402

STAGES = ("project_fwd", "project_bwd", "blend_fwd", "blend_bwd")


def workload(name):
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    wl = bench.WORKLOADS[name]
    P, V, W, H, F = wl["P"], wl["views"], wl["W"], wl["H"], wl["F"]
    g = scenes.make_gaussians(P, F=F, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    L = {k: t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs", "feature")}
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           bench.SH_DEGREE, t(c["campos"]), False, False, True) for c in cams]
    rng = np.random.default_rng(77)
    cts = [t(rng.standard_normal(s)) for s in ((V, 3, H, W), (V, F, H, W))]
    return dict(name=name, P=P, V=V, W=W, H=H, F=F, L=L, views=views, cts=cts)


def step(arm, w):
    from manigaussian_b200.gaussian_renderer import render_views
    L, cts = w["L"], w["cts"]
    for v in L.values():
        v.grad = None
    o = render_views(w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                     features_language=L["feature"], normalize_feature=False, antialiasing=(arm == "aa"))
    loss = (o["render"] * cts[0]).sum() + (o["render_embed"] * cts[1]).sum()
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


def stage_times(arm, w):
    """ms per launch of the four stages in one profiled step"""
    import torch
    from manigaussian_b200 import _binding
    torch.cuda.synchronize()
    _binding.profile_enable(True)
    _binding.profile_read()
    step(arm, w)
    torch.cuda.synchronize()
    prof = _binding.profile_read()
    _binding.profile_enable(False)
    return {k: prof[k][0] / max(prof[k][1], 1) for k in STAGES}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default="c3,mg")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_antialias needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    arms = ("off", "aa")
    result = {}
    for name in a.workloads.split(","):
        w = workload(name)
        ms = {k: [] for k in arms}
        for _ in range(a.runs):
            for arm in arms:
                ms[arm].append(timed(arm, w, a.steps, a.warmup))
        rows = {}
        for arm in arms:
            st = stage_times(arm, w)
            rows[arm] = dict(step_ms=float(np.median(ms[arm])), step_range=[min(ms[arm]), max(ms[arm])], **{k + "_ms": v for k, v in st.items()})
            r = rows[arm]
            print(f"{name:3s} {arm:4s} step {r['step_ms']:.3f} ms [{r['step_range'][0]:.3f}, {r['step_range'][1]:.3f}]  " +
                  "  ".join(f"{k} {r[k + '_ms']:.4f}" for k in STAGES) + " ms/launch", flush=True)
        result[name] = dict(P=w["P"], views=w["V"], WxH=f"{w['W']}x{w['H']}", F=w["F"], arms=rows)
        del w
        torch.cuda.empty_cache()
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "workloads": result}))


if __name__ == "__main__":
    main()
