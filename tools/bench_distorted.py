"""Distorted-pinhole views: bench.py's c3 cloud rendered through OpenCV distorted cameras against the same number of pinhole ones.

    python tools/bench_distorted.py [--steps 30] [--warmup 5] [--runs 3]

Three arms on the c3 workload (500k Gaussians, 256x256 views), each one render_views forward + backward step timed with
CUDA events over --steps steps after --warmup steps, in --runs alternated runs of one process (median and range):
  persp4   -- bench.py's 4 pinhole cameras;
  dist4    -- 4 distorted cameras at the same poses and focal lengths, a centred principal point and a Kinect-like
              rational 8-coefficient calibration;
  mixed4   -- 2 pinhole and 2 distorted cameras of those poses in one call.
It also reports the project_fwd and project_bwd stage times (ms per launch, mgs_profile_*) of one profiled step, and reads
the card name, power limit and SM clock in the same run.
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

KINECT_D = (0.45, -0.08, 0.0006, -0.0004, -0.01, 0.78, 0.02, -0.06)   # an Azure-Kinect-like rational calibration


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def setup():
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, cameras, scenes
    wl = bench.WORKLOADS["c3"]
    P, V, W, H = wl["P"], wl["views"], wl["W"], wl["H"]
    g = scenes.make_gaussians(P, F=0, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    L = {k: t(g[k]).requires_grad_() for k in ("means3D", "rotations", "scales", "opacities", "shs")}
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    persp = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           bench.SH_DEGREE, t(c["campos"]), False, False, False) for c in cams]
    # the same poses and focal lengths (W / (2 tan_fovx)), principal point at the image centre
    c2w = np.stack([np.linalg.inv(np.asarray(c["viewmatrix"], np.float64).T) for c in cams])
    K = np.stack([[[W / (2 * c["tanfovx"]), 0, (W - 1) / 2], [0, H / (2 * c["tanfovy"]), (H - 1) / 2], [0, 0, 1]] for c in cams])
    fb = cameras.build_distorted_cameras(K, np.array([KINECT_D] * V), c2w, W, H, device="cuda")
    dist = [fb.settings(i, bg, bench.SH_DEGREE, False) for i in range(V)]
    return dict(P=P, W=W, H=H, L=L, arms={"persp4": persp, "dist4": dist, "mixed4": persp[:2] + dist[2:]})


def step(s, views):
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    L = s["L"]
    o = render_views(views, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"])
    loss = (o["render"] * o["render"].detach()).sum()
    torch.autograd.grad(loss, [L["means3D"], L["scales"], L["rotations"], L["opacities"], L["shs"]])


def timed(s, views, steps, warmup):
    import torch
    for _ in range(warmup):
        step(s, views)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step(s, views)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def stages(s, views):
    import torch
    from manigaussian_b200 import _binding
    torch.cuda.synchronize()
    _binding.profile_enable(True)
    _binding.profile_read()
    step(s, views)
    torch.cuda.synchronize()
    prof = _binding.profile_read()
    _binding.profile_enable(False)
    return {k: prof[k][0] / max(prof[k][1], 1) for k in ("project_fwd", "project_bwd")}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_distorted needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    s = setup()
    ms = {k: [] for k in s["arms"]}
    for _ in range(a.runs):
        for k, views in s["arms"].items():
            ms[k].append(timed(s, views, a.steps, a.warmup))
    rows = {}
    for k, views in s["arms"].items():
        st = stages(s, views)
        rows[k] = dict(step_ms=float(np.median(ms[k])), step_range=[min(ms[k]), max(ms[k])],
                       project_fwd_ms_per_launch=st["project_fwd"], project_bwd_ms_per_launch=st["project_bwd"])
        r = rows[k]
        print(f"{k:9s} step {r['step_ms']:.3f} ms [{r['step_range'][0]:.3f}, {r['step_range'][1]:.3f}]  project_fwd "
              f"{r['project_fwd_ms_per_launch']:.4f}  project_bwd {r['project_bwd_ms_per_launch']:.4f} ms per launch", flush=True)
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "P": s["P"],
                      "WxH": f"{s['W']}x{s['H']}", "arms": rows}))


if __name__ == "__main__":
    main()
