"""Lifting 2D maps onto the cloud: gaussian_renderer.lift_views against the autograd route it replaces.

    python tools/bench_lift.py [--calls 30] [--warmup 5] [--runs 3] [--workloads c3,mg] [--widths 0,3,32,128]

Workloads are bench.py's c3 (500k Gaussians, 4 views 256x256) and mg (16k Gaussians, 1 view 128x128), each with C map
channels.  Two arms per (workload, C), each one call timed with CUDA events over --calls calls after --warmup calls, in
--runs alternated runs of one process (median and range):
  lift      -- lift_views(cameras, ..., maps) -> {"lifted" [P,C], "weight" [P]};
  autograd  -- render_views of a zero [P, C + 1] feature tensor that requires grad (normalize_feature=False), then
               torch.autograd.grad of render_embed with the maps and a ones channel as the cotangent: dL/dfeature is
               [lifted | weight], computed through a full forward and backward.
It also reports the kernel time per launch of one profiled call (mgs_profile_*: the lift kernel runs under the blend_fwd
stage; the autograd arm's blend_fwd and blend_bwd), and reads the card name, power limit and SM clock in the same run.
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


def workload(name, C):
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    wl = bench.WORKLOADS[name]
    P, V, W, H = wl["P"], wl["views"], wl["W"], wl["H"]
    g = scenes.make_gaussians(P, F=0, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    L = {k: t(g[k]) for k in ("means3D", "rotations", "scales", "opacities")}
    L["rgb"] = torch.rand(P, 3, device="cuda")
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           0, t(c["campos"]), False, False, True) for c in cams]
    maps = torch.rand(V, C, H, W, device="cuda")
    cot = torch.cat([maps, torch.ones(V, 1, H, W, device="cuda")], 1)
    return dict(name=f"{name} C={C}", P=P, V=V, W=W, H=H, C=C, L=L, views=views, maps=maps, cot=cot)


def call(arm, w):
    import torch
    from manigaussian_b200.gaussian_renderer import lift_views, render_views
    L = w["L"]
    if arm == "lift":
        return lift_views(w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"], w["maps"] if w["C"] else None)
    f = torch.zeros(w["P"], w["C"] + 1, device="cuda", requires_grad=True)
    o = render_views(w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"], pts_rgb=L["rgb"], features_language=f,
                     normalize_feature=False)
    (g,) = torch.autograd.grad(o["render_embed"], [f], w["cot"])
    return {"lifted": g[:, :w["C"]], "weight": g[:, w["C"]]}


def timed(arm, w, calls, warmup):
    import torch
    for _ in range(warmup):
        call(arm, w)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        call(arm, w)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def stages(arm, w):
    """blend_fwd (the lift kernel in the lift arm) and blend_bwd ms per launch of one profiled call"""
    import torch
    from manigaussian_b200 import _binding
    torch.cuda.synchronize()
    _binding.profile_enable(True)
    _binding.profile_read()
    call(arm, w)
    torch.cuda.synchronize()
    prof = _binding.profile_read()
    _binding.profile_enable(False)
    return {k: prof[k][0] / max(prof[k][1], 1) for k in ("blend_fwd", "blend_bwd")}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default="c3,mg")
    ap.add_argument("--widths", default="0,3,32,128")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lift needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    arms = ("lift", "autograd")
    summary = {}
    for wname in a.workloads.split(","):
        for width in a.widths.split(","):
            w = workload(wname, int(width))
            ms = {k: [] for k in arms}
            for _ in range(a.runs):
                for arm in arms:
                    ms[arm].append(timed(arm, w, a.calls, a.warmup))
            rows = {}
            for arm in arms:
                st = stages(arm, w)
                rows[arm] = dict(call_ms=float(np.median(ms[arm])), call_range=[min(ms[arm]), max(ms[arm])])
                if arm == "lift":
                    rows[arm]["lift_kernel_ms_per_launch"] = st["blend_fwd"]
                else:
                    rows[arm]["blend_fwd_ms_per_launch"], rows[arm]["blend_bwd_ms_per_launch"] = st["blend_fwd"], st["blend_bwd"]
                r = rows[arm]
                kern = " ".join(f"{k} {v:.3f}" for k, v in r.items() if k.endswith("per_launch"))
                print(f"{w['name']:12s} {arm:8s} call {r['call_ms']:.3f} ms [{r['call_range'][0]:.3f}, {r['call_range'][1]:.3f}]  "
                      f"{kern}", flush=True)
            summary[w["name"]] = dict(P=w["P"], views=w["V"], WxH=f"{w['W']}x{w['H']}", C=w["C"], arms=rows,
                                      speedup=rows["autograd"]["call_ms"] / rows["lift"]["call_ms"])
            del w
            torch.cuda.empty_cache()
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "calls": a.calls, "warmup": a.warmup, "runs": a.runs, "workloads": summary}))


if __name__ == "__main__":
    main()
