"""Cost of the alpha plane on bench.py's c3 step (render_views: 500k Gaussians, 4 views 256x256, F = 32, SH degree 1).

    python tools/bench_alpha.py [--steps 40] [--warmup 5] [--runs 3]

Three arms, each one training step (render -> loss -> backward) timed with CUDA events over --steps steps after --warmup steps,
in --runs alternated runs (the table gives the median and the range):
  off    -- render_views without alpha, colour and feature cotangents;
  alpha  -- the same with return_alpha=True and a random alpha cotangent;
  white  -- the workaround without an alpha plane: `off` plus a second render_views of the same cloud with colours 1 on a
            black background, whose red channel is alpha (projection, binning and both blends again).
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

import bench  # noqa: E402  (workload definition)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def workload():
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    wl = bench.WORKLOADS["c3"]
    P, V, W, H, F = wl["P"], wl["views"], wl["W"], wl["H"], wl["F"]
    g = scenes.make_gaussians(P, F=F, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    L = {k: t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs", "feature")}
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           bench.SH_DEGREE, t(c["campos"]), False, False, True) for c in cams]
    white_views = [v._replace(include_feature=False) for v in views]
    rng = np.random.default_rng(77)
    cts = [t(rng.standard_normal(s)) for s in ((V, 3, H, W), (V, F, H, W), (V, H, W))]
    return dict(P=P, V=V, W=W, H=H, F=F, L=L, views=views, white_views=white_views, ones=torch.ones(P, 3, device="cuda"), cts=cts)


def step(arm, w):
    from manigaussian_b200.gaussian_renderer import render_views
    L, cts = w["L"], w["cts"]
    for v in L.values():
        v.grad = None
    o = render_views(w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                     features_language=L["feature"], normalize_feature=False, return_alpha=(arm == "alpha"))
    loss = (o["render"] * cts[0]).sum() + (o["render_embed"] * cts[1]).sum()
    if arm == "alpha":
        loss = loss + (o["alpha"] * cts[2]).sum()
    elif arm == "white":
        white = render_views(w["white_views"], L["means3D"], L["rotations"], L["scales"], L["opacities"], pts_rgb=w["ones"])
        loss = loss + (white["render"][:, 0] * cts[2]).sum()
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
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_alpha needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    w = workload()
    arms = ("off", "alpha", "white")
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
        print(f"{arm:6s} step {r['step_ms']:.3f} ms [{r['step_range'][0]:.3f}, {r['step_range'][1]:.3f}]  "
              f"blend_fwd {r['blend_fwd_ms_per_view']:.3f} ms/view  blend_bwd {r['blend_bwd_ms_per_view']:.3f} ms/view", flush=True)
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "workload": "c3 render_views", "P": w["P"], "views": w["V"], "WxH": f"{w['W']}x{w['H']}", "F": w["F"],
                      "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "arms": rows}))


if __name__ == "__main__":
    main()
