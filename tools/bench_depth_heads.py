"""What the fused depth and mask heads buy: one training step with depth supervision, fused against unfused.

    python tools/bench_depth_heads.py [--workloads c3,mg] [--steps 40] [--warmup 5] [--runs 3]

Workloads are bench.py's: c3 (500k Gaussians, 4 views 256x256, F = 32) and mg (ManiGaussian's call: 16k Gaussians, one view
128x128, F = 3), SH degree 1.  Three arms, each one training step (render -> losses -> backward) timed with CUDA events over
--steps steps after --warmup steps, in --runs alternated runs (the table gives the median and the range):
  fused     -- render_views(targets={"rgb", "embed"}): today's fused colour + embedding heads, no depth supervision;
  unfused   -- render_views(return_depth=True, return_alpha=True) and the rgb / embed / depth / mask losses in PyTorch,
               the INTEGRATION.md §4 recipe (its boolean-mask mean synchronises the host);
  fused_dm  -- render_views(targets={"rgb", "embed", "depth", "mask"}): all four heads in the blend epilogue.
It also reports the blend_fwd / blend_bwd stage times per view (mgs_profile_*, CUDA events around each launch; one extra
profiled step per arm, not part of the step timing), and prints the card name, power limit and SM clock and a JSON summary.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (workload definition)
from bench_alpha import card  # noqa: E402

ARMS = ("fused", "unfused", "fused_dm")


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
    w = dict(name=name, P=P, V=V, W=W, H=H, F=F, L=L, views=views)
    from manigaussian_b200.gaussian_renderer import render_views
    with torch.no_grad():  # targets: a depth 1-5 % off the rendered one where the cloud covers the pixel, a thresholded mask
        o = render_views(views, L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=L["feature"], normalize_feature=False, return_depth=True, return_alpha=True)
    gen = torch.Generator(device="cuda").manual_seed(77)
    rnd = lambda *s: torch.rand(*s, device="cuda", generator=gen)
    d = o["depth"] / o["alpha"].clamp_min(1e-4)
    w["targets"] = {"rgb": rnd(V, 3, H, W), "embed": rnd(V, F, H, W) - 0.5,
                    "depth": torch.where(o["alpha"] > 0.3, d * (1.01 + 0.04 * rnd(V, H, W)), torch.zeros_like(d)),
                    "mask": (o["alpha"] > 0.5).float()}
    return w


def step(arm, w):
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    L, tg = w["L"], w["targets"]
    for v in L.values():
        v.grad = None
    kw = dict(features_color=L["shs"], features_language=L["feature"], normalize_feature=False)
    args = (w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"])
    if arm == "unfused":
        o = render_views(*args, return_depth=True, return_alpha=True, **kw)
        loss = ((o["render"] - tg["rgb"]) ** 2).mean() + (1 - torch.nn.functional.cosine_similarity(o["render_embed"], tg["embed"], dim=1).mean())
        d = o["depth"] / o["alpha"].clamp_min(1e-4)
        valid = (tg["depth"] > 0) & (o["alpha"] > 0.5).detach()
        loss = loss + (d - tg["depth"]).abs()[valid].mean()
        loss = loss + torch.nn.functional.binary_cross_entropy(o["alpha"].clamp(1e-4, 1 - 1e-4), tg["mask"])
    else:
        t = tg if arm == "fused_dm" else {"rgb": tg["rgb"], "embed": tg["embed"]}
        o = render_views(*args, targets=t, **kw)
        loss = o["loss_rgb"].mean() + o["loss_embed"].mean()
        if arm == "fused_dm":
            loss = loss + o["loss_depth"].mean() + o["loss_mask"].mean()
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
    ap.add_argument("--workloads", default="c3,mg")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_depth_heads needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    result = {}
    for name in a.workloads.split(","):
        w = workload(name)
        ms = {k: [] for k in ARMS}
        for _ in range(a.runs):
            for arm in ARMS:
                ms[arm].append(timed(arm, w, a.steps, a.warmup))
        rows = {}
        for arm in ARMS:
            st = blend_stages(arm, w)
            rows[arm] = dict(step_ms=float(np.median(ms[arm])), step_range=[min(ms[arm]), max(ms[arm])],
                             blend_fwd_ms_per_view=st["blend_fwd"], blend_bwd_ms_per_view=st["blend_bwd"])
            r = rows[arm]
            print(f"{name} {arm:8s} step {r['step_ms']:.3f} ms [{r['step_range'][0]:.3f}, {r['step_range'][1]:.3f}]  "
                  f"blend_fwd {r['blend_fwd_ms_per_view']:.4f} ms/view  blend_bwd {r['blend_bwd_ms_per_view']:.4f} ms/view", flush=True)
        result[name] = dict(P=w["P"], views=w["V"], WxH=f"{w['W']}x{w['H']}", F=w["F"], arms=rows)
        del w
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "workloads": result}))


if __name__ == "__main__":
    main()
