"""Cost of the optical-flow plane on a render_views training step, on bench.py's c3 shape (500k Gaussians, 4 views
256x256, SH degree 1) at F = 32, 8 and 0 feature channels.

    python tools/bench_flow.py [--steps 30] [--warmup 5] [--runs 3] [--widths 32,8,0]

Three arms per width, each one training step (render -> loss -> backward) timed with CUDA events over --steps steps after
--warmup steps, in --runs alternated runs of one process (the table gives the median and the range):
  off       -- render_views without flow: colour and feature cotangents;
  flow      -- the same with flow_xyz (next-frame means, a leaf that requires grad) and a random flow cotangent;
  features  -- what a caller had to do without the plane: per-view displacements m' - m computed in PyTorch through the
               view's projection matrix, appended to the features as F + 2 channels, one render_views call per view.
It also reports the blend_fwd / blend_bwd stage times per view (mgs_profile_*, one extra profiled step per arm, not part of
the step timing), and prints the card name, power limit and SM clock and a JSON summary.
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


def workload(F):
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    wl = bench.WORKLOADS["c3"]
    P, V, W, H = wl["P"], wl["views"], wl["W"], wl["H"]
    g = scenes.make_gaussians(P, F=F, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    L = {k: t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs") + (("feature",) if F else ())}
    rng0 = np.random.default_rng(5)
    L["next"] = t(np.asarray(g["means3D"]) + 0.01 * rng0.standard_normal(np.shape(g["means3D"]))).requires_grad_(True)
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    mk = lambda inc: [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),  # noqa: E731
                                                    bench.SH_DEGREE, t(c["campos"]), False, False, inc) for c in cams]
    rng = np.random.default_rng(77)
    cts = [t(rng.standard_normal(s)) for s in ((V, 3, H, W), (V, max(F, 1), H, W), (V, 2, H, W))]
    return dict(name=f"c3 F={F}", P=P, V=V, W=W, H=H, F=F, L=L, views=mk(F > 0), views_feat=mk(True), cts=cts)


def torch_delta(L, s):
    """per-view displacements in PyTorch: what a caller computes without the plane (pinhole views, next mean in front)"""
    import torch
    pm = s.projmatrix

    def mean(p):
        h = p @ pm[:3] + pm[3]
        ndc = h[:, :2] / (h[:, 3:4] + 1e-7)
        return torch.stack([((ndc[:, 0] + 1.0) * s.image_width - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * s.image_height - 1.0) * 0.5], 1)

    return mean(L["next"]) - mean(L["means3D"])


def step(arm, w):
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    L, cts, F = w["L"], w["cts"], w["F"]
    for v in L.values():
        v.grad = None
    feat = L.get("feature")
    if arm != "features":
        o = render_views(w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                         features_language=feat, normalize_feature=False,
                         flow_xyz=L["next"] if arm == "flow" else None)
        loss = (o["render"] * cts[0]).sum()
        if F:
            loss = loss + (o["render_embed"] * cts[1]).sum()
        if arm == "flow":
            loss = loss + (o["flow"] * cts[2]).sum()
    else:
        loss = 0.0
        for v, s in enumerate(w["views_feat"]):
            n = torch_delta(L, s)
            o = render_views([s], L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                             features_language=torch.cat([feat, n], 1) if F else n, normalize_feature=False)
            loss = loss + (o["render"][0] * cts[0][v]).sum() + (o["render_embed"][0, F:] * cts[2][v]).sum()
            if F:
                loss = loss + (o["render_embed"][0, :F] * cts[1][v]).sum()
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
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--widths", default="32,8,0")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_flow needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    arms = ("off", "flow", "features")
    summary = {}
    for width in a.widths.split(","):
        w = workload(int(width))
        name = w["name"]
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
            print(f"{name} {arm:8s} step {r['step_ms']:.3f} ms [{r['step_range'][0]:.3f}, {r['step_range'][1]:.3f}]  "
                  f"blend_fwd {r['blend_fwd_ms_per_view']:.3f} ms/view  blend_bwd {r['blend_bwd_ms_per_view']:.3f} ms/view", flush=True)
        summary[name] = dict(P=w["P"], views=w["V"], WxH=f"{w['W']}x{w['H']}", F=w["F"], arms=rows)
        del w
        torch.cuda.empty_cache()
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "step": "render_views training step", "steps": a.steps, "warmup": a.warmup, "runs": a.runs,
                      "workloads": summary}))


if __name__ == "__main__":
    main()
