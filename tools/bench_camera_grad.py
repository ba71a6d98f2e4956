"""What camera gradients cost: one render_views training step with camera gradients off and on, and the kernels that
change.

    python tools/bench_camera_grad.py [--workloads c3,mg] [--steps 40] [--warmup 5] [--runs 3] [--intrinsics]

Workloads are bench.py's: c3 (500k Gaussians, 4 views 256x256, F = 32) and mg (ManiGaussian's call: 16k Gaussians, one view
128x128, F = 3), SH degree 1.  One step is render_views(targets={"rgb", "embed"}) -> loss_rgb + loss_embed -> backward.  In
the "on" arm every view's viewmatrix, projmatrix and campos require grad, so the backward runs the CAM instantiation of
project_bwd and camera_grad_reduce_kernel and returns the camera gradients.  --intrinsics adds the "intr" arm: the "on" arm
whose views also carry their field of view as device tensors that require grad (the projection forward and backward read
it on the device, and the backward returns dL/dtan_fov as well) -- and "project_fwd" joins the profiled kernels.  It also
adds "on_batch" and "intr_batch": the same two camera set-ups as one CameraBatch of [V,...] leaf tensors (the form
cameras.camera_batch returns), whose tensors the renderer takes as they are instead of stacking per-view settings; the
difference between the settings and the batch arms is the per-view stacking and its autograd.  Step times are CUDA events over --steps steps
after --warmup steps, in --runs alternated runs (median and range).  One more step per arm runs under torch.profiler (CUDA
activities, a run of its own) for the project_bwd and reduce kernel times per launch.  The card's name, power limit and SM
clocks are read in the same run; a JSON summary is printed last.
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

ARMS = ["off", "on"]
INTR_ARMS = ["intr", "on_batch", "intr_batch"]


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
    arms = {}
    for arm in ARMS:
        if arm.endswith("_batch"):
            from manigaussian_b200.cameras import CameraBatch
            st = lambda k: torch.stack([t(c[k]) for c in cams]).requires_grad_(True)  # noqa: E731
            tf = None
            if arm == "intr_batch":
                tf = torch.tensor([[c["tanfovx"], c["tanfovy"]] for c in cams], dtype=torch.float32, device="cuda").requires_grad_()
            arms[arm] = CameraBatch(FovX=None, FovY=None, tanfovx=[c["tanfovx"] for c in cams], tanfovy=[c["tanfovy"] for c in cams],
                                    width=W, height=H, world_view_transform=st("viewmatrix"), full_proj_transform=st("projmatrix"),
                                    camera_center=st("campos"), tan_fov=tf)
            continue
        mk = (lambda x: t(x).requires_grad_(True)) if arm != "off" else t
        fov = (lambda x: torch.tensor(float(x), device="cuda", requires_grad=True)) if arm == "intr" else (lambda x: x)
        arms[arm] = [GaussianRasterizationSettings(H, W, fov(c["tanfovx"]), fov(c["tanfovy"]), bg, 1.0, mk(c["viewmatrix"]),
                                                   mk(c["projmatrix"]), bench.SH_DEGREE, mk(c["campos"]), False, False, True)
                     for c in cams]
    gen = torch.Generator(device="cuda").manual_seed(77)
    targets = {"rgb": torch.rand(V, 3, H, W, device="cuda", generator=gen),
               "embed": torch.rand(V, F, H, W, device="cuda", generator=gen) - 0.5}
    return dict(name=name, P=P, V=V, L=L, arms=arms, targets=targets)


def step(arm, w):
    from manigaussian_b200.gaussian_renderer import render_views
    L = w["L"]
    for v in L.values():
        v.grad = None
    o = render_views(w["arms"][arm], L["means3D"], L["rotations"], L["scales"], L["opacities"], features_color=L["shs"],
                     features_language=L["feature"], normalize_feature=False, targets=w["targets"])
    loss = o["loss_rgb"].mean() + o["loss_embed"].mean()
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


def kernel_times(arm, w):
    """ms per launch of the project_bwd kernels and the camera reduce in one profiled step (torch.profiler)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    step(arm, w)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(arm, w)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        for key in ("project_fwd", "project_bwd", "camera_grad_reduce"):
            if key in e.name and e.device_type.name == "CUDA":
                tot, n = out.get(key, (0.0, 0))
                out[key] = (tot + e.device_time / 1000.0, n + 1)
    return {k: dict(ms_per_launch=round(v[0] / v[1], 5), launches=v[1]) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,mg")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--intrinsics", action="store_true", help="add the arm with device-side, learnable fields of view")
    a = ap.parse_args()
    if a.intrinsics:
        ARMS.extend(INTR_ARMS)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_camera_grad: needs a CUDA device")
    summary = {"card": card(), "workloads": {}}
    for name in a.workloads.split(","):
        w = workload(name)
        times = {arm: [] for arm in ARMS}
        for _ in range(a.runs):
            for arm in ARMS:
                times[arm].append(timed(arm, w, a.steps, a.warmup))
        res = {arm: dict(median_ms=round(float(np.median(v)), 4), min_ms=round(min(v), 4), max_ms=round(max(v), 4))
               for arm, v in times.items()}
        res["kernels"] = {arm: kernel_times(arm, w) for arm in ARMS}
        summary["workloads"][name] = res
        print(f"{name}: " + "  ".join(f"{arm} {res[arm]['median_ms']:.3f} ms [{res[arm]['min_ms']:.3f}, {res[arm]['max_ms']:.3f}]"
                                      for arm in ARMS) + f"  kernels {res['kernels']}")
        del w
    summary["card_after"] = card()
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
