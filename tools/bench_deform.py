"""Cost of the fused control-graph deformation (gaussian_renderer.deform_gaussians, mgs_deform) against INTEGRATION.md
section 20's PyTorch restatement (tests/deform_ref64.py, in float32 on the GPU), on the workloads it is built for:

    python tools/bench_deform.py [--steps 20] [--warmup 5] [--runs 3] [--kernels]

  mg     ManiGaussian's size: 16,384 Gaussians on 512 nodes, k = 4 and k = 8;
  c3     500,000 Gaussians on 4,096 nodes, k = 8;
  rigid  500,000 Gaussians on 3 nodes, k = 1 (rigid segments: every Gaussian of a segment names the same node, the
         contended case of the backward's node reduction).
The Gaussians are uniform in SCENE_BOUNDS with random unit rotations; the nodes are a random subsample of them with random
rotations and 1 cm translations; the lists come from knn(node_xyz, k, queries=xyz) with weights softmax(-d^2 / 2 sigma^2)
(rigid: a random segment id with weight 1).  Each is timed forward only, and forward + backward both with all six inputs
requiring grad and next-frame only (node_rot and node_t), with CUDA events over --steps calls after --warmup calls, in
--runs runs (median and range).  The peak-memory increase over the inputs (torch.cuda.max_memory_allocated) is taken from
one call.  The lists are built once, outside the timing.  With --kernels it prints instead the fused call's device time
per kernel over --steps calls (torch.profiler, in a run of its own).  Prints the card name and power limit read in the same
run, and one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = (("mg", 16384, 512, 4), ("mg", 16384, 512, 8), ("c3", 500_000, 4096, 8), ("rigid", 500_000, 3, 1))
MODES = ("fwd", "fwd+bwd all", "fwd+bwd next")


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def inputs(label, n, nodes, k, seed=0):
    import torch
    from manigaussian_b200 import gaussian_renderer as GR, scenes
    rng = np.random.default_rng(seed)
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    xyz = t(lo + (hi - lo) * rng.random((n, 3)))
    rot = t(rng.normal(size=(n, 4)))
    rot = rot / rot.norm(dim=-1, keepdim=True)
    node_xyz = xyz[torch.from_numpy(rng.permutation(n)[:nodes]).cuda()].clone()
    node_rot = t(np.array([1.0, 0.0, 0.0, 0.0]) + 0.1 * rng.normal(size=(nodes, 4)))
    node_t = t(0.01 * rng.normal(size=(nodes, 3)))
    if label == "rigid":
        index = torch.from_numpy(rng.integers(0, nodes, (n, 1))).cuda()
        weight = torch.ones((n, 1), device="cuda")
    else:
        nn = GR.knn(node_xyz, k, queries=xyz)
        d2 = torch.where(nn["index"] >= 0, nn["dist2"], torch.full_like(nn["dist2"], float("inf")))
        sigma = float((hi - lo).max()) / nodes ** (1 / 3)
        index, weight = nn["index"], torch.softmax(-d2 / (2 * sigma ** 2), 1)
    return xyz, rot, node_xyz, node_rot, node_t, index, weight


def restatement(*a):
    from deform_ref64 import deform_ref64
    return deform_ref64(*a)


def fused(*a):
    from manigaussian_b200 import gaussian_renderer as GR
    out = GR.deform_gaussians(*a)
    return out["xyz"], out["rot"]


def call(fn, ins, mode):
    import torch
    if mode == "fwd":
        with torch.no_grad():
            return fn(*ins)
    grad = (True,) * 5 + (False, True) if mode == "fwd+bwd all" else (False, False, False, True, True, False, False)
    leaves = [t.detach().requires_grad_() if g else t for t, g in zip(ins, grad)]
    x, r = fn(*leaves)
    (x.sum() + r.sum()).backward()


def time_calls(fn, steps, warmup, runs):
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / steps)
    return float(np.median(ms)), float(min(ms)), float(max(ms))


def peak_mib(fn):
    import torch
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def kernel_us(fn, steps):
    """device time per call of each deform kernel (torch.profiler, CUDA activity only), in microseconds"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0].split("::")[-1]
        if name.startswith("deform_"):
            t = getattr(e, "self_device_time_total", None)
            out[name] = round((e.self_cuda_time_total if t is None else t) / steps, 2)
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--kernels", action="store_true",
                    help="instead of the timings: the fused call's device time per kernel (torch.profiler, a run of its own)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deform needs a CUDA device")
    info = card()
    print(info)
    rows = []
    for label, n, nodes, k in WORKLOADS:
        ins = inputs(label, n, nodes, k)
        if a.kernels:
            for mode in MODES:
                us = kernel_us(lambda: call(fused, ins, mode), a.steps)  # noqa: B023
                rows.append(dict(row=f"{label} fused {mode}", P=n, N=nodes, k=k, kernel_us=us))
                print(f"{rows[-1]['row']:32s} P={n:7d} N={nodes:5d} k={k:2d}  " + "  ".join(f"{kk} {v:.2f} us" for kk, v in us.items()))
            del ins
            continue
        for name, fn in (("fused", fused), ("restatement", restatement)):
            for mode in MODES:
                f = lambda: call(fn, ins, mode)  # noqa: E731
                med, lo, hi = time_calls(f, a.steps, a.warmup, a.runs)
                mib = peak_mib(f)
                rows.append(dict(row=f"{label} {name} {mode}", P=n, N=nodes, k=k, ms=med, ms_range=[lo, hi], peak_MiB=mib))
                print(f"{rows[-1]['row']:32s} P={n:7d} N={nodes:5d} k={k:2d}  {med:8.3f} ms  [{lo:.3f}, {hi:.3f}]"
                      f"  peak +{mib:9.1f} MiB")
        del ins
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "rows": rows}))


if __name__ == "__main__":
    main()
