"""Cost of the fused neighbour regularisers (gaussian_renderer.neighbour_regularisers, mgs_neighbour_reg) against
INTEGRATION.md section 17's PyTorch restatement, on the lists they are built for:

    python tools/bench_neighbour_reg.py [--steps 20] [--warmup 5] [--runs 3]

  mg     ManiGaussian's size: 16,384 Gaussians;
  c3     500,000 Gaussians;
each uniform in SCENE_BOUNDS with random rotations, the next frame a small deformation of it (1 mm offsets, rotations
perturbed by 0.05), on knn lists at k = 20 with weights exp(-2000 d2).  Both are timed forward only and forward + backward
(all four inputs requiring grad) with CUDA events over --steps calls after --warmup calls, in --runs runs (median and
range), and their peak-memory increase over the inputs (torch.cuda.max_memory_allocated) is taken from one call.  The
neighbour lists are built once, outside the timing.  Prints the card name and power limit read in the same run, and one
JSON line.
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


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def inputs(n, k, seed=0):
    import torch
    from manigaussian_b200 import gaussian_renderer as GR, scenes
    rng = np.random.default_rng(seed)
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    xyz = (lo + (hi - lo) * rng.random((n, 3))).astype(np.float32)
    rot = rng.normal(size=(n, 4)).astype(np.float32)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    xyz_next = xyz + np.float32(1e-3) * rng.normal(size=(n, 3)).astype(np.float32)
    rot_next = rot + np.float32(0.05) * rng.normal(size=(n, 4)).astype(np.float32)
    nn = GR.knn(t(xyz), k)
    return t(xyz), t(rot), t(xyz_next), t(rot_next), nn["index"], torch.exp(-2000.0 * nn["dist2"])


def restatement(xyz, rot, xyz_next, rot_next, j, w):
    from neighbour_reg_ref64 import integration_restatement
    return integration_restatement(xyz, rot, xyz_next, rot_next, j, w)


def fused(xyz, rot, xyz_next, rot_next, j, w):
    from manigaussian_b200 import gaussian_renderer as GR
    out = GR.neighbour_regularisers(xyz, rot, xyz_next, rot_next, j, w)
    return out["rigid"], out["rotation"], out["isometry"]


def call(fn, ins, backward):
    import torch
    if not backward:
        with torch.no_grad():
            return fn(*ins)
    leaves = [t.detach().requires_grad_() for t in ins[:4]]
    r, t, i = fn(*leaves, *ins[4:])
    (r + t + i).backward()


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    info = card()
    print(info)
    rows = []
    for label, n in (("mg", 16384), ("c3", 500_000)):
        ins = inputs(n, 20)
        for name, fn in (("fused", fused), ("restatement", restatement)):
            for backward in (False, True):
                f = lambda: call(fn, ins, backward)  # noqa: E731
                med, lo, hi = time_calls(f, a.steps, a.warmup, a.runs)
                mib = peak_mib(f)
                rows.append(dict(row=f"{label} {name} {'fwd+bwd' if backward else 'fwd'}", P=n, k=20, ms=med, ms_range=[lo, hi],
                                 peak_MiB=mib))
                print(f"{rows[-1]['row']:30s} P={n:7d} k=20  {med:8.3f} ms  [{lo:.3f}, {hi:.3f}]  peak +{mib:9.1f} MiB")
        del ins
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "rows": rows}))


if __name__ == "__main__":
    main()
