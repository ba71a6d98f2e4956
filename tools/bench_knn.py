"""Cost of the k-nearest-neighbour search (gaussian_renderer.knn, mgs_knn) on the clouds it is built for:

    python tools/bench_knn.py [--steps 20] [--warmup 5] [--runs 3]

  mg     ManiGaussian's size: 16,384 points, k = 3 and 20;
  c3     500,000 points, k = 3 and 20;
each as a uniform cloud in SCENE_BOUNDS and as a surface cloud: a depth image of the scenes.py scene rendered by this
package at sqrt(N) x sqrt(N) pixels and unprojected, one point per pixel, the pixels without depth on the camera centre
(so the surface rows also time thousands of duplicates).  A row of 20,000 copies of one point (k = 20) times the
all-duplicate case, and torch.cdist + topk at 16,384 points (k = 20) is the comparison.  Every call is timed with CUDA events
over --steps calls after --warmup calls, in --runs runs (median and range); each call includes the state allocation from
torch's caching allocator.  Prints the card name and power limit read in the same run, and one JSON line.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def surface(n, seed=0):
    """the scene's depth image at side x side pixels (side = round(sqrt(n))), unprojected"""
    import torch
    from manigaussian_b200 import rasterizer as R, scenes
    side = int(round(math.sqrt(n)))
    cam = scenes.make_camera(side, side, 0, 4)
    g = scenes.make_gaussians(16384, seed=seed)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    s = R.GaussianRasterizationSettings(side, side, cam["tanfovx"], cam["tanfovy"], t(np.zeros(3)), 1.0, t(cam["viewmatrix"]),
                                        t(cam["projmatrix"]), g["sh_degree"], t(cam["campos"]), False, False, False)
    outs, _ = R.rasterize_views_raw([s], t(g["means3D"]), None, None, t(g["opacities"]), t(g["scales"]), t(g["rotations"]), 1.0,
                                    None, t(g["shs"]), g["sh_degree"], False, return_depth=True, return_alpha=True)
    depth, alpha = (outs[0][i].double().reshape(side, side) for i in (7, 8))
    z = torch.where(alpha > 0.5, depth / alpha.clamp_min(1e-12), torch.zeros_like(depth))
    f = side / (2.0 * cam["tanfovx"])
    v, u = torch.meshgrid(torch.arange(side, device="cuda", dtype=torch.float64),
                          torch.arange(side, device="cuda", dtype=torch.float64), indexing="ij")
    c = (side - 1) / 2.0
    pc = torch.stack([(u - c) / f * z, (v - c) / f * z, z, torch.ones_like(z)], -1).reshape(-1, 4)
    pw = pc @ torch.linalg.inv(torch.from_numpy(np.asarray(cam["viewmatrix"], np.float64)).cuda())
    return pw[:, :3].float().contiguous(), int((alpha <= 0.5).sum())


def uniform(n, seed=0):
    import torch
    from manigaussian_b200 import scenes
    rng = np.random.default_rng(seed)
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    return torch.from_numpy((lo + (hi - lo) * rng.random((n, 3))).astype(np.float32)).cuda()


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


def cdist_topk(p, k):
    import torch
    d = torch.cdist(p, p)
    d.fill_diagonal_(float("inf"))
    return torch.topk(d, k, dim=1, largest=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    info = card()
    print(info)
    rows = []
    for label, n in (("mg", 16384), ("c3", 500_000)):
        sp, dup = surface(n)
        for kind, p, extra in (("uniform", uniform(n), ""), ("surface", sp, f" ({dup} on the camera centre)")):
            for k in (3, 20):
                med, lo, hi = time_calls(lambda: GR.knn(p, k), a.steps, a.warmup, a.runs)
                rows.append(dict(row=f"{label} {kind}{extra}", N=int(p.shape[0]), k=k, ms=med, ms_range=[lo, hi]))
                print(f"{rows[-1]['row']:48s} N={p.shape[0]:7d} k={k:2d}  {med:8.3f} ms  [{lo:.3f}, {hi:.3f}]")
    p = torch.tensor([[0.1, -0.2, 1.0]], device="cuda").repeat(20000, 1)
    med, lo, hi = time_calls(lambda: GR.knn(p, 20), a.steps, a.warmup, a.runs)
    rows.append(dict(row="20k duplicates of one point", N=20000, k=20, ms=med, ms_range=[lo, hi]))
    print(f"{rows[-1]['row']:48s} N=  20000 k=20  {med:8.3f} ms  [{lo:.3f}, {hi:.3f}]")
    p = uniform(16384)
    med, lo, hi = time_calls(lambda: cdist_topk(p, 20), a.steps, a.warmup, a.runs)
    rows.append(dict(row="torch.cdist + topk, mg uniform", N=16384, k=20, ms=med, ms_range=[lo, hi]))
    print(f"{rows[-1]['row']:48s} N=  16384 k=20  {med:8.3f} ms  [{lo:.3f}, {hi:.3f}]")
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "rows": rows}))


if __name__ == "__main__":
    main()
