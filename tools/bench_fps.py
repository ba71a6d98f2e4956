"""Cost of farthest-point sampling (gaussian_renderer.farthest_point_sample, mgs_fps) on the clouds it is built for, against
a device-only batched PyTorch loop of the same arithmetic:

    python tools/bench_fps.py [--steps 10] [--warmup 3] [--runs 3] [--torch-steps 2]

  mg       ManiGaussian's size: 16,384 points, n = 512, as a uniform cloud and as its surface cloud;
  c3       500,000 points, n = 512 and 4,096, uniform and surface (a 707 x 707 depth image, 499,849 points);
  policy   a batch of 32 ragged clouds of about 10,000 points (lengths 9,000 .. 10,500), n = 1,024;
  1M       1,000,000 uniform points, n = 512;
  tiers    uniform clouds on each side of the register tiers' thresholds (16,384: 4 points per thread in 8 CTAs, then 16
           in 4; 131,072: 16 points per thread in 16 CTAs, then the streaming tier), n = 512.
The uniform clouds fill SCENE_BOUNDS; the surface clouds are depth images of the scenes.py scene rendered by this package
and unprojected, one point per pixel, the pixels without depth on the camera centre (so they also hold thousands of
duplicates).  The comparison arm keeps every argmax on the device (no .item(), no host read per pick); both arms must
return identical indices and distances before anything is timed.  Each call is timed with CUDA events over --steps calls
(--torch-steps for the loop) after --warmup calls, in --runs runs (median and range), including the state and output
allocations from torch's caching allocator.  Prints the card name and power limit read in the same run, and one JSON line.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_knn import card, surface, time_calls, uniform  # noqa: E402


def torch_fps(points, n, lengths):
    """the definition as a batched PyTorch loop: points [B,P,3], lengths [B]; every op its own kernel, so nothing is fused
    into an FMA, and torch.argmax returns the first of equal maxima"""
    import torch
    B, P, _ = points.shape
    ar = torch.arange(B, device=points.device)
    ok = torch.isfinite(points).all(-1) & (torch.arange(P, device=points.device)[None] < lengths[:, None])
    d = torch.where(ok, torch.tensor(float("inf"), device=points.device), torch.tensor(-1.0, device=points.device))
    index = torch.empty((B, n), dtype=torch.int64, device=points.device)
    dist2 = torch.empty((B, n), dtype=torch.float32, device=points.device)
    x, y, z = points.unbind(-1)
    for t in range(n):
        cur = torch.argmax(d, dim=1)
        val = d[ar, cur]
        index[:, t] = torch.where(val >= 0, cur, -1)
        dist2[:, t] = torch.where(val >= 0, val, float("inf"))
        d[ar, cur] = -1.0
        s = points[ar, cur]
        dx, dy, dz = x - s[:, 0:1], y - s[:, 1:2], z - s[:, 2:3]
        D = (dx * dx + dy * dy) + dz * dz
        d = torch.where(d >= 0, torch.minimum(d, D), d)
    return index, dist2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--torch-steps", type=int, default=2)
    a = ap.parse_args()
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    info = card()
    print(info)
    rng = np.random.default_rng(0)
    cases = []
    mg_surface, dup = surface(16384)
    cases += [("mg uniform", uniform(16384)[None], None, 512),
              (f"mg surface ({dup} on the camera centre)", mg_surface[None], None, 512)]
    c3_surface, dup = surface(500_000)
    c3_uniform = uniform(500_000)[None]
    for n in (512, 4096):
        cases += [("c3 uniform", c3_uniform, None, n), (f"c3 surface ({dup} on the camera centre)", c3_surface[None], None, n)]
    lengths = torch.from_numpy(rng.integers(9_000, 10_501, 32)).cuda()
    cases.append(("policy: 32 ragged clouds of 9,000 .. 10,500", uniform(32 * 10_500, seed=1).reshape(32, 10_500, 3), lengths, 1024))
    cases.append(("1M uniform", uniform(1_000_000, seed=2)[None], None, 512))
    for P in (16384, 16385, 131072, 131073):
        cases.append((f"tier edge {P}", uniform(P, seed=P)[None], None, 512))
    rows = []
    for label, p, L, n in cases:
        B, P = p.shape[:2]
        Lt = L if L is not None else torch.full((B,), P, dtype=torch.int64, device="cuda")
        ours = lambda: GR.farthest_point_sample(p, n, lengths=L)  # noqa: E731
        loop = lambda: torch_fps(p, n, Lt)  # noqa: E731
        got, want = ours(), loop()
        torch.cuda.synchronize()
        assert torch.equal(got["index"], want[0]), f"{label}: the indices differ"
        assert torch.equal(got["dist2"], want[1]), f"{label}: the distances differ"
        med, lo, hi = time_calls(ours, a.steps, a.warmup, a.runs)
        tmed, tlo, thi = time_calls(loop, a.torch_steps, 1, a.runs)
        rows.append(dict(row=label, B=B, P=P, n=n, ms=med, ms_range=[lo, hi], torch_loop_ms=tmed, torch_loop_ms_range=[tlo, thi],
                         speedup=tmed / med, identical=True))
        print(f"{label:52s} B={B:2d} P={P:7d} n={n:4d}  {med:8.3f} ms [{lo:.3f}, {hi:.3f}]   torch loop {tmed:9.3f} ms "
              f"[{tlo:.3f}, {thi:.3f}]  x{tmed / med:6.1f}  identical")
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "torch_steps": a.torch_steps, "rows": rows}))


if __name__ == "__main__":
    main()
