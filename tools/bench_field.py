"""Field queries: gaussian_renderer.query_field on grids and random points, and a chunked float32 PyTorch evaluation of the
same definition on the GPU.

    python tools/bench_field.py [--calls 10] [--warmup 3] [--torch-calls 1] [--only mg-grid,c3-grid,random]

Workloads (the cloud is scenes.make_gaussians, seed 1234; features random normal):
  mg-grid   16k Gaussians, the 100^3 voxel centres over SCENE_BOUNDS, C = 0, 3, 32 (PerAct / GNFactor-sized voxel input);
  c3-grid   the c3 cloud (500k Gaussians), the same grid, C = 32, 128;
  random    16k Gaussians, 10^6 uniform random points in SCENE_BOUNDS, C = 32.
Per row: forward and forward + backward (random cotangents of density and features; gradients of the points and of every
Gaussian tensor), each one call timed with CUDA events over --calls calls after --warmup calls (median), and the
(bin, Gaussian) pairs per query the binning produced.  On mg-grid the torch arm evaluates the dense [Q, P] pairs in chunks
of 2048 queries (forward; forward + backward chunk by chunk with autograd.grad).  The card's name, power limit and SM clock
are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

THRESH = float(np.float32(1.0) / np.float32(255.0))


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def cloud(P, C):
    import torch
    from manigaussian_b200 import scenes
    g = scenes.make_gaussians(P, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    rng = np.random.default_rng(1)
    f = t(rng.normal(0, 1, (P, C))) if C else None
    return [t(g["means3D"]), t(g["rotations"]), t(g["scales"]), t(g["opacities"]), f]


def points(kind):
    import torch
    from manigaussian_b200 import scenes
    from manigaussian_b200.gaussian_renderer import voxel_centres
    if kind == "grid":
        return voxel_centres(scenes.SCENE_BOUNDS, 100, "cuda")[0]
    lo, hi = scenes.SCENE_BOUNDS[:3], scenes.SCENE_BOUNDS[3:]
    rng = np.random.default_rng(2)
    return torch.from_numpy((lo + (hi - lo) * rng.random((1000000, 3))).astype(np.float32)).cuda()


def ours(pts, cl, backward):
    import torch
    from manigaussian_b200.gaussian_renderer import query_field
    if not backward:
        with torch.no_grad():
            return query_field(pts, *cl)
    leaves = [x.detach().requires_grad_(True) if x is not None else None for x in [pts] + cl]
    out = query_field(*leaves)
    loss = (out["density"] * torch.cos(out["density"].detach())).sum()  # a cotangent that differs per query
    if out["features"] is not None:
        loss = loss + (out["features"] * out["features"].detach()).sum()
    return torch.autograd.grad(loss, [x for x in leaves if x is not None])


def torch_field(pts, cl, backward, chunk=2048):
    """the definition, float32, dense over [chunk, P] pairs"""
    import torch
    mu, rot, s, o, f = cl
    leaves = [x.detach().requires_grad_(backward) if x is not None else None for x in (pts, mu, rot, s, o, f)]
    grads = [torch.zeros_like(x) if (backward and x is not None) else None for x in leaves]
    x_all, mu, rot, s, o, f = leaves
    outs = []
    for a in range(0, x_all.shape[0], chunk):
        with torch.set_grad_enabled(backward):
            q = rot / rot.norm(dim=1, keepdim=True)
            r, qx, qy, qz = q.unbind(1)
            R = torch.stack([
                torch.stack([1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy + r * qz), 2 * (qx * qz - r * qy)], 1),
                torch.stack([2 * (qx * qy - r * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz + r * qx)], 1),
                torch.stack([2 * (qx * qz + r * qy), 2 * (qy * qz - r * qx), 1 - 2 * (qx * qx + qy * qy)], 1)], 1)
            A = R / s[:, :, None]
            x = x_all[a:a + chunk]
            u = torch.einsum("qpj,pkj->qpk", x[:, None, :] - mu[None], A)
            g = o.reshape(1, -1) * torch.exp(-0.5 * (u * u).sum(-1))
            g = torch.where(g >= THRESH, g, torch.zeros_like(g))
            d = g.sum(1)
            feat = g @ f if f is not None else None
        if backward:
            loss = (d * torch.cos(d.detach())).sum() + ((feat * feat.detach()).sum() if feat is not None else 0)
            live = [i for i, t in enumerate(leaves) if t is not None]
            gs = torch.autograd.grad(loss, [leaves[i] for i in live])
            for i, gi in zip(live, gs):
                grads[i] += gi
        else:
            outs.append((d, feat))
    return grads if backward else outs


def timed(fn, calls, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--torch-calls", type=int, default=1)
    ap.add_argument("--only", default="mg-grid,c3-grid,random")
    a = ap.parse_args(argv)
    import torch
    from manigaussian_b200.rasterizer import field_query_raw
    if not torch.cuda.is_available():
        raise SystemExit("bench_field needs a CUDA device")
    import bench
    rows = []
    plan = {"mg-grid": (16384, "grid", (0, 3, 32)), "c3-grid": (bench.WORKLOADS["c3"]["P"], "grid", (32, 128)),
            "random": (16384, "random", (32,))}
    for name in a.only.split(","):
        P, kind, widths = plan[name]
        pts = points(kind)
        for C in widths:
            cl = cloud(P, C)
            n = field_query_raw(pts, cl[0], cl[2], cl[1], cl[3], cl[4])[4]
            row = {"workload": name, "P": P, "Q": pts.shape[0], "C": C, "pairs_per_query": n / pts.shape[0],
                   "fwd_ms": timed(lambda: ours(pts, cl, False), a.calls, a.warmup),
                   "fwd_bwd_ms": timed(lambda: ours(pts, cl, True), a.calls, a.warmup)}
            if name == "mg-grid":
                row["torch_fwd_ms"] = timed(lambda: torch_field(pts, cl, False), a.torch_calls, 1)
                row["torch_fwd_bwd_ms"] = timed(lambda: torch_field(pts, cl, True), a.torch_calls, 1)
            rows.append(row)
            print(json.dumps(row), flush=True)
            del cl
            torch.cuda.empty_cache()
    print(json.dumps({"card": card()}))
    return rows


if __name__ == "__main__":
    main()
