"""Cost of camera rays (gaussian_renderer.camera_rays, mgs_camera_rays) in grid mode, forward and forward + backward, per camera
model, against a float32 PyTorch restatement of the same maps with the same Newton iterations:

    python tools/bench_camera_rays.py [--steps 50] [--warmup 5]

  256    V = 4 views of 256 x 256
  720p   V = 4 views of 1280 x 720
The backward asks for the pixel-independent camera gradients of a learnable pose (camera_batch) and, for fisheye and
distorted views, a learnable field of view; the restatement gets them from autograd through its iterations.  Both are timed
with CUDA events over --steps calls after --warmup calls (the forward on prebuilt views, the backward rebuilding
them from the pose each call, as a training step does), and their rays are compared (valid masks and the largest
difference of the valid rays).  At ManiGaussian's 128 x 128 the call is a single launch of microseconds: launch-bound.
Prints the card name and power limit read in the same run, and one JSON line per case.
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

MODELS = ("pinhole", "ortho", "fisheye", "distorted")
FE = (0.02, -0.01, 0.003, -0.001)
DC = (-0.05, 0.01, 0.001, -0.002, 0.0, 0.0, 0.0, 0.0)
FISHEYE_ITERS, DIST_ITERS = 16, 20  # camera.cuh's FISHEYE_RAY_ITERS and DIST_RAY_ITERS


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def _projection(model, W, H):
    import torch
    from manigaussian_b200 import cameras as C
    if model == "ortho":
        return torch.tensor(C.projection_orthographic(0.01, 100.0, 1.0, 1.0 * H / W), dtype=torch.float32, device="cuda")
    K = np.array([[0.8 * W, 0, (W - 1) / 2], [0, 0.8 * W, (H - 1) / 2], [0, 0, 1]])
    return torch.tensor(C.projection_from_intrinsics(0.1, 100.0, K[None], H, W)[0], dtype=torch.float32, device="cuda")


def _views(model, W, H, V, w2c, tf, proj):
    """V settings of the model around the origin; w2c [V,4,4] and tf [V,2] device tensors (the learnable pose and fov),
    proj the model's [4,4] projection (_projection)"""
    import torch
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    out = []
    for v in range(V):
        wvt = w2c[v].transpose(0, 1)
        kw = {}
        if model == "fisheye":
            kw["fisheye"] = ((W - 1) / 2, (H - 1) / 2) + FE + (1.4,)
        elif model == "distorted":
            kw["distortion"] = ((W - 1) / 2, (H - 1) / 2) + DC + (float("inf"),)
        tx, ty = (tf[v, 0], tf[v, 1]) if model in ("fisheye", "distorted") else ((1.0, 1.0 * H / W) if model == "ortho" else (W / (1.6 * W), H / (1.6 * W)))
        out.append(GaussianRasterizationSettings(H, W, tx, ty, torch.zeros(3, device="cuda"), 1.0, wvt, wvt @ proj.T, 0,
                                                 torch.zeros(3, device="cuda"), False, False, False, orthographic=model == "ortho", **kw))
    return out


def torch_rays(model, views, W, H):
    """the float32 PyTorch restatement: origin, direction [V,H*W,3] and valid [V,H*W] of every pixel centre"""
    import torch
    dev = views[0].viewmatrix.device
    v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32),
                          indexing="ij")
    u, v = u.reshape(-1), v.reshape(-1)
    os_, ds_, oks = [], [], []
    for s in views:
        vm = s.viewmatrix.reshape(4, 4).T  # row-major: t = vm[:3, :3] p + vm[:3, 3]
        if model in ("pinhole", "ortho"):
            pm = s.projmatrix.reshape(4, 4).T
            nx, ny = (2 * u + 1) / W - 1, (2 * v + 1) / H - 1
            A = torch.stack([pm[0, :3] - nx[:, None] * pm[3, :3], pm[1, :3] - ny[:, None] * pm[3, :3], vm[2, :3].expand(len(u), 3)], -2)
            w = pm[3, 3] + 1e-7
            b = torch.stack([nx * w - pm[0, 3], ny * w - pm[1, 3], (-vm[2, 3]).expand(len(u))], -1)
            e3 = torch.zeros_like(b)
            e3[:, 2] = 1
            sol = torch.linalg.solve(A, torch.stack([b, e3], -1))
            o, d, ok = sol[..., 0], sol[..., 1], torch.ones_like(u, dtype=torch.bool)
        else:
            fx, fy = W / (2 * s.tanfovx), H / (2 * s.tanfovy)
            lens = s.fisheye if model == "fisheye" else s.distortion
            xd, yd = (u - lens[0]) / fx, (v - lens[1]) / fy
            if model == "fisheye":
                k1, k2, k3, k4, tmax = lens[2:7]
                rho = lambda t2: 1 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)))  # noqa: E731
                d1f = lambda t2: 1 + t2 * (3 * k1 + t2 * (5 * k2 + t2 * (7 * k3 + t2 * 9 * k4)))  # noqa: E731
                td = torch.sqrt(xd * xd + yd * yd)
                ok = td <= tmax * rho(tmax * tmax)
                th = torch.clamp(td, max=tmax)
                for _ in range(FISHEYE_ITERS):
                    th = torch.clamp(th - (th * rho(th * th) - td) / d1f(th * th), 0.0, tmax)
                t2 = th * th
                tq = torch.where(t2 < 1 / 64, 1 + t2 * (1 / 3 + t2 * (2 / 15 + t2 * 17 / 315)), torch.tan(th) / torch.where(t2 > 0, th, 1))
                sc = tq / rho(t2)
                X, Y = sc * xd, sc * yd
            else:
                k1, k2, p1, p2, k3, k4, k5, k6 = lens[2:10]
                X, Y = xd, yd
                for _ in range(DIST_ITERS):
                    xx, yy, xy = X * X, Y * Y, X * Y
                    r2 = xx + yy
                    N, Q = 1 + r2 * (k1 + r2 * (k2 + r2 * k3)), 1 + r2 * (k4 + r2 * (k5 + r2 * k6))
                    N1, Q1 = k1 + r2 * (2 * k2 + r2 * 3 * k3), k4 + r2 * (2 * k5 + r2 * 3 * k6)
                    R = N / Q
                    R1 = (N1 - R * Q1) / Q
                    ex = xd - (X * R + 2 * p1 * xy + p2 * (r2 + 2 * xx))
                    ey = yd - (Y * R + p1 * (r2 + 2 * yy) + 2 * p2 * xy)
                    d00 = R + 2 * xx * R1 + 2 * p1 * Y + 6 * p2 * X
                    d01 = 2 * xy * R1 + 2 * p1 * X + 2 * p2 * Y
                    d11 = R + 2 * yy * R1 + 6 * p1 * Y + 2 * p2 * X
                    det = d00 * d11 - d01 * d01
                    X, Y = X + (d11 * ex - d01 * ey) / det, Y + (d00 * ey - d01 * ex) / det
                ok = det > 0
            Ri = torch.linalg.inv(vm[:3, :3])
            o = (-(Ri @ vm[:3, 3])).expand(len(u), 3)
            d = torch.stack([X, Y, torch.ones_like(X)], -1) @ Ri.T
        os_.append(o)
        ds_.append(d)
        oks.append(ok)
    return torch.stack(os_), torch.stack(ds_), torch.stack(oks)


def time_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_camera_rays needs a CUDA device")
    print(json.dumps({"card": card()}))
    V = 4
    for size, (W, H) in (("256", (256, 256)), ("720p", (1280, 720))):
        for model in MODELS:
            g = np.random.default_rng(0)
            w2c0 = []
            for _ in range(V):
                th = 0.3 * g.standard_normal()
                R = np.array([[math.cos(th), 0, math.sin(th)], [0, 1, 0], [-math.sin(th), 0, math.cos(th)]])
                M = np.eye(4)
                M[:3, :3], M[:3, 3] = R, [0.1, -0.05, 2.0]
                w2c0.append(M)
            w2c = torch.tensor(np.stack(w2c0), dtype=torch.float32, device="cuda").requires_grad_(True)
            tf = torch.tensor([[W / (1.6 * W), H / (1.6 * W)]] * V, dtype=torch.float32, device="cuda").requires_grad_(True)
            wo, wd = torch.randn(V, H, W, 3, device="cuda"), torch.randn(V, H, W, 3, device="cuda")

            proj = _projection(model, W, H)
            fixed = _views(model, W, H, V, w2c.detach(), tf.detach(), proj)

            def ours_fwd():
                return GR.camera_rays(fixed)

            def ours_bwd():
                out = GR.camera_rays(_views(model, W, H, V, w2c, tf, proj))
                loss = (out["origin"] * wo).nan_to_num().sum() + (out["direction"] * wd).nan_to_num().sum()
                return torch.autograd.grad(loss, [w2c, tf], allow_unused=True)

            def torch_fwd():
                with torch.no_grad():
                    return torch_rays(model, fixed, W, H)

            def torch_bwd():
                o, d, ok = torch_rays(model, _views(model, W, H, V, w2c, tf, proj), W, H)
                m = ok[..., None]
                loss = (torch.where(m, o, 0) * wo.reshape(V, -1, 3)).sum() + (torch.where(m, d, 0) * wd.reshape(V, -1, 3)).sum()
                return torch.autograd.grad(loss, [w2c, tf], allow_unused=True)

            ours = ours_fwd()
            ref = torch_fwd()
            ok = ours["valid"].reshape(V, -1)
            same_mask = bool((ok == ref[2]).all())
            diff = max(float((ours[k].reshape(V, -1, 3)[ok] - r[ok]).abs().max()) for k, r in (("origin", ref[0]), ("direction", ref[1])))
            row = dict(size=size, model=model, V=V, W=W, H=H, valid_masks_equal=same_mask, max_abs_diff=diff,
                       ours_fwd_ms=time_ms(ours_fwd, args.steps, args.warmup), torch_fwd_ms=time_ms(torch_fwd, args.steps, args.warmup),
                       ours_fwd_bwd_ms=time_ms(ours_bwd, args.steps, args.warmup),
                       torch_fwd_bwd_ms=time_ms(torch_bwd, args.steps, args.warmup))
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
