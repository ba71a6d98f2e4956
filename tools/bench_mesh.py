"""Cost of TSDF fusion and marching cubes (gaussian_renderer.tsdf_fuse / marching_cubes; mgs_tsdf_fuse,
mgs_marching_cubes_count / _emit) against device-side PyTorch restatements of the same definitions:

    python tools/bench_mesh.py [--steps 5] [--warmup 2] [--runs 3] [--torch-steps 1]

  fusion   64 views of 640 x 480 on two rings around the scenes.py scene (rendered depth / alpha where alpha > 0.5, and the
           rendered colour), pinhole and distorted (k1 = -0.05, k2 = 0.01, p1 = 0.001, p2 = -0.002), C = 0 and 3, into
           256^3 and 512^3 volumes over SCENE_BOUNDS with trunc 0.02;
  mc       the level-0 surface of the C = 3 volumes with their weights and colour, and the surface of voxelize's 256^3
           density of the same cloud at a tenth of its maximum.
The PyTorch arm of fusion projects every voxel centre per view with the same float32 map and updates the volume with
torch.where; that of marching cubes is tests/mc_ref.py (a table-driven gather) run on the device.  Before anything is timed
both arms must agree: the meshes bit for bit, the volumes on all but a reported fraction of voxels (at most 0.1 %) whose
view-pixel decisions lie at a half-integer, where the two float32 maps round differently.  Each call is timed with CUDA
events over --steps calls after --warmup calls, in --runs runs (median and range), allocations included.  Prints the card
name and power limit read in the same run, and one JSON line.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_knn import card, time_calls  # noqa: E402

W, H, TRUNC = 640, 480, 0.02
DIST = (-0.05, 0.01, 0.001, -0.002, 0.0, 0.0, 0.0, 0.0)


def scene(model):
    """(settings of 64 views, depth [64,H,W], colour [64,3,H,W]) of the scenes.py cloud"""
    import torch
    from manigaussian_b200 import gaussian_renderer as GR, scenes
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    g = scenes.make_gaussians(100_000, seed=0)
    views = []
    for r, h in enumerate((0.4, 1.2)):
        for k in range(32):
            cam = scenes.make_camera(W, H, k + 0.5 * r, 32, height=h)
            kw = {} if model == "pinhole" else dict(distortion=((W - 1) / 2.0, (H - 1) / 2.0) + DIST + (float("inf"),))
            views.append(GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], t(np.zeros(3)), 1.0, t(cam["viewmatrix"]),
                                                       t(cam["projmatrix"]), 0, t(cam["campos"]), False, False, False, **kw))
    cloud = [t(g[k]) for k in ("means3D", "rotations", "scales", "opacities")]
    rgb = t(np.random.default_rng(0).random((len(g["means3D"]), 3)))
    depth, color = [], []
    for v0 in range(0, 64, 16):
        out = GR.render_views(views[v0:v0 + 16], *cloud, pts_rgb=rgb, return_depth=True, return_alpha=True)
        d, a = out["depth"].reshape(-1, H, W), out["alpha"].reshape(-1, H, W)
        depth.append(torch.where(a > 0.5, d / a.clamp_min(1e-12), torch.zeros_like(d)).detach())
        color.append(out["render"].reshape(-1, 3, H, W).detach())
    return views, torch.cat(depth).contiguous(), torch.cat(color).contiguous(), cloud


def _map(s, x, y, z):
    """(px, py, z, ok) of float32 points under one view: screen_mean's map and cull"""
    import torch
    vm = s.viewmatrix.reshape(-1)
    tx = vm[0] * x + vm[4] * y + vm[8] * z + vm[12]
    ty = vm[1] * x + vm[5] * y + vm[9] * z + vm[13]
    tz = vm[2] * x + vm[6] * y + vm[10] * z + vm[14]
    ok = tz > 0.2
    if s.distortion is None:
        pm = s.projmatrix.reshape(-1)
        hx = pm[0] * x + pm[4] * y + pm[8] * z + pm[12]
        hy = pm[1] * x + pm[5] * y + pm[9] * z + pm[13]
        hw = pm[3] * x + pm[7] * y + pm[11] * z + pm[15]
        iw = 1.0 / (hw + 1e-7)
        px = (((hx * iw).double() + 1.0) * W - 1.0) * 0.5
        py = (((hy * iw).double() + 1.0) * H - 1.0) * 0.5
        return px.float(), py.float(), tz, ok
    cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, _ = s.distortion
    iz = 1.0 / tz
    xn, yn = tx * iz, ty * iz
    r2 = xn * xn + yn * yn
    num = 1 + r2 * (k1 + r2 * (k2 + r2 * k3))
    den = 1 + r2 * (k4 + r2 * (k5 + r2 * k6))
    rad = num / den
    xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    n1 = k1 + r2 * (2 * k2 + r2 * 3 * k3)
    q1 = k4 + r2 * (2 * k5 + r2 * 3 * k6)
    r1 = (n1 - rad * q1) / den
    d00 = rad + 2 * xn * xn * r1 + 2 * p1 * yn + 6 * p2 * xn
    d01 = 2 * xn * yn * r1 + 2 * p1 * xn + 2 * p2 * yn
    d11 = rad + 2 * yn * yn * r1 + 6 * p1 * yn + 2 * p2 * xn
    ok = ok & (d00 * d11 - d01 * d01 > 0)
    fx, fy = W / (2.0 * s.tanfovx), H / (2.0 * s.tanfovy)
    return fx * xd + cx, fy * yd + cy, tz, ok


def torch_fuse(views, depth, color, bounds, n):
    """the fusion definition as per-view PyTorch ops on the device (one thread of work per voxel and view)"""
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    pts, _ = GR.voxel_centres(bounds, n, "cuda")
    x, y, z = pts.unbind(-1)
    N = pts.shape[0]
    ts, w = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    C = 0 if color is None else color.shape[1]
    col = torch.zeros((C, N), device="cuda")
    for v, s in enumerate(views):
        px, py, tz, ok = _map(s, x, y, z)
        inside = ok & (px >= -0.5) & (px < W - 0.5) & (py >= -0.5) & (py < H - 0.5)
        i = torch.where(inside, torch.floor(px + 0.5), torch.zeros_like(px)).long().clamp_max(W - 1)
        j = torch.where(inside, torch.floor(py + 0.5), torch.zeros_like(py)).long().clamp_max(H - 1)
        pix = j * W + i
        d = depth[v].reshape(-1)[pix]
        s_ = d - tz
        upd = inside & torch.isfinite(d) & (d > 0) & (s_ >= -TRUNC)
        f = torch.clamp_max(s_ / TRUNC, 1.0)
        w1 = w + 1
        ts = torch.where(upd, (ts * w + f) / w1, ts)
        if C:
            cv = color[v].reshape(C, -1)[:, pix]
            col = torch.where(upd, (col * w + cv) / w1, col)
        w = torch.where(upd, w1, w)
    return ts.view(*n), w.view(*n), (col.view(C, *n) if C else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--torch-steps", type=int, default=1)
    a = ap.parse_args()
    import torch
    import mc_ref
    from manigaussian_b200 import gaussian_renderer as GR, scenes
    info = card()
    print(info)
    bounds = tuple(float(x) for x in scenes.SCENE_BOUNDS)
    rows, volumes = [], []
    cloud = None
    for model in ("pinhole", "distorted"):
        views, depth, color, cloud = scene(model)
        for res in (256, 512):
            for C in (0, 3):
                col = color if C else None
                ours = lambda: GR.tsdf_fuse(views, depth, bounds, res, TRUNC, color=col)  # noqa: E731
                ref = lambda: torch_fuse(views, depth, col, bounds, (res,) * 3)  # noqa: E731
                got, want = ours(), ref()
                torch.cuda.synchronize()
                off = (got["weight"] != want[1]) | ((got["tsdf"] - want[0]).abs() > 1e-4)
                if C:
                    off |= ((got["color"] - want[2]).abs() > 1e-4).any(0)
                frac = float(off.float().mean())
                assert frac <= 1e-3, f"fusion {model} {res}^3 C={C}: {100 * frac:.4f} % of the voxels differ"
                del want
                med, lo, hi = time_calls(ours, a.steps, a.warmup, a.runs)
                tmed, tlo, thi = time_calls(ref, a.torch_steps, 1, a.runs)
                label = f"fusion {model} {res}^3 C={C}"
                rows.append(dict(row=label, ms=med, ms_range=[lo, hi], torch_ms=tmed, torch_ms_range=[tlo, thi], speedup=tmed / med,
                                 voxels_differing_pct=100 * frac))
                print(f"{label:34s} {med:9.3f} ms [{lo:.3f}, {hi:.3f}]   torch {tmed:10.3f} ms [{tlo:.3f}, {thi:.3f}]  "
                      f"x{tmed / med:6.1f}  {100 * frac:.4f} % of voxels differ")
                if C:
                    volumes.append((f"mc {model} {res}^3 tsdf C=3", got))
                else:
                    del got
                torch.cuda.empty_cache()
        del depth, color
    den = GR.voxelize(bounds, 256, *cloud)["density"].detach().contiguous()
    level = 0.1 * float(den.max())
    cases = [(label, (v["tsdf"], 0.0, v["weight"], v["color"])) for label, v in volumes]
    cases.append(("mc voxelize 256^3 density", (den, level, None, None)))
    for label, (vals, lvl, wt, col) in cases:
        ours = lambda: GR.marching_cubes(vals, lvl, bounds, weight=wt, color=col)  # noqa: E731
        ref = lambda: mc_ref.marching_cubes(vals, lvl, bounds, weight=wt, color=col)  # noqa: E731
        got, want = ours(), ref()
        torch.cuda.synchronize()
        for k in ("vertices", "faces", "colors"):
            if want[k] is not None:
                g_, w_ = got[k], want[k]
                same = g_.shape == w_.shape and torch.equal(g_.view(torch.int32) if g_.dtype == torch.float32 else g_,
                                                            w_.view(torch.int32) if w_.dtype == torch.float32 else w_)
                assert same, f"{label}: {k} differ"
        nv, nf = len(got["vertices"]), len(got["faces"])
        del want
        med, lo, hi = time_calls(ours, a.steps, a.warmup, a.runs)
        tmed, tlo, thi = time_calls(ref, a.torch_steps, 1, a.runs)
        rows.append(dict(row=label, vertices=nv, faces=nf, ms=med, ms_range=[lo, hi], torch_ms=tmed, torch_ms_range=[tlo, thi],
                         speedup=tmed / med, identical=True))
        print(f"{label:34s} {med:9.3f} ms [{lo:.3f}, {hi:.3f}]   torch {tmed:10.3f} ms [{tlo:.3f}, {thi:.3f}]  "
              f"x{tmed / med:6.1f}  {nv} vertices, {nf} faces, identical")
        torch.cuda.empty_cache()
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "torch_steps": a.torch_steps, "rows": rows}))


if __name__ == "__main__":
    main()
