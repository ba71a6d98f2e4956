"""Cost of point visibility (gaussian_renderer.point_visibility, mgs_visibility_views) on three workloads:

    python tools/bench_visibility.py [--steps 20] [--warmup 5] [--runs 3]

  c3 Q=16k  -- bench.py's c3 cloud and views (500k Gaussians, 4 views 256x256), a 25^3 grid of voxel centres over SCENE_BOUNDS;
  c3 Q=1M   -- the same with a 100^3 grid (the occupancy recipe of INTEGRATION.md section 16);
  mg Q=16k  -- ManiGaussian's real size (16384 Gaussians, one view 128x128), the 25^3 grid.
Each call is timed with CUDA events over --steps calls after --warmup calls, in --runs alternated runs (median and range).
As a yardstick for a walk over the same lists, lift_views (weights only) on the same views is timed the same way.
Pairs walked: for every in-view point, its cut (the instances of its tile in front of it), counted here from a render's tile
ranges, point lists and depths (the kernel keeps no counter); the early stop at T < 1e-4 is not subtracted, so the rate is
candidate pairs per second.  Prints the card name and power limit, and one JSON line.
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


def workload(name, n):
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, gaussian_renderer as GR, scenes
    wl = bench.WORKLOADS[name]
    P, V, W, H = wl["P"], wl["views"], wl["W"], wl["H"]
    g = scenes.make_gaussians(P, F=0, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           bench.SH_DEGREE, t(c["campos"]), False, False, False) for c in cams]
    pts, _ = GR.voxel_centres(scenes.SCENE_BOUNDS, n, "cuda")
    G = dict(pts_xyz=t(g["means3D"]), rotations=t(g["rotations"]), scales=t(g["scales"]), opacity=t(g["opacities"]), shs=t(g["shs"]))
    return dict(name=f"{name} Q={n ** 3}", P=P, V=V, W=W, H=H, views=views, pts=pts, G=G)


def pairs(w, out):
    """sum over views and in-view points of the point's cut, from a render of the same views"""
    import torch
    from manigaussian_b200 import rasterizer as R
    G, P = w["G"], w["P"]
    outs, _ = R.rasterize_views_raw(w["views"], G["pts_xyz"], None, None, G["opacity"], G["scales"], G["rotations"], 1.0, None,
                                    G["shs"], bench.SH_DEGREE, False)
    torch.cuda.synchronize()
    total = 0
    for v, o in enumerate(outs):
        W, H = w["W"], w["H"]
        T = ((W + 15) // 16) * ((H + 15) // 16)
        cap, Rn = int(o[0]), o.num_rendered()

        def arr(which, name, state, a0, a1, dtype, count):
            off = R.state_array(which, name, state, a0, a1) - state.data_ptr()
            return state[off:off + count * torch.empty((), dtype=dtype).element_size()].view(dtype)

        depths = arr("geometry", "depths", o[4], P, 0, torch.float32, P).double()
        plist = arr("binning", "point_list", o[5], cap, 0, torch.int32, Rn).long()
        tiles = arr("binning", "tile_ids", o[5], cap, 0, torch.int32, Rn).long()
        ranges = arr("image", "ranges", o[6], W, H, torch.int32, 2 * T).view(T, 2).long()
        key = tiles.double() * 1e4 + depths[plist]  # depth < 1e4: the tile lists sorted one after the other
        inv = out["in_view"][v]
        uv, d = out["uv"][v][inv].double(), out["depth"][v][inv].double()
        ix = torch.clamp(torch.floor(uv[:, 0] + 0.5), max=W - 1).long()
        iy = torch.clamp(torch.floor(uv[:, 1] + 0.5), max=H - 1).long()
        tq = (iy // 16) * ((W + 15) // 16) + ix // 16
        cut = torch.searchsorted(key, tq.double() * 1e4 + d) - ranges[tq, 0]
        total += int(cut.sum())
    return total


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_visibility needs a CUDA device")
    info = card()
    print(f"card: {info}")
    rows = []
    for name, n in (("c3", 25), ("c3", 100), ("mg", 25)):
        w = workload(name, n)
        G = w["G"]
        vis = lambda: GR.point_visibility(w["views"], w["pts"], G["pts_xyz"], G["rotations"], G["scales"], G["opacity"])  # noqa: E731
        lift = lambda: GR.lift_views(w["views"], G["pts_xyz"], G["rotations"], G["scales"], G["opacity"], None)  # noqa: E731
        out = vis()
        npairs = pairs(w, out)
        inview = float(out["in_view"].float().mean())
        tv, tl = [], []
        for _ in range(a.runs):
            tv.append(timed(vis, a.steps, a.warmup))
            tl.append(timed(lift, a.steps, a.warmup))
        mv, ml = float(np.median(tv)), float(np.median(tl))
        row = dict(workload=w["name"], P=w["P"], views=w["V"], W=w["W"], H=w["H"], in_view=round(inview, 3), pairs=npairs,
                   visibility_ms=round(mv, 3), visibility_range=[round(min(tv), 3), round(max(tv), 3)],
                   pairs_per_s=float(f"{npairs / (mv * 1e-3):.3g}"), lift_views_ms=round(ml, 3),
                   lift_range=[round(min(tl), 3), round(max(tl), 3)])
        rows.append(row)
        print(f"{w['name']:>12}: point_visibility {mv:.3f} ms ({min(tv):.3f}-{max(tv):.3f}), {npairs:.3e} pairs, "
              f"{row['pairs_per_s']:.3g} pairs/s, in view {inview:.2f}; lift_views {ml:.3f} ms")
        del w, out
        torch.cuda.empty_cache()
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "rows": rows}))


if __name__ == "__main__":
    main()
