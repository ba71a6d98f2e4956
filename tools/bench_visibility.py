"""Cost of point visibility (gaussian_renderer.point_visibility, mgs_visibility_views) on three workloads:

    python tools/bench_visibility.py [--steps 20] [--warmup 5] [--runs 3] [--backward]

  c3 Q=16k  -- bench.py's c3 cloud and views (500k Gaussians, 4 views 256x256), a 25^3 grid of voxel centres over SCENE_BOUNDS;
  c3 Q=1M   -- the same with a 100^3 grid (the occupancy recipe of INTEGRATION.md section 16);
  mg Q=16k  -- ManiGaussian's real size (16384 Gaussians, one view 128x128), the 25^3 grid.
Each call is timed with CUDA events over --steps calls after --warmup calls, in --runs alternated runs (median and range).
As a yardstick for a walk over the same lists, lift_views (weights only) on the same views is timed the same way.
Pairs walked: for every in-view point, its cut (the instances of its tile in front of it), counted here from a render's tile
ranges, point lists and depths (the kernel keeps no counter); the early stop at T < 1e-4 is not subtracted, so the rate is
candidate pairs per second.  Prints the card name and power limit, and one JSON line.

--backward times point_visibility(differentiable=True) instead, forward and backward, on:
  c3 voxels   -- the c3 cloud and views with the 100^3 grid (hot tiles: ~15k points in one tile, hundreds of warps per tile
                 sending their reductions to the same blend-stage rows);
  c3 rays     -- the c3 cloud and views with 65,536 points on camera rays of view 0 at depths through the scene (RGB-D
                 free-space samples);
  mg voxels   -- ManiGaussian's size with the 25^3 grid.
The loss is sum w T + sum of uv and depth with seeded weights.  The backward is timed with CUDA events in three arms, each
with its own inputs requiring grad only where the arm asks for gradients: the points and the cloud, the cloud alone, and the
points alone.  Every arm replays the walk of every point.  The cloud arms sum the replay's terms over each warp, send them
to the Gaussians' blend-stage rows and run the per-Gaussian stage; the points arm does neither and runs the point chain
instead.  The cost of the warp sums and row reductions, hot rows included, is the difference in vis_query_bwd_kernel's
device time between the cloud arm and the points arm.  Kernel times come from torch.profiler in a pass of its own after the
timed runs (per call, summed over the views: the query backward, the point chain and the per-Gaussian stage).  The peak memory of one forward + backward is reported with and
without differentiable (the latter: the forward alone).
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


def rays(w, Q, seed=0):
    """Q points on camera rays of view 0 (uniform over the image) at depths uniform in the cloud's depth range"""
    import torch
    rng = np.random.default_rng(seed)
    s = w["views"][0]
    vm = s.viewmatrix.double().cpu().numpy().reshape(4, 4).T  # world -> view
    c2w = np.linalg.inv(vm)
    W, H = w["W"], w["H"]
    tx, ty = float(s.tanfovx), float(s.tanfovy)
    m = w["G"]["pts_xyz"].double().cpu().numpy()
    z = (m @ vm[:3, :3].T + vm[:3, 3])[:, 2]
    lo, hi = np.percentile(z[z > 0.2], [5, 95])
    u, v = rng.uniform(0, W, Q), rng.uniform(0, H, Q)
    d = rng.uniform(lo, hi, Q)
    t = np.stack([(2 * u / W - 1) * tx * d, (2 * v / H - 1) * ty * d, d], 1)
    return torch.from_numpy((t @ c2w[:3, :3].T + c2w[:3, 3]).astype(np.float32)).cuda()


# the backward's kernels, by a substring of their names in the profiler's trace
BWD_KERNELS = ("vis_query_bwd_kernel", "vis_points_bwd_kernel", "project_bwd_views")


def kernel_ms(fn, calls):
    """mean device time per call of each of BWD_KERNELS over `calls` calls of fn, from torch.profiler (CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in BWD_KERNELS}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        for k in BWD_KERNELS:
            if k in e.key:
                out[k] += us / 1e3 / calls
    return {k: round(v, 3) for k, v in out.items()}


def backward_arm(a):
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    rows = []
    for label, name, n in (("c3 voxels", "c3", 100), ("c3 rays", "c3", None), ("mg voxels", "mg", 25)):
        w = workload(name, n or 25)
        if n is None:
            w["pts"] = rays(w, 65536)
        G = w["G"]
        keys = ("pts_xyz", "rotations", "scales", "opacity")
        Q, V = w["pts"].shape[0], w["V"]
        gen = torch.Generator(device="cuda").manual_seed(0)
        wT = torch.rand(V, Q, device="cuda", generator=gen)

        def leaves(points, cloud):
            """the arm's inputs: its own clones, requiring grad only where the arm asks for gradients (the node's
            needs_input_grad is fixed at the forward from requires_grad)"""
            p = w["pts"].clone().requires_grad_(points)
            c = [G[k].clone().requires_grad_(cloud) for k in keys]
            return p, c, ([p] if points else []) + (c if cloud else [])

        arms = {"both": leaves(True, True), "cloud": leaves(False, True), "points": leaves(True, False)}

        def fwd(arm):
            p, c, _ = arms[arm]
            return GR.point_visibility(w["views"], p, *c, differentiable=True)

        def loss(out):
            return (wT * out["transmittance"]).sum() + torch.nan_to_num(out["uv"]).sum() * 1e-3 + torch.nan_to_num(out["depth"]).sum()

        def step(arm):
            return torch.autograd.grad(loss(fwd(arm)), arms[arm][2])

        def bwd(arm):
            lv = loss(fwd(arm))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            torch.autograd.grad(lv, arms[arm][2])
            e1.record()
            return e0, e1

        def timed_bwd(arm):
            for _ in range(a.warmup):
                bwd(arm)
            ev = [bwd(arm) for _ in range(a.steps)]
            torch.cuda.synchronize()
            return float(np.mean([e0.elapsed_time(e1) for e0, e1 in ev]))

        def peak(fn):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            return (torch.cuda.max_memory_allocated() - base) / 2 ** 20

        plain = lambda: GR.point_visibility(w["views"], w["pts"], *(G[k] for k in keys))  # noqa: E731
        tplain, tf = [], []
        tb = {arm: [] for arm in arms}
        for _ in range(a.runs):
            tplain.append(timed(plain, a.steps, a.warmup))
            tf.append(timed(lambda: fwd("both"), a.steps, a.warmup))
            for arm in arms:
                tb[arm].append(timed_bwd(arm))
        mem_plain = peak(plain)
        mem_diff = peak(lambda: step("both"))
        inview = float(fwd("both")["in_view"].float().mean())
        # kernel times in a pass of their own, after the timed runs: the traced calls include the forward
        kern = {arm: kernel_ms(lambda: step(arm), max(3, a.warmup)) for arm in arms}
        med = lambda x: round(float(np.median(x)), 3)  # noqa: E731
        row = dict(workload=label, P=w["P"], views=V, W=w["W"], H=w["H"], Q=Q, in_view=round(inview, 3),
                   forward_ms=med(tplain), forward_differentiable_ms=med(tf), backward_ms=med(tb["both"]),
                   backward_range=[round(min(tb["both"]), 3), round(max(tb["both"]), 3)], backward_cloud_only_ms=med(tb["cloud"]),
                   backward_points_only_ms=med(tb["points"]), kernel_ms_per_call=kern, peak_mib=round(mem_plain, 1),
                   peak_differentiable_mib=round(mem_diff, 1))
        rows.append(row)
        print(f"{label:>10}: forward {row['forward_ms']} ms (differentiable {row['forward_differentiable_ms']}), backward "
              f"{row['backward_ms']} ms (cloud only {row['backward_cloud_only_ms']}, points only {row['backward_points_only_ms']}), "
              f"peak {row['peak_mib']} / {row['peak_differentiable_mib']} MiB, in view {inview:.2f}")
        for arm in arms:
            print(f"{'':>12}{arm:>7}: " + ", ".join(f"{k} {v} ms" for k, v in kern[arm].items()))
        del w, arms
        torch.cuda.empty_cache()
    return rows


def main():
    import torch
    from manigaussian_b200 import gaussian_renderer as GR
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--backward", action="store_true", help="time point_visibility(differentiable=True), forward and backward")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_visibility needs a CUDA device")
    info = card()
    print(f"card: {info}")
    if a.backward:
        rows = backward_arm(a)
        print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "backward_rows": rows}))
        return
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
