"""What the fused L1 + SSIM head costs: one training step with the 3DGS photometric objective, fused against unfused, and the
two SSIM kernels alone.

    python tools/bench_ssim.py [--workloads mg,c3] [--steps 40] [--warmup 5] [--runs 3] [--kernel-iters 200]

Workloads are bench.py's: mg (ManiGaussian's call: 16k Gaussians, one view 128x128, F = 3) and c3 (500k Gaussians, 4 views
256x256, F = 32), SH degree 1.  Three arms, each one training step (render -> losses -> backward) timed with CUDA events over
--steps steps after --warmup steps, in --runs alternated runs (the table gives the median and the range):
  fused       -- render_views(targets={"rgb", "embed"}): the fused colour + embedding heads, no photometric objective;
  fused_ssim  -- render_views(targets=..., ssim=True) and 0.8 loss_l1 + 0.2 (1 - ssim) on top of the same heads;
  torch_ssim  -- render_views() and the same four losses in PyTorch: the reference's l1_loss and ssim (five grouped conv2d
                 calls) on the returned image, with the default cuDNN settings (TF32 allowed), as users run it.  (The fused
                 path returns its images detached, so a PyTorch SSIM on them could not train: the unfused render is the
                 alternative a user has.)
The two kernels alone (mgs_ssim / mgs_ssim_backward on the workload's [V,3,H,W] images) are timed with CUDA events over
--kernel-iters launches, with the bytes they must move: forward reads x, g and writes the partials (60 B per pixel),
backward reads the partials, x, g and writes the cotangent (72 B per pixel).  The card's name, power limit and SM clock are
read in the same run, and a JSON summary is printed last.
"""
import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (workload definition)
from bench_alpha import card  # noqa: E402

ARMS = ("fused", "fused_ssim", "torch_ssim")


def workload(name):
    import torch
    from manigaussian_b200 import GaussianRasterizationSettings, scenes
    wl = bench.WORKLOADS[name]
    P, V, W, H, F = wl["P"], wl["views"], wl["W"], wl["H"], wl["F"]
    g = scenes.make_gaussians(P, F=F, sh_degree=bench.SH_DEGREE, seed=1234)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    L = {k: t(g[k]).requires_grad_(True) for k in ("means3D", "rotations", "scales", "opacities", "shs", "feature")}
    bg = torch.zeros(3, device="cuda")
    cams = [scenes.make_camera(W, H, v, V) for v in range(V)]
    views = [GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], bg, 1.0, t(c["viewmatrix"]), t(c["projmatrix"]),
                                           bench.SH_DEGREE, t(c["campos"]), False, False, True) for c in cams]
    gen = torch.Generator(device="cuda").manual_seed(77)
    targets = {"rgb": torch.rand(V, 3, H, W, device="cuda", generator=gen),
               "embed": torch.rand(V, F, H, W, device="cuda", generator=gen) - 0.5}
    return dict(name=name, P=P, V=V, W=W, H=H, F=F, L=L, views=views, targets=targets)


_WINDOW = {}


def torch_ssim(img1, img2):
    """the reference's ssim (utils/loss_utils.py: window 11, sigma 1.5, size_average) on [B,C,H,W]"""
    import torch
    import torch.nn.functional as F
    C = img1.shape[1]
    w = _WINDOW.get((C, img1.device))
    if w is None:
        gauss = torch.tensor([math.exp(-(i - 5) ** 2 / 4.5) for i in range(11)])
        gauss = gauss / gauss.sum()
        w = _WINDOW[(C, img1.device)] = (gauss[:, None] @ gauss[None, :]).expand(C, 1, 11, 11).contiguous().to(img1.device)
    mu1, mu2 = F.conv2d(img1, w, padding=5, groups=C), F.conv2d(img2, w, padding=5, groups=C)
    s1 = F.conv2d(img1 * img1, w, padding=5, groups=C) - mu1 ** 2
    s2 = F.conv2d(img2 * img2, w, padding=5, groups=C) - mu2 ** 2
    s12 = F.conv2d(img1 * img2, w, padding=5, groups=C) - mu1 * mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 ** 2 + mu2 ** 2 + c1) * (s1 + s2 + c2))).mean()


def step(arm, w):
    import torch
    from manigaussian_b200.gaussian_renderer import render_views
    L, tg = w["L"], w["targets"]
    for v in L.values():
        v.grad = None
    kw = dict(features_color=L["shs"], features_language=L["feature"], normalize_feature=False)
    args = (w["views"], L["means3D"], L["rotations"], L["scales"], L["opacities"])
    if arm == "torch_ssim":
        o = render_views(*args, **kw)
        x = o["render"]
        loss = ((x - tg["rgb"]) ** 2).mean() + (1 - torch.nn.functional.cosine_similarity(o["render_embed"], tg["embed"], dim=1).mean())
        loss = loss + 0.8 * (x - tg["rgb"]).abs().mean() + 0.2 * (1 - torch_ssim(x, tg["rgb"]))
    else:
        o = render_views(*args, targets=tg, ssim=arm == "fused_ssim", **kw)
        loss = o["loss_rgb"].mean() + o["loss_embed"].mean()
        if arm == "fused_ssim":
            loss = loss + 0.8 * o["loss_l1"].mean() + 0.2 * (1 - o["ssim"].mean())
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


def ssim_stages(w):
    """ssim_fwd / ssim_bwd ms per launch (= per view) of one profiled fused_ssim step"""
    import torch
    from manigaussian_b200 import _binding
    torch.cuda.synchronize()
    _binding.profile_enable(True)
    _binding.profile_read()
    step("fused_ssim", w)
    torch.cuda.synchronize()
    prof = _binding.profile_read()
    _binding.profile_enable(False)
    return {k: prof[k][0] / max(prof[k][1], 1) for k in ("ssim_fwd", "ssim_bwd", "blend_fwd", "blend_bwd")}


def kernels_alone(w, iters):
    """the two kernels on the workload's [V,3,H,W] images: ms per launch and achieved GB/s of the bytes they must move"""
    import torch
    from manigaussian_b200 import _binding as B
    V, H, W = w["V"], w["H"], w["W"]
    gen = torch.Generator(device="cuda").manual_seed(5)
    x, g = (torch.rand(V, 3, H, W, device="cuda", generator=gen) for _ in range(2))
    terms, acc = torch.empty(V, 9, H, W, device="cuda"), torch.empty(V, 2, device="cuda")
    scale, cot = torch.ones(V, 2, device="cuda"), torch.empty_like(x)
    L, st = B.lib(), torch.cuda.current_stream().cuda_stream
    calls = {
        "ssim_fwd": lambda: L.mgs_ssim(V, 3, H, W, x.data_ptr(), g.data_ptr(), terms.data_ptr(), acc.data_ptr(), st),
        "ssim_bwd": lambda: L.mgs_ssim_backward(V, 3, H, W, x.data_ptr(), g.data_ptr(), terms.data_ptr(), scale.data_ptr(), None,
                                                cot.data_ptr(), st),
    }
    bytes_px = {"ssim_fwd": 60, "ssim_bwd": 72}
    out = {}
    for k, fn in calls.items():
        for _ in range(10):
            B.check(fn(), k)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        nbytes = bytes_px[k] * V * H * W
        out[k] = dict(ms=ms, bytes=nbytes, GBps=nbytes / (ms * 1e-3) / 1e9)
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="mg,c3")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ssim needs a CUDA device")
    info = card()
    print("card:", info, "cudnn.allow_tf32:", torch.backends.cudnn.allow_tf32, flush=True)
    result = {}
    for name in a.workloads.split(","):
        w = workload(name)
        ms = {k: [] for k in ARMS}
        for _ in range(a.runs):
            for arm in ARMS:
                ms[arm].append(timed(arm, w, a.steps, a.warmup))
        rows = {arm: dict(step_ms=float(np.median(ms[arm])), step_range=[min(ms[arm]), max(ms[arm])]) for arm in ARMS}
        for arm in ARMS:
            r = rows[arm]
            print(f"{name} {arm:10s} step {r['step_ms']:.3f} ms [{r['step_range'][0]:.3f}, {r['step_range'][1]:.3f}]", flush=True)
        stages = ssim_stages(w)
        kern = kernels_alone(w, a.kernel_iters)
        print(f"{name} stages in the fused_ssim step (ms per view): " + ", ".join(f"{k} {v:.4f}" for k, v in stages.items()), flush=True)
        for k, r in kern.items():
            print(f"{name} {k} alone: {r['ms'] * 1e3:.1f} us, {r['bytes'] / 1e6:.2f} MB, {r['GBps']:.0f} GB/s", flush=True)
        result[name] = dict(P=w["P"], views=w["V"], WxH=f"{w['W']}x{w['H']}", F=w["F"], arms=rows, stages_ms_per_view=stages,
                            kernels_alone=kern)
        del w
    info["after"] = card()["power.limit, clocks.sm, clocks.max.sm"]
    print(json.dumps({"card": info, "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "workloads": result}))


if __name__ == "__main__":
    main()
