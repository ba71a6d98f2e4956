"""Timeline of the blend CTAs of one c3 step (variant library built with -DMGS_CTA_LOG, MGS_VARIANT=ctalog):
per kernel launch the start/end of the launch, the duration distribution of its CTAs (one warp forward, two warps
backward at F <= 32), how long the longest
CTA alone runs (the kernel's critical path) and how much the launches of different views overlap.
Run on a GPU box: MGS_VARIANT=ctalog MGS_NVCC_DEFINES=-DMGS_CTA_LOG MGS_NO_BUILD=1 python tools/cta_timeline.py [c3]"""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from manigaussian_b200 import _binding

wl = dict(bench.WORKLOADS[sys.argv[1] if len(sys.argv) > 1 else "c3"])
P, V, F = wl["P"], wl["views"], wl["F"]
M = (bench.SH_DEGREE + 1) ** 2
g, cams, cts = bench.host_inputs(wl, 0, 1)
G, C, T = bench.to_device(g, cams, cts, torch)
flat, acc = bench.make_packed(P, F, M, torch)
L = _binding.lib()
cap = 1 << 16
log = torch.zeros((cap, 4), dtype=torch.int64, device="cuda")
cnt = torch.zeros((1,), dtype=torch.int32, device="cuda")
L.mgs_debug_set_cta_log.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint]
for _ in range(5):
    bench.run_step_views(G, C, T, flat, acc, None, F, wl["depth"])
torch.cuda.synchronize()
L.mgs_debug_set_cta_log(log.data_ptr(), cnt.data_ptr(), cap)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
bench.run_step_views(G, C, T, flat, acc, None, F, wl["depth"])
e1.record()
torch.cuda.synchronize()
L.mgs_debug_set_cta_log(None, None, 0)
n = int(cnt.item())
a = log[:n].cpu().numpy().view(np.uint64)
t0, t1 = a[:, 0].astype(np.int64), a[:, 1].astype(np.int64)
kind = (a[:, 2] & 0xff).astype(np.int64)
length = (a[:, 2] >> 32).astype(np.int64)
sm = (a[:, 3] & 0xffffffff).astype(np.int64)
base = t0.min()
out = {"step_ms": e0.elapsed_time(e1), "ctas_logged": n, "kernels": []}
for k, name in ((0, "blend_fwd"), (1, "blend_bwd")):
    sel = np.where(kind == k)[0]
    if sel.size == 0:
        continue
    # split the CTAs of this kind into launches: a launch's CTAs share a list-length multiset; use start-time clustering by
    # sorting on t0 and cutting into V groups of equal size (each launch logs the same number of CTAs on this workload)
    order = sel[np.argsort(t0[sel], kind="stable")]
    dur = (t1 - t0)[sel] / 1e3
    out[name] = {"ctas": int(sel.size), "span_us": float((t1[sel].max() - t0[sel].min()) / 1e3),
                 "sum_cta_us": float(dur.sum()), "mean_cta_us": float(dur.mean()), "max_cta_us": float(dur.max()),
                 "p50_cta_us": float(np.percentile(dur, 50)), "p90_cta_us": float(np.percentile(dur, 90)),
                 "first_start_us": float((t0[sel].min() - base) / 1e3), "last_end_us": float((t1[sel].max() - base) / 1e3),
                 "avg_resident_ctas_per_sm": float(dur.sum() / ((t1[sel].max() - t0[sel].min()) / 1e3) / torch.cuda.get_device_properties(0).multi_processor_count),
                 "us_per_list_entry_p50": float(np.percentile(dur / np.maximum(length[sel], 1), 50))}
    # occupancy over time: CTAs of this kind resident, sampled every 20 us
    ts = np.arange(t0[sel].min(), t1[sel].max(), 20000)
    res = [int(((t0[sel] <= t) & (t1[sel] > t)).sum()) for t in ts]
    out[name]["resident_ctas_every_20us"] = res
    # the ten longest CTAs: start, duration, list length
    top = sel[np.argsort(-(t1 - t0)[sel])[:10]]
    out[name]["longest"] = [{"start_us": float((t0[i] - base) / 1e3), "dur_us": float((t1[i] - t0[i]) / 1e3), "len": int(length[i]), "sm": int(sm[i])} for i in top]
print(json.dumps(out))
