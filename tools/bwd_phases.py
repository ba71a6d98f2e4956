"""Where a two-warp backward blend CTA spends a chunk: clock64() cycles per chunk and phase, for one view of a workload
(variant library built with -DMGS_BWD_PHASES; blend_common.cuh names the phases).  The companion's phases and the walker's
are laps of two warps that run at the same time, so each role's phases add up to that role's loop, not to each other.
Also prints blend_bwd's time per launch (CUDA events; the phase stamps cost a little of it).
Run on a GPU box, e.g. with the timing-only switches of blend_bwd.cu added to the defines:
  MGS_VARIANT=phases MGS_NVCC_DEFINES=-DMGS_BWD_PHASES python tools/bwd_phases.py [c3] [steps]"""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from manigaussian_b200 import _binding

PHASES = ["queue", "record_wait", "row_issue", "row_wait", "done_wait", "gemm23", "flush", "companion_loop",
          "full_wait", "gemm1", "walk", "walker_loop", "chunks", "ctas"]

wl = dict(bench.WORKLOADS[sys.argv[1] if len(sys.argv) > 1 else "c3"])
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
P, F = wl["P"], wl["F"]
M = (bench.SH_DEGREE + 1) ** 2
g, cams, cts = bench.host_inputs(wl, 0, 1)
G, C, T = bench.to_device(g, cams, cts, torch)
C, T = C[:1], T[:1]  # one view
flat, acc = bench.make_packed(P, F, M, torch)
L = _binding.lib()
L.mgs_debug_set_bwd_phases.argtypes = [ctypes.c_void_p]
L.mgs_profile_stage_name.restype = ctypes.c_char_p
ph = torch.zeros((len(PHASES),), dtype=torch.int64, device="cuda")
for _ in range(5):
    bench.run_step_views(G, C, T, flat, acc, None, F, wl["depth"])
torch.cuda.synchronize()
ns = L.mgs_profile_num_stages()
tot = (ctypes.c_float * ns)()
cnt = (ctypes.c_int * ns)()
L.mgs_profile_read(tot, cnt)  # drop what the warm-up recorded
L.mgs_profile_enable(1)
L.mgs_debug_set_bwd_phases(ph.data_ptr())
for _ in range(steps):
    bench.run_step_views(G, C, T, flat, acc, None, F, wl["depth"])
torch.cuda.synchronize()
L.mgs_debug_set_bwd_phases(None)
L.mgs_profile_enable(0)
L.mgs_profile_read(tot, cnt)
stage = {L.mgs_profile_stage_name(i).decode(): tot[i] / cnt[i] for i in range(ns) if cnt[i] > 0}
v = ph.cpu().numpy().view(np.uint64).astype(np.float64)
chunks = v[PHASES.index("chunks")]
out = {"workload": wl, "steps": steps, "variant": os.environ.get("MGS_VARIANT", ""),
       "defines": os.environ.get("MGS_NVCC_DEFINES", ""), "gpu": torch.cuda.get_device_name(0),
       "blend_bwd_ms_per_launch": round(stage.get("blend_bwd", float("nan")), 4),
       "chunks_per_launch": chunks / steps, "ctas_per_launch": v[PHASES.index("ctas")] / steps,
       "cycles_per_chunk": {n: round(v[i] / max(chunks, 1), 1) for i, n in enumerate(PHASES[:-2])}}
print(json.dumps(out))
