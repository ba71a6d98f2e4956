"""bench.py at another feature width: measures the cost of F > 32 (channel groups of 32, DESIGN.md section 4).

    python tools/bench_features.py F [bench.py arguments...]
    python tools/bench_features.py 64 --gpus 1 --steps 40 --warmup 5 --no-cpu-baseline --no-c5 --no-e2e

Runs bench.py's own harness unchanged, with the feature width of every workload (default c3) replaced by F, and prints
the same JSON line (`config.feature_channels` = F; per-stage times under `measured.stage_ms_per_launch`).  Only the
product build (`--impl ours`) is supported above 32 channels: the compiled reference is built for at most 32.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main(argv):
    if not argv or not argv[0].isdigit():
        raise SystemExit(__doc__)
    F, rest = int(argv[0]), argv[1:]
    if F > 32 and "reference" in rest:
        raise SystemExit("the compiled reference is built for at most 32 feature channels")
    for wl in bench.WORKLOADS.values():
        wl["F"] = F
    sys.argv = [os.path.join(ROOT, "bench.py")] + rest
    return bench.main()


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
