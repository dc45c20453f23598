"""Threshold search (similarity.sim_range) against the top-k search (similarity.sim_topk, k = 10) on the same inputs.

    python tools/sim_range_bench.py [--reps 5]

Workloads: 10k queries x 100k gallery rows x 512 dims of synthetic descriptors (synthetic.descriptors: unit rows, 1 % of
the gallery planted as noisy copies of queries) at thresholds 0.5, 0.8 and 0.95, and the 100k gallery joined with itself
at 0.5 (the reference's similarity_wtrain.pth).  Each timed sim_range call is followed by a timed sim_topk call on the
same inputs, so both see the same clocks; CUDA events around each call, after two untimed calls of each.  Prints one
JSON line per workload (median ms per call, candidate pairs examined, pairs returned) with the GPU's name and power
limit."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from dcr_b200 import _lib, similarity, synthetic  # noqa: E402


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown"}


def candidates(q: torch.Tensor, g: torch.Tensor, t: float, pairs: int) -> int:
    """candidate pairs the exact re-score examined (counts[1] of the C call)"""
    lib = _lib.load()
    counts = (C.c_int64 * 2)()
    cap = pairs
    for _ in range(2):
        nbytes = lib.dcr_sim_range_workspace_size(q.shape[0], g.shape[0], q.shape[1], cap)
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=q.device)
        off = torch.empty(q.shape[0] + 1, dtype=torch.int64, device=q.device)
        idx = torch.empty(max(cap, 1), dtype=torch.int64, device=q.device)
        val = torch.empty(max(cap, 1), dtype=torch.float32, device=q.device)
        rc = lib.dcr_sim_range(q.data_ptr(), q.shape[0], g.data_ptr(), g.shape[0], q.shape[1], t, 0, 1, off.data_ptr(),
                               idx.data_ptr(), val.data_ptr(), cap, counts, similarity._aligned_ptr(ws), nbytes,
                               torch.cuda.current_stream().cuda_stream)
        if rc == _lib.ERR_CAPACITY:
            cap = int(counts[1])
            continue
        _lib.check(rc, "dcr_sim_range")
        return int(counts[1])
    raise RuntimeError("capacity retry did not fit")


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    info = gpu_info()
    q, g = synthetic.descriptors(10000, 100000, 512, seed=2)
    q, g = q.cuda(), g.cuda()
    for name, qq, gg, t in [("10k x 100k x 512", q, g, 0.5), ("10k x 100k x 512", q, g, 0.8),
                            ("10k x 100k x 512", q, g, 0.95), ("100k self-join x 512", g, g, 0.5)]:
        for _ in range(2):
            similarity.sim_range(qq, gg, t)
            similarity.sim_topk(qq, gg, 10)
        ms_range, ms_topk = [], []
        for _ in range(args.reps):
            ms, res = timed(lambda: similarity.sim_range(qq, gg, t))
            ms_range.append(ms)
            ms_topk.append(timed(lambda: similarity.sim_topk(qq, gg, 10))[0])
        pairs = int(res[1].numel())
        line = {"workload": name, "threshold": t, "sim_range_ms": round(statistics.median(ms_range), 3),
                "sim_topk10_ms": round(statistics.median(ms_topk), 3),
                "ratio": round(statistics.median(ms_range) / statistics.median(ms_topk), 3),
                "candidates": candidates(qq, gg, t, pairs), "pairs": pairs, **info}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
