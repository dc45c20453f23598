"""Threshold search under the split score ('splitloss'): dcr_sim_range_split against the split top-k and against the
per-part composition it replaces.

The composition is rebuilt from public entries: one sim_range per part at the same threshold, then the union of the
per-part pairs with the maximum per pair.  A pair reaches the threshold under the split score exactly when its best part
does, and fp32 rounding is monotonic, so the composition's CSR must be bit-identical to the fused search's.  In every
repetition the three calls alternate in one process: the fused threshold search, sim_topk_split(k=10) on the same
inputs, and the composition (where it runs).  The threshold is the median over the queries of their third-best split
score, so a query has about three pairs.  Times are medians of CUDA-event intervals.  Prints one JSON line per workload
with the candidates and pairs, the card name and its power limit.

    python tools/sim_range_split_bench.py [--reps 5] [--only a,b]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dcr_b200 import _lib, similarity, synthetic  # noqa: E402
from tools.sim_split_bench import token_like  # noqa: E402


def composition(q, g, t, c):
    """sim_range per part, then the union of the pairs with the maximum per pair, as one CSR."""
    nq, d = q.shape
    ng, p = g.shape[0], d // c
    keys, vals = [], []
    for j in range(c):
        off, idx, val = similarity.sim_range(q[:, j * p:(j + 1) * p].contiguous(), g[:, j * p:(j + 1) * p].contiguous(), t)
        rows = torch.repeat_interleave(torch.arange(nq, device=q.device), off[1:] - off[:-1])
        keys.append(rows * ng + idx)
        vals.append(val)
    keys, vals = torch.cat(keys), torch.cat(vals)
    uniq, inv = torch.unique(keys, sorted=True, return_inverse=True)
    best = torch.full((uniq.numel(),), -float("inf"), device=q.device).scatter_reduce(0, inv, vals, "amax")
    counts = torch.bincount(uniq // ng, minlength=nq)
    off = torch.zeros(nq + 1, dtype=torch.int64, device=q.device)
    off[1:] = torch.cumsum(counts, 0)
    return off, uniq % ng, best


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


WORKLOADS = {
    # name: (nq, ng, C, p, data, run the composition)
    "a": (10000, 100000, 4, 128, "descriptors", True),
    "b": (2000, 20000, 197, 384, "tokens", True),          # ViT-S/16 tokens
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    args = ap.parse_args()
    name, power = card()
    for w in args.only.split(","):
        nq, ng, c, p, kind, with_base = WORKLOADS[w]
        d = c * p
        if kind == "descriptors":
            q, g = synthetic.descriptors(nq, ng, d, seed=1)
            q, g = q.cuda(), g.cuda()
        else:
            q, g = token_like(nq, c, p, 2), token_like(ng, c, p, 3)
        topk = lambda: similarity.sim_topk_split(q, g, 10, c)  # noqa: E731
        s10, _ = topk()
        t = float(s10[:, 2].median())
        fused = lambda: similarity.sim_range_split(q, g, t, c)  # noqa: E731
        base = lambda: composition(q, g, t, c)  # noqa: E731
        want = fused()
        n_pairs = int(want[0][-1])
        # the candidate count: the capacity a call with max_pairs = 0 asks for
        lib = _lib.load()
        cnt = (C.c_int64 * 2)()
        nbytes = lib.dcr_sim_range_split_workspace_size(nq, ng, d, c, 0)
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device="cuda")
        off = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
        rc = lib.dcr_sim_range_split(q.data_ptr(), nq, g.data_ptr(), ng, d, c, t, 0, 1, off.data_ptr(), None, None, 0, cnt,
                                     similarity._aligned_ptr(ws), nbytes, torch.cuda.current_stream().cuda_stream)
        n_cand = int(cnt[1]) if rc in (0, _lib.ERR_CAPACITY) else -1
        del ws
        if with_base:
            timed(base)
        t_range, t_topk, t_base, same = [], [], [], True
        for _ in range(args.reps):
            ms, got = timed(fused)
            t_range.append(ms)
            same_fused = all(torch.equal(x, y) for x, y in zip(got, want))
            t_topk.append(timed(topk)[0])
            if with_base:
                ms, comp = timed(base)
                t_base.append(ms)
                same &= (torch.equal(comp[0], want[0]) and torch.equal(comp[1], want[1])
                         and torch.equal(comp[2].view(torch.int32), want[2].view(torch.int32)))
            assert same_fused, "the fused search returned different bits on a repeated call"
        rec = {"workload": w, "nq": nq, "ng": ng, "parts": c, "part_len": p, "data": kind, "threshold": t,
               "candidates": n_cand, "pairs": n_pairs, "pairs_per_query": round(n_pairs / nq, 2),
               "range_split_ms": round(median(t_range), 3), "topk_split_k10_ms": round(median(t_topk), 3),
               "range_over_topk": round(median(t_range) / median(t_topk), 2),
               "composition_ms": round(median(t_base), 3) if with_base else "not measured",
               "composition_bit_identical": same if with_base else "not measured",
               "card": name, "power_limit": power}
        print(json.dumps(rec), flush=True)
        del q, g, want
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
