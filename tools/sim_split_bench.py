"""Split-score top-k ('splitloss'): the fused sweep of dcr_sim_topk_split against the per-part composition it replaces.

The composition is rebuilt from public entries: one dcr_sim_topk per part, then dcr_split_rescore over the union of the
per-part lists (C * k <= 4096 candidates per query).  Where both run, the two paths alternate in one process and their
outputs must be bit-identical.  Prints one JSON line per workload: median ms, TFLOP/s as 2 nq ng d / t (against the
989 TFLOP/s dense bf16 peak of the H100 SXM), the fallback counts, the card name and its power limit.

    python tools/sim_split_bench.py [--reps 5] [--only a,b,c]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dcr_b200 import _lib, similarity  # noqa: E402

PEAK = 989.0


def composition(q, g, k, c):
    """The per-part composition: sim_topk per part, then the exact split score of the union of the lists."""
    nq, d = q.shape
    p = d // c
    cand = torch.empty((nq, c * k), dtype=torch.int64, device=q.device)
    for j in range(c):
        _, idx = similarity.sim_topk(q[:, j * p:(j + 1) * p].contiguous(), g[:, j * p:(j + 1) * p].contiguous(), k)
        cand[:, j * k:(j + 1) * k] = idx
    out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    lib = _lib.load()
    rc = lib.dcr_split_rescore(q.data_ptr(), g.data_ptr(), nq, d, c, 0, cand.data_ptr(), c * k, k, out_s.data_ptr(),
                               out_i.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "dcr_split_rescore")
    return out_s, out_i


def token_like(n, c, p, seed):
    """Per-token-like rows: every part a shared direction plus noise of the same size, the whole row unit-norm."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    mean = torch.nn.functional.normalize(torch.randn(c, p, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)), dim=1)
    out = torch.empty((n, c * p), device="cuda")
    for s in range(0, n, 256):
        x = torch.randn(min(256, n - s), c, p, device="cuda", generator=gen)
        x = mean + torch.nn.functional.normalize(x, dim=2)
        out[s:s + x.shape[0]] = torch.nn.functional.normalize(x.reshape(x.shape[0], c * p), dim=1)
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


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
    # name: (nq, ng, C, p, k, data, run the composition)
    "a": (10000, 100000, 4, 128, 10, "random", True),
    "b": (2000, 20000, 197, 384, 1, "tokens", True),       # ViT-S/16 tokens; top-1 keeps the composition's re-score
    "b10": (2000, 20000, 197, 384, 10, "tokens", False),   # ... at top-10 the composition re-reads 1,970 rows per query
    "c": (1000, 5000, 785, 768, 10, "tokens", False),      # ViT-B/8 tokens: C * k = 7,850, beyond the composition
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    args = ap.parse_args()
    name, power = card()
    for w in args.only.split(","):
        nq, ng, c, p, k, kind, with_base = WORKLOADS[w]
        d = c * p
        if kind == "random":
            q = torch.nn.functional.normalize(torch.randn(nq, d, device="cuda"), dim=1)
            g = torch.nn.functional.normalize(torch.randn(ng, d, device="cuda"), dim=1)
        else:
            q, g = token_like(nq, c, p, 2), token_like(ng, c, p, 3)
        fused = lambda: similarity.sim_topk_split(q, g, k, c)  # noqa: E731
        base = lambda: composition(q, g, k, c)  # noqa: E731
        timed(fused)
        if with_base:
            timed(base)
        t_new, t_base, same = [], [], True
        stats = None
        for _ in range(args.reps):
            t, (s1, i1) = timed(fused)
            t_new.append(t)
            stats = similarity.sim_topk_stats()
            if with_base:
                t, (s0, i0) = timed(base)
                t_base.append(t)
                same &= bool(torch.equal(i0, i1)) and bool(torch.equal(s0.view(torch.int32), s1.view(torch.int32)))
        flop = 2.0 * nq * ng * d
        rec = {"workload": w, "nq": nq, "ng": ng, "parts": c, "part_len": p, "k": k, "data": kind,
               "fused_ms": round(median(t_new), 3), "fused_tflops": round(flop / median(t_new) / 1e9, 1),
               "fused_kernel_ms": round(stats["kernel_ms"], 3), "n_second": stats["n_second"],
               "n_flagged": stats["n_flagged"], "peak_tflops": PEAK, "card": name, "power_limit": power}
        if with_base:
            rec.update({"composition_ms": round(median(t_base), 3),
                        "composition_tflops": round(flop / median(t_base) / 1e9, 1),
                        "speedup": round(median(t_base) / median(t_new), 2), "bit_identical": same})
        print(json.dumps(rec), flush=True)
        del q, g
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
