"""Top-k and threshold search under the cross split score ('splitloss', --stype cross): the fused sweep
(dcr_sim_topk_cross / dcr_sim_range_cross) against the composition it replaces.

The composition is a private copy of the host code the cross top-k used before the fused sweep existed, built from public
entries: candidates from dcr_sim_topk over the part matrices, then dcr_split_rescore(cross = 1).
  single pass   one sim_topk over [nq C, p] x [ng C, p] with k' = (k - 1) C + 1 (only while k' <= 16)
  per part      one sim_topk per gallery part, [nq C, p] x [ng, p] with k' = k (only while C^2 k <= 4096)
Both report the bits of dcr_split_rescore, as the fused search does, so every output pair is compared bit for bit.

Workloads (as in the table of DESIGN.md section 3):
  a   10k x 100k x 512, C = 4, k = 10      fused vs the per-part composition
  b   1k x 10k ViT-S/16 tokens, k = 1      fused vs the single-pass composition
  c   b at k = 10                          fused only (the composition refuses 197^2 * 10 candidates)
  d   sim_range_split(cross=True) on a at tau = the median third-best cross score, vs sim_topk_split(cross=True, k=10)
Every shape is warmed up first; in each of --reps repetitions the compared calls alternate in one process.  Times are
medians of CUDA-event intervals.  One JSON line per workload, with the fused path's fallback counts and the card's
name, power limit and SM clock read in the same process.

    python tools/sim_cross_bench.py [--reps 5] [--only a,b,c,d]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dcr_b200 import _lib, similarity, synthetic  # noqa: E402
from tools.sim_split_bench import token_like  # noqa: E402


def composition(q, g, k, c):
    """The cross top-k as the host used to compose it: per-part candidates from sim_topk, then dcr_split_rescore."""
    lib = _lib.load()
    nq, d = q.shape
    ng, p = g.shape[0], d // c
    kk = (k - 1) * c + 1
    if kk <= 16:
        kk = min(kk, ng * c)
        _, idx = similarity.sim_topk(q.view(nq * c, p), g.view(ng * c, p), kk)
        cand = (idx // c).reshape(nq, c * kk).contiguous()
    else:
        if c * c * k > 4096:
            raise _lib.DcrError(f"composition: {c} parts x top-{k} needs {c * c * k} candidates per query (max 4096)")
        kq = min(k, ng)
        cand = torch.full((nq, c, c, k), -1, dtype=torch.int64, device=q.device)
        qparts = q.view(nq * c, p)
        for b in range(c):
            _, idx = similarity.sim_topk(qparts, g[:, b * p:(b + 1) * p].contiguous(), kq)
            cand[:, :, b, :kq] = idx.view(nq, c, kq)
        cand = cand.reshape(nq, c * c * k).contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    rc = lib.dcr_split_rescore(q.data_ptr(), g.data_ptr(), nq, d, c, 1, cand.data_ptr(), cand.shape[1], k,
                               out_s.data_ptr(), out_i.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "dcr_split_rescore")
    return out_s, out_i


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
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = (x.strip() for x in out.strip().split(","))
    except Exception:  # noqa: BLE001
        name, power, sm, sm_max = torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"
    return {"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def same_bits(x, y):
    return all(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                           b.view(torch.int32) if b.dtype == torch.float32 else b) for a, b in zip(x, y))


WORKLOADS = {
    # name: (nq, ng, C, p, data, k)
    "a": (10000, 100000, 4, 128, "descriptors", 10),
    "b": (1000, 10000, 197, 384, "tokens", 1),      # ViT-S/16 tokens
    "c": (1000, 10000, 197, 384, "tokens", 10),
    "d": (10000, 100000, 4, 128, "descriptors", 10),
}


def data(w):
    nq, ng, c, p, kind, _ = WORKLOADS[w]
    if kind == "descriptors":
        q, g = synthetic.descriptors(nq, ng, c * p, seed=1)
        return q.cuda(), g.cuda()
    return token_like(nq, c, p, 2), token_like(ng, c, p, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    args = ap.parse_args()
    for w in args.only.split(","):
        nq, ng, c, p, kind, k = WORKLOADS[w]
        q, g = data(w)
        fused = lambda: similarity.sim_topk_split(q, g, k, c, cross=True)  # noqa: E731
        rec = {"workload": w, "nq": nq, "ng": ng, "parts": c, "part_len": p, "data": kind, "k": k}
        want = fused()                                             # warm-up
        st = similarity.sim_topk_stats()
        rec.update(fused_n_second=st["n_second"], fused_n_flagged=st["n_flagged"])
        if w == "d":
            t = float(want[0][:, 2].median())
            rng = lambda: similarity.sim_range_split(q, g, t, c, cross=True)  # noqa: E731
            r0 = rng()
            t_range, t_topk, same = [], [], True
            for _ in range(args.reps):
                ms, got = timed(rng)
                t_range.append(ms)
                same &= same_bits(got, r0)
                t_topk.append(timed(fused)[0])
            rec.update(threshold=t, pairs=int(r0[0][-1]), range_ms=round(median(t_range), 3),
                       topk_k10_ms=round(median(t_topk), 3), range_over_topk=round(median(t_range) / median(t_topk), 2),
                       range_repeat_bit_identical=same)
        else:
            base = (lambda: composition(q, g, k, c)) if w in ("a", "b") else None
            if base:
                timed(base)                                        # warm-up
            t_fused, t_base, same, flagged = [], [], True, 0
            for _ in range(args.reps):
                ms, got = timed(fused)
                t_fused.append(ms)
                flagged = max(flagged, similarity.sim_topk_stats()["n_flagged"])
                same &= same_bits(got, want)
                if base:
                    ms, comp = timed(base)
                    t_base.append(ms)
                    same &= same_bits(comp, want)
            rec.update(fused_ms=round(median(t_fused), 3), fused_max_n_flagged=flagged,
                       composition_ms=round(median(t_base), 3) if base else "refused",
                       fused_over_composition=round(median(t_fused) / median(t_base), 3) if base else None,
                       bit_identical=same)
        rec.update(card())
        print(json.dumps(rec), flush=True)
        del q, g, want
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
