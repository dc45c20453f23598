"""Gallery-sharded threshold search (dist.sharded_range) at several world sizes.

    torchrun --nproc_per_node N tools/sim_range_scaling.py [--reps 10] [--backend auto|nccl|gloo]
    python tools/sim_range_scaling.py                 (world size 1, no process group)

Every rank generates the same seeded inputs (synthetic.descriptors(10000, 100000, 512, seed=2), as
tools/sim_range_bench.py) and keeps its contiguous gallery shard (dist.shard_bounds).  Cases: the 10k queries against
the 100k gallery at threshold 0.5, and the gallery joined with itself at 0.5 (every rank passes all 100k rows as
queries).  Rank 0 prints one JSON line per case: the median per-call time over --reps calls (CUDA events on each rank
after two untimed calls; the slowest rank's median) next to rank 0's median of similarity.sim_range on the whole gallery,
timed alternately with the sharded calls, the bytes each rank sends (header + message, the largest over the
ranks) and receives, and whether rank 0's CSR is bit-identical to similarity.sim_range on the whole gallery in one
process.  With fewer GPUs than ranks the ranks share cards over gloo (--backend auto): that run checks the result, it
does not measure scaling.

--num-chunks C [--cross] measures the split-score forms instead (dist.sharded_range(num_chunks=C, cross=...), compared
with similarity.sim_range_split(..., cross=...) on the whole gallery), on the workloads of the cross table in DESIGN.md
section 3: (a) synthetic.descriptors(10000, 100000, 512, seed=1) in C parts, and 1k x 10k ViT-S/16 token rows
(tools/sim_split_bench.token_like, 197 parts of 384: one per token, whatever C is).  Their threshold is the median over
the queries of the third-best score under the same form (sim_topk_split, k = 3, on the whole gallery, on every rank):
a few pairs per query.  Those lines also carry the score, the part count, the threshold, and the SM clock (current and
maximum, read after the timed calls).

    python tools/sim_range_scaling.py --num-chunks 4 --cross --reps 5
    torchrun --nproc_per_node 2 tools/sim_range_scaling.py --num-chunks 4 --cross --reps 5"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as tdist  # noqa: E402

from dcr_b200 import dist as ddist  # noqa: E402
from dcr_b200 import similarity, synthetic  # noqa: E402


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown"}


def sm_clock() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        sm, sm_max = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"sm_clock": "unknown", "sm_clock_max": "unknown"}


def split_cases(num_chunks: int, cross: bool):
    """(name, queries, gallery, threshold, parts) of the split-score workloads, each made when it is reached."""
    from tools.sim_split_bench import token_like

    def case(name, make, c):
        q, g = make()
        v, _ = similarity.sim_topk_split(q, g, 3, c, cross=cross)
        return name, q, g, float(v[:, 2].median()), c

    yield case("10k x 100k x 512", lambda: tuple(x.cuda() for x in synthetic.descriptors(10000, 100000, 512, seed=1)),
               num_chunks)
    yield case("1k x 10k ViT-S/16 tokens (197 x 384)", lambda: (token_like(1000, 197, 384, 2),
                                                                token_like(10000, 197, 384, 3)), 197)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--backend", default="auto", choices=["auto", "nccl", "gloo"])
    ap.add_argument("--num-chunks", type=int, default=1, help="the split score over this many parts (default: dot product)")
    ap.add_argument("--cross", action="store_true", help="the cross split score (needs --num-chunks >= 2)")
    args = ap.parse_args()
    if args.cross and args.num_chunks < 2:
        ap.error("--cross needs --num-chunks C >= 2")
    split = args.num_chunks > 1
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("sim_range_scaling: no CUDA device")
    backend = args.backend if args.backend != "auto" else ("nccl" if n_dev >= world else "gloo")
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")) % n_dev)
    torch.cuda.set_device(dev)
    if world > 1:
        tdist.init_process_group(backend, device_id=dev if backend == "nccl" else None)
    sent = []

    def allgather(send, recv, nbytes, stream):
        sent.append(nbytes)
        tdist.all_gather_into_tensor(ddist.device_bytes(recv, nbytes * world, dev), ddist.device_bytes(send, nbytes, dev))
        return 0

    def dot_cases():
        q, g = synthetic.descriptors(10000, 100000, 512, seed=2)
        q, g = q.to(dev), g.to(dev)
        yield "10k x 100k x 512", q, g, 0.5, 1
        yield "100k self-join x 512", g, g, 0.5, 1

    for name, qq, g, t, c in (split_cases(args.num_chunks, args.cross) if split else dot_cases()):
        lo, hi = ddist.shard_bounds(g.shape[0], rank, world)
        shard = g[lo:hi].contiguous()

        def single():
            if split:
                return similarity.sim_range_split(qq, g, t, c, cross=args.cross)
            return similarity.sim_range(qq, g, t)

        def call():
            return ddist.sharded_range(qq, shard, t, lo, allgather=allgather if world > 1 else None, world=world,
                                       num_chunks=c, cross=args.cross)

        for _ in range(2):
            res = call()
        ms, ms_single = [], []
        for _ in range(args.reps):
            if world > 1:
                tdist.barrier()
            sent.clear()
            t_call, res = timed(call)
            ms.append(t_call)
            if rank == 0:   # the single-process search on the whole gallery, alternated with the sharded calls
                ms_single.append(timed(single)[0])
        per_rank = torch.tensor([statistics.median(ms), float(sum(sent))], dtype=torch.float64, device=dev)
        if world > 1:
            tdist.all_reduce(per_rank, op=tdist.ReduceOp.MAX)
        if rank == 0:
            want = single()
            identical = all(torch.equal(x, y) for x, y in zip(res, want))
            bytes_sent = int(per_rank[1]) if world > 1 else 0
            rec = {"workload": name, "threshold": t, "world": world, "backend": backend if world > 1 else None,
                   "ranks_per_gpu": -(-world // n_dev), "median_ms": round(float(per_rank[0]), 3),
                   "single_process_ms": round(statistics.median(ms_single), 3),
                   "bytes_sent_per_rank": bytes_sent, "bytes_received_per_rank": bytes_sent * world,
                   "pairs": int(res[1].numel()), "identical_to_world1": identical, **gpu_info()}
            if split:
                rec.update(score="cross" if args.cross else "aligned", parts=c, **sm_clock())
            print(json.dumps(rec), flush=True)
        del qq, g, shard, res
        torch.cuda.empty_cache()
    if world > 1:
        tdist.barrier()
        tdist.destroy_process_group()


if __name__ == "__main__":
    main()
