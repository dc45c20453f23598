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
does not measure scaling."""
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
    args = ap.parse_args()
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
    q, g = synthetic.descriptors(10000, 100000, 512, seed=2)
    q, g = q.to(dev), g.to(dev)
    lo, hi = ddist.shard_bounds(g.shape[0], rank, world)
    shard = g[lo:hi].contiguous()
    sent = []

    def allgather(send, recv, nbytes, stream):
        sent.append(nbytes)
        tdist.all_gather_into_tensor(ddist.device_bytes(recv, nbytes * world, dev), ddist.device_bytes(send, nbytes, dev))
        return 0

    for name, qq, t in [("10k x 100k x 512", q, 0.5), ("100k self-join x 512", g, 0.5)]:
        call = lambda: ddist.sharded_range(qq, shard, t, lo, allgather=allgather if world > 1 else None, world=world)
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
                ms_single.append(timed(lambda: similarity.sim_range(qq, g, t))[0])
        per_rank = torch.tensor([statistics.median(ms), float(sum(sent))], dtype=torch.float64, device=dev)
        if world > 1:
            tdist.all_reduce(per_rank, op=tdist.ReduceOp.MAX)
        if rank == 0:
            want = similarity.sim_range(qq, g, t)
            identical = all(torch.equal(x, y) for x, y in zip(res, want))
            bytes_sent = int(per_rank[1]) if world > 1 else 0
            print(json.dumps({"workload": name, "threshold": t, "world": world, "backend": backend if world > 1 else None,
                              "ranks_per_gpu": -(-world // n_dev), "median_ms": round(float(per_rank[0]), 3),
                              "single_process_ms": round(statistics.median(ms_single), 3),
                              "bytes_sent_per_rank": bytes_sent, "bytes_received_per_rank": bytes_sent * world,
                              "pairs": int(res[1].numel()), "identical_to_world1": identical, **gpu_info()}), flush=True)
    if world > 1:
        tdist.barrier()
        tdist.destroy_process_group()


if __name__ == "__main__":
    main()
