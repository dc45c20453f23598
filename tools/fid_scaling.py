"""FID of two synthetic 299x299 image sets sharded over the ranks: every rank embeds its share with the Inception
network, the float64 statistics are all-gathered and merged (ActivationStatistics.all_reduce_), and the Frechet distance
is taken on every rank.

    torchrun --nproc-per-node N tools/fid_scaling.py --gen 50000 --real 50000 [--precision fast|parity|exact]

The images come in fixed blocks of --block images, each generated from its own seed (set, global block index); the
blocks are dealt to the ranks contiguously.  The union over the ranks is the same set for every N, so the FID printed
here can be compared across N.  Prints one JSON line: world size, images/s, ms per step (CUDA events around whole
steps after --warmup untimed ones, maximum over the ranks), the FID, and the all-gather + merge time of the two sets on
its own (nothing is exchanged at world size 1), with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from dcr_b200 import fid, nets  # noqa: E402
from dcr_b200.dist import shard_bounds  # noqa: E402
from dcr_b200.retrieval import extract_features  # noqa: E402
from oracle import models as om  # noqa: E402

SIZE = 299


def block_images(set_id: int, block: int, n: int, device) -> torch.Tensor:
    """uint8 [n, 299, 299, 3] low-frequency random fields plus pixel noise, seeded by (set, global block index)."""
    g = torch.Generator(device=device).manual_seed(1_000_003 * (set_id + 1) + block)
    img = 0.4 * torch.rand((n, 3, 1, 1), device=device, generator=g)
    for res, amp in ((4, 0.35), (16, 0.3), (64, 0.25)):
        field = torch.rand((n, 3, res, res), device=device, generator=g)
        gain = amp * torch.rand((n, 1, 1, 1), device=device, generator=g)
        img = img + gain * torch.nn.functional.interpolate(field, size=(SIZE, SIZE), mode="bilinear", align_corners=False)
    img = img + (0.04 + 0.02 * set_id) * torch.randn((n, 3, SIZE, SIZE), device=device, generator=g)
    return (img.clamp_(0, 1) * 255.0).round_().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def rank_blocks(total: int, block: int, rank: int, world: int):
    """[(global block index, images)] of this rank: a contiguous run of the blocks (dist.shard_bounds)."""
    n_blocks = (total + block - 1) // block
    lo, hi = shard_bounds(n_blocks, rank, world)
    return [(b, min(block, total - b * block)) for b in range(lo, hi)]


def shard_images(set_id: int, total: int, block: int, rank: int, world: int, device) -> torch.Tensor:
    blocks = rank_blocks(total, block, rank, world)
    out = torch.empty((sum(n for _, n in blocks), SIZE, SIZE, 3), dtype=torch.uint8, device=device)
    s = 0
    for b, n in blocks:
        out[s:s + n] = block_images(set_id, b, n, device)
        s += n
    return out


def gpu_facts(index: int):
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in q.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(index), None


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--gen", type=int, default=50000)
    ap.add_argument("--real", type=int, default=50000)
    ap.add_argument("--precision", default="fast", choices=["fast", "parity", "exact"])
    ap.add_argument("--batch", type=int, default=200)
    ap.add_argument("--block", type=int, default=500, help="images per seeded block (keep it fixed when comparing N)")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--backend", default="nccl", choices=["nccl", "gloo"],
                    help="gloo lets several ranks share one GPU: that checks the sharding and the FID across N on a "
                         "single card, but its times are not a scaling measurement")
    args = ap.parse_args()

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if args.backend == "gloo":
        local %= torch.cuda.device_count()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group(args.backend, device_id=dev if args.backend == "nccl" else None)
    net = nets.build_fid_inception(om.make_inception_state_dict(0), max_batch=args.batch, precision=args.precision)
    real = shard_images(0, args.real, args.block, rank, world, dev)
    gen = shard_images(1, args.gen, args.block, rank, world, dev)
    chunk = max(args.batch, net.max_batch) * 8        # the accumulate chunk of fid.statistics_of_images
    exchange = []

    def statistics(imgs):
        st = fid.ActivationStatistics(net.out_dim, dev)
        for s in range(0, imgs.shape[0], chunk):
            st.update(extract_features(net, imgs[s:s + chunk], args.batch))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if world > 1:
            st.all_reduce_()
        e1.record()
        exchange.append((e0, e1))
        return st.finalize()

    def step():
        exchange.clear()
        m1, s1 = statistics(real)
        m2, s2 = statistics(gen)
        return fid.frechet_distance(m1, s1, m2, s2)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        step()
    barrier()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    xms = 0.0
    t0.record()
    for _ in range(args.steps):
        value = step()
        torch.cuda.synchronize()
        xms += sum(a.elapsed_time(b) for a, b in exchange)
    t1.record()
    barrier()
    ms = torch.tensor([t0.elapsed_time(t1) / args.steps, xms / args.steps], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    fids = torch.tensor([value], device=dev, dtype=torch.float64)
    if world > 1:
        allf = torch.empty(world, device=dev, dtype=torch.float64)
        dist.all_gather_into_tensor(allf, fids)
        fids = allf
    if rank == 0:
        name, limit = gpu_facts(local)
        n = args.gen + args.real
        print(json.dumps({"world_size": world, "images": n, "images_per_s": n / (float(ms[0]) / 1e3),
                          "ms_per_step": float(ms[0]), "allgather_merge_ms": float(ms[1]), "fid": value,
                          "fid_identical_on_all_ranks": bool((fids == fids[0]).all()), "precision": args.precision,
                          "backend": args.backend if world > 1 else None, "batch": args.batch, "block": args.block,
                          "steps": args.steps, "warmup": args.warmup,
                          "gpu": name, "power_limit": limit}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
