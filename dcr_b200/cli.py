"""Drop-in command line for the retrieval hot path of diff_retrieval.py (same flags, same defaults):

    python -m dcr_b200.cli --arch resnet50_disc --similarity_metric dotproduct --pt_style sscd \
        --query_dir <generations> --val_dir <training images>          (README.md:55 of the reference)

What it does is the `if args.rank == 0:` block diff_retrieval.py:375-483 restricted to the hot path: embed both folders,
L2-normalise, top-1 (and top-`num_matches`... the reference hard-codes top-10 for its galleries, :621) matches, background
top-2, the printed statistics dictionary, and optionally FID (:597-600).  Plots, CLIP score, complexity statistics and
wandb are out of scope (DESIGN.md section 9).  Flags that the reference parses but never reads are accepted and ignored.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch


def bool_flag(s):                                   # utils_ret.py:463-474
    falsy, truthy = {"off", "false", "0"}, {"on", "true", "1"}
    if s.lower() in falsy:
        return False
    if s.lower() in truthy:
        return True
    raise argparse.ArgumentTypeError("invalid value for a boolean flag")


def build_parser() -> argparse.ArgumentParser:
    """Mirror of the module-level parser, diff_retrieval.py:124-181."""
    p = argparse.ArgumentParser("Generic image retrieval given a path")
    p.add_argument("--query_dir", type=str, required=True, help="The inferences")
    p.add_argument("--val_dir", type=str, required=True, help="The train data")
    p.add_argument("--pt_style", default="sscd", type=str)
    p.add_argument("-a", "--arch", metavar="ARCH", default="resnet50")
    p.add_argument("-j", "--workers", default=4, type=int, metavar="N")
    p.add_argument("-b", "--batch-size", default=128, type=int, metavar="N")
    p.add_argument("--world-size", default=-1, type=int)
    p.add_argument("--rank", default=-1, type=int)
    p.add_argument("--dist-url", default="tcp://224.66.41.62:23456", type=str)
    p.add_argument("--dist-backend", default="nccl", type=str)
    p.add_argument("--seed", default=None, type=int)
    p.add_argument("--gpu", default=None, type=int)
    p.add_argument("--multiprocessing-distributed", action="store_true")
    p.add_argument("--multiscale", default=False, type=bool_flag)
    p.add_argument("--pretrained", default="", type=str)
    p.add_argument("--similarity_metric", default="dotproduct", type=str)
    p.add_argument("--num_loss_chunks", default=1, type=int)
    p.add_argument("--numpatches", default=1, type=int)
    p.add_argument("--isvit", action="store_true")
    p.add_argument("--layer", default=1, type=int)
    p.add_argument("--stype", default="", type=str, choices=["", "cross"])
    p.add_argument("--keephead", action="store_true")
    p.add_argument("--keeppredictor", action="store_true")
    p.add_argument("-ssp", "--sim_save_path", type=str, default="./similarityscores/")
    p.add_argument("--einsum_chunks", default=30, type=int)
    p.add_argument("--dontsave", action="store_true")
    p.add_argument("--num_matches", default=4, type=int)
    p.add_argument("--imsize", default=224, type=int)
    p.add_argument("--noeval", action="store_true")
    # additions of this implementation (all optional)
    p.add_argument("--weights", default="", type=str, help="state_dict / TorchScript file of the descriptor model "
                   "(default: the reference's hard-coded ./pretrainedmodels/ paths)")
    p.add_argument("--precision", default="fast", choices=["fast", "bf16x3", "parity", "exact"],
                   help="fast: bf16 tensor cores; bf16x3 / parity: 3- / 6-term split-bf16 tensor cores (fp32-level); exact: float64 accumulation")
    p.add_argument("--topk", default=10, type=int, help="matches kept per query (reference: 1 for the statistics, 10 for the galleries)")
    p.add_argument("--sim_threshold", default=None, type=float,
                   help="also write every pair scoring at least this much (matches.pth, and matches_wtrain.pth for the "
                        "gallery self-join): sparse CSR in place of the reference's similarity*.pth matrices; "
                        "--sim_threshold=-inf gives every pair.  Dot-product metric, one process")
    p.add_argument("--fid_weights", default="", type=str, help="pt_inception-2015-12-05 state_dict; enables FID")
    return p


SSCD_FILES = {  # diff_retrieval.py:277-283
    "resnet50": "./pretrainedmodels/sscd_disc_mixup.torchscript.pt",
    "resnet50_im": "./pretrainedmodels/sscd_imagenet_mixup.torchscript.pt",
    "resnet50_disc": "./pretrainedmodels/sscd_disc_large.torchscript.pt",
}


def load_state_dict(path: str):
    if not os.path.exists(path):
        raise FileNotFoundError(f"model weights not found: {path} (pass --weights)")
    try:
        return torch.jit.load(path, map_location="cpu").state_dict()
    except Exception:
        obj = torch.load(path, map_location="cpu")
        return obj.get("state_dict", obj) if isinstance(obj, dict) else obj.state_dict()


def build_model(args):
    from . import nets, retrieval
    if args.pt_style == "sscd":
        if args.arch not in SSCD_FILES:
            raise NotImplementedError("This model type does not exist/supported for SSCD")      # :285
        sd = load_state_dict(args.weights or SSCD_FILES[args.arch])
        if args.multiscale:                                                                   # utils_ret.py:676-698
            return [nets.build_sscd_resnet50(sd, max_batch=384, precision=args.precision, scale_factor=s)
                    for s in retrieval.MULTI_SCALES]
        return nets.build_sscd_resnet50(sd, max_batch=384, precision=args.precision)
    if args.pt_style == "dino":
        if args.arch not in ("vit_small", "vit_base", "vit_base8"):                             # :251-257
            raise NotImplementedError("--pt_style dino: --arch vit_small (dino_vits16), vit_base (dino_vitb16) and "
                                      "vit_base8 (dino_vitb8) are implemented; resnet50 / vit_base_cifar10 are not")
        sd = load_state_dict(args.weights or args.pretrained)
        # splitloss on a ViT: global_pool='' (:258-263) -> one descriptor part per token (utils_ret.py:728-737)
        pool = "" if args.similarity_metric == "splitloss" else "token"
        kw = dict(max_batch=64 if args.arch == "vit_base8" else 256, precision=args.precision, global_pool=pool,
                  n_last_layers=max(1, args.layer))                                             # utils_ret.py:732,745
        if args.multiscale:                                                                   # utils_ret.py:676-698
            return [nets.build_dino_vit(sd, scale_factor=s, **kw) for s in retrieval.MULTI_SCALES]
        return nets.build_dino_vit(sd, **kw)
    if args.pt_style == "clip":
        # diff_retrieval.py:264-271 loads clip.load({'vit_large': 'ViT-L/14', 'vit_base': 'ViT-B/16', 'resnet50': 'RN50x16'}[arch]);
        # the descriptor is `model.encode_image(samples)` (the branch utils_ret.py:725-726 spells out).  The ViT image
        # towers are built from the CLIP state_dict; the ResNet tower (RN50x16) is not.
        if args.arch not in ("vit_base", "vit_large"):
            raise NotImplementedError("--pt_style clip: --arch vit_base (ViT-B/16) and vit_large (ViT-L/14) are implemented")
        sd = load_state_dict(args.weights or args.pretrained)
        if args.multiscale or args.similarity_metric == "splitloss":
            raise NotImplementedError("--pt_style clip supports the dot-product metric at the native input size")
        return nets.build_clip_visual(sd, max_batch=64 if args.arch == "vit_large" else 256, precision=args.precision)
    raise NotImplementedError(f"--pt_style {args.pt_style} is outside the embed->match hot path (DESIGN.md section 9)")


def main(argv=None) -> int:
    """diff_retrieval.py:183-221: parse, then one worker -- or, with --multiprocessing-distributed, one worker per GPU."""
    args = build_parser().parse_args(argv)
    assert os.path.isdir(args.query_dir), "Query dir doesnt exist, skipping!"                   # :185
    if args.similarity_metric == "splitlosscross":                                            # :186-188
        args.similarity_metric, args.stype = "splitloss", "cross"
    if args.similarity_metric not in ("dotproduct", "splitloss"):
        raise NotImplementedError(f"--similarity_metric {args.similarity_metric}")
    if args.dist_url == "env://" and args.world_size == -1:                                   # :204-205
        args.world_size = int(os.environ["WORLD_SIZE"])
    args.distributed = args.world_size > 1 or args.multiprocessing_distributed               # :207
    if args.sim_threshold is not None:
        if args.similarity_metric == "splitloss":
            raise NotImplementedError("--sim_threshold is implemented for --similarity_metric dotproduct")
        if args.distributed:
            raise NotImplementedError("--sim_threshold runs in one process (no sharded threshold search)")
    ngpus_per_node = torch.cuda.device_count()
    if args.multiprocessing_distributed:                                                     # :210-216
        args.world_size = ngpus_per_node * max(1, args.world_size)
        import torch.multiprocessing as mp
        mp.spawn(main_worker, nprocs=ngpus_per_node, args=(ngpus_per_node, args))
        return 0
    return main_worker(args.gpu, ngpus_per_node, args)


def _init_distributed(gpu, ngpus_per_node, args) -> None:
    """diff_retrieval.py:237-246 (and utils_ret.init_distributed_mode for the env:// launch)."""
    import torch.distributed as dist
    if args.dist_url == "env://" and args.rank == -1:
        args.rank = int(os.environ["RANK"])
    if args.multiprocessing_distributed:
        args.rank = max(0, args.rank) * ngpus_per_node + gpu          # global rank among all the processes (:240-243)
    if args.gpu is None:                                              # env:// launch (torchrun): one GPU per local rank
        args.gpu = int(os.environ.get("LOCAL_RANK", args.rank % max(1, ngpus_per_node)))
    torch.cuda.set_device(args.gpu)
    dist.init_process_group(backend=args.dist_backend, init_method=args.dist_url, world_size=args.world_size,
                            rank=args.rank, device_id=torch.device("cuda", args.gpu) if args.dist_backend == "nccl" else None)
    dist.barrier()


def main_worker(gpu, ngpus_per_node, args) -> int:
    """diff_retrieval.py:224-483 restricted to the hot path.  Distributed runs shard BOTH image sets contiguously over
    the ranks (the reference shards the gallery loader with a DistributedSampler, :345-348, and funnels every batch to
    rank 0); every rank embeds its shards, scores all queries against its gallery shard and the per-shard top-k lists
    are all-gathered and merged (dcr_b200/dist.py) -- same result as the single-process run, on every rank.  With
    --fid_weights the FID statistics are sharded the same way and their float64 states merged over the ranks."""
    args.gpu = gpu
    if args.multiprocessing_distributed and args.gpu != 0:                                    # :229-232
        import builtins
        builtins.print = lambda *a, **k: None
    if args.gpu is not None:
        print("Use GPU: {} for training".format(args.gpu))
    rank, world = 0, 1
    if args.distributed:
        import torch.distributed as dist
        _init_distributed(gpu, ngpus_per_node, args)
        rank, world = dist.get_rank(), dist.get_world_size()
    elif args.gpu is not None:
        torch.cuda.set_device(args.gpu)
    from . import data, retrieval, similarity
    from . import dist as ddist
    split = args.num_loss_chunks if args.similarity_metric == "splitloss" else 1
    net = build_model(args)
    first = net[0] if isinstance(net, (list, tuple)) else net
    if args.similarity_metric == "splitloss" and args.pt_style == "dino":
        split = first.tokens                                              # args.numpatches = feats.shape[1] (utils_ret.py:736, :394-395)
    cross = split > 1 and args.stype == "cross"
    q_files = data.list_images(args.query_dir)
    v_files = data.list_images(args.val_dir)
    print(f"train: {len(v_files)} imgs / query: {len(q_files)} imgs")                         # :367
    qlo, qhi = ddist.shard_bounds(len(q_files), rank, world)
    vlo, vhi = ddist.shard_bounds(len(v_files), rank, world)
    query_u8 = data.load_files_u8(q_files[qlo:qhi], workers=args.workers)
    values_u8 = data.load_files_u8(v_files[vlo:vhi], workers=args.workers)
    k = min(args.topk, len(v_files))
    if world == 1:
        # splitloss: the reference never defines sim2 on that branch (:393-403) and stops at :412; background statistics
        # are only produced for the dot-product metric
        out = retrieval.run_retrieval(net, query_u8, values_u8, k=k, with_background=(split == 1), num_loss_chunks=split,
                                      cross=cross, threshold=args.sim_threshold)
    else:
        if split > 1:
            raise NotImplementedError("--similarity_metric splitloss runs on one GPU (the sharded path merges dot-product lists)")
        embed = retrieval.extract_features_multiscale if isinstance(net, (list, tuple)) else retrieval.extract_features
        gf = similarity.l2_normalize_(embed(net, values_u8))                                    # :386, :388
        qf = similarity.l2_normalize_(embed(net, query_u8))                                     # :387, :389
        q_sizes = [b - a for a, b in (ddist.shard_bounds(len(q_files), r, world) for r in range(world))]
        v_sizes = [b - a for a, b in (ddist.shard_bounds(len(v_files), r, world) for r in range(world))]
        main_v, main_l = ddist.sharded_topk(qf, gf, k, vlo, ddist.cuda_local_topk, ddist.cuda_merge, query_sizes=q_sizes)
        bg, _ = ddist.sharded_topk(gf, gf, min(2, len(v_files)), vlo, ddist.cuda_local_topk, ddist.cuda_merge,
                                   query_sizes=v_sizes)                                         # :403, :418
        out = {"values": main_v, "indices": main_l, "bg_values": bg[:, -1],
               "stats": retrieval.retrieval_stats(main_v[:, 0], bg[:, -1])}
    fid_val = None
    if args.fid_weights and world > 1:
        # every rank embeds its shard of both folders; the fp64 statistics are merged over the ranks (dcr_b200/fid.py)
        from . import fid, nets
        inc = nets.build_fid_inception(load_state_dict(args.fid_weights), max_batch=50)
        m1, s1 = fid.compute_statistics_of_path(args.val_dir, inc, 50, num_workers=args.workers, distributed=True)
        m2, s2 = fid.compute_statistics_of_path(args.query_dir, inc, 50, num_workers=args.workers, distributed=True)
        fid_val = fid.frechet_distance(m1, s1, m2, s2)
    if rank == 0:                                                                             # :375 only rank 0 writes
        dp = os.sep.join(os.path.normpath(args.query_dir).split(os.sep)[-3:])                  # :378
        save = f"ret_plots/{dp}/images/{args.pt_style}_{args.arch}_{args.similarity_metric}{args.stype}/"   # :408
        os.makedirs(save, exist_ok=True)
        torch.save({"values": out["values"].cpu(), "indices": out["indices"].cpu(), "query_files": q_files,
                    "gallery_files": v_files}, os.path.join(save, "topk.pth"))
        # torch.sparse_csr_tensor(d["crow_indices"], d["col_indices"], d["values"], size=d["size"]) rebuilds a matrix;
        # with --sim_threshold=-inf, .to_dense() of matches.pth is the reference's query-major similarity.pth (:414)
        for key, name, n_rows in (("matches", "matches.pth", len(q_files)), ("bg_matches", "matches_wtrain.pth", len(v_files))):
            if key in out:
                offsets, idx, scores = out[key]
                torch.save({"crow_indices": offsets.cpu(), "col_indices": idx.cpu(), "values": scores.cpu(),
                            "size": (n_rows, len(v_files)), "threshold": args.sim_threshold}, os.path.join(save, name))
        print("Simscores @x% part done")                                                     # :470
        print(out["stats"])
        if args.fid_weights:
            if fid_val is None:
                from . import fid, nets
                inc = nets.build_fid_inception(load_state_dict(args.fid_weights), max_batch=50)
                fid_val = fid.fid_from_images(inc, fid.load_resized(args.val_dir), fid.load_resized(args.query_dir))   # :597-600
            print({"fid": fid_val})
            out["stats"]["fid"] = fid_val
        with open(os.path.join(save, "stats.json"), "w") as f:
            json.dump(out["stats"], f)
    if args.distributed:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
