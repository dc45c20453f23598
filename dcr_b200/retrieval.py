"""Embed -> normalise -> similarity -> top-k: the host-side mirror of diff_retrieval.py's `main_worker` hot path.

    extract_features(net, images)        utils_ret.py:704-787 (single process: H2D per batch, forward, rows kept on GPU)
    retrieve(query, gallery, k)          diff_retrieval.py:388-389 (normalize) + :402,:411,:417 (mm, T, topk)
    background_similarity(gallery)       diff_retrieval.py:403,:418-419
    retrieval_stats(main_v, bg_v)        diff_retrieval.py:442-454 (same keys as the wandb/print dict :456-483)
    run_retrieval(...)                   the `if args.rank == 0:` block :375-419 end to end

Differences from the reference, all deliberate (SURVEY.md appendix B): features stay on the GPU (the reference moves
every batch to the CPU, utils_ret.py:786, and runs mm/topk there); the full [Q,G] / [G,G] matrices are never
built or saved; `torch.argsort(-sim)` (:405, result unused) is not computed; ties are ordered by lowest index.
"""
from __future__ import annotations

from typing import Dict, Iterable, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .nets import DcrNet
from .similarity import l2_normalize_, sim_range, sim_topk, sim_topk_split


@torch.no_grad()
def extract_features(net: DcrNet, images: torch.Tensor, batch_size: Optional[int] = None,
                     two_in_flight: Optional[bool] = None) -> torch.Tensor:
    """images: uint8 [N,H,W,3], either already on the GPU or on the host (pinned memory makes the copies async).
    Returns fp32 [N, D] on the GPU.  Host batches are copied on a side stream into a ring of staging buffers so the H2D
    transfer of batch i+1 overlaps the forward pass of batch i (the reference copies synchronously per batch,
    utils_ret.py:711-712).  With more than one batch, consecutive batches alternate between the network and a fork of
    it (same weights, own activations: DcrNet.twin) on two streams: the persistent kernels of one forward pass fill the
    SMs the other leaves idle at its wave tails and pipeline ramps (+15 % images/s on the SSCD ResNet-50, batch 256,
    tools/dual_stream.py).  Rows are bit-identical either way; `two_in_flight=False` keeps everything on one stream."""
    if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[-1] != 3:
        raise _lib.DcrError("extract_features expects uint8 [N,H,W,3]")
    bs = net.max_batch if batch_size is None else min(batch_size, net.max_batch)
    n = images.shape[0]
    dev = net.device
    out = torch.empty((n, net.out_dim), dtype=torch.float32, device=dev)
    if n == 0:
        return out
    dual = (n > bs) if two_in_flight is None else (bool(two_in_flight) and n > bs)
    main = torch.cuda.current_stream(dev)
    execs = [(net, main)]
    if dual:
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(main)          # the fork's buffers / `out` may still be in use by work queued on the caller's stream
        try:
            execs.append((net.twin(), side))
        except _lib.DcrError:           # no memory for a second set of activations: one forward pass at a time
            dual = False
    starts = list(range(0, n, bs))
    if images.is_cuda:
        for i, s in enumerate(starts):
            ex, st = execs[i % len(execs)]
            with torch.cuda.stream(st):
                out[s:s + bs] = ex(images[s:s + bs])
        if dual:
            main.wait_stream(side)
        return out
    copy = torch.cuda.Stream(device=dev)
    n_slots = 2 * len(execs)
    stage = [torch.empty((bs,) + tuple(images.shape[1:]), dtype=torch.uint8, device=dev) for _ in range(n_slots)]
    # The staging blocks come from the caller's stream's allocator pool: a previous call's forward passes (still queued
    # there -- the host runs far ahead of the GPU) may be reading the very same memory.  The copy stream must not write
    # into them before everything already queued on that stream has finished.
    copy.wait_stream(main)
    ready = [torch.cuda.Event() for _ in range(n_slots)]
    freed = [torch.cuda.Event() for _ in range(n_slots)]
    for i, s in enumerate(starts):
        b = min(bs, n - s)
        slot = i % n_slots
        ex, st = execs[i % len(execs)]
        with torch.cuda.stream(copy):
            if i >= n_slots:
                copy.wait_event(freed[slot])
            stage[slot][:b].copy_(images[s:s + b], non_blocking=True)
            ready[slot].record(copy)
        st.wait_event(ready[slot])
        with torch.cuda.stream(st):
            out[s:s + b] = ex(stage[slot][:b])
            freed[slot].record(st)
    if dual:
        main.wait_stream(side)
    # the staging buffers go back to the caller's pool on return: everything that touched them is ordered before `main` now
    main.wait_stream(copy)
    return out


MULTI_SCALES = (1.0, 1.0 / 2 ** 0.5, 0.5)       # utils_ret.py:678 "we use 3 different scales"


@torch.no_grad()
def extract_features_multiscale(nets_by_scale, images: torch.Tensor, batch_size: Optional[int] = None) -> torch.Tensor:
    """`extract_features(..., multiscale=True)` (utils_ret.py:676-698, :714-715): the mean over the three scales of the
    model's descriptor.  `nets_by_scale`: one network per entry of MULTI_SCALES, built with
    `build_sscd_resnet50(sd, scale_factor=s)` (the bilinear resize of the transformed crop is fused into the first
    kernel).  The reference then divides the whole batch tensor by ITS Frobenius norm (`v /= v.norm()`, :697) -- one
    scalar per loader batch, which the per-row normalisation of diff_retrieval.py:388-389 removes again; it is not
    applied here.  Convolutional trunks only (a ViT would need interpolated position embeddings)."""
    if len(nets_by_scale) != len(MULTI_SCALES):
        raise _lib.DcrError(f"extract_features_multiscale needs {len(MULTI_SCALES)} networks (scales {MULTI_SCALES})")
    out = None
    for net in nets_by_scale:
        f = extract_features(net, images, batch_size)
        out = f if out is None else out.add_(f)
    return out.div_(float(len(nets_by_scale)))


def retrieve(query_features: torch.Tensor, gallery_features: torch.Tensor, k: int = 1, normalize: bool = True,
             index_base: int = 0, index_stride: int = 1) -> Tuple[torch.Tensor, torch.Tensor]:
    """(values [Q,k], indices [Q,k]) == torch.mm(normalize(G), normalize(Q).T).T.topk(k)  (diff_retrieval.py:388-417)."""
    q = query_features.float().contiguous()
    g = gallery_features.float().contiguous()
    if normalize:                      # never modify the caller's tensors
        q = l2_normalize_(q.clone())
        g = l2_normalize_(g.clone())
    return sim_topk(q, g, k, index_base=index_base, index_stride=index_stride)


def background_similarity(gallery_features: torch.Tensor, normalize: bool = True) -> torch.Tensor:
    """bg_v of diff_retrieval.py:403,418-419: per gallery row, the second largest similarity to the gallery (the largest
    being the row itself)."""
    g = gallery_features.float().contiguous()
    if normalize:
        g = l2_normalize_(g.clone())
    v, _ = sim_topk(g, g, 2)
    return v[:, -1]


def retrieval_stats(main_v: torch.Tensor, bg_v: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """Same keys and numpy calls as diff_retrieval.py:442-454 (computed on the host on Q / G scalars)."""
    x0 = main_v.detach().float().cpu().numpy().reshape(-1)
    st = {"sim_mean": float(np.mean(x0)), "sim_std": float(np.std(x0)), "sim_75pc": float(np.percentile(x0, 75)),
          "sim_90pc": float(np.percentile(x0, 90)), "sim_95pc": float(np.percentile(x0, 95)),
          "sim_gt_05pc": float(np.sum(x0 > 0.5) / x0.shape[0])}
    if bg_v is not None:
        x1 = bg_v.detach().float().cpu().numpy().reshape(-1)
        st.update({"bg_mean": float(np.mean(x1)), "bg_std": float(np.std(x1)), "bg_75pc": float(np.percentile(x1, 75)),
                   "bg_90pc": float(np.percentile(x1, 90)), "bg_95pc": float(np.percentile(x1, 95))})
    return st


def run_retrieval(net: DcrNet, query_images: torch.Tensor, gallery_images: torch.Tensor, k: int = 1,
                  with_background: bool = False, batch_size: Optional[int] = None,
                  num_loss_chunks: int = 1, cross: bool = False, threshold: Optional[float] = None) -> Dict[str, object]:
    """Embed both image sets and match them (the rank-0 block of diff_retrieval.py:386-419).  With a threshold, also
    every pair scoring at least that much (sim_range, CSR): out["matches"] (query x gallery, the entries of the
    reference's similarity.pth, :402, :414) and, with the background, out["bg_matches"] (the gallery self-join, diagonal
    included, as similarity_wtrain.pth, :403, :415).  Dot-product metric only."""
    if threshold is not None and num_loss_chunks > 1:
        raise NotImplementedError("a similarity threshold is implemented for the dot-product metric only")
    if isinstance(net, (list, tuple)):                                      # multiscale=args.multiscale (:386-387)
        values_features = extract_features_multiscale(net, gallery_images, batch_size)
        query_features = extract_features_multiscale(net, query_images, batch_size)
    else:
        values_features = extract_features(net, gallery_images, batch_size)   # :386
        query_features = extract_features(net, query_images, batch_size)     # :387
    l2_normalize_(values_features)                                           # :388
    l2_normalize_(query_features)                                            # :389
    if num_loss_chunks > 1:                                                  # :393-400 ('splitloss', aligned parts)
        main_v, main_l = sim_topk_split(query_features, values_features, k, num_loss_chunks, cross=cross)
    else:
        main_v, main_l = sim_topk(query_features, values_features, k)         # :402, :411, :417
    out = {"values": main_v, "indices": main_l, "query_features": query_features,
           "gallery_features": values_features}
    bg_v = None
    if with_background:
        bg, _ = sim_topk(values_features, values_features, 2)                 # :403, :418
        bg_v = bg[:, -1]                                                      # :419
        out["bg_values"] = bg_v
    if threshold is not None:
        out["matches"] = sim_range(query_features, values_features, threshold)
        if with_background:
            out["bg_matches"] = sim_range(values_features, values_features, threshold)
    out["stats"] = retrieval_stats(main_v[:, 0], bg_v)
    return out
