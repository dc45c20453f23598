"""Gallery-sharded retrieval over torch.distributed (one process per GPU, NCCL over NVLink/NVSwitch).

The reference's multi-GPU path (diff_retrieval.py:237-246, 288-317, 345-348; utils_ret.py:762-786) shards only the
gallery *loader* with a DistributedSampler, all_gathers (index, feats) after every batch and funnels everything to
rank 0, which then does the similarity alone (and it dead-locks as committed -- SURVEY.md 3.2).  Here each rank keeps
its 1/N of the gallery descriptors resident, every rank scores ALL queries against its shard with the fused kernel,
and one all-gather of the [Q,k] (score, index) pairs + a merge gives every rank the global top-k:

    rank r: embeds gallery rows [r*G/N, (r+1)*G/N) and queries [r*Q/N, (r+1)*Q/N)
    all_gather_into_tensor(query descriptors, f32)      Q*D*4 bytes total            (one collective)
    local fused sim+top-k with global index = base + local
    all_gather_into_tensor(packed (score, index))       N*Q*k*12 bytes               (one collective)
    merge N lists -> top-k by (score desc, index asc)   == top-k over the concatenated gallery

There is no data-path collective inside the kernels: the exchange is two small all-gathers per run (message sizes
are KBs..MBs, latency bound), so NCCL is the right tool.  The functions take the local scorer / merger as arguments
so the sharding logic is testable on CPU with the oracle under the gloo backend (tests/test_dist_cpu.py).

The threshold search has the same shape (`sharded_range`, C entry `dcr_sim_range_sharded`): each rank searches all
queries against its shard, a fixed-size header per rank is all-gathered first so that every rank reaches the same
outcome, then the CSR pieces, padded to the largest, and a device merge places them into the CSR of the whole gallery.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous shard [lo, hi) of n items for `rank`; sizes differ by at most one."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def all_gather_rows(x: torch.Tensor, sizes: Optional[list] = None) -> torch.Tensor:
    """Concatenate row blocks of every rank (blocks may differ in length by one).  One collective into one pre-sized
    buffer (`all_gather_into_tensor`): equal blocks land in place, ragged blocks are padded to the longest and compacted
    afterwards.  Descriptors travel as float32: the scores are float64-accumulated products of the float32 inputs, and
    rounding the queries to bf16 for the wire (3x fewer bytes of a transfer that is already < 0.5 ms over NVLink at
    50k x 512) would change them."""
    world = dist.get_world_size()
    if world == 1:
        return x
    if sizes is None:
        n = torch.tensor([x.shape[0]], device=x.device, dtype=torch.int64)
        ns = torch.empty(world, device=x.device, dtype=torch.int64)
        dist.all_gather_into_tensor(ns, n)
        sizes = [int(v) for v in ns.tolist()]
    mx = max(sizes)
    x = x.contiguous()
    if x.shape[0] != mx:
        pad = torch.zeros((mx,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        pad[:x.shape[0]] = x
        x = pad
    buf = torch.empty((world * mx,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(buf, x)
    if all(s == mx for s in sizes):
        return buf
    return torch.cat([buf[r * mx:r * mx + s] for r, s in enumerate(sizes)], dim=0)


def _pack_topk(s: torch.Tensor, i: torch.Tensor) -> torch.Tensor:
    """(scores f32 [Q,k], indices i64 [Q,k]) -> one int32 [Q,k,3] message: score bits, index low / high words."""
    iv = i.contiguous().view(torch.int32).view(i.shape[0], i.shape[1], 2)
    return torch.cat([s.contiguous().view(torch.int32).unsqueeze(-1), iv], dim=-1).contiguous()


def _unpack_topk(p: torch.Tensor):
    s = p[..., 0].contiguous().view(torch.float32)
    i = p[..., 1:].contiguous().view(torch.int64).squeeze(-1)
    return s, i


def sharded_topk(query_local: torch.Tensor, gallery_local: torch.Tensor, k: int, gallery_base: int,
                 local_topk: Callable, merge: Callable, query_sizes: Optional[list] = None
                 ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Global top-k for ALL queries on every rank.  query_local: this rank's block of query descriptors;
    gallery_local: this rank's gallery shard whose first row has global index `gallery_base`.
    local_topk(q, g, k, index_base) -> (scores [Q,k], idx [Q,k]); merge(scores [N,Q,k], idx [N,Q,k], k) -> ([Q,k],[Q,k])."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    q_all = all_gather_rows(query_local, query_sizes) if world > 1 else query_local
    kk = min(k, gallery_local.shape[0])
    s, i = local_topk(q_all, gallery_local, kk, gallery_base)
    if kk < k:   # a shard smaller than k: pad with empty entries
        pad_s = torch.full((s.shape[0], k - kk), float("-inf"), dtype=s.dtype, device=s.device)
        pad_i = torch.full((i.shape[0], k - kk), -1, dtype=i.dtype, device=i.device)
        s, i = torch.cat([s, pad_s], 1), torch.cat([i, pad_i], 1)
    if world == 1:
        return s, i
    # ONE collective for the per-shard lists: (score, index) packed into 12 bytes per entry
    msg = _pack_topk(s, i)
    allmsg = torch.empty((world * msg.shape[0],) + tuple(msg.shape[1:]), dtype=msg.dtype, device=msg.device)
    dist.all_gather_into_tensor(allmsg, msg)                   # rank-major concatenation along dim 0
    ss, ii = _unpack_topk(allmsg.view((world,) + tuple(msg.shape)))
    return merge(ss.contiguous(), ii.contiguous(), k)


def cuda_local_topk(q, g, k, index_base):
    from .similarity import sim_topk
    return sim_topk(q, g, k, index_base=index_base)


def split_local_topk(num_chunks: int, cross: bool = False) -> Callable:
    """local_topk of sharded_topk under the 'splitloss' similarity (similarity.sim_topk_split, aligned or cross parts)."""
    def local(q, g, k, index_base):
        from .similarity import sim_topk_split
        return sim_topk_split(q, g, k, num_chunks, cross=cross, index_base=index_base)
    return local


def cuda_merge(scores, idx, k):
    from .similarity import topk_merge
    return topk_merge(scores, idx, k)


def sharded_topk_c(query_all: torch.Tensor, gallery_local: torch.Tensor, k: int, gallery_base: int,
                   allgather: Optional[Callable] = None, world: Optional[int] = None, index_stride: int = 1
                   ) -> Tuple[torch.Tensor, torch.Tensor]:
    """The same exchange through the C entry `dcr_sim_topk_sharded` (include/dcr_b200.h): local fused top-k, ONE all-gather
    of the packed lists, merge -- all enqueued by the library on the current stream.  `query_all`: every query descriptor
    (already all-gathered); `allgather(send_ptr, recv_ptr, bytes_per_rank, stream_ptr) -> int` performs the collective
    (default: torch.distributed.all_gather_into_tensor over uint8 views of the two device buffers)."""
    import ctypes as C
    from . import _lib
    from .similarity import _aligned_ptr, _check_cuda_f32
    lib = _lib.load()
    q = _check_cuda_f32("query_all", query_all)
    g = _check_cuda_f32("gallery_local", gallery_local)
    if world is None:
        world = dist.get_world_size() if dist.is_initialized() else 1
    nq, d = q.shape
    ng = g.shape[0]
    cb = _allgather_callback(allgather, world, q.device, "sharded_topk_c")
    with torch.cuda.device(q.device):
        nbytes = lib.dcr_sim_topk_sharded_workspace_size(nq, ng, d, k, world)
        if nbytes == 0:
            raise _lib.DcrError(f"dcr_sim_topk_sharded_workspace_size: {_lib.last_error()}")
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=q.device)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
        st = torch.cuda.current_stream().cuda_stream
        rc = lib.dcr_sim_topk_sharded(q.data_ptr(), nq, g.data_ptr(), ng, d, k, gallery_base, index_stride, world,
                                      C.cast(cb, C.c_void_p), None, out_s.data_ptr(), out_i.data_ptr(), _aligned_ptr(ws), nbytes, st)
        _lib.check(rc, "dcr_sim_topk_sharded")
        torch.cuda.current_stream().synchronize()    # the workspace and the views above die with this frame
    return out_s, out_i


def _allgather_callback(allgather: Optional[Callable], world: int, device: torch.device, what: str):
    """The C callback (_lib.ALLGATHER_FN) the sharded entries call: `allgather(send_ptr, recv_ptr, bytes_per_rank,
    stream_ptr) -> int`, by default torch.distributed.all_gather_into_tensor over zero-copy uint8 views of the library's
    device buffers.  An exception becomes a non-zero return: it never unwinds through the C frame.  Keep the returned
    object alive for the duration of the call."""
    holders = []

    def default_allgather(send, recv, nbytes, stream):
        sv = device_bytes(send, nbytes, device)
        rv = device_bytes(recv, nbytes * world, device)
        holders.extend([sv, rv])
        dist.all_gather_into_tensor(rv, sv)
        return 0

    fn = allgather or default_allgather

    def trampoline(send, recv, nbytes, ctx, stream):
        try:
            return int(fn(send, recv, nbytes, stream))
        except Exception as e:                      # never unwind through the C frame
            print(f"dcr_b200.dist.{what}: all-gather callback raised {e!r}")
            return 1

    from . import _lib
    return _lib.ALLGATHER_FN(trampoline)


def sharded_range(query_all: torch.Tensor, gallery_local: torch.Tensor, threshold: float, gallery_base: int, *,
                  allgather: Optional[Callable] = None, world: Optional[int] = None, index_stride: int = 1,
                  num_chunks: int = 1, cross: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Threshold search over a gallery sharded across ranks, through the C entry `dcr_sim_range_sharded`
    (include/dcr_b200.h): every rank searches ALL queries against its shard (global index of local row j =
    gallery_base + index_stride * j), the CSR pieces are exchanged and merged on the device, and every rank returns
    (offsets i64[Q+1], indices i64[P], scores f32[P]) -- bit for bit what similarity.sim_range returns for the union of
    the shards.  `query_all`: every query descriptor (a query-sharded caller all-gathers them first with
    all_gather_rows).  `gallery_local` may have 0 rows; that rank still takes part in the exchanges.  `allgather` as in
    sharded_topk_c (default: torch.distributed.all_gather_into_tensor).  The capacities start where sim_range's do; when
    some rank needs more, every rank gets DCR_ERR_CAPACITY with the needs and retries once, together.
    num_chunks > 1: the 'splitloss' score over that many aligned parts (`dcr_sim_range_split_sharded`), bit for bit
    what similarity.sim_range_split returns for the union of the shards.  cross=True with num_chunks > 1: the cross
    score (`--stype cross`, `dcr_sim_range_cross_sharded`), bit for bit what similarity.sim_range_split(cross=True)
    returns for the union of the shards; with num_chunks = 1 it is the dot product.  Every rank must pass the same
    num_chunks and cross: ranks computing different scores raise DcrError ("disagree") instead of merging."""
    import ctypes as C
    from . import _lib
    from .similarity import _aligned_ptr, _check_cuda_f32
    lib = _lib.load()
    q = _check_cuda_f32("query_all", query_all)
    g = _check_cuda_f32("gallery_local", gallery_local)
    if world is None:
        world = dist.get_world_size() if dist.is_initialized() else 1
    nq, d = q.shape
    ng = g.shape[0]
    # a gallery of another dim or device is this rank's failure: it goes to the library as a missing gallery, so that
    # every rank returns the error instead of this one leaving its peers in the exchange
    g_ok = g.shape[1] == d and g.device == q.device
    g_ptr = (g.data_ptr() if ng > 0 else None) if g_ok else None
    cb = _allgather_callback(allgather, world, q.device, "sharded_range")
    split = num_chunks > 1
    what = ("dcr_sim_range_cross_sharded" if cross else "dcr_sim_range_split_sharded") if split else "dcr_sim_range_sharded"
    counts = (C.c_int64 * 3)()
    local_cap = out_cap = max(1 << 20, 16 * nq)   # sim_range's start; the exact needs come back with ERR_CAPACITY
    with torch.cuda.device(q.device):
        offsets = torch.empty(nq + 1, dtype=torch.int64, device=q.device)
        for attempt in range(2):
            # 0 (invalid arguments) is passed on: the library reports the reason on every rank
            if split:
                nbytes = getattr(lib, what + "_workspace_size")(nq, ng if g_ok else 1, d, num_chunks, world, local_cap)
            else:
                nbytes = lib.dcr_sim_range_sharded_workspace_size(nq, ng if g_ok else 1, d, world, local_cap)
            ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=q.device) if nbytes else None
            out_i = torch.empty(out_cap, dtype=torch.int64, device=q.device)
            out_s = torch.empty(out_cap, dtype=torch.float32, device=q.device)
            st = torch.cuda.current_stream().cuda_stream
            args = (gallery_base, index_stride, world, C.cast(cb, C.c_void_p), None, offsets.data_ptr(),
                    out_i.data_ptr() or None, out_s.data_ptr() or None, out_cap, local_cap, counts,
                    _aligned_ptr(ws) if ws is not None else None, nbytes, st)
            if split:
                rc = getattr(lib, what)(q.data_ptr(), nq, g_ptr, ng if g_ok else 1, d, num_chunks, float(threshold), *args)
            else:
                rc = lib.dcr_sim_range_sharded(q.data_ptr(), nq, g_ptr, ng if g_ok else 1, d, float(threshold), *args)
            if rc == _lib.ERR_CAPACITY and attempt == 0:
                local_cap, out_cap = int(counts[1]), int(counts[2])   # agreed by every rank: all retry together
                continue
            if rc != 0 and not g_ok:
                raise _lib.DcrError(f"{what}: gallery_local {tuple(g.shape)} on {g.device} does not "
                                    f"match query_all {tuple(q.shape)} on {q.device} ({_lib.last_error()})")
            _lib.check(rc, what)
            break
    n = int(counts[0])
    if n < out_cap:   # do not keep the whole capacity alive behind the result
        out_i, out_s = out_i[:n].clone(), out_s[:n].clone()
    return offsets, out_i, out_s


def device_bytes(ptr: int, nbytes: int, device: torch.device) -> torch.Tensor:
    """Zero-copy uint8 tensor over a raw device pointer (the library's workspace), for handing it to torch.distributed."""
    iface = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 2}
    holder = type("_DevicePtr", (), {"__cuda_array_interface__": iface})()
    return torch.as_tensor(holder, device=device)
