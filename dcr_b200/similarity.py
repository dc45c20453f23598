"""Host mirror of the reference's similarity / top-k step.

The reference has no function boundary here -- it is inline tensor code in `main_worker`:

    values_features = nn.functional.normalize(values_features, dim=1, p=2)      diff_retrieval.py:388
    query_features  = nn.functional.normalize(query_features,  dim=1, p=2)      diff_retrieval.py:389
    sim = torch.mm(values_features, query_features.T)                            diff_retrieval.py:402
    main_v, main_l = sim.T.topk(1, axis=1, largest=True)                         diff_retrieval.py:411,417
    bg_v = (values @ values.T).T.topk(2, axis=1)[0][:, -1]                       diff_retrieval.py:403,418-419

`sim_topk(query, gallery, k)` returns exactly what `torch.mm(gallery, query.T).T.topk(k, dim=1)` would (values,
indices), with a defined tie rule (lowest gallery index first) and without materialising the [Q,G] matrix.
`sim_range(query, gallery, threshold)` returns the entries of that matrix that reach a threshold, as CSR.
All compute happens in libdcr_b200.so on the tensors' CUDA device.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import torch

from . import _lib


def _check_cuda_f32(name: str, t: torch.Tensor) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise _lib.DcrError(f"{name} must be a CUDA tensor (dcr_b200 has no CPU compute path)")
    if t.dtype != torch.float32:
        raise _lib.DcrError(f"{name} must be float32, got {t.dtype}")
    if t.dim() != 2:
        raise _lib.DcrError(f"{name} must be 2-D [N, D], got shape {tuple(t.shape)}")
    return t.contiguous()


_ws_cache: dict = {}


def _workspace(nbytes: int, device: torch.device) -> torch.Tensor:
    key = (device.type, device.index)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=device)
        _ws_cache[key] = ws
    return ws


def _aligned_ptr(t: torch.Tensor, align: int = 256) -> int:
    p = t.data_ptr()
    return (p + align - 1) // align * align


def l2_normalize_(x: torch.Tensor, eps: float = 1e-12) -> torch.Tensor:
    """In-place `nn.functional.normalize(x, dim=1, p=2)` (diff_retrieval.py:388-389)."""
    lib = _lib.load()
    x = _check_cuda_f32("x", x)
    with torch.cuda.device(x.device):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.dcr_l2_normalize(x.data_ptr(), x.shape[0], x.shape[1], eps, st), "dcr_l2_normalize")
    return x


def sim_topk(query: torch.Tensor, gallery: torch.Tensor, k: int = 1, *, index_base: int = 0,
             index_stride: int = 1) -> Tuple[torch.Tensor, torch.Tensor]:
    """values f32[Q,k], indices i64[Q,k] of the k largest <query_i, gallery_j>, ties -> lowest j."""
    lib = _lib.load()
    q = _check_cuda_f32("query", query)
    g = _check_cuda_f32("gallery", gallery)
    if q.device != g.device:
        raise _lib.DcrError("query and gallery must be on the same device")
    if q.shape[1] != g.shape[1]:
        raise _lib.DcrError(f"descriptor dims differ: {q.shape[1]} vs {g.shape[1]}")
    nq, d = q.shape
    ng = g.shape[0]
    with torch.cuda.device(q.device):
        nbytes = lib.dcr_sim_topk_workspace_size(nq, ng, d, k)
        if nbytes == 0:
            raise _lib.DcrError(f"dcr_sim_topk_workspace_size: {_lib.last_error()}")
        ws = _workspace(nbytes, q.device)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
        st = torch.cuda.current_stream().cuda_stream
        rc = lib.dcr_sim_topk(q.data_ptr(), nq, g.data_ptr(), ng, d, k, index_base, index_stride, out_s.data_ptr(),
                              out_i.data_ptr(), _aligned_ptr(ws), nbytes, st)
        _lib.check(rc, "dcr_sim_topk")
    return out_s, out_i


def sim_range(query: torch.Tensor, gallery: torch.Tensor, threshold: float, *, index_base: int = 0,
              index_stride: int = 1) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Every (query i, gallery j) pair with score >= threshold, in CSR form: (offsets i64[Q+1], indices i64[P],
    scores f32[P]); row i is indices[offsets[i]:offsets[i+1]], gallery rows ascending, reported as
    index_base + index_stride * j.  Scores are bit for bit the ones sim_topk reports for the same pairs; NaN scores are
    never reported, threshold = -inf reports every pair.  The threshold is taken as fp32 (what the comparison sees).
    Replaces the score matrices the reference saves (diff_retrieval.py:402-403, 414-415) without forming them."""
    lib = _lib.load()
    q = _check_cuda_f32("query", query)
    g = _check_cuda_f32("gallery", gallery)
    if q.device != g.device:
        raise _lib.DcrError("query and gallery must be on the same device")
    if q.shape[1] != g.shape[1]:
        raise _lib.DcrError(f"descriptor dims differ: {q.shape[1]} vs {g.shape[1]}")
    threshold = float(threshold)
    if math.isnan(threshold):
        raise _lib.DcrError("sim_range: threshold is NaN")
    nq, d = q.shape
    ng = g.shape[0]
    counts = (C.c_int64 * 2)()
    cap = max(1 << 20, 16 * nq)   # a modest start; the exact need is known after the counting pass
    with torch.cuda.device(q.device):
        offsets = torch.empty(nq + 1, dtype=torch.int64, device=q.device)
        for attempt in range(2):
            nbytes = lib.dcr_sim_range_workspace_size(nq, ng, d, cap)
            if nbytes == 0:
                raise _lib.DcrError(f"dcr_sim_range_workspace_size: {_lib.last_error()}")
            ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=q.device)
            out_i = torch.empty(cap, dtype=torch.int64, device=q.device)
            out_s = torch.empty(cap, dtype=torch.float32, device=q.device)
            st = torch.cuda.current_stream().cuda_stream
            rc = lib.dcr_sim_range(q.data_ptr(), nq, g.data_ptr(), ng, d, threshold, index_base, index_stride,
                                   offsets.data_ptr(), out_i.data_ptr(), out_s.data_ptr(), cap, counts, _aligned_ptr(ws),
                                   nbytes, st)
            if rc == _lib.ERR_CAPACITY and attempt == 0:
                cap = int(counts[1])   # the candidate count is a fixed function of the inputs: this capacity fits
                continue
            _lib.check(rc, "dcr_sim_range")
            break
    n = int(counts[0])
    if n < cap:   # do not keep the whole capacity alive behind the result
        out_i, out_s = out_i[:n].clone(), out_s[:n].clone()
    return offsets, out_i, out_s


def sim_topk_split(q: torch.Tensor, g: torch.Tensor, k: int, num_chunks: int, cross: bool = False
                   ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Top-k under the 'splitloss' similarity of diff_retrieval.py:393-400 (--similarity_metric splitloss,
    --num_loss_chunks C): score(q, g) = max_c <q_c, g_c> over the C equal parts of the descriptors.
    One fused similarity+top-k pass per part (the true top-k is contained in the union of the per-part top-k lists),
    then dcr_split_rescore evaluates the exact split score of the <= C*k candidates per query and selects.
    cross=True is `--stype cross` (einsum_in_chunks :643-662): score = max over every (gallery part, query part) pair.
    Candidates then come from ONE fused pass over the part matrices [Q*C, D/C] x [G*C, D/C] with
    k' = (k-1)*C + 1 rows per query part (fewer than k' part-rows can beat the best part-row of a true top-k gallery row)
    while k' <= 16, otherwise from one pass per gallery part with k' = k (no limit on the number of parts)."""
    lib = _lib.load()
    if num_chunks == 1:
        return sim_topk(q, g, k)
    if cross:
        return _sim_topk_cross(lib, q, g, k, num_chunks)
    if not (q.is_cuda and g.is_cuda):
        raise _lib.DcrError("sim_topk_split needs CUDA tensors")
    q = q.contiguous().float()
    g = g.contiguous().float()
    nq, d = q.shape
    if d % num_chunks or (d // num_chunks) % 4:
        raise _lib.DcrError(f"splitloss: descriptor dim {d} must split into {num_chunks} parts of a multiple of 4 dims")
    if num_chunks * k > 4096:
        raise _lib.DcrError("splitloss: num_chunks * k must be <= 4096")
    p = d // num_chunks
    cand = torch.empty((nq, num_chunks * k), dtype=torch.int64, device=q.device)
    for c in range(num_chunks):
        _, idx = sim_topk(q[:, c * p:(c + 1) * p].contiguous(), g[:, c * p:(c + 1) * p].contiguous(), k)
        cand[:, c * k:(c + 1) * k] = idx
    out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    with torch.cuda.device(q.device):
        st = torch.cuda.current_stream().cuda_stream
        rc = lib.dcr_split_rescore(q.data_ptr(), g.data_ptr(), nq, d, num_chunks, 0, cand.data_ptr(), num_chunks * k, k,
                                   out_s.data_ptr(), out_i.data_ptr(), st)
        _lib.check(rc, "dcr_split_rescore")
    return out_s, out_i


def _sim_topk_cross(lib, q: torch.Tensor, g: torch.Tensor, k: int, c: int) -> Tuple[torch.Tensor, torch.Tensor]:
    if not (q.is_cuda and g.is_cuda):
        raise _lib.DcrError("sim_topk_split needs CUDA tensors")
    q = q.contiguous().float()
    g = g.contiguous().float()
    nq, d = q.shape
    ng = g.shape[0]
    if d % c or (d // c) % 4:
        raise _lib.DcrError(f"splitloss: descriptor dim {d} must split into {c} parts of a multiple of 4 dims")
    kk = (k - 1) * c + 1
    p = d // c
    if kk <= 16:
        # one fused pass over the part matrices: a gallery row of the true top-k is reached through its best
        # (query part, gallery part) pair, and fewer than (k-1)*c + 1 part-rows can beat that part-row
        kk = min(kk, ng * c)
        _, idx = sim_topk(q.view(nq * c, p), g.view(ng * c, p), kk)            # rows of the part matrices
        cand = (idx // c).reshape(nq, c * kk).contiguous()                      # gallery rows the part-rows belong to
    else:
        # any number of parts (the reference default topk = 10 with num_loss_chunks >= 2, diff_retrieval.py:643-662):
        # one fused pass per GALLERY part against all query parts with k' = k.  Within the list of the pair
        # (query part a, gallery part b) every row that beats a true top-k row also beats it in the cross score, so
        # the union of the c*c per-pair top-k lists contains the true top-k.
        if c * c * k > 4096:
            raise _lib.DcrError(f"splitloss cross: {c} parts x top-{k} needs {c * c * k} candidates per query (max 4096)")
        kq = min(k, ng)
        cand = torch.full((nq, c, c, k), -1, dtype=torch.int64, device=q.device)
        qparts = q.view(nq * c, p)
        for b in range(c):
            _, idx = sim_topk(qparts, g[:, b * p:(b + 1) * p].contiguous(), kq)   # [nq*c, kq] gallery rows
            cand[:, :, b, :kq] = idx.view(nq, c, kq)
        cand = cand.reshape(nq, c * c * k).contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=q.device)
    with torch.cuda.device(q.device):
        st = torch.cuda.current_stream().cuda_stream
        rc = lib.dcr_split_rescore(q.data_ptr(), g.data_ptr(), nq, d, c, 1, cand.data_ptr(), cand.shape[1], k,
                                   out_s.data_ptr(), out_i.data_ptr(), st)
        _lib.check(rc, "dcr_split_rescore")
    return out_s, out_i


def sim_topk_stats() -> dict:
    lib = _lib.load()
    arr = (C.c_int * 8)()
    lib.dcr_sim_topk_last_stats(arr)
    keys = ["cta_group", "grid", "smem_bytes", "stages", "kp", "cap", "n_flagged", "d_pad"]
    st = dict(zip(keys, list(arr)))
    st["kernel_ms"] = float(lib.dcr_sim_topk_last_kernel_ms())
    st["n_second"] = int(lib.dcr_sim_topk_last_second_pass())
    st["sm_mhz"] = float(lib.dcr_sim_topk_last_sm_mhz())
    st["epilogue_sets"] = int(lib.dcr_sim_topk_last_epilogue_sets())
    return st


def kernel_launch_count() -> int:
    return int(_lib.load().dcr_kernel_launch_count())


def topk_merge(scores: torch.Tensor, idx: torch.Tensor, k_out: Optional[int] = None
               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Merge per-shard results: scores/idx [nlists, Q, k_in] -> [Q, k_out] by (score desc, idx asc)."""
    lib = _lib.load()
    if not (scores.is_cuda and idx.is_cuda):
        raise _lib.DcrError("topk_merge needs CUDA tensors")
    scores = scores.contiguous().float()
    idx = idx.contiguous().long()
    nl, nq, k_in = scores.shape
    k_out = k_in if k_out is None else k_out
    out_s = torch.empty((nq, k_out), dtype=torch.float32, device=scores.device)
    out_i = torch.empty((nq, k_out), dtype=torch.int64, device=scores.device)
    with torch.cuda.device(scores.device):
        st = torch.cuda.current_stream().cuda_stream
        rc = lib.dcr_topk_merge(scores.data_ptr(), idx.data_ptr(), nq, nl, k_in, k_out, out_s.data_ptr(),
                                out_i.data_ptr(), st)
        _lib.check(rc, "dcr_topk_merge")
    return out_s, out_i
