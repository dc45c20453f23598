// Threshold search for sm_90a (dcr_sim_range): every pair scoring at least tau, exact, in CSR form.  It replaces the saved
// score matrices of diff_retrieval.py:402-403, 414-415 and the threshold of :454.  Stage 1 and the fused sweep are the
// top-k search's (sim_sweep.cuh): the sweep's epilogue compares each approximate score against a per-row threshold that
// no qualifying pair can fall below, and the candidates are re-scored with the same fp64 dot product.
#include <algorithm>
#include <cmath>

#include "../../include/dcr_b200.h"
#include "dcr_internal.cuh"
#include "sim_sweep.cuh"

namespace dcr {

namespace {

// ------------------------------------------------------------------------------------------------------------
// Threshold search (dcr_sim_range): every pair with fp32(exact score) >= tau, in CSR form.
//   1. range_threshold_kernel  per query row the candidate threshold t_i on the approximate score: no pair whose fp32
//                              exact score reaches tau has an approximate score below t_i (row_bound)
//   2. sim_range_kernel<*, 0>  count sweep: candidates per (segment slot, row)
//   3. range_slot_scan_kernel + exclusive_scan_kernel: per row, the slots' offsets in gallery order; the rows' offsets
//   4. sim_range_kernel<*, 1>  emit sweep: the same decisions again, each row's candidates written in ascending order
//   5. range_rescore_kernel    exact scores in pieces of kRangePiece candidates of one row, stable compaction to the
//                              pairs that reach tau
//   6. exclusive_scan_kernel over the pieces, range_output_kernel / range_row_offsets_kernel: the CSR arrays
// Everything is a fixed function of the inputs (no atomics decide an order), so every call returns the same bits.
// Under the split score (sim_range_split, n_parts > 0) the same steps run on the split operands: the sweep folds the
// parts into a running maximum (fused_tile_mma_split), the bound is split_row_bound and the re-score takes the maximum
// of the per-part exact dot products (DESIGN.md section 3).  Under the cross split score (sim_range_cross) the sweep walks
// every (query part, gallery part) pair (fused_tile_mma_split<., true>), the bound is cross_row_bound and the re-score
// folds every pair (cross_exact_scores).
constexpr int kRangePiece = 512;   // candidates of one row re-scored by one block

struct RangeParams : SweepHead {
  int stages;
  const int* bias_flag;
  const float* col_bias;
  const float* thr;            // [nq] candidate threshold t_i
  int* seg;                    // [n_slots][128] count sweep: candidates; emit sweep: offset inside the row
  const long long* row_cand;   // [nq + 1] emit sweep: first candidate of each row
  int* cand_idx;               // emit sweep: local gallery rows
  int kb_part;                 // split score: k-blocks per descriptor part (kSplit kernels only)
};

// Candidate columns of one 32-column chunk of an accumulator row: bit c is set when the approximate score of column
// col0 + c is not below t (NaN included: the exact score decides) and c < n_valid.  Columns past the gallery are cut by
// n_valid rather than by mask_tail: at t = -inf their -inf would pass.
template <bool kBias>
DCR_DEVICE uint32_t range_hits(const uint32_t (&r)[32], const float* sb, float t, int n_valid) {
  float v[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) v[c] = __uint_as_float(r[c]);
  if constexpr (kBias) {   // the same fp32 additions as scan_chunk
#pragma unroll
    for (int c = 0; c < 32; c += 4) {
      const float4 b = *reinterpret_cast<const float4*>(sb + c);
      v[c] += b.x; v[c + 1] += b.y; v[c + 2] += b.z; v[c + 3] += b.w;
    }
  }
  uint32_t m = 0;
#pragma unroll
  for (int c = 0; c < 32; ++c) m |= static_cast<uint32_t>(!(v[c] < t)) << c;
  if (n_valid < 32) m &= n_valid <= 0 ? 0u : (1u << n_valid) - 1u;
  return m;
}

// The fused sweep of the threshold search: the work decomposition, pipeline and k-loop of sim_topk_kernel with one
// consumer warpgroup, an epilogue that compares every accumulator column against its row's threshold, and no warm-up.
// kEmit = 0 counts the candidates of every (segment slot, row); kEmit = 1 writes them at the offsets the scan derived
// from those counts.  Both make the same decisions: same tiles, same wgmma sequence, same thresholds.
// kSplit: the split score.  A tile's approximate score is the maximum over the descriptor parts (fused_tile_mma_split),
// and range_hits sees that maximum.  The running maximum and the part accumulator of a 128-column tile would take 256
// registers per thread, so two consumer warpgroups each own one 64-column half of every tile, as in the split top-k.
// After each tile the halves trade their per-row hit counts through shared memory: the lower half's columns come first
// in the row, so both halves count the same total and the emit sweep writes the row in ascending column order.
// kCross: the cross split score, the same kernel with the cross schedule of the part pairs.
template <bool kBias, bool kEmit, bool kSplit = false, bool kCross = false>
__global__ void __launch_bounds__(32 + 128 * (kSplit ? 2 : 1), 1)
    sim_range_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_g,
                     const RangeParams p) {
  static_assert(!kSplit || !kBias, "the split score is not centred");
  static_assert(!kCross || kSplit, "the cross score is a split score");
  constexpr int kSets = kSplit ? 2 : 1;
  constexpr int kSetCols = kBlockN / kSets;
  if (((p.bias_flag != nullptr) && (*p.bias_flag != 0)) != kBias) return;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // the pipeline, then barriers, then 4 kSets transpose buffers (split: then the halves' hit counts [2][2][128])
  const FusedPipe pp(smem_raw, p.num_kb, p.stream_a, p.stages, 0);
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31;
  pp.init(&tmap_q, &tmap_g, p.stages, 4 * kSets);
  const long long n_units = gridDim.x;
  const long long unit = blockIdx.x;
  SegWalker w(p.n_qtiles, p.n_gtiles, p.gchunk, p.n_chunks, unit, n_units);
  if (warp == 4 * kSets) {
    fused_producer<kCross>(pp, &tmap_q, &tmap_g, p.stages, w, [](const SegWalker&) { return 0; }, p.kb_part);
  } else {
    const uint32_t set = kSplit ? warp >> 2 : 0;                    // column half of every tile (split)
    const uint32_t row = (kSplit ? warp & 3 : warp) * 32 + lane;   // query row inside the tile
    const uint32_t xacc = smem_u32(pp.tail) + warp * kAccXposeWarpBytes;
    // [tile parity][set][row]: tile n writes buffer n & 1, so a half that runs ahead never overwrites a count the
    // other half has yet to read (it first passes the barrier of tile n + 1)
    int* half_cnt = reinterpret_cast<int*>(pp.tail + 4 * kSets * kAccXposeWarpBytes);
    const uint32_t a_base = smem_u32(pp.stream_a ? pp.smem_b + kBTileBytes : pp.smem_a);
    const uint32_t b_base = smem_u32(pp.smem_b) + set * kSetCols * 128;
    PipeState st(p.stages);
    uint32_t seg = 0;
    uint32_t tile_no = 0;   // tiles swept so far (split: the parity of the hit-count buffer)
    while (w.next()) {
      const int qrow = w.qi * kBlockM + static_cast<int>(row);
      const bool row_ok = qrow < p.nq;
      const float t = row_ok ? p.thr[qrow] : INFINITY;
      const size_t sr = static_cast<size_t>(slot_index(w.chunk, static_cast<int>(unit), w.qi, 0, static_cast<int>(n_units),
                                                       p.n_qtiles, 1)) * kBlockM + row;
      int cnt = 0;
      int* out = nullptr;
      if (kEmit && row_ok) out = p.cand_idx + p.row_cand[qrow] + p.seg[sr];
      if (!pp.stream_a) mbar_wait(pp.a_full, seg & 1);
#pragma unroll 1
      for (int j = 0; j < w.ntiles; ++j) {
        if constexpr (kSplit) {
          WgAcc<kSetCols> acc;
          fused_tile_mma_split<kSetCols, kCross>(acc, st, pp, a_base, b_base, p.kb_part, j == w.ntiles - 1, lane);
          const int gcol0 = (w.g_begin + j) * kBlockN + static_cast<int>(set) * kSetCols;
          uint32_t hits[kSetCols / 32];
          int mine = 0;
#pragma unroll
          for (int ch = 0; ch < kSetCols / 32; ++ch) {
            uint32_t r[32];
            acc.rows32(ch, r, xacc, lane);
            const int col0 = gcol0 + ch * 32;
            hits[ch] = range_hits<false>(r, nullptr, t, row_ok ? p.ng - col0 : 0);
            mine += __popc(hits[ch]);
          }
          int* hc = half_cnt + (tile_no & 1) * 2 * kBlockM;
          hc[set * kBlockM + row] = mine;
          named_bar_sync(1, 128 * kSets);
          const int lower = hc[row], both = lower + hc[kBlockM + row];
          ++tile_no;
          if constexpr (kEmit) {
            if (mine) {
              int* o = out + (set ? lower : 0);
#pragma unroll
              for (int ch = 0; ch < kSetCols / 32; ++ch)
                for (uint32_t h = hits[ch]; h; h &= h - 1) *o++ = gcol0 + ch * 32 + __ffs(h) - 1;   // ascending columns
            }
            if (both) out += both;
          } else {
            cnt += both;
          }
        } else {
          WgAcc<kBlockN> acc;
          fused_tile_mma(acc, st, pp, a_base, b_base, j == w.ntiles - 1, lane);
          const int gcol0 = (w.g_begin + j) * kBlockN;
#pragma unroll
          for (int ch = 0; ch < kBlockN / 32; ++ch) {
            uint32_t r[32];
            acc.rows32(ch, r, xacc, lane);
            const int col0 = gcol0 + ch * 32;
            const uint32_t hits = range_hits<kBias>(r, kBias ? p.col_bias + col0 : nullptr, t, row_ok ? p.ng - col0 : 0);
            if constexpr (kEmit) {
              for (uint32_t h = hits; h; h &= h - 1) *out++ = col0 + __ffs(h) - 1;   // ascending columns
            } else {
              cnt += __popc(hits);
            }
          }
        }
      }
      ++seg;
      if (!kEmit && set == 0) p.seg[sr] = cnt;   // split: both halves hold the row's total
    }
  }
  __syncthreads();
}

// t_i = tau - q.mu - eps - slack - margin, rounded down at every step.  fp32(s) >= tau needs s >= tau - half an fp32 ulp
// (margin), hence approximate score >= t_i (row_bound).  A warp per query row.
// kSplit: the split score, with eps and slack from split_row_bound (q.mu = 0; d_pad = n_parts * p_pad).  A NaN part norm
// makes eps and t_i NaN, and !(a < NaN) keeps every column of that row: the exact re-score decides them all.
// kCross: the cross split score, eps and slack from cross_row_bound.
template <bool kSplit, bool kCross = false>
__global__ void __launch_bounds__(128)
    range_threshold_kernel(const float* __restrict__ q, int nq, int d, int d_pad, int n_parts, float tau,
                           const float* __restrict__ q_norm_hat, const float* __restrict__ q_norm_res,
                           const float* __restrict__ q_norm_x, const unsigned int* __restrict__ g_max,
                           const float* __restrict__ mu, const float* __restrict__ nu, const int* __restrict__ nu_flag,
                           float* __restrict__ thr) {
  const int row = blockIdx.x * 4 + static_cast<int>(threadIdx.x >> 5);
  const uint32_t lane = threadIdx.x & 31;
  if (row >= nq) return;
  const RowBound rb = [&] {
    if constexpr (kCross)
      return cross_row_bound(n_parts, d / n_parts, d_pad / n_parts, row, q_norm_hat, q_norm_res, q_norm_x, g_max, lane);
    else if constexpr (kSplit)
      return split_row_bound(n_parts, d / n_parts, d_pad / n_parts, row, q_norm_hat, q_norm_res, q_norm_x, g_max, lane);
    else
      return row_bound(q + static_cast<size_t>(row) * d, d, d_pad, row, q_norm_hat, q_norm_res, q_norm_x, g_max, mu, nu,
                       nu_flag, lane);
  }();
  if (lane == 0) {
    const double margin = isfinite(tau) ? fabs(static_cast<double>(tau)) * 1.2e-7 + 1e-45 : 0.0;
    double t = __dsub_rd(static_cast<double>(tau), rb.qmu);
    t = __dsub_rd(t, static_cast<double>(rb.eps));
    t = __dsub_rd(t, rb.slack);
    t = __dsub_rd(t, margin);
    thr[row] = __double2float_rd(t);
  }
}

// Per query row (a thread each): walk the row's segment slots in gallery order -- chunk by chunk, and inside a chunk unit
// by unit (a unit's tiles follow the previous unit's) -- replacing each count by the row's candidates before it.
__global__ void __launch_bounds__(256)
    range_slot_scan_kernel(int* __restrict__ seg, int nq, int n_qtiles, int n_gtiles, int gchunk, int n_chunks,
                           int n_units, long long* __restrict__ row_cnt, long long* __restrict__ row_pieces) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= nq) return;
  const int qi = row / kBlockM, r = row % kBlockM;
  int acc = 0;
  for (int chunk = 0; chunk < n_chunks; ++chunk) {
    const int ncg = min(gchunk, n_gtiles - chunk * gchunk);
    const long long T = static_cast<long long>(n_qtiles) * ncg;
    const int u_lo = static_cast<int>(owner_unit(static_cast<long long>(qi) * ncg, T, n_units));
    const int u_hi = static_cast<int>(owner_unit(static_cast<long long>(qi + 1) * ncg - 1, T, n_units));
    for (int u = u_lo; u <= u_hi; ++u) {
      const size_t sr = static_cast<size_t>(slot_index(chunk, u, qi, 0, n_units, n_qtiles, 1)) * kBlockM + r;
      const int c = seg[sr];
      seg[sr] = acc;
      acc += c;
    }
  }
  row_cnt[row] = acc;
  row_pieces[row] = (acc + kRangePiece - 1) / kRangePiece;
}

// out[0..n] = exclusive prefix sums of in[0..n-1] (out[n] = total), one block: thread t sums a contiguous run, the runs'
// sums are scanned in shared memory, then each thread writes its run.  Fixed association.
template <typename T>
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(const T* __restrict__ in, long long n, long long* __restrict__ out) {
  __shared__ long long part[32];
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  const long long per = (n + 1023) / 1024;
  const long long lo = min(n, tid * per), hi = min(n, lo + per);
  long long s = 0;
  for (long long i = lo; i < hi; ++i) s += in[i];
  long long incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long v = __shfl_up_sync(kFull, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) part[wp] = incl;
  __syncthreads();
  if (wp == 0) {
    long long x = part[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long v = __shfl_up_sync(kFull, x, o);
      if (lane >= o) x += v;
    }
    part[lane] = x;   // inclusive over warps
  }
  __syncthreads();
  long long run = incl - s + (wp > 0 ? part[wp - 1] : 0);
  for (long long i = lo; i < hi; ++i) {
    out[i] = run;
    run += in[i];
  }
  if (tid == 0) out[n] = part[31];
}

// piece w: row, first candidate and candidate count (row_piece[0] = 0 <= w < row_piece[nq])
DCR_DEVICE void range_piece(long long w, const long long* __restrict__ row_cand, const long long* __restrict__ row_piece,
                            int nq, int& row, long long& start, int& n) {
  int lo = 0, hi = nq;   // row_piece[lo] <= w < row_piece[hi]
  while (hi - lo > 1) {
    const int mid = lo + (hi - lo) / 2;
    if (row_piece[mid] <= w) lo = mid;
    else hi = mid;
  }
  row = lo;
  start = row_cand[lo] + (w - row_piece[lo]) * kRangePiece;
  n = static_cast<int>(min(static_cast<long long>(kRangePiece), row_cand[lo + 1] - start));
}

// Exact scores of one piece (exact_dot: the values dcr_sim_topk reports), then a stable in-place
// compaction of the pairs with fp32 score >= tau.  piece_kept[w] = pairs kept.
// kSplit: the split score, bit for bit what dcr_split_rescore reports.  A split row is far wider than shared memory, so the
// query is staged one part at a time: per part, stage the query part, prefetch that part of the piece's candidates, and
// fold the part's exact_dot into the candidate's fp64 running maximum (-inf, then parts 0, 1, ..: the order of
// split_rescore_kernel); the maximum is rounded to fp32 once.
// kCross: the cross split score, every (query part, gallery part) pair folded by cross_exact_scores, `staged` query parts
// in shared memory at a time.
template <bool kSplit, bool kCross = false>
__global__ void __launch_bounds__(kRescoreThreads)
    range_rescore_kernel(const float* __restrict__ q, const float* __restrict__ g, int nq, int d, int n_parts, float tau,
                         const long long* __restrict__ row_cand, const long long* __restrict__ row_piece,
                         int* __restrict__ cand_idx, float* __restrict__ cand_score, int* __restrict__ piece_kept,
                         int staged) {
  static_assert(!kCross || kSplit, "the cross score is a split score");
  extern __shared__ __align__(16) uint8_t sm[];
  const int tid = threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const int warp = tid >> 5;
  int row, n;
  long long start;
  range_piece(blockIdx.x, row_cand, row_piece, nq, row, start, n);
  int* ci = cand_idx + start;
  float* cs = cand_score + start;
  if constexpr (kCross) {
    double* best = reinterpret_cast<double*>(sm);   // [kRangePiece] the piece's exact scores
    double* qs = best + kRangePiece;                // the staged query parts, then the warps' running maxima
    cross_exact_scores<kRescoreThreads>(q + static_cast<size_t>(row) * d, g, d, n_parts, staged, ci, n, best, qs,
                                        qs + static_cast<size_t>(staged) * (d / n_parts));
    for (int c = tid; c < n; c += kRescoreThreads) cs[c] = static_cast<float>(best[c]);
  } else if constexpr (kSplit) {
    double* best = reinterpret_cast<double*>(sm);   // [kRangePiece] running maxima of the piece's candidates
    double* qs = best + kRangePiece;                // [d / n_parts] the query part, widened
    const int pl = d / n_parts;
    for (int c = tid; c < n; c += kRescoreThreads) best[c] = -INFINITY;
    const float* qsrc = q + static_cast<size_t>(row) * d;
    const float* gp = g;   // part `part` of gallery row 0
    for (int part = 0; part < n_parts; ++part, qsrc += pl, gp += pl) {
      __syncthreads();   // the previous part's readers of qs are done (and the maxima initialised)
      for (int c = tid * 4; c < pl; c += kRescoreThreads * 4) {
        const float4 v = *reinterpret_cast<const float4*>(qsrc + c);
        *reinterpret_cast<double2*>(qs + c) = make_double2(static_cast<double>(v.x), static_cast<double>(v.y));
        *reinterpret_cast<double2*>(qs + c + 2) = make_double2(static_cast<double>(v.z), static_cast<double>(v.w));
      }
      for (int c = warp; c < n; c += kRescoreThreads / 32) {   // a warp per candidate, a lane per 128-byte line
        const float* gr = gp + static_cast<size_t>(ci[c]) * d;
        for (int l = static_cast<int>(lane) * 32; l < pl; l += 32 * 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(gr + l));
      }
      __syncthreads();
      for (int c = 2 * warp; c < n; c += 2 * (kRescoreThreads / 32)) {
        const float* g0 = gp + static_cast<size_t>(ci[c]) * d;
        double v0, v1 = 0.0;
        if (c + 1 < n) exact_dot<2>(qs, g0, gp + static_cast<size_t>(ci[c + 1]) * d, pl, lane, v0, v1);
        else exact_dot<1>(qs, g0, nullptr, pl, lane, v0, v1);
        if (lane == 0) {
          best[c] = fmax(best[c], v0);
          if (c + 1 < n) best[c + 1] = fmax(best[c + 1], v1);
        }
      }
    }
    __syncthreads();
    for (int c = tid; c < n; c += kRescoreThreads) cs[c] = static_cast<float>(best[c]);
  } else {
    double* qs = reinterpret_cast<double*>(sm);   // [d] the query row, widened once
    for (int c = tid; c < d; c += kRescoreThreads) qs[c] = static_cast<double>(q[static_cast<size_t>(row) * d + c]);
    __syncthreads();
    for (int c = 2 * warp; c < n; c += 2 * (kRescoreThreads / 32)) {
      double v0, v1 = 0.0;
      if (c + 1 < n) exact_dot<2>(qs, g + static_cast<size_t>(ci[c]) * d, g + static_cast<size_t>(ci[c + 1]) * d, d, lane, v0, v1);
      else exact_dot<1>(qs, g + static_cast<size_t>(ci[c]) * d, nullptr, d, lane, v0, v1);
      if (lane == 0) {
        cs[c] = static_cast<float>(v0);
        if (c + 1 < n) cs[c + 1] = static_cast<float>(v1);
      }
    }
  }
  __syncthreads();
  // round by round: every read of a round happens before the barrier inside group_scan, every write after it, and a
  // round writes only below the positions later rounds read
  int kept = 0;
  for (int c0 = 0; c0 < n; c0 += kRescoreThreads) {
    const int c = c0 + tid;
    int idx = 0;
    float s = 0.f;
    bool keep = false;
    if (c < n) {
      idx = ci[c];
      s = cs[c];
      keep = s >= tau;   // NaN never
    }
    int total;
    const int pos = kept + group_scan<kRescoreThreads>(keep ? 1 : 0, total);
    if (keep) {
      ci[pos] = idx;
      cs[pos] = s;
    }
    kept += total;
  }
  if (tid == 0) piece_kept[blockIdx.x] = kept;
}

// piece w's kept pairs -> the output at piece_excl[w] (global gallery indices)
__global__ void __launch_bounds__(256)
    range_output_kernel(const long long* __restrict__ row_cand, const long long* __restrict__ row_piece, int nq,
                        const long long* __restrict__ piece_excl, const int* __restrict__ cand_idx,
                        const float* __restrict__ cand_score, long long g_index_base, long long g_index_stride,
                        long long* __restrict__ out_idx, float* __restrict__ out_scores) {
  int row, n;
  long long start;
  range_piece(blockIdx.x, row_cand, row_piece, nq, row, start, n);
  const long long o = piece_excl[blockIdx.x];
  const int kept = static_cast<int>(piece_excl[blockIdx.x + 1] - o);
  for (int j = threadIdx.x; j < kept; j += blockDim.x) {
    out_idx[o + j] = g_index_base + g_index_stride * cand_idx[start + j];
    out_scores[o + j] = cand_score[start + j];
  }
}

// row i starts at the output position of its first piece (rows without candidates: of the next row's first piece)
__global__ void range_row_offsets_kernel(const long long* __restrict__ row_piece, const long long* __restrict__ piece_excl,
                                         int nq, long long* __restrict__ row_offsets) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= nq; i += gridDim.x * blockDim.x)
    row_offsets[i] = piece_excl[row_piece[i]];
}

constexpr long long kMaxRangePairs = 1ll << 40;   // capacity accepted by the planner (keeps the byte counts in range)

struct RangePlan {
  SweepGeometry geo;
  int n_parts;   // split score: descriptor parts; 0 = dot product
  bool cross;    // the cross split score (n_parts >= 2)
  int nq_pad, n_qtiles, n_units, n_slots, stages;
  size_t smem_bytes;
  long long max_pieces;   // pieces of kRangePiece candidates when max_pairs candidates fill the rows worst
  size_t total;           // workspace bytes
};

// The threshold search's workspace: the operands, the per-row thresholds, the slot counts / offsets, the row and piece
// scans, and the candidates with their scores
struct RangeBuffers {
  Operands ops;
  float* thr;
  int* seg;
  long long *row_cnt, *row_cand, *row_pcnt, *row_piece;
  int* cand_idx;
  float* cand_score;
  int* piece_kept;
  long long* piece_excl;
};

RangeBuffers carve_range(const RangePlan& rp, int nq, int d, long long max_pairs, Carve& w) {
  RangeBuffers b;
  if (rp.n_parts) {
    b.ops = carve_split_operands(w, rp.nq_pad, rp.geo, rp.n_parts);   // no centring: no flag
  } else {
    b.ops = carve_operands(w, rp.nq_pad, rp.geo, d);
    b.ops.qflag = w.take<int>(4);
  }
  b.thr = w.take<float>(nq);
  b.seg = w.take<int>(static_cast<size_t>(rp.n_slots) * kBlockM);
  b.row_cnt = w.take<long long>(nq);
  b.row_cand = w.take<long long>(static_cast<size_t>(nq) + 1);
  b.row_pcnt = w.take<long long>(nq);
  b.row_piece = w.take<long long>(static_cast<size_t>(nq) + 1);
  b.cand_idx = w.take<int>(max_pairs);
  b.cand_score = w.take<float>(max_pairs);
  b.piece_kept = w.take<int>(rp.max_pieces);
  b.piece_excl = w.take<long long>(static_cast<size_t>(rp.max_pieces) + 1);
  return b;
}

// n_parts = 0: the dot product (sim_range); >= 2: the split score over n_parts parts (sim_range_split; cross:
// sim_range_cross)
const char* range_name(int n_parts, bool cross) {
  return n_parts ? (cross ? "sim_range_cross" : "sim_range_split") : "sim_range";
}

int make_range_plan(int nq, int ng, int d, int n_parts, bool cross, long long max_pairs, int num_sms, size_t max_smem,
                    RangePlan* rp) {
  const char* who = range_name(n_parts, cross);
  DCR_REQUIRE(nq >= 1 && ng >= 1 && d >= 1, "%s: empty problem (nq=%d ng=%d d=%d)", who, nq, ng, d);
  if (n_parts) {
    DCR_REQUIRE(n_parts >= 1 && d % n_parts == 0 && (d / n_parts) % 4 == 0,
                "%s: d=%d must split into %d parts whose length is a multiple of 4", who, d, n_parts);
    const int p = d / n_parts;
    DCR_REQUIRE(p <= kMaxDim, "%s: part length %d > %d not supported", who, p, kMaxDim);
    DCR_REQUIRE(static_cast<long long>(n_parts) * ((p + kBlockK - 1) / kBlockK * kBlockK) <= (1ll << 30),
                "%s: %d parts of %d padded to 64 exceed 2^30 columns", who, n_parts, p);
  } else {
    DCR_REQUIRE(d <= kMaxDim, "sim_range: descriptor dim %d > %d not supported", d, kMaxDim);
    DCR_REQUIRE(d % 4 == 0, "sim_range: descriptor dim %d is not a multiple of 4", d);
  }
  DCR_REQUIRE(max_pairs >= 0 && max_pairs <= kMaxRangePairs, "%s: max_pairs=%lld outside [0, 2^40]", who, max_pairs);
  rp->n_parts = n_parts;
  rp->cross = n_parts && cross;
  if (n_parts) {
    plan_split_geometry(ng, n_parts, d / n_parts, &rp->geo);
    // the threshold sweep keeps no candidate lists in shared memory, so a query tile of up to 512 part-padded columns
    // stays resident as in the dot product (the split top-k always streams it)
    rp->geo.stream_a = rp->geo.num_kb > kMaxKB ? 1 : 0;
  } else {
    plan_geometry(ng, d, &rp->geo);
  }
  const SweepGeometry& g = rp->geo;
  rp->n_qtiles = (nq + kBlockM - 1) / kBlockM;
  rp->nq_pad = rp->n_qtiles * kBlockM;
  // shared memory: the pipeline, then the accumulator transposes of 4 warps per consumer warpgroup (split: two
  // warpgroups, then their per-tile hit counts)
  const size_t tail = n_parts ? 8 * kAccXposeWarpBytes + 2 * 2 * kBlockM * sizeof(int) : 4 * kAccXposeWarpBytes;
  auto smem = [&](int st) { return FusedPipe::smem_bytes(g.num_kb, g.stream_a, st, 0, tail); };
  int stages = 2;
  DCR_REQUIRE(max_smem >= smem(stages), "%s: not enough shared memory (%zu B) for d=%d", who, max_smem, d);
  while (stages < 8 && max_smem >= smem(stages + 1)) ++stages;
  rp->stages = stages;
  rp->smem_bytes = smem(stages);
  // every unit owns at least one tile of every chunk (the last chunk is the smallest): every slot the scan walks is written
  const int last = g.n_gtiles - (g.n_chunks - 1) * g.gchunk;
  rp->n_units = static_cast<int>(std::min<long long>(num_sms, static_cast<long long>(rp->n_qtiles) * last));
  rp->n_slots = g.n_chunks * (rp->n_units + rp->n_qtiles);
  rp->max_pieces = max_pairs / kRangePiece + nq;
  Carve size;
  carve_range(*rp, nq, d, max_pairs, size);
  rp->total = size.bytes;
  return 0;
}

size_t range_workspace_size(int nq, int ng, int d, int n_parts, bool cross, long long max_pairs) {
  const DeviceInfo* di = device_info();
  RangePlan rp;
  if (make_range_plan(nq, ng, d, n_parts, cross, max_pairs, di ? di->num_sms : 132, di ? di->max_smem_optin : 232448, &rp) != 0)
    return 0;
  return rp.total;
}

// The whole search.  n_parts = 0: the dot product (sim_range); >= 2: the split score (sim_range_split; cross:
// sim_range_cross).
int range_search(const float* q, int nq, const float* g, int ng, int d, int n_parts, bool cross, float threshold,
                 long long g_index_base, long long g_index_stride, long long* row_offsets, long long* out_idx,
                 float* out_scores, long long max_pairs, long long* counts, void* ws, size_t ws_bytes,
                 cudaStream_t stream) {
  const char* who = range_name(n_parts, cross);
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  if (int rc = require_sm90a(di, who)) return rc;
  DCR_REQUIRE(!std::isnan(threshold), "%s: threshold is NaN", who);
  DCR_REQUIRE(g_index_stride >= 1, "%s: g_index_stride=%lld < 1", who, g_index_stride);
  RangePlan rp;
  if (int rc = make_range_plan(nq, ng, d, n_parts, cross, max_pairs, di->num_sms, di->max_smem_optin, &rp)) return rc;
  DCR_REQUIRE(ws != nullptr && ws_bytes >= rp.total, "%s: workspace too small (%zu < %zu)", who, ws_bytes, rp.total);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "%s: workspace must be 256-byte aligned", who);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0,
              "%s: q/g must be 16-byte aligned", who);
  const SweepGeometry& geo = rp.geo;
  Carve w{static_cast<uint8_t*>(ws)};
  const RangeBuffers b = carve_range(rp, nq, d, max_pairs, w);
  const Operands& o = b.ops;
  const int pl = n_parts ? d / n_parts : d;   // the length of one exact dot product (a part, or the whole row)
  if (n_parts) {
    if (int rc = prepare_split_operands(q, nq, rp.nq_pad, g, ng, n_parts, pl, geo, di, o, stream)) return rc;
  } else {
    if (int rc = prepare_operands(q, nq, rp.nq_pad, g, ng, d, geo, di, o, stream)) return rc;
  }
  auto threshold_kernel = rp.cross ? range_threshold_kernel<true, true>
                                   : (n_parts ? range_threshold_kernel<true> : range_threshold_kernel<false>);
  if (int rc = launch(threshold_kernel, (nq + 3) / 4, 128, 0, stream,
                      who, q, nq, d, geo.d_pad, n_parts, threshold, o.qnh, o.qnr, o.qnx, o.gmax, o.mu, o.nu, o.qflag, b.thr))
    return rc;

  CUtensorMap tq, tg;
  RangeParams p;
  if (int rc = sweep_setup(geo, nq, rp.n_qtiles, ng, geo.gchunk, geo.n_chunks, o.qb, o.gb, &p, &tq, &tg)) return rc;
  p.stages = rp.stages;
  p.bias_flag = o.qflag;
  p.col_bias = o.bias;
  p.thr = b.thr;
  p.seg = b.seg;
  p.row_cand = b.row_cand;
  p.cand_idx = b.cand_idx;
  p.kb_part = n_parts ? geo.num_kb / n_parts : 0;
  auto sweep = [&](auto off, auto on, auto split, auto cross_split) {
    if (rp.cross) return launch(cross_split, rp.n_units, 32 + 128 * 2, rp.smem_bytes, stream, who, tq, tg, p);
    if (n_parts) return launch(split, rp.n_units, 32 + 128 * 2, rp.smem_bytes, stream, who, tq, tg, p);
    return launch_sweep(off, on, rp.n_units, 32 + 128, rp.smem_bytes, stream, who, tq, tg, p);
  };
  if (int rc = sweep(sim_range_kernel<false, false>, sim_range_kernel<true, false>, sim_range_kernel<false, false, true>,
                     sim_range_kernel<false, false, true, true>))
    return rc;
  if (int rc = launch(range_slot_scan_kernel, (nq + 255) / 256, 256, 0, stream, who, b.seg, nq, rp.n_qtiles,
                      geo.n_gtiles, geo.gchunk, geo.n_chunks, rp.n_units, b.row_cnt, b.row_pcnt))
    return rc;
  if (int rc = exclusive_scan_i64(b.row_cnt, nq, b.row_cand, stream)) return rc;
  if (int rc = exclusive_scan_i64(b.row_pcnt, nq, b.row_piece, stream)) return rc;
  long long h_tot[2] = {0, 0};   // candidates, pieces
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_tot, b.row_cand + nq, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_tot + 1, b.row_piece + nq, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  const long long n_cand = h_tot[0], n_pieces = h_tot[1];
  counts[0] = 0;
  counts[1] = n_cand;
  if (n_cand > max_pairs)
    return set_error(DCR_ERR_CAPACITY, "%s: %lld candidate pairs exceed max_pairs=%lld (call again with that capacity)",
                     who, n_cand, max_pairs);

  if (n_pieces > 0) {
    if (int rc = sweep(sim_range_kernel<false, true>, sim_range_kernel<true, true>, sim_range_kernel<false, true, true>,
                       sim_range_kernel<false, true, true, true>))
      return rc;
    // split: the piece's running maxima, then one query part; cross: then the staged query parts and the warps' running
    // maxima; dot product: the whole query row
    const int staged = rp.cross ? cross_staged_parts(n_parts, pl) : 0;
    const size_t rescore_smem =
        (rp.cross ? static_cast<size_t>(kRangePiece) + cross_stage_doubles(staged, pl, kRescoreThreads / 32)
                  : (n_parts ? static_cast<size_t>(kRangePiece) + pl : static_cast<size_t>(d))) * 8;
    auto rescore_kernel = rp.cross ? range_rescore_kernel<true, true>
                                   : (n_parts ? range_rescore_kernel<true> : range_rescore_kernel<false>);
    if (int rc = launch(rescore_kernel, static_cast<unsigned>(n_pieces), kRescoreThreads, rescore_smem, stream, who, q, g,
                        nq, d, n_parts, threshold, b.row_cand, b.row_piece, b.cand_idx, b.cand_score, b.piece_kept, staged))
      return rc;
  }
  if (int rc = launch(exclusive_scan_kernel<int>, 1, 1024, 0, stream, who, b.piece_kept, n_pieces, b.piece_excl))
    return rc;
  if (n_pieces > 0) {
    if (int rc = launch(range_output_kernel, static_cast<unsigned>(n_pieces), 256, 0, stream, who, b.row_cand,
                        b.row_piece, nq, b.piece_excl, b.cand_idx, b.cand_score, g_index_base, g_index_stride, out_idx,
                        out_scores))
      return rc;
  }
  if (int rc = launch(range_row_offsets_kernel, grid_for(nq + 1, 256, di->num_sms), 256, 0, stream, who, b.row_piece,
                      b.piece_excl, nq, row_offsets))
    return rc;
  long long h_pairs = 0;
  DCR_CUDA_CHECK(cudaMemcpyAsync(&h_pairs, b.piece_excl + n_pieces, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  counts[0] = h_pairs;
  return 0;
}

}  // namespace

size_t sim_range_workspace_size(int nq, int ng, int d, long long max_pairs) {
  return range_workspace_size(nq, ng, d, 0, false, max_pairs);
}

int sim_range(const float* q, int nq, const float* g, int ng, int d, float threshold, long long g_index_base,
              long long g_index_stride, long long* row_offsets, long long* out_idx, float* out_scores, long long max_pairs,
              long long* counts, void* ws, size_t ws_bytes, cudaStream_t stream) {
  return range_search(q, nq, g, ng, d, 0, false, threshold, g_index_base, g_index_stride, row_offsets, out_idx, out_scores,
                      max_pairs, counts, ws, ws_bytes, stream);
}

// one part is the dot product itself: the dot-product search, whose bits the split score must reproduce
size_t sim_range_split_workspace_size(int nq, int ng, int d, int n_parts, long long max_pairs, bool cross) {
  if (n_parts < 1) {
    set_error(-1, "%s: n_parts=%d < 1", range_name(1, cross), n_parts);
    return 0;
  }
  return range_workspace_size(nq, ng, d, n_parts == 1 ? 0 : n_parts, cross, max_pairs);
}

int sim_range_split(const float* q, int nq, const float* g, int ng, int d, int n_parts, float threshold,
                    long long g_index_base, long long g_index_stride, long long* row_offsets, long long* out_idx,
                    float* out_scores, long long max_pairs, long long* counts, void* ws, size_t ws_bytes,
                    cudaStream_t stream, bool cross) {
  DCR_REQUIRE(n_parts >= 1, "%s: n_parts=%d < 1", range_name(1, cross), n_parts);
  return range_search(q, nq, g, ng, d, n_parts == 1 ? 0 : n_parts, cross, threshold, g_index_base, g_index_stride, row_offsets,
                      out_idx, out_scores, max_pairs, counts, ws, ws_bytes, stream);
}

int exclusive_scan_i64(const long long* in, long long n, long long* out, cudaStream_t stream) {
  return launch(exclusive_scan_kernel<long long>, 1, 1024, 0, stream, "exclusive_scan_i64", in, n, out);
}

}  // namespace dcr
