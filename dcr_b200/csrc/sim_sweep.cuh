// The fused similarity sweep shared by the top-k search (sim_topk.cu) and the threshold search (sim_range.cu): tile
// constants, the work decomposition, the TMA / wgmma pipeline of the sweep kernels, the error bound of its approximate
// scores, the group collectives and the one fp64 dot product every exact score comes from.  Device code here is inline
// only (no kernel), so each search compiles its own kernels against one definition.  Stage 1 -- the bf16 operands and
// their norms -- and the sweep's host side are defined in sim_sweep.cu.
#pragma once
#include <cuda_bf16.h>

#include <algorithm>

#include "host_util.cuh"
#include "ptx.cuh"

namespace dcr {

constexpr int kBlockM = 128;      // query rows per CTA
constexpr int kBlockN = 128;      // gallery rows per tile (accumulator columns: 128 registers per thread with one warpgroup)
constexpr int kBlockK = 64;       // bf16 elements per 128-byte swizzled smem row
constexpr int kMaxKB = 8;         // d_pad <= 512: the query tile stays resident in shared memory; larger: streamed
constexpr int kMaxDim = 8192;     // largest descriptor dimension accepted
constexpr uint32_t kFull = 0xffffffffu;
constexpr int kATileBytes = kBlockM * kBlockK * 2;  // 16 KB
constexpr int kBTileBytes = kBlockN * kBlockK * 2;  // 16 KB
constexpr int kRescoreThreads = 128;   // block size of the exact re-score kernels

// The leading parameters of both sweep kernels (SimParams, RangeParams), in this order
struct SweepHead {
  int nq, ng;
  int num_kb;          // d_pad / 64
  int stream_a;        // 1 (d_pad > 512): query k-blocks travel with the gallery k-blocks instead of staying resident
  int n_qtiles;        // ceil(nq / 128)
  int n_gtiles;        // ceil(ng / 128)
  int gchunk;          // gallery tiles per L2-sized chunk (all units sweep chunk c before chunk c+1)
  int n_chunks;
};

// Work decomposition shared by the three warp roles and rescore_select_kernel: for every gallery chunk c (chunks are
// L2-sized so that the units, which all sweep chunk c at about the same time, share its tiles in L2) the
// (q-tile, g-tile-in-chunk) grid is linearised q-major into T tiles and cut into n_units equal contiguous ranges, unit u
// owning [u*T/U, (u+1)*T/U); a unit's range is walked as segments = maximal runs inside one q-tile.

// owner unit of linear tile t
DCR_DEVICE long long owner_unit(long long t, long long T, long long U) { return ((t + 1) * U + T - 1) / T - 1; }

// Candidate slot of the segment (chunk, unit, q-tile qi) and epilogue set: the q-tiles of a unit's range never lie below
// those of the previous unit, so unit + qi is distinct within a chunk and below n_units + n_qtiles.
DCR_DEVICE int slot_index(int chunk, int unit, int qi, int set, int n_units, int n_qtiles, int n_sets) {
  return (chunk * (n_units + n_qtiles) + unit + qi) * n_sets + set;
}

// Thresholds carry over from chunk to chunk: `carried` says that this unit finished a segment of the same q-tile before
// (its final per-row thresholds are valid lower bounds, so no warm-up replay is needed).
struct SegWalker {
  int n_qtiles, n_gtiles, gchunk, n_chunks;
  long long unit, n_units;
  // current segment
  int chunk, qi, g_begin, ntiles;
  bool carried;
  // state
  long long t, t_end;
  int ncg, g_lo;
  int tag[4];
  __device__ SegWalker(int nq_t, int ng_t, int gc, int nc, long long u, long long nu)
      : n_qtiles(nq_t), n_gtiles(ng_t), gchunk(gc), n_chunks(nc), unit(u), n_units(nu), chunk(-1), t(0), t_end(0) {
    tag[0] = tag[1] = tag[2] = tag[3] = -1;
  }
  __device__ bool next() {
    if (chunk >= 0) {   // close the previous segment
      const int s4 = qi & 3;
      if (s4 == 0) tag[0] = qi; else if (s4 == 1) tag[1] = qi; else if (s4 == 2) tag[2] = qi; else tag[3] = qi;
    }
    while (t >= t_end) {
      ++chunk;
      if (chunk >= n_chunks) return false;
      g_lo = chunk * gchunk;
      ncg = min(gchunk, n_gtiles - g_lo);
      const long long T = static_cast<long long>(n_qtiles) * ncg;
      t = unit * T / n_units;
      t_end = (unit + 1) * T / n_units;
    }
    qi = static_cast<int>(t / ncg);
    g_begin = g_lo + static_cast<int>(t % ncg);
    const long long seg_end = min(t_end, static_cast<long long>(qi + 1) * ncg);
    ntiles = static_cast<int>(seg_end - t);
    const int s4 = qi & 3;
    const int tg = s4 == 0 ? tag[0] : (s4 == 1 ? tag[1] : (s4 == 2 ? tag[2] : tag[3]));
    carried = (tg == qi);
    t = seg_end;
    return true;
  }
};

// Shared-memory pipeline of a fused sweep (sim_topk_kernel, sim_range_kernel), from the 1024-byte aligned base:
//   resident mode: [num_kb x 16 KB query tile][stages x gallery tile]; streamed mode (d_pad > 512, the query tile no
//   longer fits): [stages x (gallery tile | 16 KB query k-block)] -- twice the L2->SMEM traffic per FLOP
// followed by `list_bytes` of the caller's own, the barriers, and whatever the caller puts after them (`tail`).
struct FusedPipe {
  // The layout, written once: the kernels place it at the aligned shared-memory base (B = uint8_t*), the planners at
  // offset 0 (B = size_t), where `tail` is the size of the pipeline
  template <class B>
  struct Layout {
    int stage_bytes;
    B smem_b, lists, bars, tail;
    __host__ __device__ Layout(B base, int num_kb, bool stream_a, int stages, size_t list_bytes) {
      stage_bytes = kBTileBytes + (stream_a ? kATileBytes : 0);
      smem_b = base + (stream_a ? 0 : num_kb * kATileBytes);
      lists = smem_b + stages * stage_bytes;
      bars = lists + list_bytes;
      tail = bars + 32 * sizeof(uint64_t);
    }
  };
  // dynamic shared memory of a launch: the alignment slack, the pipeline, and tail_bytes after it
  static size_t smem_bytes(int num_kb, int stream_a, int stages, size_t list_bytes, size_t tail_bytes) {
    return 1024 + Layout<size_t>(0, num_kb, stream_a != 0, stages, list_bytes).tail + tail_bytes;
  }

  bool stream_a;
  int num_kb, stage_bytes;
  uint8_t* smem_a;     // num_kb x 16 KB (resident mode)
  uint8_t* smem_b;     // stages x stage_bytes
  uint8_t* lists;
  uint64_t *b_full, *b_empty, *a_full, *a_empty;
  uint8_t* tail;
  DCR_DEVICE FusedPipe(uint8_t* smem_raw, int nkb, int stream, int stages, size_t list_bytes) {
    // all tile bases 1024-byte aligned for the 128B swizzle
    smem_a = smem_align1024(smem_raw);
    stream_a = stream != 0;
    num_kb = nkb;
    const Layout<uint8_t*> L(smem_a, num_kb, stream_a, stages, list_bytes);
    stage_bytes = L.stage_bytes;
    smem_b = L.smem_b;
    lists = L.lists;
    uint64_t* bars = reinterpret_cast<uint64_t*>(L.bars);
    b_full = bars;          // [stages]
    b_empty = bars + 8;     // [stages]
    a_full = bars + 16;
    a_empty = bars + 17;
    tail = L.tail;
  }
  // producer warp = consumer_warps (the last warp); every thread of the CTA calls this
  DCR_DEVICE void init(const CUtensorMap* tq, const CUtensorMap* tg, int stages, uint32_t consumer_warps) const {
    const uint32_t warp = threadIdx.x >> 5;
    if (warp == consumer_warps && elect_one()) {
      tma_prefetch_desc(tq);
      tma_prefetch_desc(tg);
    }
    if (warp == 0 && elect_one()) {
      for (int s = 0; s < stages; ++s) {
        mbar_init(&b_full[s], 1);
        mbar_init(&b_empty[s], consumer_warps);   // one arrive per consumer warp
      }
      mbar_init(a_full, 1);
      mbar_init(a_empty, consumer_warps);
      fence_mbar_init();
    }
    __syncthreads();
  }
};

// TMA producer of a fused sweep.  The whole warp walks the loop (warp-uniform values stay in uniform registers) and one
// elected lane issues.  Per segment: the query tile (resident mode), then warm + ntiles gallery tiles of num_kb k-blocks,
// the first `warm` of them replayed from the segment start; warm_of(walker) says how many.
// kCross: the cross split score (DESIGN.md section 3).  A tile is n_parts^2 part pairs of kb_part k-blocks each, gallery
// part b outer and query part a inner: step (b, a, kin) loads gallery k-block b kb_part + kin and, streamed, query k-block
// a kb_part + kin.  Three nested int loops: the n_parts^2 kb_part steps of a tile are never one count.
template <bool kCross = false, class WarmOf>
DCR_DEVICE void fused_producer(const FusedPipe& pp, const CUtensorMap* tq, const CUtensorMap* tg, int stages, SegWalker& w,
                               WarmOf warm_of, int kb_part = 0) {
  uint32_t seg = 0;
  PipeState st(stages);
  while (w.next()) {
    const int qi = w.qi, g_begin = w.g_begin, ntiles = w.ntiles;
    const int warm = warm_of(w);
    const int q_row = qi * kBlockM;
    if (!pp.stream_a) {   // resident query tile
      mbar_wait(pp.a_empty, (seg & 1) ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(pp.a_full, pp.num_kb * kATileBytes);
        for (int kb = 0; kb < pp.num_kb; ++kb)
          tma_load_2d(pp.smem_a + kb * kATileBytes, tq, pp.a_full, kb * kBlockK, q_row, kEvictNormal);
      }
      __syncwarp();
    }
    for (int j = 0; j < warm + ntiles; ++j) {
      const int gi = g_begin + (j < warm ? j : j - warm);
      const int g_row = gi * kBlockN;
      // one stage: gallery k-block gkb, and with a streamed query tile query k-block qkb
      auto issue = [&](int gkb, int qkb) {
        const uint32_t s = st.s, ph = st.ph;
        mbar_wait(&pp.b_empty[s], ph ^ 1);
        if (elect_one()) {
          mbar_arrive_expect_tx(&pp.b_full[s], pp.stage_bytes);
          tma_load_2d(pp.smem_b + s * pp.stage_bytes, tg, &pp.b_full[s], gkb * kBlockK, g_row, kEvictNormal);
          if (pp.stream_a)
            tma_load_2d(pp.smem_b + s * pp.stage_bytes + kBTileBytes, tq, &pp.b_full[s], qkb * kBlockK, q_row, kEvictNormal);
        }
        __syncwarp();
      };
      if constexpr (kCross) {
        for (int gkb0 = 0; gkb0 < pp.num_kb; gkb0 += kb_part)
          for (int qkb0 = 0; qkb0 < pp.num_kb; qkb0 += kb_part)
            for (int kin = 0; kin < kb_part; ++kin, st.next()) issue(gkb0 + kin, qkb0 + kin);
      } else {
        for (int kb = 0; kb < pp.num_kb; ++kb, st.next()) issue(kb, kb);
      }
    }
    ++seg;
  }
}

// One 128-row accumulator tile of a consumer warpgroup: the wgmma k-loop over the pipeline stages.  The stage of k-block
// kb is released once wgmma_wait<1> in k-block kb+1 has seen its MMAs complete; `last` also releases the resident query
// tile (last tile of the segment).  a_base / b_base: shared addresses of the query tile and of this warpgroup's columns
// of gallery stage 0.
template <int kCols>
DCR_DEVICE void fused_tile_mma(WgAcc<kCols>& acc, PipeState& st, const FusedPipe& pp, uint32_t a_base, uint32_t b_base,
                               bool last, uint32_t lane) {
  const uint32_t a_step = pp.stream_a ? 0u : static_cast<uint32_t>(kATileBytes);   // per k-block (resident query tile)
  uint32_t prev_s = 0;
  for (int kb = 0; kb < pp.num_kb; ++kb, st.next()) {
    const uint32_t s = st.s;
    mbar_wait(&pp.b_full[s], st.ph);
    const uint32_t a_addr = a_base + (pp.stream_a ? s * static_cast<uint32_t>(pp.stage_bytes) : static_cast<uint32_t>(kb) * a_step);
    const uint32_t b_addr = b_base + s * static_cast<uint32_t>(pp.stage_bytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k) acc.mma(a_addr + 32 * k, wgmma_desc_sw128(b_addr + 32 * k), (kb | k) != 0);
    wgmma_commit();
    wgmma_wait<1>();
    if (kb > 0 && lane == 0) mbar_arrive(&pp.b_empty[prev_s]);
    prev_s = s;
  }
  wgmma_wait<0>();
  acc.fence_regs();
  if (lane == 0) {
    mbar_arrive(&pp.b_empty[prev_s]);
    if (!pp.stream_a && last) mbar_arrive(pp.a_empty);
  }
}

// The same k-loop under the split score (descriptors cut into parts of kb_part k-blocks each, DESIGN.md section 3): each
// part's first k-block overwrites the part accumulator, and after its last one the accumulator is folded into `best`,
// the running element-wise maximum over the parts (fmaxf: a NaN part is ignored, as in the exact split score).  A part
// boundary waits for every MMA in flight, because the fold reads the accumulator, and then releases both stages it held.
// kCross: the cross split score, the same fold over the n_parts^2 part pairs in fused_producer<true>'s order (gallery part
// outer, query part inner); a resident query tile supplies query part a's k-blocks.
template <int kCols, bool kCross = false>
DCR_DEVICE void fused_tile_mma_split(WgAcc<kCols>& best, PipeState& st, const FusedPipe& pp, uint32_t a_base,
                                     uint32_t b_base, int kb_part, bool last, uint32_t lane) {
  const uint32_t a_step = pp.stream_a ? 0u : static_cast<uint32_t>(kATileBytes);
  WgAcc<kCols> part;
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int i = 0; i < kCols / 2; ++i) best.d[s][i] = -INFINITY;
  uint32_t prev_s = 0;
  bool held = false;   // stage prev_s is still read by an MMA that may be in flight
  int kin = 0;         // k-block within the current part
  // one k-block of the current part (pair), whose query k-block is kb
  auto step = [&](int kb) {
    const uint32_t s = st.s;
    mbar_wait(&pp.b_full[s], st.ph);
    const uint32_t a_addr = a_base + (pp.stream_a ? s * static_cast<uint32_t>(pp.stage_bytes) : static_cast<uint32_t>(kb) * a_step);
    const uint32_t b_addr = b_base + s * static_cast<uint32_t>(pp.stage_bytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k) part.mma(a_addr + 32 * k, wgmma_desc_sw128(b_addr + 32 * k), (kin | k) != 0);
    wgmma_commit();
    if (++kin == kb_part) {
      wgmma_wait<0>();
      part.fence_regs();
      if (lane == 0) {
        if (held) mbar_arrive(&pp.b_empty[prev_s]);
        mbar_arrive(&pp.b_empty[s]);
      }
      held = false;
      kin = 0;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < kCols / 2; ++i) best.d[h][i] = fmaxf(best.d[h][i], part.d[h][i]);
    } else {
      wgmma_wait<1>();
      if (held && lane == 0) mbar_arrive(&pp.b_empty[prev_s]);
      held = true;
      prev_s = s;
    }
  };
  if constexpr (kCross) {
    for (int gkb0 = 0; gkb0 < pp.num_kb; gkb0 += kb_part)
      for (int qkb0 = 0; qkb0 < pp.num_kb; qkb0 += kb_part)
        for (int i = 0; i < kb_part; ++i, st.next()) step(qkb0 + i);
  } else {
    for (int kb = 0; kb < pp.num_kb; ++kb, st.next()) step(kb);
  }
  if (lane == 0 && !pp.stream_a && last) mbar_arrive(pp.a_empty);   // num_kb is a whole number of parts: nothing held
}

// ------------------------------------------------------------------------------------------------------------
// The exact dot product: fp64 accumulate with one fixed association.  Lane l owns the elements l*4 + 128*i (float4
// granules), accumulates them in ascending order with fma, then a fixed xor butterfly from 16 down to 1.  Every exact
// score -- the top-k re-score and its brute-force path, split_rescore, the threshold search -- comes from here, so all of
// them report bit-identical values for the same pair.
//   TQ     the query row: fp32, or already widened to fp64 in shared memory (the widening is exact; the re-score kernels
//          are bound by the fp64 pipe -- per gallery row 512 fma plus 1024 fp32->fp64 conversions -- and this halves the
//          conversions)
//   kRows  gallery rows scored at once: out0 = q . b0, and with two rows out1 = q . b1 (one row leaves out1 alone)
DCR_DEVICE void query_granule(const float* __restrict__ a, int c, double (&x)[4]) {
#pragma unroll
  for (int e = 0; e < 4; ++e) x[e] = static_cast<double>(a[c + e]);
}
DCR_DEVICE void query_granule(const double* __restrict__ a, int c, double (&x)[4]) {
  const double2 a01 = *reinterpret_cast<const double2*>(a + c);
  const double2 a23 = *reinterpret_cast<const double2*>(a + c + 2);
  x[0] = a01.x;
  x[1] = a01.y;
  x[2] = a23.x;
  x[3] = a23.y;
}

// one granule: acc + x0 v.x + x1 v.y + x2 v.z + x3 v.w, each step an fma, in that order
DCR_DEVICE double fma_granule(const double (&x)[4], float4 v, double acc) {
  acc = fma(x[0], static_cast<double>(v.x), acc);
  acc = fma(x[1], static_cast<double>(v.y), acc);
  acc = fma(x[2], static_cast<double>(v.z), acc);
  return fma(x[3], static_cast<double>(v.w), acc);
}

template <int kRows, typename TQ>
DCR_DEVICE void exact_dot(const TQ* __restrict__ a_smem, const float* __restrict__ b0, const float* __restrict__ b1, int d,
                          uint32_t lane, double& out0, double& out1) {
  static_assert(kRows == 1 || kRows == 2, "one or two gallery rows");
  double acc0 = 0.0, acc1 = 0.0;   // acc1: second row
  bool all_loads_first = false;
  if constexpr (kRows == 2) all_loads_first = (d & 127) == 0 && d <= 512;
  if (all_loads_first) {
    if constexpr (kRows == 2) {
      // every lane owns d/128 whole 16-byte granules of each row: all (up to eight) loads are issued before the first
      // fma -- written as a loop, each 128-column step waited for its own two loads (40 serial memory latencies per query)
      float4 v0[4], v1[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i * 128 < d) {
          v0[i] = *reinterpret_cast<const float4*>(b0 + lane * 4 + i * 128);
          v1[i] = *reinterpret_cast<const float4*>(b1 + lane * 4 + i * 128);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i * 128 < d) {
          double x[4];
          query_granule(a_smem, lane * 4 + i * 128, x);
          acc0 = fma_granule(x, v0[i], acc0);
          acc1 = fma_granule(x, v1[i], acc1);
        }
      }
    }
  } else {
    for (int c = lane * 4; c < d; c += 128) {
      if (c + 3 < d) {
        float4 v[kRows];
        v[0] = *reinterpret_cast<const float4*>(b0 + c);
        if constexpr (kRows == 2) v[1] = *reinterpret_cast<const float4*>(b1 + c);
        double x[4];
        query_granule(a_smem, c, x);
        acc0 = fma_granule(x, v[0], acc0);
        if constexpr (kRows == 2) acc1 = fma_granule(x, v[1], acc1);
      } else {
        for (int e = c; e < d; ++e) {
          acc0 = fma(static_cast<double>(a_smem[e]), static_cast<double>(b0[e]), acc0);
          if constexpr (kRows == 2) acc1 = fma(static_cast<double>(a_smem[e]), static_cast<double>(b1[e]), acc1);
        }
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    acc0 += __shfl_xor_sync(kFull, acc0, off);
    if constexpr (kRows == 2) acc1 += __shfl_xor_sync(kFull, acc1, off);
  }
  out0 = acc0;
  if constexpr (kRows == 2) out1 = acc1;
}

// Collectives of a group.  Every thread of the group calls them; the 128-wide forms go through a 4-entry shared array.
template <int kThreads>
DCR_DEVICE void group_sync() {
  if constexpr (kThreads == 32) __syncwarp();
  else __syncthreads();
}

// float or double; fmax ignores NaN
template <int kThreads, typename T>
DCR_DEVICE T group_max(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(kFull, v, o));
  if constexpr (kThreads > 32) {
    __shared__ T part[4];
    __syncthreads();   // the previous call's readers are done
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    v = fmax(fmax(part[0], part[1]), fmax(part[2], part[3]));
  }
  return v;
}

// exclusive prefix sum over the group in thread order; total = the group's sum
template <int kThreads>
DCR_DEVICE int group_scan(int v, int& total) {
  const int lane = threadIdx.x & 31;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(kFull, incl, o);
    if (lane >= o) incl += t;
  }
  total = __shfl_sync(kFull, incl, 31);
  if constexpr (kThreads == 32) {
    return incl - v;
  } else {
    __shared__ int part[4];
    const int w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) part[w] = total;
    __syncthreads();
    for (int i = 0; i < w; ++i) incl += part[i];
    total = part[0] + part[1] + part[2] + part[3];
    return incl - v;
  }
}

// How far an approximate score of the fused sweeps can lie from the exact one, for query row qrow.  Whole warp; q is the
// query row (fp32 in global memory or already widened to fp64 in shared memory: the same values).
//   eps   bounds |tensor-core score of (bf16 q', bf16 (g-mu)) (+ the column offset nu.(g-mu)) - q.(g-mu)| from the
//         measured norms (DESIGN.md section 4): bf16 rounding of both operands, fp32 accumulation, fp32 roundings of
//         q - nu, g - mu, the offset and its addition
//   qmu   q . mu in fp64: the constant the centred approximate scores are offset by
//   slack covers the fp64 rounding of an exact score and of q.mu themselves (each a d-term dot of vectors no longer than
//         (|q'| + |nu|), (|g'| + |mu|)): irrelevant next to eps except when the centred gallery is (nearly) zero -- all
//         rows identical -- and eps with it
// So the fp64 score of a pair whose approximate score is a satisfies  s <= a + eps + qmu + slack  and
// s >= a - eps + qmu - slack.
struct RowBound {
  float eps;
  double qmu, slack;
};
template <typename TQ>
DCR_DEVICE RowBound row_bound(const TQ* __restrict__ q, int d, int d_pad, int qrow, const float* __restrict__ q_norm_hat,
                              const float* __restrict__ q_norm_res, const float* __restrict__ q_norm_x,
                              const unsigned int* __restrict__ g_max, const float* __restrict__ mu,
                              const float* __restrict__ nu, const int* __restrict__ nu_flag, uint32_t lane) {
  const float g_norm = __uint_as_float(g_max[0]), g_res = __uint_as_float(g_max[1]);
  const float qh = q_norm_hat[qrow], qr = q_norm_res[qrow], qx = q_norm_x[qrow];
  float eps = 1.001f * (qh * g_res + qr * g_norm) + d_pad * 2.4e-7f * qh * (g_norm + g_res) + 1e-30f;
  float nun = 0.f, mun = 0.f;   // |nu|, |mu| (upper bounds)
  {
    float acc = 0.f;
    if (nu && nu_flag && *nu_flag)
      for (int c = lane; c < d; c += 32) acc += nu[c] * nu[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    nun = sqrtf(acc) * 1.001f;
    eps += 3e-7f * (qx + nun) * g_norm;
  }
  double qmu = 0.0;
  {
    float mu2 = 0.f;
    for (int c = lane; c < d; c += 32) {
      qmu = fma(static_cast<double>(q[c]), static_cast<double>(mu[c]), qmu);
      mu2 = fmaf(mu[c], mu[c], mu2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      qmu += __shfl_xor_sync(kFull, qmu, o);
      mu2 += __shfl_xor_sync(kFull, mu2, o);
    }
    mun = sqrtf(mu2) * 1.001f;
  }
  RowBound rb;
  rb.eps = eps;
  rb.qmu = qmu;
  rb.slack = 4.6e-16 * (d + 8) * static_cast<double>(qx + nun) * static_cast<double>(g_norm + mun);
  return rb;
}

// The same bound under the split score, whose operands are not centred (qmu = 0).  Part c of a pair is a p-term dot
// product accumulated over p_pad, bounded as above from the part's own norms (q_norm_*[qrow * n_parts + c], g_max[2c],
// g_max[2c + 1]), and |max_c a_c - max_c s_c| <= max_c |a_c - s_c|: the bound is the largest over the parts.  A NaN
// part norm makes eps NaN, so the certificate fails rather than leave that part unbounded.  Whole warp.
DCR_DEVICE RowBound split_row_bound(int n_parts, int p, int p_pad, int qrow, const float* __restrict__ q_norm_hat,
                                    const float* __restrict__ q_norm_res, const float* __restrict__ q_norm_x,
                                    const unsigned int* __restrict__ g_max, uint32_t lane) {
  float eps = 0.f;
  double slack = 0.0;
  bool nan = false;
  for (int c = static_cast<int>(lane); c < n_parts; c += 32) {
    const float g_norm = __uint_as_float(g_max[2 * c]), g_res = __uint_as_float(g_max[2 * c + 1]);
    const size_t i = static_cast<size_t>(qrow) * n_parts + c;
    const float qh = q_norm_hat[i], qr = q_norm_res[i], qx = q_norm_x[i];
    const float e = 1.001f * (qh * g_res + qr * g_norm) + p_pad * 2.4e-7f * qh * (g_norm + g_res) + 3e-7f * qx * g_norm + 1e-30f;
    nan |= (e != e);
    eps = fmaxf(eps, e);
    slack = fmax(slack, 4.6e-16 * (p + 8) * static_cast<double>(qx) * static_cast<double>(g_norm));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    eps = fmaxf(eps, __shfl_xor_sync(kFull, eps, o));
    slack = fmax(slack, __shfl_xor_sync(kFull, slack, o));
  }
  RowBound rb;
  rb.eps = __any_sync(kFull, nan) ? __int_as_float(0x7fc00000) : eps;
  rb.qmu = 0.0;
  rb.slack = slack;
  return rb;
}

// The same bound under the cross split score: the approximate score of pair (a, b) is the bf16 dot product of query part a
// with gallery part b, bounded by the part formula above from query part a's norms and gallery part b's maxima, and
// |max_ab a_ab - max_ab s_ab| <= max_ab |a_ab - s_ab|.  The exact maximum over the n_parts^2 pairs (lane-strided over a,
// a broadcast walk over b): it is the tightest bound the norms allow, at n_parts^2 / 32 steps per lane, small next to the
// sweep's n_parts^2 k-blocks per tile.  A NaN part norm makes eps NaN.  Whole warp.
DCR_DEVICE RowBound cross_row_bound(int n_parts, int p, int p_pad, int qrow, const float* __restrict__ q_norm_hat,
                                    const float* __restrict__ q_norm_res, const float* __restrict__ q_norm_x,
                                    const unsigned int* __restrict__ g_max, uint32_t lane) {
  float eps = 0.f;
  double slack = 0.0;
  bool nan = false;
  for (int a = static_cast<int>(lane); a < n_parts; a += 32) {
    const size_t i = static_cast<size_t>(qrow) * n_parts + a;
    const float qh = q_norm_hat[i], qr = q_norm_res[i], qx = q_norm_x[i];
    for (int b = 0; b < n_parts; ++b) {
      const float g_norm = __uint_as_float(g_max[2 * b]), g_res = __uint_as_float(g_max[2 * b + 1]);
      const float e = 1.001f * (qh * g_res + qr * g_norm) + p_pad * 2.4e-7f * qh * (g_norm + g_res) + 3e-7f * qx * g_norm + 1e-30f;
      nan |= (e != e);
      eps = fmaxf(eps, e);
      slack = fmax(slack, 4.6e-16 * (p + 8) * static_cast<double>(qx) * static_cast<double>(g_norm));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    eps = fmaxf(eps, __shfl_xor_sync(kFull, eps, o));
    slack = fmax(slack, __shfl_xor_sync(kFull, slack, o));
  }
  RowBound rb;
  rb.eps = __any_sync(kFull, nan) ? __int_as_float(0x7fc00000) : eps;
  rb.qmu = 0.0;
  rb.slack = slack;
  return rb;
}

// Exact cross split scores of the gallery rows rows[0 .. n) against query row q (d = n_parts * pl values): best[c] = the
// fmax fold from -inf of exact_dot(q_a, g_b) over query part a outer, gallery part b inner -- the order of
// split_rescore_kernel's cross branch.  The query is staged `staged` parts at a time in qs (fp64, [staged][pl]); for each
// candidate the warp walks the gallery parts once per staged group, scoring part b against every staged query part while
// it sits in L1, so a row is read from L2 about ceil(n_parts / staged) times instead of n_parts times.  Per group the warp
// keeps each staged part's running maximum over b in part_max ([warp][2][staged]) and folds them into best in part order:
// exact_dot never returns -0 (its sums start at +0 and round to nearest) and fmax ignores NaN, so on its values fmax is
// associative and this grouping is the bits of the single chain.  Every thread of the group calls this.
template <int kThreads>
DCR_DEVICE void cross_exact_scores(const float* __restrict__ q, const float* __restrict__ g, int d, int n_parts, int staged,
                                   const int* __restrict__ rows, int n, double* __restrict__ best, double* __restrict__ qs,
                                   double* __restrict__ part_max) {
  constexpr int kWarps = kThreads / 32;
  const int tid = static_cast<int>(threadIdx.x) % kThreads;
  const uint32_t lane = threadIdx.x & 31;
  const int warp = tid >> 5;
  const int pl = d / n_parts;
  double* pm = part_max + warp * 2 * staged;
  for (int c = tid; c < n; c += kThreads) best[c] = -INFINITY;
  for (int a0 = 0; a0 < n_parts; a0 += staged) {
    const int na = min(staged, n_parts - a0);
    group_sync<kThreads>();   // the previous group's readers of qs are done (and best initialised)
    const float* qsrc = q + static_cast<size_t>(a0) * pl;
    for (int c = tid * 4; c < na * pl; c += kThreads * 4) {   // pl % 4 == 0
      const float4 v = *reinterpret_cast<const float4*>(qsrc + c);
      *reinterpret_cast<double2*>(qs + c) = make_double2(static_cast<double>(v.x), static_cast<double>(v.y));
      *reinterpret_cast<double2*>(qs + c + 2) = make_double2(static_cast<double>(v.z), static_cast<double>(v.w));
    }
    group_sync<kThreads>();
    for (int c = 2 * warp; c < n; c += 2 * kWarps) {
      const bool two = c + 1 < n;
      const float* g0 = g + static_cast<size_t>(rows[c]) * d;
      const float* g1 = two ? g + static_cast<size_t>(rows[c + 1]) * d : g0;
      for (int i = static_cast<int>(lane); i < 2 * staged; i += 32) pm[i] = -INFINITY;
      for (int l = static_cast<int>(lane) * 32; l < pl; l += 32 * 32) {   // part 0 of both rows, a lane per 128-byte line
        asm volatile("prefetch.global.L2 [%0];" ::"l"(g0 + l));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(g1 + l));
      }
      __syncwarp();
      for (int b = 0; b < n_parts; ++b) {
        const size_t off = static_cast<size_t>(b) * pl;
        if (b + 1 < n_parts)
          for (int l = static_cast<int>(lane) * 32; l < pl; l += 32 * 32) {
            asm volatile("prefetch.global.L2 [%0];" ::"l"(g0 + off + pl + l));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(g1 + off + pl + l));
          }
        for (int a = 0; a < na; ++a) {
          double v0, v1 = 0.0;
          if (two) exact_dot<2>(qs + static_cast<size_t>(a) * pl, g0 + off, g1 + off, pl, lane, v0, v1);
          else exact_dot<1>(qs + static_cast<size_t>(a) * pl, g0 + off, nullptr, pl, lane, v0, v1);
          if (lane == 0) {
            pm[a] = fmax(pm[a], v0);
            if (two) pm[staged + a] = fmax(pm[staged + a], v1);
          }
        }
      }
      __syncwarp();
      if (lane == 0) {
        for (int a = 0; a < na; ++a) {
          best[c] = fmax(best[c], pm[a]);
          if (two) best[c + 1] = fmax(best[c + 1], pm[staged + a]);
        }
      }
      __syncwarp();
    }
  }
  group_sync<kThreads>();
}

// Query parts the cross re-score stages at once (cross_exact_scores) within kCrossStageBytes of shared memory, counting
// each part's fp64 values and the running maxima of four warps; at least one part.
constexpr size_t kCrossStageBytes = 44 * 1024;
inline int cross_staged_parts(int n_parts, int pl) {
  const size_t per_part = (static_cast<size_t>(pl) + 8) * sizeof(double);
  return static_cast<int>(std::max<size_t>(1, std::min<size_t>(n_parts, kCrossStageBytes / per_part)));
}
// fp64 values cross_exact_scores needs at qs for `staged` parts of pl values, with kWarps warps' running maxima after them
__host__ __device__ inline size_t cross_stage_doubles(int staged, int pl, int warps) {
  return static_cast<size_t>(staged) * pl + 2 * static_cast<size_t>(warps) * staged;
}

// ------------------------------------------------------------------------------------------------------------
// host side, defined in sim_sweep.cu

// tiles, padding and gallery chunking of a fused sweep
struct SweepGeometry {
  int d_pad, num_kb, ng_pad, n_gtiles, rows_per_qtile;
  int stream_a;           // d_pad > 512: query tile streamed with the gallery k-blocks
  int gchunk, n_chunks;   // preferred gallery chunking (a top-k pass may use fewer chunks)
};
void plan_geometry(int ng, int d, SweepGeometry* geo);

// Stage 1 of both searches: the centres, the decision whether to centre the queries, and the bf16 operands with the
// norms their error bound needs.
struct Operands {
  __nv_bfloat16 *qb, *gb;   // [nq_pad, d_pad], [ng_pad, d_pad]
  float *qnh, *qnr, *qnx;   // per query row, see to_bf16_rows_kernel
  unsigned int* gmax;       // [2]
  double* colsum;           // [2 d] scratch
  float *mu, *nu, *bias;    // gallery centre, query centre, per-gallery-row offset nu.(g - mu)
  int* qflag;               // device flag: query centring on / off (placed by the caller)
};
// the operand buffers of both searches, cut from the caller's workspace
Operands carve_operands(Carve& w, int nq_pad, const SweepGeometry& geo, int d);
int prepare_operands(const float* q, int nq, int nq_pad, const float* g, int ng, int d, const SweepGeometry& geo,
                     const DeviceInfo* di, const Operands& o, cudaStream_t stream);

// Stage 1 under the split score: rows of n_parts parts of p values, each part zero-padded to p_pad = ceil64(p) so that a
// part boundary is a k-block boundary (d_pad = n_parts * p_pad).  No centring.  Norms per part: qnh / qnr / qnx hold
// [nq_pad][n_parts], gmax [n_parts][2] the gallery maxima of each part; mu, nu, bias, colsum and qflag stay unused.
void plan_split_geometry(int ng, int n_parts, int p, SweepGeometry* geo);
Operands carve_split_operands(Carve& w, int nq_pad, const SweepGeometry& geo, int n_parts);
int prepare_split_operands(const float* q, int nq, int nq_pad, const float* g, int ng, int n_parts, int p,
                           const SweepGeometry& geo, const DeviceInfo* di, const Operands& o, cudaStream_t stream);

// The head of a sweep over the first n_qtiles query tiles of qb against gb, and the tensor maps of both operands
int sweep_setup(const SweepGeometry& geo, int nq, int n_qtiles, int ng, int gchunk, int n_chunks, const __nv_bfloat16* qb,
                const __nv_bfloat16* gb, SweepHead* head, CUtensorMap* tq, CUtensorMap* tg);

// Both query-centring variants of a sweep kernel are launched; the one that does not match the device-side decision
// (Operands::qflag) returns at once, so the choice needs no host synchronisation.
template <class P>
int launch_sweep(void (*off)(CUtensorMap, CUtensorMap, P), void (*on)(CUtensorMap, CUtensorMap, P), int grid, int block,
                 size_t smem, cudaStream_t stream, const char* who, const CUtensorMap& tq, const CUtensorMap& tg,
                 const P& p) {
  if (int rc = launch(off, grid, block, smem, stream, who, tq, tg, p)) return rc;
  return launch(on, grid, block, smem, stream, who, tq, tg, p);
}

}  // namespace dcr
