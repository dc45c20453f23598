// Fused all-pairs similarity + per-query top-k for sm_90a.
//
// Replaces (reference = somepago/DCR):
//   diff_retrieval.py:402      sim = torch.mm(values_features, query_features.T)          (fp32, [G,Q], CPU/MKL)
//   diff_retrieval.py:417,613,621   simscores.topk(k, axis=1, largest=True)               k in {1,10}
//   diff_retrieval.py:403,418-419   sim2 = mm(values, values.T); topk(2)[...,-1]           (same kernel, Q:=G, k=2)
//   embedding_search/similarity_search.py:62-63   features @ batch.T ; max(dim=0)
//
// The [Q,G] score matrix is never written.  Three stages, all on the caller's stream:
//   1. to_bf16_rows_kernel   fp32 descriptors -> zero-padded bf16 rows + per-row norms of the rounding residual
//                            (sim_sweep.cu, shared with the threshold search in sim_range.cu)
//   2. sim_topk_kernel       wgmma bf16 GEMM (fp32 accumulate in registers) whose epilogue keeps, per query, the
//                            kp (>= k) best approximate scores of its gallery segment (threshold filter on the
//                            accumulator registers, warp-cooperative compaction in shared memory)
//   3. rescore_select_kernel exact re-score (fp64 accumulate, fixed order) of the <= slots*kp candidates per query,
//                            final order (score desc, gallery index asc), plus a per-query certificate that no
//                            non-candidate can reach the k-th exact score.  One kernel body, two widths: a warp per
//                            query when a q-tile has few candidate slots, the whole 128-thread block otherwise; both
//                            compute the same values.  Queries failing the certificate are recomputed by brute force in
//                            fp64 (exact_scan_kernel / exact_select_kernel).
// Result: indices identical to ranking all G exact dot products with ties broken by lowest index.
#include <algorithm>
#include <type_traits>

#include "../../include/dcr_b200.h"
#include "dcr_internal.cuh"
#include "sim_sweep.cuh"

namespace dcr {

namespace {

constexpr int kKPMax = 32;        // max candidates kept per (query, segment)
constexpr int kWarmTiles = 4;     // tiles replayed at the start of every segment to seed the threshold
constexpr int kMaxSlotsPerQuery = 512;  // (chunk, unit) segments that may cover one q-tile

struct SimParams : SweepHead {
  int kp;              // candidates kept per (query, segment): 8, 16 or 32
  int cap;             // shared-memory list capacity per query row (kp + 16 .. 64)
  int stages;          // B pipeline depth
  uint2* cand;         // [n_slots][rows_per_qtile][kKPMax]   (score bits, local gallery row)
  int* cand_cnt;       // [n_slots][rows_per_qtile]
  float* cand_thr;     // [n_slots][rows_per_qtile]
  const int* bias_flag;    // device flag: 0 = ignore col_bias (query centring switched off for this data)
  const float* col_bias;   // [ng_pad] per-gallery-row score offset nu.(g-mu) added to every accumulator column
  const float* thr_init;   // per query row: start thresholds (second-chance pass); null = seed by warm-up replay
  unsigned int* gthr;      // [nq_pad] per query row: best threshold any unit has reached so far, as an order-preserving
                           // unsigned key (0 = none)
  unsigned long long* clk; // [4] clock64 / globaltimer at the start and end of CTA 0 (SM clock under this kernel); null = off
  int kb_part;             // split score: k-blocks per descriptor part (kSplit kernels only; n_parts = num_kb / kb_part)
};

// second-chance pass: copy the bf16 rows of the flagged queries into a compact matrix (zero rows up to n_pad)
__global__ void gather_rows_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ rows, int n, int n_pad,
                                   int d_pad, __nv_bfloat16* __restrict__ dst) {
  const int chunks = d_pad / 8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
       i < static_cast<long long>(n_pad) * chunks; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / chunks), c = static_cast<int>(i % chunks);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < n) v = *reinterpret_cast<const uint4*>(src + static_cast<size_t>(rows[r]) * d_pad + c * 8);
    *reinterpret_cast<uint4*>(dst + static_cast<size_t>(r) * d_pad + c * 8) = v;
  }
}

// ------------------------------------------------------------------------------------------------------------
// stage 2 helpers

DCR_DEVICE unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// order-preserving float <-> unsigned key (0 is below every float): thresholds are shared with atomicMax
DCR_DEVICE unsigned int thr_key(float f) {
  const unsigned int b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
DCR_DEVICE float thr_from_key(unsigned int k) {
  if (k == 0) return -INFINITY;
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

DCR_DEVICE float max8(const float* v) {
  return fmaxf(fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3])), fmaxf(fmaxf(v[4], v[5]), fmaxf(v[6], v[7])));
}

// Keep the kp best of lane L's n (kp < n <= 64) list entries, stored at list[j * 128] (j = 0..n-1); returns the
// kp-th best score, which becomes that row's new threshold.  Whole warp cooperates: lane l ranks entries l and
// l+32 against all n keys (broadcast shared-memory reads), winners are rewritten in rank order (sorted list).
DCR_DEVICE float compact_one(uint2* list, int n, int kp, uint32_t lane) {
  const uint2 none = make_uint2(0xff800000u, 0xffffffffu);  // -inf
  const int l0 = static_cast<int>(lane), l1 = l0 + 32;
  const uint2 e0 = (l0 < n) ? list[l0 * 128] : none;
  const uint2 e1 = (l1 < n) ? list[l1 * 128] : none;
  const float k0 = __uint_as_float(e0.x), k1 = __uint_as_float(e1.x);
  int r0 = 0, r1 = 0;
  const float* keys = reinterpret_cast<const float*>(list);   // key j at keys[j * 256]
  if (n <= 32) {
#pragma unroll 4
    for (int j = 0; j < n; ++j) {
      const float kj = keys[j * 256];
      r0 += (kj > k0) || (kj == k0 && j < l0);
    }
  } else {
#pragma unroll 4
    for (int j = 0; j < n; ++j) {
      const float kj = keys[j * 256];
      r0 += (kj > k0) || (kj == k0 && j < l0);
      r1 += (kj > k1) || (kj == k1 && j < l1);
    }
  }
  __syncwarp();
  if (l0 < n && r0 < kp) list[r0 * 128] = e0;
  if (l1 < n && r1 < kp) list[r1 * 128] = e1;
  __syncwarp();
  return keys[(kp - 1) * 256];
}

DCR_DEVICE void compact_warp(uint2* warp_list, unsigned need, int kp, float& thr, int& cnt, uint32_t lane) {
  __syncwarp();   // make every lane's list stores visible to the lanes that will rank them
  while (need) {
    const int L = __ffs(need) - 1;
    need &= need - 1;
    const int n = __shfl_sync(kFull, cnt, L);
    const float t = compact_one(warp_list + L, n, kp, lane);
    if (static_cast<int>(lane) == L) {
      thr = t;
      cnt = kp;
    }
  }
}

DCR_DEVICE void st_shared_v2_if(uint32_t saddr, uint32_t a, uint32_t b, bool p) {
  asm volatile(
      "{\n\t.reg .pred q;\n\t"
      "setp.ne.b32 q, %3, 0;\n\t"
      "@q st.shared.v2.b32 [%0], {%1, %2};\n\t}\n" ::"r"(saddr),
      "r"(a), "r"(b), "r"(static_cast<uint32_t>(p))
      : "memory");
}

// One 32-column chunk of the accumulator row held by this thread.  The common case (no lane of the warp has a
// score above its threshold) costs a max-tree, one compare and one vote.  Otherwise the 8-column sub-chunks that
// contain a hit are appended to the row lists with predicated stores (no per-lane branching).
template <bool kMaskTail>
DCR_DEVICE void scan_chunk(const uint32_t (&r)[32], const float* sb, int gcol0, int ng, float& thr, int& cnt,
                           uint32_t my_list_saddr, uint2* warp_list, int kp, int cap, uint32_t lane) {
  float v[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) v[c] = __uint_as_float(r[c]);
  if (sb) {   // warp-uniform
#pragma unroll
    for (int c = 0; c < 32; c += 4) {
      const float4 b = *reinterpret_cast<const float4*>(sb + c);
      v[c] += b.x; v[c + 1] += b.y; v[c + 2] += b.z; v[c + 3] += b.w;
    }
  }
#pragma unroll
  for (int c = 0; c < 32; ++c)
    if (kMaskTail && gcol0 + c >= ng) v[c] = -INFINITY;
  float s[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) s[i] = max8(v + 8 * i);
  const float m = fmaxf(fmaxf(s[0], s[1]), fmaxf(s[2], s[3]));
  if (__any_sync(kFull, m > thr)) {
#pragma unroll
    for (int sub = 0; sub < 4; ++sub) {
      if (__any_sync(kFull, s[sub] > thr)) {
        uint32_t addr = my_list_saddr + static_cast<uint32_t>(cnt) * 1024u;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float x = v[sub * 8 + c];
          const bool h = x > thr;
          st_shared_v2_if(addr, __float_as_uint(x), static_cast<uint32_t>(gcol0 + sub * 8 + c), h);
          addr += h ? 1024u : 0u;
        }
        cnt = static_cast<int>((addr - my_list_saddr) >> 10);
        const unsigned need = __ballot_sync(kFull, cnt > cap - 8);
        if (need) compact_warp(warp_list, need, kp, thr, cnt, lane);
      }
    }
  }
}

// last gallery tile only: columns past the end of the gallery never win (-inf survives the offset add)
DCR_DEVICE void mask_tail(uint32_t (&r)[32], int gcol0, int ng) {
#pragma unroll
  for (int c = 0; c < 32; ++c)
    if (gcol0 + c >= ng) r[c] = 0xff800000u;
}

// Warm-up chunk: running maxima of 32 column slots (slot = column mod 32); no candidates are recorded.
template <bool kMaskTail>
DCR_DEVICE void warm_chunk(const uint32_t (&r)[32], const float* sb, int gcol0, int ng, float (&slot)[32]) {
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    float x = __uint_as_float(r[c]);
    if (sb) x += sb[c];
    if (kMaskTail && gcol0 + c >= ng) x = -INFINITY;
    slot[c] = fmaxf(slot[c], x);
  }
}

// Seed of a segment's threshold from the warm-up maxima: fold the 32 slot maxima into `groups` >= kp disjoint groups;
// the smallest group maximum is exceeded by at least groups-1 already-seen scores, so it is a safe (never too high
// for kp) start.  Segments shorter than the warm-up still get a valid bound.
DCR_DEVICE float seed_threshold(float (&slot)[32], int kp) {
  int groups = 32;
  if (kp <= 16) {
#pragma unroll
    for (int c = 0; c < 16; ++c) slot[c] = fmaxf(slot[c], slot[c + 16]);
    groups = 16;
  }
  if (kp <= 8) {
#pragma unroll
    for (int c = 0; c < 8; ++c) slot[c] = fmaxf(slot[c], slot[c + 8]);
    groups = 8;
  }
  if (kp <= 4) {
#pragma unroll
    for (int c = 0; c < 4; ++c) slot[c] = fmaxf(slot[c], slot[c + 4]);
    groups = 4;
  }
  float lo = slot[0];
#pragma unroll
  for (int c = 1; c < 32; ++c)
    if (c < groups) lo = fminf(lo, slot[c]);
  // strictly below the smallest group maximum so that the maxima themselves are recorded
  float thr = (lo == -INFINITY) ? -INFINITY : __uint_as_float(__float_as_uint(lo) + (lo > 0.f ? -1 : (lo < 0.f ? 1 : 0)));
  if (lo == 0.f) thr = -1e-30f;
  return thr;
}

// ------------------------------------------------------------------------------------------------------------
// stage 2: the fused kernel.  One CTA per work unit; kSets consumer warpgroups (warps 0 .. 4 kSets - 1) each issue the
// wgmma for their column range of every 128 x 128 tile (fp32 accumulators in registers) and filter it; the last warp is
// the TMA producer.
//
// Work decomposition: the (q-tile, g-tile) grid is linearised q-major into T = n_qtiles * n_gtiles tiles and cut
// into gridDim equal contiguous ranges.  A unit's range is walked as "segments" (maximal runs inside one
// q-tile); per segment the query tile is loaded once (A stays resident) and the thresholds are seeded by
// replaying the first kWarmTiles tiles.  Segment (unit u, q-tile i) owns candidate slot u + i.
// kBias: compiled with / without the per-column offset path of query centring.  Both variants are launched; the one
// that does not match the device-side decision (p.bias_flag) exits at once -- no host synchronisation needed.
// kSplit: the split score (sim_topk_split): every tile's approximate score is the maximum over the descriptor parts
// (fused_tile_mma_split); the filter and the lists see that maximum.  Built with kSets = 2 and without kBias only.
// kCross: the cross split score (sim_topk_cross), the same kernel with the cross schedule of the part pairs.
template <bool kBias, int kSets, bool kSplit = false, bool kCross = false>
__global__ void __launch_bounds__(32 + 128 * kSets, 1)
    sim_topk_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_g,
                    const SimParams p) {
  static_assert(!kSplit || (kSets == 2 && !kBias), "the split score runs on column halves, uncentred");
  static_assert(!kCross || kSplit, "the cross score is a split score");
  if (((p.bias_flag != nullptr) && (*p.bias_flag != 0)) != kBias) return;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int kSetCols = kBlockN / kSets;
  // the pipeline, then [kSets][cap][128] candidate lists, barriers, carried thresholds and transpose buffers
  const FusedPipe pp(smem_raw, p.num_kb, p.stream_a, p.stages, static_cast<size_t>(kSets) * p.cap * 128 * 8);
  const bool stream_a = pp.stream_a;
  uint2* cand = reinterpret_cast<uint2*>(pp.lists);   // [kSets][cap][128]
  float* carry = reinterpret_cast<float*>(pp.tail);   // [kSets][4][128] thresholds carried to the next chunk, by q-tile & 3
  uint8_t* acc_xpose = reinterpret_cast<uint8_t*>(carry + kSets * 4 * kBlockM);   // [4 kSets warps] accumulator transposes

  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31;
  constexpr uint32_t kProducerWarp = 4 * kSets;

  pp.init(&tmap_q, &tmap_g, p.stages, kProducerWarp);
  if (p.clk && blockIdx.x == 0 && threadIdx.x == 0) {
    p.clk[0] = clock64();
    p.clk[1] = global_timer_ns();
  }

  // this unit's tile range
  const long long n_units = gridDim.x;
  const long long unit = blockIdx.x;
  const int rows_per_qtile = kBlockM;

  if (warp == kProducerWarp) {
    // ===================================== TMA producer =====================================
    SegWalker w(p.n_qtiles, p.n_gtiles, p.gchunk, p.n_chunks, unit, n_units);
    fused_producer<kCross>(pp, &tmap_q, &tmap_g, p.stages, w,
                           [&](const SegWalker& s) { return (p.thr_init || s.carried) ? 0 : min(kWarmTiles, s.ntiles); },
                           p.kb_part);
  } else {
    // ===================================== consumer warpgroups =====================================
    // kSets = 2: two warps per 32-row block, each owning one column half ("set") of every tile and its own candidate
    // lists / slot -- the filter is issue- and latency-bound with a single warp per sub-partition.
    const uint32_t quad = warp & 3;             // rows quad*32 .. +31 of the tile
    const uint32_t set = warp >> 2;             // column range [set * kSetCols, (set + 1) * kSetCols) of every tile
    const uint32_t row = quad * 32 + lane;      // query row inside this CTA's tile
    uint2* set_list = cand + set * p.cap * 128;
    const uint32_t my_list = smem_u32(set_list + row);
    uint2* warp_list = set_list + quad * 32;
    const uint32_t xacc = smem_u32(acc_xpose) + warp * kAccXposeWarpBytes;
    float* my_carry = carry + set * 4 * kBlockM;
    const int kp = p.kp, cap = p.cap;
    const float* colbias = kBias ? p.col_bias : nullptr;
    const uint32_t a_base = smem_u32(stream_a ? pp.smem_b + kBTileBytes : pp.smem_a);
    const uint32_t b_base = smem_u32(pp.smem_b) + set * kSetCols * 128;
    PipeState st(p.stages);
    uint32_t seg = 0;
    SegWalker w(p.n_qtiles, p.n_gtiles, p.gchunk, p.n_chunks, unit, n_units);
    while (w.next()) {
      const int qi = w.qi, g_begin = w.g_begin, ntiles = w.ntiles;
      const int warm = (p.thr_init || w.carried) ? 0 : min(kWarmTiles, ntiles);
      float thr = -INFINITY;
      if (p.thr_init) {
        const int qrow_g = qi * rows_per_qtile + static_cast<int>(row);
        thr = qrow_g < p.nq ? p.thr_init[qrow_g] : INFINITY;   // padding rows collect nothing
      }
      // a threshold this row reached on an earlier gallery chunk is a valid (and usually tight) start here
      if (w.carried) thr = fmaxf(thr, my_carry[(qi & 3) * kBlockM + row]);
      int cnt = 0;
      // Threshold sharing: a threshold ANY unit reached for this query row (kp recorded scores above it exist somewhere
      // in the gallery) is a valid drop bound for every other unit sweeping the same query tile.  Read once per tile
      // (the load is issued before the main loop), published when it has risen.
      const int qrow_s = qi * rows_per_qtile + static_cast<int>(row);
      unsigned int* gslot = qrow_s < p.nq ? p.gthr + qrow_s : nullptr;
      float published = gslot ? thr_from_key(*reinterpret_cast<volatile unsigned int*>(gslot)) : INFINITY;
      if (gslot) thr = fmaxf(thr, published);
      if (!stream_a) mbar_wait(pp.a_full, seg & 1);

      // one accumulator tile: warm-up tiles only track column-slot maxima, the others feed the candidate lists.  Two
      // separate loops so that the 32 slot registers are dead while the lists are live.
      auto tile = [&](auto warm_tag, int gi, bool last, float (&slot)[32]) {
        constexpr bool kWarm = decltype(warm_tag)::value;
        const int gcol0 = gi * kBlockN + static_cast<int>(set) * kSetCols;
        const bool tail = gcol0 + kSetCols > p.ng;
        const float* sb = kBias ? colbias + gcol0 : nullptr;   // per-column offsets: warp-uniform (broadcast) loads
        unsigned int shared_key = 0;
        if (!kWarm && gslot) shared_key = *reinterpret_cast<volatile unsigned int*>(gslot);
        WgAcc<kSetCols> acc;
        if constexpr (kSplit) fused_tile_mma_split<kSetCols, kCross>(acc, st, pp, a_base, b_base, p.kb_part, last, lane);
        else fused_tile_mma(acc, st, pp, a_base, b_base, last, lane);
        if (!kWarm && gslot) {
          if (thr > published) {   // risen since the last publication (compaction): let the other units know
            atomicMax(gslot, thr_key(thr));
            published = thr;
          }
          const float other = thr_from_key(shared_key);
          if (other > thr) {
            thr = other;
            published = other;
          }
        }
#pragma unroll
        for (int ch = 0; ch < kSetCols / 32; ++ch) {
          uint32_t r[32];
          acc.rows32(ch, r, xacc, lane);
          if (tail) mask_tail(r, gcol0 + ch * 32, p.ng);
          if constexpr (kWarm) warm_chunk<false>(r, sb ? sb + ch * 32 : nullptr, gcol0 + ch * 32, p.ng, slot);
          else scan_chunk<false>(r, sb ? sb + ch * 32 : nullptr, gcol0 + ch * 32, p.ng, thr, cnt, my_list, warp_list, kp, cap, lane);
        }
      };
      if (warm > 0) {
        float slot[32];
#pragma unroll
        for (int c = 0; c < 32; ++c) slot[c] = -INFINITY;
#pragma unroll 1
        for (int j = 0; j < warm; ++j) tile(std::true_type{}, g_begin + j, false, slot);
        thr = seed_threshold(slot, kp);
      }
      {
        float unused[32];
#pragma unroll 1
        for (int j = 0; j < ntiles; ++j) tile(std::false_type{}, g_begin + j, j == ntiles - 1, unused);
      }
      ++seg;
      // ---- flush this segment's lists: final compaction to kp, then coalesced copy to the slot ----
      __syncwarp();
      {
        const unsigned need = __ballot_sync(kFull, cnt > kp);
        if (need) compact_warp(warp_list, need, kp, thr, cnt, lane);
      }
      __syncwarp();
      my_carry[(qi & 3) * kBlockM + row] = thr;
      if (gslot && thr > published) atomicMax(gslot, thr_key(thr));
      const int slot = slot_index(w.chunk, static_cast<int>(unit), qi, static_cast<int>(set), static_cast<int>(n_units),
                                  p.n_qtiles, kSets);
      const size_t slot_row0 = static_cast<size_t>(slot) * rows_per_qtile + quad * 32;
      for (int L = 0; L < 32; ++L) {
        const int n = __shfl_sync(kFull, cnt, L);
        if (static_cast<int>(lane) < n) p.cand[(slot_row0 + L) * kKPMax + lane] = warp_list[L + lane * 128];
      }
      p.cand_cnt[slot_row0 + lane] = cnt;
      p.cand_thr[slot_row0 + lane] = thr;
      __syncwarp();
    }
  }

  // teardown
  __syncthreads();
  if (p.clk && blockIdx.x == 0 && threadIdx.x == 0) {
    p.clk[2] = clock64();
    p.clk[3] = global_timer_ns();
  }
}

// order (score desc, index asc)
DCR_DEVICE bool better(double s, long long i, double bs, long long bi) { return (s > bs) || (s == bs && i < bi); }

// block-wide arg-best over (key desc, index asc) of kWarps warps; every thread passes its local best (pos < 0 = none) and
// receives the block's
template <int kWarps>
struct BlockBest {
  double key[kWarps];
  long long idx[kWarps];
  int pos[kWarps];
};
template <int kWarps>
DCR_DEVICE void block_argbest(double& bs, long long& bi, int& bp, BlockBest<kWarps>* sb, uint32_t lane, uint32_t warp) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double os = __shfl_xor_sync(kFull, bs, off);
    const long long oi = __shfl_xor_sync(kFull, bi, off);
    const int op = __shfl_xor_sync(kFull, bp, off);
    if (op >= 0 && (bp < 0 || better(os, oi, bs, bi))) {
      bs = os;
      bi = oi;
      bp = op;
    }
  }
  if (lane == 0) {
    sb->key[warp] = bs;
    sb->idx[warp] = bi;
    sb->pos[warp] = bp;
  }
  __syncthreads();
  bs = sb->key[0];
  bi = sb->idx[0];
  bp = sb->pos[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w)
    if (sb->pos[w] >= 0 && (bp < 0 || better(sb->key[w], sb->idx[w], bs, bi))) {
      bs = sb->key[w];
      bi = sb->idx[w];
      bp = sb->pos[w];
    }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------------------
// stage 3: exact re-score, selection and certificate.  A group of kThreads threads serves one query: a warp (kThreads =
// 32, four queries per block, no block-wide barrier) or the whole 128-thread block.  Both widths run this one body, so
// they gather the same candidates and compute the same eps, exact scores, order and certificate.
//   1. gather the (gallery row, approximate score) candidates of every segment slot of this query's q-tile
//   2. prune: with A_k the k-th largest approximate score, a candidate below A_k - 2*eps cannot be in the exact
//      top-k (its exact score is < A_k - eps <= the exact scores of the k best-approximate candidates)
//   3. exact fp64 scores of the survivors, selection by (score desc, index asc)
//   4. certificate against the rows the fused kernel dropped; failures are appended to `flagged` together with
//      a threshold for the second-chance pass (thr_next).
// kSplit: the split score.  The exact score of a candidate is the maximum over the parts of exact_dot over that part, the
// query staged in shared memory one part at a time (rows are far wider than shared memory), and the bound is
// split_row_bound.
// kCross: the cross split score.  The exact score folds every (query part, gallery part) pair (cross_exact_scores, the
// query staged several parts at a time) and the bound is cross_row_bound.
struct RescoreParams {
  const float* q;                   // the caller's query rows [*][d]
  const float* g;                   // [ng][d]
  int nq;                           // queries of this pass: rows of the (possibly compacted) matrix the fused kernel saw
  int d, d_pad, k;
  int n_qtiles, n_gtiles, gchunk, n_chunks, n_units, n_sets;   // the fused pass's work decomposition
  int max_cand;                     // candidates one query may gather (sizes its shared memory)
  const uint2* cand;                // the fused pass's slots: SimParams::cand, cand_cnt, cand_thr
  const int* cand_cnt;
  const float* cand_thr;
  const int* qmap;                  // pass row -> caller's row; null = identity
  const float* mu;                  // gallery centre
  const float* nu;                  // query centre, used when *nu_flag != 0; null = none
  const int* nu_flag;
  const float* q_norm_hat;          // per caller row, from stage 1
  const float* q_norm_res;
  const float* q_norm_x;
  const unsigned int* g_max;        // [2] from stage 1
  long long g_index_base, g_index_stride;
  float* out_scores;                // [*][k] by caller row
  long long* out_idx;
  int* flagged;                     // caller rows whose certificate failed, counted by *n_flagged
  int* n_flagged;
  float* thr_next;                  // per flagged entry: start threshold of the second-chance pass; null = last pass
  int n_parts;                      // split score (kSplit): descriptor parts of d / n_parts values; q_norm_* per part
  int staged;                       // cross split score (kCross): query parts staged at once (cross_staged_parts)
};

// One query's shared memory: the query row widened to fp64, then four arrays of max_cand entries.  Every part is a
// multiple of 16 bytes, so the four queries of a 32-wide block lie back to back.
struct RescoreSmem {
  size_t sc, ci, ap, kc, bytes;   // byte offsets of: exact scores (fp64), candidate rows, approximate scores, survivor rows
  __host__ __device__ RescoreSmem(int d, int max_cand) {
    const size_t d2 = (static_cast<size_t>(d) + 1) & ~size_t(1), mc = (static_cast<size_t>(max_cand) + 3) & ~size_t(3);
    sc = d2 * 8;
    ci = sc + mc * 8;
    ap = ci + mc * 4;
    kc = ap + mc * 4;
    bytes = kc + mc * 4;
  }
};

template <int kThreads, bool kSplit = false, bool kCross = false>
__global__ void __launch_bounds__(kRescoreThreads) rescore_select_kernel(const RescoreParams p) {
  static_assert(!kCross || kSplit, "the cross score is a split score");
  constexpr int kWarps = kThreads / 32;
  extern __shared__ __align__(16) uint8_t sm[];
  const int tid = static_cast<int>(threadIdx.x) % kThreads;
  const uint32_t lane = threadIdx.x & 31;
  const int warp = tid >> 5;   // warp of the group
  const int grp = static_cast<int>(threadIdx.x) / kThreads;
  // crow indexes the (possibly compacted) query matrix the fused kernel saw; qrow is the caller's row
  const int crow = blockIdx.x * (kRescoreThreads / kThreads) + grp;
  if (crow >= p.nq) return;   // whole groups leave; nothing below synchronises across groups
  const RescoreSmem L(kCross ? static_cast<int>(cross_stage_doubles(p.staged, p.d / p.n_parts, kWarps))
                             : (kSplit ? p.d / p.n_parts : p.d),
                      p.max_cand);
  uint8_t* base = sm + grp * L.bytes;
  double* qs = reinterpret_cast<double*>(base);          // [d] the query row, widened once ([d / n_parts]: one part;
                                                         // cross: the staged parts and the warps' running maxima)
  double* sc = reinterpret_cast<double*>(base + L.sc);   // exact scores of the survivors
  int* ci = reinterpret_cast<int*>(base + L.ci);         // gallery rows of all candidates
  float* ap = reinterpret_cast<float*>(base + L.ap);     // approximate scores
  int* kc = reinterpret_cast<int*>(base + L.kc);         // gallery rows of the survivors
  const int d = p.d, k = p.k;
  const int qrow = p.qmap ? p.qmap[crow] : crow;
  // the query row: requested first, consumed after the slot walk below has issued its own loads (one memory round trip for
  // both instead of one after the other).  Thread t owns the 16-byte granules t, t + kThreads, ... of the first 512 dims.
  constexpr int kQv = 512 / (4 * kThreads);
  float4 qv[kQv];
#pragma unroll
  for (int i = 0; i < kQv; ++i) {
    const int c = (i * kThreads + tid) * 4;
    if (!kSplit && c < d) qv[i] = *reinterpret_cast<const float4*>(p.q + static_cast<size_t>(qrow) * d + c);   // d % 4 == 0
  }

  // ---- the (chunk, unit, set) slots that cover this q-tile, in rounds: lane c owns chunk c0 + c (every warp of the group
  // holds the same 32 chunks), then thread t owns slot s0 + t; prefix sums of the slot counts place the entries ----
  const int qi = crow / kBlockM, r = crow % kBlockM;
  int n = 0;
  bool overflow = false;
  float thr = -INFINITY;
  for (int c0 = 0; c0 < p.n_chunks; c0 += 32) {
    const int chunk = c0 + static_cast<int>(lane);
    int u_lo = 0, n_cs = 0;   // this lane's chunk: first unit whose range covers q-tile qi, and the chunk's slot count
    if (chunk < p.n_chunks) {
      const int ncg = min(p.gchunk, p.n_gtiles - chunk * p.gchunk);
      const long long T = static_cast<long long>(p.n_qtiles) * ncg;
      u_lo = static_cast<int>(owner_unit(static_cast<long long>(qi) * ncg, T, p.n_units));
      n_cs = (static_cast<int>(owner_unit(static_cast<long long>(qi + 1) * ncg - 1, T, p.n_units)) - u_lo + 1) * p.n_sets;
    }
    int n_slots;
    const int first = group_scan<32>(n_cs, n_slots);
    const int nc = min(32, p.n_chunks - c0);
    for (int s0 = 0; s0 < n_slots; s0 += kThreads) {
      const int s = s0 + tid;
      int slot = -1;
      for (int c = 0; c < nc; ++c) {
        const int rel = s - __shfl_sync(kFull, first, c), cnt = __shfl_sync(kFull, n_cs, c), lo = __shfl_sync(kFull, u_lo, c);
        if (rel >= 0 && rel < cnt) slot = slot_index(c0 + c, lo + rel / p.n_sets, qi, rel % p.n_sets, p.n_units, p.n_qtiles, p.n_sets);
      }
      int cc = 0;
      if (slot >= 0) {
        const size_t sr = static_cast<size_t>(slot) * kBlockM + r;
        cc = p.cand_cnt[sr];
        thr = fmaxf(thr, p.cand_thr[sr]);
      }
      int n_round;
      const int off = n + group_scan<kThreads>(cc, n_round);
      overflow |= n + n_round > p.max_cand;   // cannot happen: plan_pass sizes max_cand for kp entries in every slot
      if (!overflow) {
        // each warp copies its own threads' slots, a lane per entry (kKPMax = 32 entries per slot)
        const int nsl = min(32, n_slots - s0 - warp * 32);
#pragma unroll 4
        for (int j = 0; j < nsl; ++j) {
          const int c_j = __shfl_sync(kFull, cc, j), off_j = __shfl_sync(kFull, off, j), slot_j = __shfl_sync(kFull, slot, j);
          if (static_cast<int>(lane) < c_j) {
            const uint2 e = p.cand[(static_cast<size_t>(slot_j) * kBlockM + r) * kKPMax + lane];
            ci[off_j + lane] = static_cast<int>(e.y);
            ap[off_j + lane] = __uint_as_float(e.x);
          }
        }
      }
      n += n_round;
    }
  }
  if (overflow) n = 0;   // k >= 1: the certificate fails and the query is flagged
  thr = group_max<kThreads>(thr);
  if constexpr (!kSplit) {
#pragma unroll
    for (int i = 0; i < kQv; ++i) {
      const int c = (i * kThreads + tid) * 4;
      if (c < d) {
        *reinterpret_cast<double2*>(qs + c) = make_double2(static_cast<double>(qv[i].x), static_cast<double>(qv[i].y));
        *reinterpret_cast<double2*>(qs + c + 2) = make_double2(static_cast<double>(qv[i].z), static_cast<double>(qv[i].w));
      }
    }
    for (int c = 512 + tid; c < d; c += kThreads) qs[c] = static_cast<double>(p.q[static_cast<size_t>(qrow) * d + c]);
  }
  group_sync<kThreads>();

  // certificate: every gallery row that is not a candidate has approximate centred score <= thr, hence exact score
  // q.g <= thr + eps + q.mu + slack (row_bound; split_row_bound for the split score)
  const RowBound rb = [&] {
    if constexpr (kCross)
      return cross_row_bound(p.n_parts, d / p.n_parts, p.d_pad / p.n_parts, qrow, p.q_norm_hat, p.q_norm_res, p.q_norm_x,
                             p.g_max, lane);
    else if constexpr (kSplit)
      return split_row_bound(p.n_parts, d / p.n_parts, p.d_pad / p.n_parts, qrow, p.q_norm_hat, p.q_norm_res, p.q_norm_x,
                             p.g_max, lane);
    else
      return row_bound(qs, d, p.d_pad, qrow, p.q_norm_hat, p.q_norm_res, p.q_norm_x, p.g_max, p.mu, p.nu, p.nu_flag, lane);
  }();
  const float eps = rb.eps;
  const double qmu = rb.qmu;
  const bool closed = thr > -INFINITY;   // some segment dropped rows
  const double bound = static_cast<double>(thr) + static_cast<double>(eps) + qmu + rb.slack;

  // ---- prune by approximate score: A_k by rank counting (n is a few dozen: one pass instead of k arg-max rounds) ----
  const int kk = min(k, n);
  float a_k = -INFINITY;
  for (int c = tid; c < n; c += kThreads) {
    const float v = ap[c];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float o = ap[j];
      rank += (o > v) || (o == v && j < c);
    }
    if (rank == kk - 1) a_k = v;
  }
  a_k = group_max<kThreads>(a_k);
  const float cut = a_k - 2.f * eps - 1e-6f * fabsf(a_k);
  int m = 0;
  for (int c0 = 0; c0 < n; c0 += kThreads) {
    const int c = c0 + tid;
    const bool keep = c < n && (n <= k || ap[c] >= cut);
    int kept;
    const int pos = m + group_scan<kThreads>(keep ? 1 : 0, kept);
    if (keep) kc[pos] = ci[c];
    m += kept;
  }
  group_sync<kThreads>();
  if constexpr (kCross) {
    const int pl = d / p.n_parts;
    cross_exact_scores<kThreads>(p.q + static_cast<size_t>(qrow) * d, p.g, d, p.n_parts, p.staged, kc, m, sc, qs,
                                 qs + static_cast<size_t>(p.staged) * pl);
  } else if constexpr (kSplit) {
    // ---- exact split scores of the survivors: per part, stage the query part, prefetch that part of every survivor, then
    // fold each part's dot product into the running maximum (the order of split_rescore_kernel: -inf, then parts 0, 1, ..)
    const int pl = d / p.n_parts;
    for (int c = tid; c < m; c += kThreads) sc[c] = -INFINITY;
    for (int part = 0; part < p.n_parts; ++part) {
      group_sync<kThreads>();   // the previous part's readers of qs are done
      const float* qsrc = p.q + static_cast<size_t>(qrow) * d + static_cast<size_t>(part) * pl;
      for (int c = tid * 4; c < pl; c += kThreads * 4) {
        const float4 v = *reinterpret_cast<const float4*>(qsrc + c);
        *reinterpret_cast<double2*>(qs + c) = make_double2(static_cast<double>(v.x), static_cast<double>(v.y));
        *reinterpret_cast<double2*>(qs + c + 2) = make_double2(static_cast<double>(v.z), static_cast<double>(v.w));
      }
      const int lines = (pl * 4 + 127) / 128;
      for (int t = tid; t < m * lines; t += kThreads) {
        const float* ptr = p.g + static_cast<size_t>(kc[t / lines]) * d + static_cast<size_t>(part) * pl + (t % lines) * 32;
        asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
      }
      group_sync<kThreads>();
      for (int c = 2 * warp; c < m; c += 2 * kWarps) {
        const float* g0 = p.g + static_cast<size_t>(kc[c]) * d + static_cast<size_t>(part) * pl;
        double v0, v1 = 0.0;
        if (c + 1 < m) exact_dot<2>(qs, g0, p.g + static_cast<size_t>(kc[c + 1]) * d + static_cast<size_t>(part) * pl, pl, lane, v0, v1);
        else exact_dot<1>(qs, g0, nullptr, pl, lane, v0, v1);
        if (lane == 0) {
          sc[c] = fmax(sc[c], v0);
          if (c + 1 < m) sc[c + 1] = fmax(sc[c + 1], v1);
        }
      }
    }
    group_sync<kThreads>();
  } else {
    // every surviving row's cache lines are requested at once (L2 prefetch): the dot products below then wait for L2, not
    // for one DRAM round trip per pair of rows
    {
      const int lines = (d * 4 + 127) / 128;
      for (int t = tid; t < m * lines; t += kThreads) {
        const float* ptr = p.g + static_cast<size_t>(kc[t / lines]) * d + (t % lines) * 32;
        asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
      }
    }

    // ---- exact scores of the survivors (two rows in flight per warp), then selection by (score desc, index asc) ----
    for (int c = 2 * warp; c < m; c += 2 * kWarps) {
      double v0, v1 = 0.0;
      if (c + 1 < m) exact_dot<2>(qs, p.g + static_cast<size_t>(kc[c]) * d, p.g + static_cast<size_t>(kc[c + 1]) * d, d, lane, v0, v1);
      else exact_dot<1>(qs, p.g + static_cast<size_t>(kc[c]) * d, nullptr, d, lane, v0, v1);
      if (lane == 0) {
        sc[c] = v0;
        if (c + 1 < m) sc[c + 1] = v1;
      }
    }
    group_sync<kThreads>();
  }
  const int km = min(k, m);
  double kth = -INFINITY;
  for (int c = tid; c < m; c += kThreads) {
    const double v = sc[c];
    const int iv = kc[c];
    int rank = 0;
    for (int j = 0; j < m; ++j) {
      const double o = sc[j];
      const int io = kc[j];
      rank += (o > v) || (o == v && (io < iv || (io == iv && j < c)));   // candidate rows are distinct; j < c only for safety
    }
    if (rank < km) {
      p.out_scores[static_cast<size_t>(qrow) * k + rank] = static_cast<float>(v);
      p.out_idx[static_cast<size_t>(qrow) * k + rank] = p.g_index_base + p.g_index_stride * iv;
      if (rank == km - 1) kth = v;
    }
  }
  kth = group_max<kThreads>(kth);   // one thread holds it (NaN -> -inf: flagged)
  if (tid == 0) {
    const bool ok = (n >= k) && (m >= k) && (!closed || kth > bound);
    if (!ok) {
      const int pos = atomicAdd(p.n_flagged, 1);
      p.flagged[pos] = qrow;
      if (p.thr_next) {
        // every row of the true top-k has exact score >= kth, hence centred approximate score >= kth - q.mu - eps
        float t = -INFINITY;
        if (m >= k && kth > -INFINITY) {
          const double lo = kth - qmu - static_cast<double>(eps);
          t = static_cast<float>(lo) - 2e-6f * fabsf(static_cast<float>(lo)) - 1e-7f;
        }
        p.thr_next[pos] = t;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// 'splitloss' similarity (diff_retrieval.py:393-400): descriptors are cut into n_chunks equal parts and the score of
// a pair is the MAXIMUM over the parts of the per-part dot products.  The top-k under that score is contained in the
// union of the per-part top-k lists (if a row is in the true top-k through its best part c, fewer than k rows beat it
// in part c), so the host runs the fused kernel once per part and this kernel finishes: per query, de-duplicate the
// n_cand candidate rows, evaluate max_c <q_c, g_c> exactly (float64, the same fixed-order dot as the re-score
// kernel), and select k by (score desc, row asc).
__global__ void __launch_bounds__(128)
    split_rescore_kernel(const float* __restrict__ q, const float* __restrict__ g, int d, int n_chunks, int cross,
                         const long long* __restrict__ cand, int n_cand, int k, float* __restrict__ out_scores,
                         long long* __restrict__ out_idx) {
  extern __shared__ __align__(16) uint8_t sm[];
  // only ONE query part is staged at a time (per-token splitloss on ViT outputs has d = 197 * 384 floats per row)
  const int p = d / n_chunks;
  float* qs = reinterpret_cast<float*>(sm);                              // [p]
  double* sc = reinterpret_cast<double*>(sm + ((p * 4 + 15) & ~15));      // [n_cand]
  long long* ci = reinterpret_cast<long long*>(sc + n_cand);              // [n_cand], -1 = duplicate / taken
  __shared__ BlockBest<4> s_bb;
  const int qrow = blockIdx.x;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = threadIdx.x; c < n_cand; c += blockDim.x) ci[c] = cand[static_cast<size_t>(qrow) * n_cand + c];
  __syncthreads();
  // duplicates (a row that made the list of several parts): keep the first occurrence
  for (int c = threadIdx.x; c < n_cand; c += blockDim.x) {
    const long long v = ci[c];
    bool dup = v < 0;                                                     // negative = empty slot of the caller's list
    for (int j = 0; j < c; ++j) dup |= (ci[j] == v);   // ci is not modified before the barrier below
    sc[c] = dup ? 1.0 : 0.0;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < n_cand; c += blockDim.x) {
    if (sc[c] != 0.0) ci[c] = -1;
    sc[c] = -INFINITY;
  }
  __syncthreads();
  for (int qp = 0; qp < n_chunks; ++qp) {
    for (int c = threadIdx.x; c < p; c += blockDim.x) qs[c] = q[static_cast<size_t>(qrow) * d + qp * p + c];
    __syncthreads();
    for (int c = warp; c < n_cand; c += 4) {
      if (ci[c] < 0) continue;   // warp-uniform
      double best = sc[c];
      if (cross) {   // 'cross' (einsum_in_chunks, diff_retrieval.py:652-654): every gallery part against every query part
        for (int part = 0; part < n_chunks; ++part) {
          double v;
          exact_dot<1>(qs, g + static_cast<size_t>(ci[c]) * d + part * p, nullptr, p, lane, v, v);
          best = fmax(best, v);
        }
      } else {
        double v;
        exact_dot<1>(qs, g + static_cast<size_t>(ci[c]) * d + qp * p, nullptr, p, lane, v, v);
        best = fmax(best, v);
      }
      if (lane == 0) sc[c] = best;   // ranked on the float64 value (as dcr_sim_topk), reported as fp32
    }
    __syncthreads();
  }
  for (int round = 0; round < k; ++round) {
    double bs = -INFINITY;
    long long bi = 0x7fffffffffffffffLL;
    int bp = -1;
    for (int c = threadIdx.x; c < n_cand; c += blockDim.x)
      if (ci[c] >= 0 && (bp < 0 || better(sc[c], ci[c], bs, bi))) {
        bs = sc[c];
        bi = ci[c];
        bp = c;
      }
    block_argbest(bs, bi, bp, &s_bb, lane, warp);
    if (threadIdx.x == 0) {
      out_scores[static_cast<size_t>(qrow) * k + round] = bp >= 0 ? static_cast<float>(bs) : -INFINITY;
      out_idx[static_cast<size_t>(qrow) * k + round] = bp >= 0 ? bi : -1;
      if (bp >= 0) ci[bp] = -1;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------------------
// brute-force exact path for flagged queries (batch of <= kExactBatch): scores[f][g] in fp64, then select.
constexpr int kExactBatch = 32;

__global__ void __launch_bounds__(256)
    exact_scan_kernel(const float* __restrict__ q, const float* __restrict__ g, int ng, int d,
                      const int* __restrict__ flagged, int f_begin, const int* __restrict__ n_flagged,
                      double* __restrict__ scores, int batch) {
  extern __shared__ __align__(16) uint8_t sm[];
  float* qs = reinterpret_cast<float*>(sm);  // [nb][d]
  const int nb = min(batch, *n_flagged - f_begin);
  if (nb <= 0) return;
  for (int i = threadIdx.x; i < nb * d; i += blockDim.x) {
    const int f = i / d, c = i % d;
    qs[i] = q[static_cast<size_t>(flagged[f_begin + f]) * d + c];
  }
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const int warps = (blockDim.x >> 5) * gridDim.x;
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < ng; row += warps) {
    const float* gr = g + static_cast<size_t>(row) * d;
    for (int f = 0; f < nb; ++f) {
      double v;
      exact_dot<1>(qs + f * d, gr, nullptr, d, lane, v, v);
      if (lane == 0) scores[static_cast<size_t>(f) * ng + row] = v;
    }
  }
}

// the same under the split score: scores[f][g] = max over the parts of exact_dot over that part (the order of
// split_rescore_kernel), the batch's query parts staged one part at a time.  kCross: the cross split score, query part
// `part` against every gallery part b in ascending order (split_rescore_kernel's cross branch: query part outer).
template <bool kCross>
__global__ void __launch_bounds__(256)
    split_scan_kernel(const float* __restrict__ q, const float* __restrict__ g, int ng, int d, int n_parts,
                      const int* __restrict__ flagged, int f_begin, const int* __restrict__ n_flagged,
                      double* __restrict__ scores, int batch) {
  extern __shared__ __align__(16) uint8_t sm[];
  float* qs = reinterpret_cast<float*>(sm);  // [nb][pl]
  const int nb = min(batch, *n_flagged - f_begin);
  if (nb <= 0) return;
  const int pl = d / n_parts;
  const uint32_t lane = threadIdx.x & 31;
  const int warps = (blockDim.x >> 5) * gridDim.x;
  for (int part = 0; part < n_parts; ++part) {
    __syncthreads();   // the previous part's readers are done
    for (int i = threadIdx.x; i < nb * pl; i += blockDim.x) {
      const int f = i / pl, c = i % pl;
      qs[i] = q[static_cast<size_t>(flagged[f_begin + f]) * d + static_cast<size_t>(part) * pl + c];
    }
    __syncthreads();
    for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < ng; row += warps) {
      if constexpr (kCross) {
        const float* gr = g + static_cast<size_t>(row) * d;
        for (int f = 0; f < nb; ++f) {
          double s = part == 0 ? -INFINITY : scores[static_cast<size_t>(f) * ng + row];
          for (int b = 0; b < n_parts; ++b) {
            double v;
            exact_dot<1>(qs + f * pl, gr + static_cast<size_t>(b) * pl, nullptr, pl, lane, v, v);
            s = fmax(s, v);
          }
          if (lane == 0) scores[static_cast<size_t>(f) * ng + row] = s;
        }
      } else {
        const float* gr = g + static_cast<size_t>(row) * d + static_cast<size_t>(part) * pl;
        for (int f = 0; f < nb; ++f) {
          double v;
          exact_dot<1>(qs + f * pl, gr, nullptr, pl, lane, v, v);
          if (lane == 0) {
            double& s = scores[static_cast<size_t>(f) * ng + row];
            s = fmax(part == 0 ? -INFINITY : s, v);
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256)
    exact_select_kernel(double* __restrict__ scores, int ng, int k, const int* __restrict__ flagged, int f_begin,
                        const int* __restrict__ n_flagged, long long g_index_base, long long g_index_stride,
                        float* __restrict__ out_scores, long long* __restrict__ out_idx) {
  const int f = blockIdx.x;
  if (f_begin + f >= *n_flagged) return;
  const int qrow = flagged[f_begin + f];
  double* s = scores + static_cast<size_t>(f) * ng;
  __shared__ BlockBest<8> s_bb;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int round = 0; round < k; ++round) {
    double bs = -INFINITY;
    long long bi = -1;
    int bp = -1;   // = bi: the position is the gallery row
    for (int c = threadIdx.x; c < ng; c += blockDim.x) {
      const double v = s[c];
      if (!(v != v) && (bp < 0 || v > bs)) {   // NaN skipped; ascending c per thread => first (lowest index) max kept
        bs = v;
        bi = bp = c;
      }
    }
    block_argbest(bs, bi, bp, &s_bb, lane, warp);
    if (threadIdx.x == 0) {
      if (bp < 0) {   // every remaining score is NaN (NaN query row, or k > number of non-NaN scores)
        out_scores[static_cast<size_t>(qrow) * k + round] = __int_as_float(0x7fc00000);
        out_idx[static_cast<size_t>(qrow) * k + round] = -1;
      } else {
        out_scores[static_cast<size_t>(qrow) * k + round] = static_cast<float>(bs);
        out_idx[static_cast<size_t>(qrow) * k + round] = g_index_base + g_index_stride * bi;
        s[bp] = __longlong_as_double(0x7ff8000000000000LL);  // NaN marks "taken"
      }
    }
    __syncthreads();
  }
}

// launch geometry of one fused pass over nq queries
struct PassPlan {
  int nq, nq_pad, n_qtiles, n_units, n_slots, kp, cap, stages, max_cand;
  int n_sets;             // epilogue warp sets = candidate slots per segment (column halves with their own lists)
  int gchunk, n_chunks;   // gallery tiles per L2-sized chunk for this pass
  size_t smem_bytes;
};

struct SimPlan : SweepGeometry {
  int n_parts;   // split score: descriptor parts (plan_split_geometry); 0 = dot product
  bool cross;    // the cross split score (n_parts >= 2)
  int max_sets;  // upper bound for PassPlan::n_sets (1 or 2)
  int kp0, kp1;           // candidates kept by the first pass / by the second-chance pass (0 = no second pass)
  PassPlan p0, p1;        // p1 is sized for the worst case (every query flagged)
  size_t total;           // workspace bytes
};

int plan_pass(int nq, int kp, const SimPlan& sp, int num_sms, size_t max_smem, int d, int k, PassPlan* pp) {
  pp->nq = nq;
  pp->n_qtiles = (nq + sp.rows_per_qtile - 1) / sp.rows_per_qtile;
  pp->nq_pad = pp->n_qtiles * sp.rows_per_qtile;
  pp->kp = kp;
  // ---- shared memory: the pipeline with n_sets x cap KB of lists, then carried thresholds (4 KB, whatever n_sets) and
  // the accumulator transposes of 4 n_sets warps ----
  auto smem = [&](int st, int cp, int sets) {
    return FusedPipe::smem_bytes(sp.num_kb, sp.stream_a, st, static_cast<size_t>(sets) * cp * 128 * 8,
                                 4096 + static_cast<size_t>(sets) * 4 * kAccXposeWarpBytes);
  };
  auto fits = [&](int st, int cp, int sets) { return max_smem >= smem(st, cp, sets); };
  // two epilogue warp sets whenever their lists (at least kp + 8 entries per row and set) fit next to 3 B stages
  int sets = (sp.max_sets >= 2 && fits(3, kp + 8, 2)) ? 2 : 1;
  DCR_REQUIRE(!sp.n_parts || sets == 2, "sim_topk_split: not enough shared memory (%zu B) for two column halves", max_smem);
  int cap = kp + (sets == 2 ? 8 : 16);
  if (!fits(2, cap, sets)) cap = kp + 8;   // d = 512 with k > 10: the resident query tile leaves room for 8 spare entries
  const int cap_max = std::max(cap, 64);
  int stages = 2;
  DCR_REQUIRE(fits(stages, cap, sets), "sim_topk: not enough shared memory (%zu B) for d=%d k=%d", max_smem, d, k);
  // priorities: 3 B stages, then list capacity up to 64 (fewer compactions), then more stages (up to 8)
  if (fits(3, cap, sets)) stages = 3;
  while (cap < cap_max && fits(stages, cap + 1, sets)) ++cap;
  while (stages < 8 && fits(stages + 1, cap, sets)) ++stages;
  pp->cap = cap;
  pp->stages = stages;
  pp->n_sets = sets;
  pp->smem_bytes = smem(stages, cap, sets);

  // ---- gallery chunking and work units ----
  pp->gchunk = sp.gchunk;
  pp->n_chunks = sp.n_chunks;
  int units = 1;
  long long span_total = 0;
  for (;;) {
    const long long T = static_cast<long long>(pp->n_qtiles) * pp->gchunk;   // tiles of one (full) gallery chunk
    units = num_sms;
    if (T < units) units = static_cast<int>(std::max<long long>(1, T));
    // per chunk a q-tile is covered by at most ceil(tiles_in_chunk / (T_c / units)) + 1 units
    span_total = 0;
    for (int c = 0; c < pp->n_chunks; ++c) {
      const int ncg = std::min(pp->gchunk, sp.n_gtiles - c * pp->gchunk);
      const long long Tc = static_cast<long long>(pp->n_qtiles) * ncg;
      const long long per_unit = std::max<long long>(1, Tc / units);
      long long span = (ncg + per_unit - 1) / per_unit + 1;
      if (span > units) span = units;
      span_total += span * sets;
    }
    // the re-score kernel keeps every candidate of a query in shared memory (20 B each): few queries spread over all
    // units and many chunks would not fit -> use fewer chunks for such a pass
    if (pp->n_chunks == 1 || (span_total <= kMaxSlotsPerQuery && span_total * kp * 20 <= 150 * 1024)) break;
    pp->n_chunks = (pp->n_chunks + 1) / 2;
    pp->gchunk = (sp.n_gtiles + pp->n_chunks - 1) / pp->n_chunks;
    pp->n_chunks = (sp.n_gtiles + pp->gchunk - 1) / pp->gchunk;
  }
  pp->n_units = units;
  pp->n_slots = pp->n_chunks * (units + pp->n_qtiles) * sets;
  DCR_REQUIRE(span_total <= kMaxSlotsPerQuery, "sim_topk: %lld candidate slots per query tile (max %d)", span_total,
              kMaxSlotsPerQuery);
  pp->max_cand = static_cast<int>(span_total) * kp;
  return 0;
}

struct PassBuffers {
  uint2* cand;
  int* ccnt;
  float* cthr;
};

// The top-k search's workspace: the operands, the second pass's compacted queries, the candidate slots (sized for the
// larger pass), the flagged queries and the brute-force scores
struct TopkBuffers {
  Operands ops;   // ops.qflag is counts + 2
  __nv_bfloat16* qb1;
  PassBuffers pb;
  int *flag0, *flag1;
  float* thr1;
  int* counts;   // [0] flagged by pass 0, [1] flagged by pass 1, [2] the query-centring flag
  unsigned long long* clk;
  unsigned int* gthr;
  double* exact;
};

TopkBuffers carve_topk(const SimPlan& pl, int nq, int ng, int d, Carve& w) {
  TopkBuffers b;
  b.ops = pl.n_parts ? carve_split_operands(w, pl.p0.nq_pad, pl, pl.n_parts) : carve_operands(w, pl.p0.nq_pad, pl, d);
  b.qb1 = w.take<__nv_bfloat16>(pl.kp1 ? static_cast<size_t>(pl.p1.nq_pad) * pl.d_pad : 0);
  const size_t slot_rows = static_cast<size_t>(std::max(pl.p0.n_slots, pl.kp1 ? pl.p1.n_slots : 0)) * pl.rows_per_qtile;   // n_slots counts sets
  b.pb.cand = w.take<uint2>(slot_rows * kKPMax);
  b.pb.ccnt = w.take<int>(slot_rows);
  b.pb.cthr = w.take<float>(slot_rows);
  b.flag0 = w.take<int>(nq);
  b.flag1 = w.take<int>(nq);
  b.thr1 = w.take<float>(nq);
  b.counts = w.take<int>(4);
  b.clk = w.take<unsigned long long>(4);
  b.gthr = w.take<unsigned int>(std::max(pl.p0.nq_pad, pl.kp1 ? pl.p1.nq_pad : 0));
  b.exact = w.take<double>(static_cast<size_t>(kExactBatch) * ng);
  return b;
}

// n_parts = 0: the dot product; >= 1: the split score over n_parts parts (sim_topk_split; cross: sim_topk_cross)
const char* topk_name(int n_parts, bool cross) { return n_parts ? (cross ? "sim_topk_cross" : "sim_topk_split") : "sim_topk"; }

int make_plan(int nq, int ng, int d, int k, int n_parts, bool cross, int num_sms, size_t max_smem, SimPlan* pl) {
  const char* who = topk_name(n_parts, cross);
  DCR_REQUIRE(nq >= 1 && ng >= 1 && d >= 1, "%s: empty problem (nq=%d ng=%d d=%d)", who, nq, ng, d);
  if (n_parts) {
    DCR_REQUIRE(n_parts >= 1 && d % n_parts == 0 && (d / n_parts) % 4 == 0,
                "%s: d=%d must split into %d parts whose length is a multiple of 4", who, d, n_parts);
    const int p = d / n_parts;
    DCR_REQUIRE(p <= kMaxDim, "%s: part length %d > %d not supported", who, p, kMaxDim);
    DCR_REQUIRE(static_cast<long long>(n_parts) * ((p + kBlockK - 1) / kBlockK * kBlockK) <= (1ll << 30),
                "%s: %d parts of %d padded to 64 exceed 2^30 columns", who, n_parts, p);
  } else {
    DCR_REQUIRE(d <= kMaxDim, "sim_topk: descriptor dim %d > %d not supported", d, kMaxDim);
  }
  DCR_REQUIRE(k >= 1 && k <= 16, "%s: k=%d outside [1,16]", who, k);
  DCR_REQUIRE(k <= ng, "%s: k=%d > gallery size %d", who, k, ng);
  pl->n_parts = n_parts;
  pl->cross = n_parts && cross;
  if (n_parts) plan_split_geometry(ng, n_parts, d / n_parts, pl);
  else plan_geometry(ng, d, pl);
  // Two consumer warpgroups (two warps per 32-row block, each with its own lists for one column half) when few
  // candidates are kept (k <= 2: each segment keeps 2 x 4 candidates); with larger k the lists of two sets only fit with
  // a small capacity.  The split score always runs on column halves: the running maximum of a 128-column tile next to its
  // part accumulator would not fit a thread's registers.
  pl->max_sets = (k <= 2 || n_parts) ? 2 : 1;
  // first pass keeps few candidates per (query, segment) -- enough unless many gallery rows sit within the error
  // bound of the k-th score; such queries get a second chance with 32 candidates before the brute-force path
  // k in 6..10 keeps 12 (two spare candidates per segment keep the second-chance pass rare)
  const int kp0 = (k <= 2) ? 4 : (k <= 5 ? 8 : (k <= 10 ? 12 : 32));   // k <= kp0 <= kKPMax for every k <= 16
  pl->kp0 = kp0;
  pl->kp1 = (kp0 < kKPMax) ? kKPMax : 0;
  if (int rc = plan_pass(nq, pl->kp0, *pl, num_sms, max_smem, d, k, &pl->p0)) return rc;
  if (pl->kp1) {
    if (plan_pass(nq, pl->kp1, *pl, num_sms, max_smem, d, k, &pl->p1) != 0) pl->kp1 = 0;   // does not fit: skip
  }
  Carve size;
  carve_topk(*pl, nq, ng, d, size);
  pl->total = size.bytes;
  return 0;
}

// one fused pass: qb (bf16, padded) x gb (bf16, centred, padded) -> candidate slots
int launch_fused(const SimPlan& pl, const PassPlan& pp, const __nv_bfloat16* qb, const __nv_bfloat16* gb, int ng,
                 const PassBuffers& pb, const float* col_bias, const int* bias_flag, const float* thr_init,
                 unsigned long long* clk, unsigned int* gthr, cudaStream_t stream) {
  CUtensorMap tq, tg;
  SimParams p;
  if (int rc = sweep_setup(pl, pp.nq, pp.n_qtiles, ng, pp.gchunk, pp.n_chunks, qb, gb, &p, &tq, &tg)) return rc;
  p.kp = pp.kp;
  p.cap = pp.cap;
  p.stages = pp.stages;
  p.cand = pb.cand;
  p.cand_cnt = pb.ccnt;
  p.cand_thr = pb.cthr;
  p.col_bias = col_bias;
  p.bias_flag = bias_flag;
  p.thr_init = thr_init;
  p.clk = clk;
  p.gthr = gthr;
  p.kb_part = pl.n_parts ? pl.num_kb / pl.n_parts : 0;
  DCR_CUDA_CHECK(cudaMemsetAsync(gthr, 0, static_cast<size_t>(pp.nq_pad) * 4, stream));
  if (pl.cross)
    return launch(sim_topk_kernel<false, 2, true, true>, pp.n_units, 32 + 128 * 2, pp.smem_bytes, stream, "sim_topk_cross", tq,
                  tg, p);
  if (pl.n_parts)
    return launch(sim_topk_kernel<false, 2, true>, pp.n_units, 32 + 128 * 2, pp.smem_bytes, stream, "sim_topk_split", tq, tg, p);
  const bool two = pp.n_sets == 2;
  return launch_sweep(two ? sim_topk_kernel<false, 2> : sim_topk_kernel<false, 1>,
                      two ? sim_topk_kernel<true, 2> : sim_topk_kernel<true, 1>, pp.n_units, 32 + 128 * pp.n_sets,
                      pp.smem_bytes, stream, "sim_topk", tq, tg, p);
}

// The whole search: stage 1, the fused pass, the exact re-score, the second-chance pass and the brute-force path.
// n_parts = 0: the dot product (sim_topk); >= 1: the split score over n_parts parts (sim_topk_split; cross: sim_topk_cross).
int topk_search(const float* q, int nq, const float* g, int ng, int d, int n_parts, bool cross, int k,
                long long g_index_base, long long g_index_stride, float* out_scores, long long* out_idx, void* ws,
                size_t ws_bytes, cudaStream_t stream, SimStats* stats) {
  const char* who = topk_name(n_parts, cross);
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  if (int rc = require_sm90a(di, who)) return rc;
  SimPlan pl;
  if (int rc = make_plan(nq, ng, d, k, n_parts, cross, di->num_sms, di->max_smem_optin, &pl)) return rc;
  DCR_REQUIRE(ws != nullptr && ws_bytes >= pl.total, "%s: workspace too small (%zu < %zu)", who, ws_bytes, pl.total);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "%s: workspace must be 256-byte aligned", who);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0 && d % 4 == 0,
              "%s: q/g must be 16-byte aligned with d %% 4 == 0 (d=%d)", who, d);
  Carve w{static_cast<uint8_t*>(ws)};
  TopkBuffers b = carve_topk(pl, nq, ng, d, w);
  DCR_CUDA_CHECK(cudaMemsetAsync(b.counts, 0, 16, stream));
  const int pl_len = n_parts ? d / n_parts : d;   // the length of one exact dot product (a part, or the whole row)
  if (n_parts) {
    if (int rc = prepare_split_operands(q, nq, pl.p0.nq_pad, g, ng, n_parts, pl_len, pl, di, b.ops, stream)) return rc;
  } else {
    b.ops.qflag = b.counts + 2;
    if (int rc = prepare_operands(q, nq, pl.p0.nq_pad, g, ng, d, pl, di, b.ops, stream)) return rc;
  }
  const Operands& o = b.ops;

  // CUDA events around the first fused pass only (thread-local, created once): bench.py's roofline numerator
  // (events belong to the device that was current when they were created: one pair per device)
  static thread_local cudaEvent_t ev_tab[64][2] = {};
  cudaEvent_t& ev0 = ev_tab[di->device][0];
  cudaEvent_t& ev1 = ev_tab[di->device][1];
  if (!ev0) {
    DCR_CUDA_CHECK(cudaEventCreate(&ev0));
    DCR_CUDA_CHECK(cudaEventCreate(&ev1));
  }
  DCR_CUDA_CHECK(cudaEventRecord(ev0, stream));
  if (int rc = launch_fused(pl, pl.p0, o.qb, o.gb, ng, b.pb, o.bias, o.qflag, nullptr, b.clk, b.gthr, stream)) return rc;
  DCR_CUDA_CHECK(cudaEventRecord(ev1, stream));

  auto rescore = [&](const PassPlan& pp, const int* qmap, int* flagged, int* n_flagged, float* thr_next) -> int {
    RescoreParams rp;
    rp.q = q, rp.g = g, rp.nq = pp.nq, rp.d = d, rp.d_pad = pl.d_pad, rp.k = k;
    rp.n_qtiles = pp.n_qtiles, rp.n_gtiles = pl.n_gtiles, rp.gchunk = pp.gchunk, rp.n_chunks = pp.n_chunks;
    rp.n_units = pp.n_units, rp.n_sets = pp.n_sets, rp.max_cand = pp.max_cand;
    rp.cand = b.pb.cand, rp.cand_cnt = b.pb.ccnt, rp.cand_thr = b.pb.cthr, rp.qmap = qmap;
    rp.mu = o.mu, rp.nu = o.nu, rp.nu_flag = o.qflag;
    rp.q_norm_hat = o.qnh, rp.q_norm_res = o.qnr, rp.q_norm_x = o.qnx, rp.g_max = o.gmax;
    rp.g_index_base = g_index_base, rp.g_index_stride = g_index_stride, rp.out_scores = out_scores, rp.out_idx = out_idx;
    rp.flagged = flagged, rp.n_flagged = n_flagged, rp.thr_next = thr_next, rp.n_parts = n_parts;
    rp.staged = pl.cross ? cross_staged_parts(n_parts, pl_len) : 0;
    // one warp per query when a q-tile's candidate slots fit a lane each and four queries' rows fit a block's shared memory
    // (the block-wide form spends its time on barriers for such small candidate sets).  The cross score always takes the
    // block form: each survivor costs n_parts^2 part dot products, which four warps share.
    const size_t per_query =
        RescoreSmem(pl.cross ? static_cast<int>(cross_stage_doubles(rp.staged, pl_len, kRescoreThreads / 32)) : pl_len,
                    pp.max_cand).bytes;
    const bool warp_form = !pl.cross && pp.kp > 0 && pp.max_cand / pp.kp <= 32 && pp.n_chunks <= 32 &&
                           4 * per_query <= 56 * 1024 && !tuning_flag("DCR_SIM_RESCORE_BLOCK");
    const int per_block = warp_form ? kRescoreThreads / 32 : 1;
    const size_t smem = per_block * per_query;
    auto kern = pl.cross ? rescore_select_kernel<kRescoreThreads, true, true>
                : n_parts ? (warp_form ? rescore_select_kernel<32, true> : rescore_select_kernel<kRescoreThreads, true>)
                          : (warp_form ? rescore_select_kernel<32> : rescore_select_kernel<kRescoreThreads>);
    return launch(kern, (pp.nq + per_block - 1) / per_block, kRescoreThreads, smem, stream, who, rp);
  };
  if (int rc = rescore(pl.p0, nullptr, b.flag0, b.counts + 0, b.thr1)) return rc;

  int h_counts[2] = {0, 0};
  unsigned long long h_clk[4] = {0, 0, 0, 0};
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_counts, b.counts, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_clk, b.clk, 32, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  int n_second = 0;
  const int* exact_list = b.flag0;
  int n_exact = h_counts[0];
  if (h_counts[0] > 0 && pl.kp1) {
    // second chance: the flagged queries alone, 32 candidates per (query, segment)
    n_second = h_counts[0];
    PassPlan p1;
    if (int rc = plan_pass(n_second, pl.kp1, pl, di->num_sms, di->max_smem_optin, d, k, &p1)) return rc;
    if (int rc = launch(gather_rows_kernel, std::min(di->num_sms * 8, (p1.nq_pad * (pl.d_pad / 8) + 255) / 256), 256, 0,
                        stream, who, o.qb, b.flag0, n_second, p1.nq_pad, pl.d_pad, b.qb1))
      return rc;
    if (int rc = launch_fused(pl, p1, b.qb1, o.gb, ng, b.pb, o.bias, o.qflag, b.thr1, nullptr, b.gthr, stream)) return rc;
    if (int rc = rescore(p1, b.flag0, b.flag1, b.counts + 1, nullptr)) return rc;
    DCR_CUDA_CHECK(cudaMemcpyAsync(h_counts, b.counts, 8, cudaMemcpyDeviceToHost, stream));
    DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
    exact_list = b.flag1;
    n_exact = h_counts[1];
  }

  // brute-force fp64 path for the queries whose certificate still fails (ties beyond 32 candidates, NaNs, ...)
  if (n_exact > 0) {
    // queries per brute-force launch: as many as fit in shared memory next to each other (32 up to d = 1536; under the
    // split score the rows are staged one part at a time)
    const int ex_batch = std::max(1, std::min<int>(kExactBatch, static_cast<int>(192 * 1024 / (static_cast<size_t>(pl_len) * 4))));
    const size_t ex_smem = static_cast<size_t>(ex_batch) * pl_len * 4;
    const int* n_dev = (exact_list == b.flag0) ? b.counts + 0 : b.counts + 1;
    for (int done = 0; done < n_exact; done += ex_batch) {
      const int rc = n_parts ? launch(pl.cross ? split_scan_kernel<true> : split_scan_kernel<false>, di->num_sms * 2, 256,
                                      ex_smem, stream, who, q, g, ng, d, n_parts, exact_list, done, n_dev, b.exact, ex_batch)
                             : launch(exact_scan_kernel, di->num_sms * 2, 256, ex_smem, stream, who, q, g, ng, d, exact_list,
                                      done, n_dev, b.exact, ex_batch);
      if (rc) return rc;
      if (int rc = launch(exact_select_kernel, ex_batch, 256, 0, stream, who, b.exact, ng, k, exact_list, done, n_dev,
                          g_index_base, g_index_stride, out_scores, out_idx))
        return rc;
    }
    DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  }

  if (stats) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ev0, ev1) != cudaSuccess) ms = 0.f;
    stats->kernel_ms = ms;
    stats->sm_mhz = (h_clk[3] > h_clk[1]) ? static_cast<float>(static_cast<double>(h_clk[2] - h_clk[0]) * 1e3 /
                                                               static_cast<double>(h_clk[3] - h_clk[1]))
                                          : 0.f;
    stats->n_sets = pl.p0.n_sets;
    stats->cta_group = 1;   // one CTA per work unit (the field stays for callers that read it)
    stats->grid = pl.p0.n_units;
    stats->smem_bytes = static_cast<int>(pl.p0.smem_bytes);
    stats->stages = pl.p0.stages;
    stats->kp = pl.p0.kp;
    stats->cap = pl.p0.cap;
    stats->n_flagged = n_exact;
    stats->n_second = n_second;
    stats->d_pad = pl.d_pad;
  }
  return 0;
}

}  // namespace

int split_rescore(const float* q, const float* g, int nq, int d, int n_chunks, int cross, const long long* cand, int n_cand,
                  int k, float* out_scores, long long* out_idx, cudaStream_t stream) {
  DCR_REQUIRE(nq >= 1 && d >= 1 && n_chunks >= 1 && d % n_chunks == 0 && (d / n_chunks) % 4 == 0,
              "split_rescore: d=%d must split into %d parts whose length is a multiple of 4", d, n_chunks);
  DCR_REQUIRE(n_cand >= k && k >= 1 && n_cand <= 4096, "split_rescore: need k <= n_cand <= 4096 (k=%d n_cand=%d)", k, n_cand);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0,
              "split_rescore: q/g must be 16-byte aligned");
  const size_t smem = ((static_cast<size_t>(d / n_chunks) * 4 + 15) & ~size_t(15)) + static_cast<size_t>(n_cand) * 16;
  return launch(split_rescore_kernel, nq, 128, smem, stream, "split_rescore", q, g, d, n_chunks, cross, cand, n_cand, k,
                out_scores, out_idx);
}

namespace {
size_t workspace_size(int nq, int ng, int d, int n_parts, bool cross, int k) {
  const DeviceInfo* di = device_info();
  SimPlan pl;
  if (make_plan(nq, ng, d, k, n_parts, cross, di ? di->num_sms : 132, di ? di->max_smem_optin : 232448, &pl) != 0)
    return 0;
  return pl.total;
}
}  // namespace

size_t sim_topk_workspace_size(int nq, int ng, int d, int k) { return workspace_size(nq, ng, d, 0, false, k); }

int sim_topk(const float* q, int nq, const float* g, int ng, int d, int k, long long g_index_base,
             long long g_index_stride, float* out_scores, long long* out_idx, void* ws, size_t ws_bytes,
             cudaStream_t stream, SimStats* stats) {
  return topk_search(q, nq, g, ng, d, 0, false, k, g_index_base, g_index_stride, out_scores, out_idx, ws, ws_bytes, stream, stats);
}

// one part is the dot product itself: the dot-product search, whose bits the split score must reproduce
size_t sim_topk_split_workspace_size(int nq, int ng, int d, int n_parts, int k, bool cross) {
  if (n_parts == 1) return workspace_size(nq, ng, d, 0, false, k);
  if (n_parts < 1) {
    set_error(-1, "%s: n_parts=%d < 1", topk_name(1, cross), n_parts);
    return 0;
  }
  return workspace_size(nq, ng, d, n_parts, cross, k);
}

int sim_topk_split(const float* q, int nq, const float* g, int ng, int d, int n_parts, int k, long long g_index_base,
                   long long g_index_stride, float* out_scores, long long* out_idx, void* ws, size_t ws_bytes,
                   cudaStream_t stream, SimStats* stats, bool cross) {
  DCR_REQUIRE(n_parts >= 1, "%s: n_parts=%d < 1", topk_name(1, cross), n_parts);
  return topk_search(q, nq, g, ng, d, n_parts == 1 ? 0 : n_parts, cross, k, g_index_base, g_index_stride, out_scores,
                     out_idx, ws, ws_bytes, stream, stats);
}

}  // namespace dcr
