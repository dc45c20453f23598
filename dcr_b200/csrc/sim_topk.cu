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
//
// The same stages 1 and 2 also serve the threshold search (sim_range: every pair scoring at least tau, exact, in CSR
// form; it replaces the saved score matrices of diff_retrieval.py:402-403, 414-415 and the threshold of :454): the
// fused sweep's epilogue then compares each approximate score against a per-row threshold that no qualifying pair can
// fall below, and the candidates are re-scored with the same fp64 dot products.
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <type_traits>

#include "../../include/dcr_b200.h"
#include "dcr_internal.cuh"
#include "host_util.cuh"
#include "ptx.cuh"

namespace dcr {

namespace {

constexpr int kBlockM = 128;      // query rows per CTA
constexpr int kBlockN = 128;      // gallery rows per tile (accumulator columns: 128 registers per thread with one warpgroup)
constexpr int kBlockK = 64;       // bf16 elements per 128-byte swizzled smem row
constexpr int kMaxKB = 8;         // d_pad <= 512: the query tile stays resident in shared memory; larger: streamed
constexpr int kMaxDim = 8192;     // largest descriptor dimension accepted
constexpr int kKPMax = 32;        // max candidates kept per (query, segment)
constexpr int kWarmTiles = 4;     // tiles replayed at the start of every segment to seed the threshold
constexpr uint32_t kFull = 0xffffffffu;
constexpr int kATileBytes = kBlockM * kBlockK * 2;  // 16 KB
constexpr int kBTileBytes = kBlockN * kBlockK * 2;  // 16 KB
constexpr int kMaxSlotsPerQuery = 512;  // (chunk, unit) segments that may cover one q-tile

struct SimParams {
  int nq, ng;
  int num_kb;          // d_pad / 64
  int stream_a;        // 1 (d_pad > 512): query k-blocks travel with the gallery k-blocks instead of staying resident
  int n_qtiles;        // ceil(nq / 128)
  int n_gtiles;        // ceil(ng / 128)
  int gchunk;          // gallery tiles per L2-sized chunk (all units sweep chunk c before chunk c+1)
  int n_chunks;
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
};

// ------------------------------------------------------------------------------------------------------------
// stage 1: fp32 rows -> bf16 rows (zero padded to [n_pad, d_pad]) + norms needed by the error bound
//   norms[0][r] = ||bf16(x_r)||, norms[1][r] = ||x_r - bf16(x_r)||, gmax[0] = max_r ||x_r||, gmax[1] = max_r residual
// mu (optional): a vector subtracted from every row before rounding (gallery centring: q.g = q.(g-mu) + q.mu and the
// second term does not depend on g, so the ranking is unchanged while the bf16 rounding error now scales with the
// SPREAD of the gallery instead of its norm).
template <int kIter>
__global__ void __launch_bounds__(256) to_bf16_rows_kernel(const float* __restrict__ x, int n, int d, int n_pad, int d_pad,
                                    const float* __restrict__ mu, __nv_bfloat16* __restrict__ out,
                                    float* __restrict__ norm_hat, float* __restrict__ norm_res,
                                    float* __restrict__ norm_x, unsigned int* __restrict__ gmax,
                                    const float* __restrict__ nu, float* __restrict__ bias_out,
                                    const int* __restrict__ mu_flag, const int* __restrict__ nu_flag) {
  if (mu_flag && *mu_flag == 0) mu = nullptr;   // device-side decision (centre_decision_kernel)
  if (nu_flag && *nu_flag == 0) nu = nullptr;
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  // gmax: one global atomic per BLOCK (100k same-address atomics, one per row, serialise in L2 and dominated this kernel)
  __shared__ unsigned int s_gmax[2];
  if (threadIdx.x < 2) s_gmax[threadIdx.x] = 0u;
  __syncthreads();
  unsigned int w_nx = 0u, w_nr = 0u;   // this warp's running maxima (lane 0)
  for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < n_pad; row += gridDim.x * warps_per_block) {
    float s_hat = 0.f, s_res = 0.f, s_x = 0.f;
    double s_bias = 0.0;   // nu . (x - mu) in fp64: the per-gallery-row score offset of query centring
    __nv_bfloat16* o = out + static_cast<size_t>(row) * d_pad;
    if (row < n) {
      const float* xr = x + static_cast<size_t>(row) * d;
      // kIter float4 loads per lane issued back to back (the row's whole HBM read is in flight before the first value
      // is used: the kernel is a pure stream, 12 B/element read+written, and was latency bound with one load at a time)
      for (int c0 = 0; c0 < d_pad; c0 += 128 * kIter) {
        float4 v[kIter];
#pragma unroll
        for (int i = 0; i < kIter; ++i) {
          const int c = c0 + i * 128 + lane * 4;
          v[i] = (c + 3 < d) ? *reinterpret_cast<const float4*>(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);   // d % 4 == 0
        }
#pragma unroll
        for (int i = 0; i < kIter; ++i) {
          const int c = c0 + i * 128 + lane * 4;
          if (c >= d_pad) continue;
          if (c + 3 < d) {
            if (mu) {
              const float4 m = *reinterpret_cast<const float4*>(mu + c);
              v[i].x -= m.x; v[i].y -= m.y; v[i].z -= m.z; v[i].w -= m.w;
            }
            if (nu) {
              const float4 u = *reinterpret_cast<const float4*>(nu + c);
              s_bias = fma(static_cast<double>(u.x), static_cast<double>(v[i].x), s_bias);
              s_bias = fma(static_cast<double>(u.y), static_cast<double>(v[i].y), s_bias);
              s_bias = fma(static_cast<double>(u.z), static_cast<double>(v[i].z), s_bias);
              s_bias = fma(static_cast<double>(u.w), static_cast<double>(v[i].w), s_bias);
            }
          }
          const __nv_bfloat16 h0 = __float2bfloat16_rn(v[i].x), h1 = __float2bfloat16_rn(v[i].y);
          const __nv_bfloat16 h2 = __float2bfloat16_rn(v[i].z), h3 = __float2bfloat16_rn(v[i].w);
          const float f0 = __bfloat162float(h0), f1 = __bfloat162float(h1), f2 = __bfloat162float(h2), f3 = __bfloat162float(h3);
          s_hat += f0 * f0 + f1 * f1 + f2 * f2 + f3 * f3;
          s_res += (v[i].x - f0) * (v[i].x - f0) + (v[i].y - f1) * (v[i].y - f1) + (v[i].z - f2) * (v[i].z - f2) + (v[i].w - f3) * (v[i].w - f3);
          s_x += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
          uint2 pk;
          pk.x = static_cast<uint32_t>(__bfloat16_as_ushort(h0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h1)) << 16);
          pk.y = static_cast<uint32_t>(__bfloat16_as_ushort(h2)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h3)) << 16);
          *reinterpret_cast<uint2*>(o + c) = pk;
        }
      }
    } else {
      for (int c = lane * 2; c < d_pad; c += 64) *reinterpret_cast<uint32_t*>(o + c) = 0u;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s_hat += __shfl_xor_sync(kFull, s_hat, off);
      s_res += __shfl_xor_sync(kFull, s_res, off);
      s_x += __shfl_xor_sync(kFull, s_x, off);
      s_bias += __shfl_xor_sync(kFull, s_bias, off);
    }
    if (lane == 0 && bias_out) bias_out[row] = (row < n) ? static_cast<float>(s_bias) : 0.f;
    if (lane == 0 && row < n) {
      // 1.0001: cover the fp32 rounding of the squared sums so the stored values are upper bounds
      float nh = sqrtf(s_hat) * 1.0001f, nr = sqrtf(s_res) * 1.0001f, nx = sqrtf(s_x) * 1.0001f;
      if (norm_hat) norm_hat[row] = nh;
      if (norm_res) norm_res[row] = nr;
      if (norm_x) norm_x[row] = nx;
      w_nx = max(w_nx, __float_as_uint(nx));     // non-negative floats order like their bit patterns
      w_nr = max(w_nr, __float_as_uint(nr));
    }
  }
  if (gmax) {
    if (lane == 0) {
      atomicMax(&s_gmax[0], w_nx);
      atomicMax(&s_gmax[1], w_nr);
    }
    __syncthreads();
    if (threadIdx.x < 2) atomicMax(gmax + threadIdx.x, s_gmax[threadIdx.x]);
  }
}

// column sums of x[n, d] accumulated in double; mean = sum / n afterwards (rows r*row_stride, r < n: any fixed vector works
// as the centre, so a strided sample of the gallery is enough).  A thread owns one 16-byte column group and a slice of the
// block's rows (independent loads, four in flight), the slices meet in shared memory and the block does ONE atomicAdd per
// column instead of every block adding all d columns (hundreds of thousands of same-address double atomics).
constexpr int kColSumThreads = 512;
__global__ void __launch_bounds__(kColSumThreads)
    col_sum_kernel(const float* __restrict__ x, int n, int row_stride, int d, double* __restrict__ sums,
                   double* __restrict__ sq_sums) {
  __shared__ double red[kColSumThreads][8];
  const int groups = d >> 2;                                   // d % 4 == 0 (checked by the caller)
  const int G = min(groups, kColSumThreads), S = kColSumThreads / G;
  const int tg = threadIdx.x % G, sl = threadIdx.x / G;         // threads with sl >= S idle (G does not divide the block)
  const int rows_per_block = (n + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(n, r0 + rows_per_block);
  for (int cg = tg; cg < groups; cg += G) {
    double da[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) da[e] = 0.0;
    if (sl < S) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f), acc2 = make_float4(0.f, 0.f, 0.f, 0.f);
      int cnt = 0;
#pragma unroll 4
      for (int r = r0 + sl; r < r1; r += S) {
        const float4 v = *reinterpret_cast<const float4*>(x + static_cast<size_t>(r) * row_stride * d + cg * 4);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        acc2.x += v.x * v.x; acc2.y += v.y * v.y; acc2.z += v.z * v.z; acc2.w += v.w * v.w;
        if (++cnt == 256) {   // flush the fp32 partials into the double accumulators every 256 rows
          da[0] += acc.x; da[1] += acc.y; da[2] += acc.z; da[3] += acc.w;
          da[4] += acc2.x; da[5] += acc2.y; da[6] += acc2.z; da[7] += acc2.w;
          acc = make_float4(0.f, 0.f, 0.f, 0.f);
          acc2 = make_float4(0.f, 0.f, 0.f, 0.f);
          cnt = 0;
        }
      }
      da[0] += acc.x; da[1] += acc.y; da[2] += acc.z; da[3] += acc.w;
      da[4] += acc2.x; da[5] += acc2.y; da[6] += acc2.z; da[7] += acc2.w;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) red[threadIdx.x][e] = da[e];
    __syncthreads();
    if (sl == 0 && r1 > r0) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        double t = 0.0;
        for (int s2 = 0; s2 < S; ++s2) t += red[s2 * G + tg][e];   // fixed order within the block
        if (e < 4) atomicAdd(sums + cg * 4 + e, t);
        else if (sq_sums) atomicAdd(sq_sums + cg * 4 + (e - 4), t);
      }
    }
    __syncthreads();
  }
}
__global__ void col_mean_finish_kernel(const double* __restrict__ sums, int n, int d, float* __restrict__ mu) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < d) mu[c] = static_cast<float>(sums[c] / n);
}
// Query centring pays only when the centred queries are much shorter than the queries themselves (the bf16 error
// bound shrinks by ||q-nu|| / ||q||) -- and costs a per-column offset in the fused epilogue.  flag = 1 when the
// mean squared norm of the centred sample is below 1/16 of the uncentred one (a 4x tighter bound).
__global__ void __launch_bounds__(256)
    centre_decision_kernel(const double* __restrict__ sums, const double* __restrict__ sq_sums, int n, int d,
                           int* __restrict__ flag) {
  __shared__ double s_m2[8], s_nu2[8];
  double m2 = 0.0, nu2 = 0.0;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    m2 += sq_sums[c] / n;
    const double m = sums[c] / n;
    nu2 += m * m;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    m2 += __shfl_xor_sync(kFull, m2, off);
    nu2 += __shfl_xor_sync(kFull, nu2, off);
  }
  if ((threadIdx.x & 31) == 0) {
    s_m2[threadIdx.x >> 5] = m2;
    s_nu2[threadIdx.x >> 5] = nu2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    m2 = nu2 = 0.0;
    for (int w = 0; w < 8; ++w) {
      m2 += s_m2[w];
      nu2 += s_nu2[w];
    }
    *flag = (m2 - nu2 < m2 / 16.0) ? 1 : 0;
  }
}

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

// Shared-memory pipeline of a fused sweep (sim_topk_kernel, sim_range_kernel):
//   resident mode: [num_kb x 16 KB query tile][stages x gallery tile]; streamed mode (d_pad > 512, the query tile no
//   longer fits): [stages x (gallery tile | 16 KB query k-block)] -- twice the L2->SMEM traffic per FLOP
// followed by `list_bytes` of the caller's own, the barriers, and whatever the caller puts after them (`tail`).
struct FusedPipe {
  bool stream_a;
  int num_kb, stage_bytes;
  uint8_t* smem_a;     // num_kb x 16 KB (resident mode)
  uint8_t* smem_b;     // stages x stage_bytes
  uint8_t* lists;
  uint64_t *b_full, *b_empty, *a_full, *a_empty;
  uint8_t* tail;
  DCR_DEVICE FusedPipe(uint8_t* smem_raw, int nkb, int stream, int stages, size_t list_bytes) {
    // all tile bases 1024-byte aligned for the 128B swizzle
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    stream_a = stream != 0;
    num_kb = nkb;
    stage_bytes = kBlockN * kBlockK * 2 + (stream_a ? kATileBytes : 0);
    smem_a = smem;
    smem_b = smem_a + (stream_a ? 0 : num_kb * kATileBytes);
    lists = smem_b + stages * stage_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(lists + list_bytes);
    b_full = bars;          // [stages]
    b_empty = bars + 8;     // [stages]
    a_full = bars + 16;
    a_empty = bars + 17;
    tail = reinterpret_cast<uint8_t*>(bars + 32);
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
template <class WarmOf>
DCR_DEVICE void fused_producer(const FusedPipe& pp, const CUtensorMap* tq, const CUtensorMap* tg, int stages, SegWalker& w,
                               WarmOf warm_of) {
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
      for (int kb = 0; kb < pp.num_kb; ++kb, st.next()) {
        const uint32_t s = st.s, ph = st.ph;
        mbar_wait(&pp.b_empty[s], ph ^ 1);
        if (elect_one()) {
          mbar_arrive_expect_tx(&pp.b_full[s], pp.stage_bytes);
          tma_load_2d(pp.smem_b + s * pp.stage_bytes, tg, &pp.b_full[s], kb * kBlockK, g_row, kEvictNormal);
          if (pp.stream_a)
            tma_load_2d(pp.smem_b + s * pp.stage_bytes + kBTileBytes, tq, &pp.b_full[s], kb * kBlockK, q_row, kEvictNormal);
        }
        __syncwarp();
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
template <bool kBias, int kSets>
__global__ void __launch_bounds__(32 + 128 * kSets, 1)
    sim_topk_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_g,
                    const SimParams p) {
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
    fused_producer(pp, &tmap_q, &tmap_g, p.stages, w,
                   [&](const SegWalker& s) { return (p.thr_init || s.carried) ? 0 : min(kWarmTiles, s.ntiles); });
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
        fused_tile_mma(acc, st, pp, a_base, b_base, last, lane);
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

// ------------------------------------------------------------------------------------------------------------
// exact dot product, fp64 accumulate, fixed association: lane l owns elements l*4 + 128*i (float4 granules),
// accumulates them in order, then a fixed xor-butterfly.  Used by both the re-score and the brute-force path so
// that the two produce bit-identical values.
DCR_DEVICE double exact_dot_warp(const float* __restrict__ a_smem, const float* __restrict__ b, int d, uint32_t lane) {
  double acc = 0.0;
  for (int c = lane * 4; c < d; c += 128) {
    if (c + 3 < d) {
      const float4 bv = *reinterpret_cast<const float4*>(b + c);
      acc = fma(static_cast<double>(a_smem[c]), static_cast<double>(bv.x), acc);
      acc = fma(static_cast<double>(a_smem[c + 1]), static_cast<double>(bv.y), acc);
      acc = fma(static_cast<double>(a_smem[c + 2]), static_cast<double>(bv.z), acc);
      acc = fma(static_cast<double>(a_smem[c + 3]), static_cast<double>(bv.w), acc);
    } else {
      for (int e = c; e < d; ++e) acc = fma(static_cast<double>(a_smem[e]), static_cast<double>(b[e]), acc);
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(kFull, acc, off);
  return acc;
}

// Same values, same association as exact_dot_warp with the query row already widened to fp64 in shared memory (the widening
// is exact): the re-score kernel is bound by the fp64 pipe -- per gallery row 512 fma plus 1024 fp32->fp64 conversions --
// and this halves the conversions.
DCR_DEVICE double exact_dot_warp_qd(const double* __restrict__ a_smem, const float* __restrict__ b, int d, uint32_t lane) {
  double acc = 0.0;
  for (int c = lane * 4; c < d; c += 128) {
    if (c + 3 < d) {
      const float4 bv = *reinterpret_cast<const float4*>(b + c);
      const double2 a01 = *reinterpret_cast<const double2*>(a_smem + c);
      const double2 a23 = *reinterpret_cast<const double2*>(a_smem + c + 2);
      acc = fma(a01.x, static_cast<double>(bv.x), acc);
      acc = fma(a01.y, static_cast<double>(bv.y), acc);
      acc = fma(a23.x, static_cast<double>(bv.z), acc);
      acc = fma(a23.y, static_cast<double>(bv.w), acc);
    } else {
      for (int e = c; e < d; ++e) acc = fma(a_smem[e], static_cast<double>(b[e]), acc);
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(kFull, acc, off);
  return acc;
}

// order (score desc, index asc)
DCR_DEVICE bool better(double s, long long i, double bs, long long bi) { return (s > bs) || (s == bs && i < bi); }

// block-wide arg-best over (key desc, index asc) of 128 threads; every thread passes its local best (pos < 0 = none)
struct BlockBest {
  double key[4];
  long long idx[4];
  int pos[4];
};
DCR_DEVICE void block_argbest(double& bs, long long& bi, int& bp, BlockBest* sb, uint32_t lane, uint32_t warp) {
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
  for (int w = 1; w < 4; ++w)
    if (sb->pos[w] >= 0 && (bp < 0 || better(sb->key[w], sb->idx[w], bs, bi))) {
      bs = sb->key[w];
      bi = sb->idx[w];
      bp = sb->pos[w];
    }
  __syncthreads();
}

// two rows, each with exactly the association of exact_dot_warp_qd; both rows' loads are issued before the first fma
DCR_DEVICE void exact_dot_warp_qd2(const double* __restrict__ a_smem, const float* __restrict__ b0,
                                   const float* __restrict__ b1, int d, uint32_t lane, double& out0, double& out1) {
  double acc0 = 0.0, acc1 = 0.0;
  if ((d & 127) == 0 && d <= 512) {
    // every lane owns d/128 whole 16-byte granules of each row: all (up to eight) loads are issued before the first fma --
    // written as a loop, each 128-column step waited for its own two loads (40 serial memory latencies per query)
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
        const double2 a01 = *reinterpret_cast<const double2*>(a_smem + lane * 4 + i * 128);
        const double2 a23 = *reinterpret_cast<const double2*>(a_smem + lane * 4 + i * 128 + 2);
        acc0 = fma(a01.x, static_cast<double>(v0[i].x), acc0);
        acc0 = fma(a01.y, static_cast<double>(v0[i].y), acc0);
        acc0 = fma(a23.x, static_cast<double>(v0[i].z), acc0);
        acc0 = fma(a23.y, static_cast<double>(v0[i].w), acc0);
        acc1 = fma(a01.x, static_cast<double>(v1[i].x), acc1);
        acc1 = fma(a01.y, static_cast<double>(v1[i].y), acc1);
        acc1 = fma(a23.x, static_cast<double>(v1[i].z), acc1);
        acc1 = fma(a23.y, static_cast<double>(v1[i].w), acc1);
      }
    }
  } else {
    for (int c = lane * 4; c < d; c += 128) {
      if (c + 3 < d) {
        const float4 v0 = *reinterpret_cast<const float4*>(b0 + c);
        const float4 v1 = *reinterpret_cast<const float4*>(b1 + c);
        const double2 a01 = *reinterpret_cast<const double2*>(a_smem + c);
        const double2 a23 = *reinterpret_cast<const double2*>(a_smem + c + 2);
        acc0 = fma(a01.x, static_cast<double>(v0.x), acc0);
        acc0 = fma(a01.y, static_cast<double>(v0.y), acc0);
        acc0 = fma(a23.x, static_cast<double>(v0.z), acc0);
        acc0 = fma(a23.y, static_cast<double>(v0.w), acc0);
        acc1 = fma(a01.x, static_cast<double>(v1.x), acc1);
        acc1 = fma(a01.y, static_cast<double>(v1.y), acc1);
        acc1 = fma(a23.x, static_cast<double>(v1.z), acc1);
        acc1 = fma(a23.y, static_cast<double>(v1.w), acc1);
      } else {
        for (int e = c; e < d; ++e) {
          acc0 = fma(a_smem[e], static_cast<double>(b0[e]), acc0);
          acc1 = fma(a_smem[e], static_cast<double>(b1[e]), acc1);
        }
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    acc0 += __shfl_xor_sync(kFull, acc0, off);
    acc1 += __shfl_xor_sync(kFull, acc1, off);
  }
  out0 = acc0;
  out1 = acc1;
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
constexpr int kRescoreThreads = 128;   // block size of both widths

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

template <int kThreads>
__global__ void __launch_bounds__(kRescoreThreads) rescore_select_kernel(const RescoreParams p) {
  constexpr int kWarps = kThreads / 32;
  extern __shared__ __align__(16) uint8_t sm[];
  const int tid = static_cast<int>(threadIdx.x) % kThreads;
  const uint32_t lane = threadIdx.x & 31;
  const int warp = tid >> 5;   // warp of the group
  const int grp = static_cast<int>(threadIdx.x) / kThreads;
  // crow indexes the (possibly compacted) query matrix the fused kernel saw; qrow is the caller's row
  const int crow = blockIdx.x * (kRescoreThreads / kThreads) + grp;
  if (crow >= p.nq) return;   // whole groups leave; nothing below synchronises across groups
  const RescoreSmem L(p.d, p.max_cand);
  uint8_t* base = sm + grp * L.bytes;
  double* qs = reinterpret_cast<double*>(base);          // [d] the query row, widened once
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
    if (c < d) qv[i] = *reinterpret_cast<const float4*>(p.q + static_cast<size_t>(qrow) * d + c);   // d % 4 == 0
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
#pragma unroll
  for (int i = 0; i < kQv; ++i) {
    const int c = (i * kThreads + tid) * 4;
    if (c < d) {
      *reinterpret_cast<double2*>(qs + c) = make_double2(static_cast<double>(qv[i].x), static_cast<double>(qv[i].y));
      *reinterpret_cast<double2*>(qs + c + 2) = make_double2(static_cast<double>(qv[i].z), static_cast<double>(qv[i].w));
    }
  }
  for (int c = 512 + tid; c < d; c += kThreads) qs[c] = static_cast<double>(p.q[static_cast<size_t>(qrow) * d + c]);
  group_sync<kThreads>();

  // certificate: every gallery row that is not a candidate has approximate centred score <= thr, hence exact score
  // q.g <= thr + eps + q.mu + slack (row_bound)
  const RowBound rb = row_bound(qs, d, p.d_pad, qrow, p.q_norm_hat, p.q_norm_res, p.q_norm_x, p.g_max, p.mu, p.nu,
                                p.nu_flag, lane);
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
  // every surviving row's cache lines are requested at once (L2 prefetch): the dot products below then wait for L2, not for
  // one DRAM round trip per pair of rows
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
    if (c + 1 < m) exact_dot_warp_qd2(qs, p.g + static_cast<size_t>(kc[c]) * d, p.g + static_cast<size_t>(kc[c + 1]) * d, d, lane, v0, v1);
    else v0 = exact_dot_warp_qd(qs, p.g + static_cast<size_t>(kc[c]) * d, d, lane);
    if (lane == 0) {
      sc[c] = v0;
      if (c + 1 < m) sc[c + 1] = v1;
    }
  }
  group_sync<kThreads>();
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
  __shared__ BlockBest s_bb;
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
        for (int part = 0; part < n_chunks; ++part)
          best = fmax(best, exact_dot_warp(qs, g + static_cast<size_t>(ci[c]) * d + part * p, p, lane));
      } else {
        best = fmax(best, exact_dot_warp(qs, g + static_cast<size_t>(ci[c]) * d + qp * p, p, lane));
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
      const double v = exact_dot_warp(qs + f * d, gr, d, lane);
      if (lane == 0) scores[static_cast<size_t>(f) * ng + row] = v;
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
  __shared__ double s_best[8];
  __shared__ int s_besti[8];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int round = 0; round < k; ++round) {
    double bs = -INFINITY;
    int bi = -1;
    for (int c = threadIdx.x; c < ng; c += blockDim.x) {
      const double v = s[c];
      if (!(v != v) && (bi < 0 || v > bs)) {   // ascending c per thread => first (lowest index) max kept
        bs = v;
        bi = c;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double os = __shfl_xor_sync(kFull, bs, off);
      const int oi = __shfl_xor_sync(kFull, bi, off);
      if (oi >= 0 && (bi < 0 || os > bs || (os == bs && oi < bi))) {
        bs = os;
        bi = oi;
      }
    }
    if (lane == 0) {
      s_best[warp] = bs;
      s_besti[warp] = bi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < 8; ++w)
        if (s_besti[w] >= 0 && (s_besti[0] < 0 || s_best[w] > s_best[0] ||
                                (s_best[w] == s_best[0] && s_besti[w] < s_besti[0]))) {
          s_best[0] = s_best[w];
          s_besti[0] = s_besti[w];
        }
      if (s_besti[0] < 0) {   // every remaining score is NaN (NaN query row, or k > number of non-NaN scores)
        out_scores[static_cast<size_t>(qrow) * k + round] = __int_as_float(0x7fc00000);
        out_idx[static_cast<size_t>(qrow) * k + round] = -1;
      } else {
        out_scores[static_cast<size_t>(qrow) * k + round] = static_cast<float>(s_best[0]);
        out_idx[static_cast<size_t>(qrow) * k + round] = g_index_base + g_index_stride * s_besti[0];
        s[s_besti[0]] = __longlong_as_double(0x7ff8000000000000LL);  // NaN marks "taken"
      }
    }
    __syncthreads();
  }
}

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
constexpr int kRangePiece = 512;   // candidates of one row re-scored by one block

struct RangeParams {
  int nq, ng;
  int num_kb, stream_a, n_qtiles, n_gtiles, gchunk, n_chunks, stages;   // as SimParams
  const int* bias_flag;
  const float* col_bias;
  const float* thr;            // [nq] candidate threshold t_i
  int* seg;                    // [n_slots][128] count sweep: candidates; emit sweep: offset inside the row
  const long long* row_cand;   // [nq + 1] emit sweep: first candidate of each row
  int* cand_idx;               // emit sweep: local gallery rows
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
template <bool kBias, bool kEmit>
__global__ void __launch_bounds__(32 + 128, 1)
    sim_range_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_g,
                     const RangeParams p) {
  if (((p.bias_flag != nullptr) && (*p.bias_flag != 0)) != kBias) return;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const FusedPipe pp(smem_raw, p.num_kb, p.stream_a, p.stages, 0);   // then barriers, then 4 transpose buffers
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31;
  pp.init(&tmap_q, &tmap_g, p.stages, 4);
  const long long n_units = gridDim.x;
  const long long unit = blockIdx.x;
  SegWalker w(p.n_qtiles, p.n_gtiles, p.gchunk, p.n_chunks, unit, n_units);
  if (warp == 4) {
    fused_producer(pp, &tmap_q, &tmap_g, p.stages, w, [](const SegWalker&) { return 0; });
  } else {
    const uint32_t row = warp * 32 + lane;   // query row inside the tile
    const uint32_t xacc = smem_u32(pp.tail) + warp * kAccXposeWarpBytes;
    const uint32_t a_base = smem_u32(pp.stream_a ? pp.smem_b + kBTileBytes : pp.smem_a);
    const uint32_t b_base = smem_u32(pp.smem_b);
    PipeState st(p.stages);
    uint32_t seg = 0;
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
      ++seg;
      if (!kEmit) p.seg[sr] = cnt;
    }
  }
  __syncthreads();
}

// t_i = tau - q.mu - eps - slack - margin, rounded down at every step.  fp32(s) >= tau needs s >= tau - half an fp32 ulp
// (margin), hence approximate score >= t_i (row_bound).  A warp per query row.
__global__ void __launch_bounds__(128)
    range_threshold_kernel(const float* __restrict__ q, int nq, int d, int d_pad, float tau,
                           const float* __restrict__ q_norm_hat, const float* __restrict__ q_norm_res,
                           const float* __restrict__ q_norm_x, const unsigned int* __restrict__ g_max,
                           const float* __restrict__ mu, const float* __restrict__ nu, const int* __restrict__ nu_flag,
                           float* __restrict__ thr) {
  const int row = blockIdx.x * 4 + static_cast<int>(threadIdx.x >> 5);
  const uint32_t lane = threadIdx.x & 31;
  if (row >= nq) return;
  const RowBound rb = row_bound(q + static_cast<size_t>(row) * d, d, d_pad, row, q_norm_hat, q_norm_res, q_norm_x, g_max,
                                mu, nu, nu_flag, lane);
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

// Exact scores of one piece (the association of exact_dot_warp: the values dcr_sim_topk reports), then a stable in-place
// compaction of the pairs with fp32 score >= tau.  piece_kept[w] = pairs kept.
__global__ void __launch_bounds__(kRescoreThreads)
    range_rescore_kernel(const float* __restrict__ q, const float* __restrict__ g, int nq, int d, float tau,
                         const long long* __restrict__ row_cand, const long long* __restrict__ row_piece,
                         int* __restrict__ cand_idx, float* __restrict__ cand_score, int* __restrict__ piece_kept) {
  extern __shared__ __align__(16) uint8_t sm[];
  double* qs = reinterpret_cast<double*>(sm);   // [d] the query row, widened once
  const int tid = threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const int warp = tid >> 5;
  int row, n;
  long long start;
  range_piece(blockIdx.x, row_cand, row_piece, nq, row, start, n);
  for (int c = tid; c < d; c += kRescoreThreads) qs[c] = static_cast<double>(q[static_cast<size_t>(row) * d + c]);
  __syncthreads();
  int* ci = cand_idx + start;
  float* cs = cand_score + start;
  for (int c = 2 * warp; c < n; c += 2 * (kRescoreThreads / 32)) {
    double v0, v1 = 0.0;
    if (c + 1 < n) exact_dot_warp_qd2(qs, g + static_cast<size_t>(ci[c]) * d, g + static_cast<size_t>(ci[c + 1]) * d, d, lane, v0, v1);
    else v0 = exact_dot_warp_qd(qs, g + static_cast<size_t>(ci[c]) * d, d, lane);
    if (lane == 0) {
      cs[c] = static_cast<float>(v0);
      if (c + 1 < n) cs[c + 1] = static_cast<float>(v1);
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

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// launch geometry of one fused pass over nq queries
struct PassPlan {
  int nq, nq_pad, n_qtiles, n_units, n_slots, kp, cap, stages, max_cand;
  int n_sets;             // epilogue warp sets = candidate slots per segment (column halves with their own lists)
  int gchunk, n_chunks;   // gallery tiles per L2-sized chunk for this pass
  size_t smem_bytes;
};

struct SimPlan {
  int d_pad, num_kb, ng_pad, n_gtiles, rows_per_qtile;
  int stream_a;  // d_pad > 512: query tile streamed with the gallery k-blocks
  int max_sets;  // upper bound for PassPlan::n_sets (1 or 2)
  int gchunk, n_chunks;   // preferred gallery chunking (a pass may use fewer chunks)
  int kp0, kp1;           // candidates kept by the first pass / by the second-chance pass (0 = no second pass)
  PassPlan p0, p1;        // p1 is sized for the worst case (every query flagged)
  // workspace offsets
  size_t off_qb, off_qb1, off_gb, off_qnh, off_qnr, off_qnx, off_gmax, off_colsum, off_mu, off_cand, off_cnt, off_thr,
      off_flag0, off_flag1, off_thr1, off_counts, off_exact, off_nu, off_bias, off_clk, off_gthr;
  size_t total;
};

int plan_pass(int nq, int kp, const SimPlan& sp, int num_sms, size_t max_smem, int d, int k, PassPlan* pp) {
  pp->nq = nq;
  pp->n_qtiles = (nq + sp.rows_per_qtile - 1) / sp.rows_per_qtile;
  pp->nq_pad = pp->n_qtiles * sp.rows_per_qtile;
  pp->kp = kp;
  // ---- shared memory: resident A + stages*B + n_sets * cap KB of lists + barriers + carried thresholds ----
  const size_t a_bytes = sp.stream_a ? 0 : static_cast<size_t>(sp.num_kb) * kATileBytes;
  const size_t b_tile = static_cast<size_t>(kBlockN) * kBlockK * 2 + (sp.stream_a ? kATileBytes : 0);
  const size_t fixed = 1024 /*align slack*/ + 256 /*barriers*/ + 4096 /*carried thresholds*/;
  auto per_set = [&](int cp) { return static_cast<size_t>(cp) * 1024 + 4 * kAccXposeWarpBytes; };   // lists + transposes
  auto fits = [&](int st, int cp, int sets) { return max_smem >= a_bytes + st * b_tile + per_set(cp) * sets + fixed; };
  // two epilogue warp sets whenever their lists (at least kp + 8 entries per row and set) fit next to 3 B stages
  int sets = (sp.max_sets >= 2 && fits(3, kp + 8, 2)) ? 2 : 1;
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
  pp->smem_bytes = fixed + a_bytes + stages * b_tile + per_set(cap) * sets;

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

// tiles, padding and gallery chunking of a fused sweep (both entry points)
void plan_geometry(int ng, int d, SimPlan* pl) {
  pl->d_pad = static_cast<int>(align_up(d, kBlockK));
  pl->num_kb = pl->d_pad / kBlockK;
  pl->stream_a = pl->num_kb > kMaxKB ? 1 : 0;
  pl->rows_per_qtile = kBlockM;
  pl->n_gtiles = (ng + kBlockN - 1) / kBlockN;
  pl->ng_pad = pl->n_gtiles * kBlockN;
  // gallery chunks of ~40 MB of bf16 rows: the units sweep one chunk at a time so that it stays L2 resident
  const long long chunk_bytes = 40ll << 20;
  int gchunk = static_cast<int>(std::max<long long>(16, chunk_bytes / (static_cast<long long>(kBlockN) * pl->d_pad * 2)));
  int n_chunks = (pl->n_gtiles + gchunk - 1) / gchunk;
  if (n_chunks > 64) n_chunks = 64;
  gchunk = (pl->n_gtiles + n_chunks - 1) / n_chunks;   // equal chunks
  n_chunks = (pl->n_gtiles + gchunk - 1) / gchunk;
  pl->gchunk = gchunk;
  pl->n_chunks = n_chunks;
}

int make_plan(int nq, int ng, int d, int k, int num_sms, size_t max_smem, SimPlan* pl) {
  DCR_REQUIRE(nq >= 1 && ng >= 1 && d >= 1, "sim_topk: empty problem (nq=%d ng=%d d=%d)", nq, ng, d);
  DCR_REQUIRE(d <= kMaxDim, "sim_topk: descriptor dim %d > %d not supported", d, kMaxDim);
  DCR_REQUIRE(k >= 1 && k <= 16, "sim_topk: k=%d outside [1,16]", k);
  DCR_REQUIRE(k <= ng, "sim_topk: k=%d > gallery size %d", k, ng);
  plan_geometry(ng, d, pl);
  // Two consumer warpgroups (two warps per 32-row block, each with its own lists for one column half) when few
  // candidates are kept (k <= 2: each segment keeps 2 x 4 candidates); with larger k the lists of two sets only fit with
  // a small capacity.
  pl->max_sets = k <= 2 ? 2 : 1;
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
  const PassPlan& big = pl->p0;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  pl->off_qb = take(static_cast<size_t>(big.nq_pad) * pl->d_pad * 2);
  pl->off_qb1 = take(pl->kp1 ? static_cast<size_t>(pl->p1.nq_pad) * pl->d_pad * 2 : 0);
  pl->off_gb = take(static_cast<size_t>(pl->ng_pad) * pl->d_pad * 2);
  pl->off_qnh = take(static_cast<size_t>(big.nq_pad) * 4);
  pl->off_qnr = take(static_cast<size_t>(big.nq_pad) * 4);
  pl->off_qnx = take(static_cast<size_t>(big.nq_pad) * 4);
  pl->off_gmax = take(16);
  pl->off_colsum = take(static_cast<size_t>(d) * 16);   // column sums + column sums of squares
  pl->off_mu = take(static_cast<size_t>(d) * 4);
  pl->off_nu = take(static_cast<size_t>(d) * 4);
  pl->off_bias = take(static_cast<size_t>(pl->ng_pad) * 4);
  const size_t slot_rows = static_cast<size_t>(std::max(pl->p0.n_slots, pl->kp1 ? pl->p1.n_slots : 0)) * pl->rows_per_qtile;   // n_slots counts sets
  pl->off_cand = take(slot_rows * kKPMax * 8);
  pl->off_cnt = take(slot_rows * 4);
  pl->off_thr = take(slot_rows * 4);
  pl->off_flag0 = take(static_cast<size_t>(nq) * 4);
  pl->off_flag1 = take(static_cast<size_t>(nq) * 4);
  pl->off_thr1 = take(static_cast<size_t>(nq) * 4);
  pl->off_counts = take(16);
  pl->off_clk = take(32);
  pl->off_gthr = take(static_cast<size_t>(std::max(big.nq_pad, pl->kp1 ? pl->p1.nq_pad : 0)) * 4);
  pl->off_exact = take(static_cast<size_t>(kExactBatch) * ng * 8);
  pl->total = off;
  return 0;
}


struct PassBuffers {
  uint2* cand;
  int* ccnt;
  float* cthr;
};

// one fused pass: qb (bf16, padded) x gb (bf16, centred, padded) -> candidate slots
int launch_fused(const SimPlan& pl, const PassPlan& pp, const __nv_bfloat16* qb, const __nv_bfloat16* gb, int ng,
                 const PassBuffers& pb, const float* col_bias, const int* bias_flag, const float* thr_init,
                 unsigned long long* clk, unsigned int* gthr, cudaStream_t stream) {
  CUtensorMap tq, tg;
  if (int rc = make_tmap_2d_bf16(&tq, qb, pp.nq_pad, pl.d_pad, pl.d_pad, kBlockM, kBlockK)) return rc;
  if (int rc = make_tmap_2d_bf16(&tg, gb, pl.ng_pad, pl.d_pad, pl.d_pad, kBlockN, kBlockK)) return rc;
  SimParams p;
  p.nq = pp.nq;
  p.ng = ng;
  p.num_kb = pl.num_kb;
  p.stream_a = pl.stream_a;
  p.n_qtiles = pp.n_qtiles;
  p.n_gtiles = pl.n_gtiles;
  p.gchunk = pp.gchunk;
  p.n_chunks = pp.n_chunks;
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
  DCR_CUDA_CHECK(cudaMemsetAsync(gthr, 0, static_cast<size_t>(pp.nq_pad) * 4, stream));
  auto launch = [&](auto kern) -> int {
    DCR_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(pp.smem_bytes)));
    kern<<<pp.n_units, 32 + 128 * pp.n_sets, pp.smem_bytes, stream>>>(tq, tg, p);
    count_launch();
    DCR_CUDA_CHECK(cudaGetLastError());
    return 0;
  };
  // both variants are launched; the one that does not match the device flag (query centring on / off) returns at once
  if (pp.n_sets == 2) {
    if (int rc = launch(sim_topk_kernel<false, 2>)) return rc;
    return launch(sim_topk_kernel<true, 2>);
  }
  if (int rc = launch(sim_topk_kernel<false, 1>)) return rc;
  return launch(sim_topk_kernel<true, 1>);
}

// Stage 1 of both entry points: the centres, the decision whether to centre the queries, and the bf16 operands with the
// norms their error bound needs.
struct Operands {
  __nv_bfloat16 *qb, *gb;   // [nq_pad, d_pad], [ng_pad, d_pad]
  float *qnh, *qnr, *qnx;   // per query row, see to_bf16_rows_kernel
  unsigned int* gmax;       // [2]
  double* colsum;           // [2 d] scratch
  float *mu, *nu, *bias;    // gallery centre, query centre, per-gallery-row offset nu.(g - mu)
  int* qflag;               // device flag: query centring on / off
};

int prepare_operands(const float* q, int nq, int nq_pad, const float* g, int ng, int d, const SimPlan& pl,
                     const DeviceInfo* di, const Operands& o, cudaStream_t stream) {
  DCR_CUDA_CHECK(cudaMemsetAsync(o.gmax, 0, 16, stream));
  const int conv_blocks = di->num_sms * 8;
  auto sampled_mean = [&](const float* x, int n, float* out, bool decide) -> int {
    // any fixed vector works as a centre, so a strided sample of <= 8192 rows is enough
    DCR_CUDA_CHECK(cudaMemsetAsync(o.colsum, 0, static_cast<size_t>(d) * 16, stream));
    const int row_stride = std::max(1, n / 8192);
    const int n_sample = (n + row_stride - 1) / row_stride;
    col_sum_kernel<<<std::max(1, std::min((n_sample + 63) / 64, di->num_sms)), kColSumThreads, 0, stream>>>(
        x, n_sample, row_stride, d, o.colsum, decide ? o.colsum + d : nullptr);
    count_launch();
    col_mean_finish_kernel<<<(d + 255) / 256, 256, 0, stream>>>(o.colsum, n_sample, d, out);
    count_launch();
    if (decide) {
      centre_decision_kernel<<<1, 256, 0, stream>>>(o.colsum, o.colsum + d, n_sample, d, o.qflag);
      count_launch();
    }
    return 0;
  };
  if (int rc = sampled_mean(g, ng, o.mu, false)) return rc;    // gallery centre mu (always used)
  if (int rc = sampled_mean(q, nq, o.nu, true)) return rc;     // query centre nu + the decision whether to use it
  // q' = q - nu, g' = g - mu:  q.g = q'.g' + nu.g' + q.mu  -- the tensor cores see only the centred parts, nu.g' is a
  // per-gallery-row offset added to the accumulator columns, q.mu a per-query constant that cannot change the ranking
  // d_pad <= 256: 2 loads per lane cover the row; otherwise 4 per round (512 dims = one round)
  auto convert = (pl.d_pad <= 256) ? to_bf16_rows_kernel<2> : to_bf16_rows_kernel<4>;
  convert<<<conv_blocks, 256, 0, stream>>>(q, nq, d, nq_pad, pl.d_pad, o.nu, o.qb, o.qnh, o.qnr, o.qnx, nullptr,
                                           nullptr, nullptr, o.qflag, nullptr);
  count_launch();
  convert<<<conv_blocks, 256, 0, stream>>>(g, ng, d, pl.ng_pad, pl.d_pad, o.mu, o.gb, nullptr, nullptr, nullptr,
                                           o.gmax, o.nu, o.bias, nullptr, o.qflag);
  count_launch();
  DCR_CUDA_CHECK(cudaGetLastError());
  return 0;
}

constexpr long long kMaxRangePairs = 1ll << 40;   // capacity accepted by the planner (keeps the byte counts in range)

struct RangePlan {
  SimPlan geo;   // plan_geometry fields only
  int nq_pad, n_qtiles, n_units, n_slots, stages;
  size_t smem_bytes;
  long long max_pieces;   // pieces of kRangePiece candidates when max_pairs candidates fill the rows worst
  size_t off_qb, off_gb, off_qnh, off_qnr, off_qnx, off_gmax, off_colsum, off_mu, off_nu, off_bias, off_flag, off_thr,
      off_seg, off_row_cnt, off_row_cand, off_row_pcnt, off_row_piece, off_cand_idx, off_cand_score, off_piece_kept,
      off_piece_excl;
  size_t total;
};

int make_range_plan(int nq, int ng, int d, long long max_pairs, int num_sms, size_t max_smem, RangePlan* rp) {
  DCR_REQUIRE(nq >= 1 && ng >= 1 && d >= 1, "sim_range: empty problem (nq=%d ng=%d d=%d)", nq, ng, d);
  DCR_REQUIRE(d <= kMaxDim, "sim_range: descriptor dim %d > %d not supported", d, kMaxDim);
  DCR_REQUIRE(d % 4 == 0, "sim_range: descriptor dim %d is not a multiple of 4", d);
  DCR_REQUIRE(max_pairs >= 0 && max_pairs <= kMaxRangePairs, "sim_range: max_pairs=%lld outside [0, 2^40]", max_pairs);
  plan_geometry(ng, d, &rp->geo);
  const SimPlan& g = rp->geo;
  rp->n_qtiles = (nq + kBlockM - 1) / kBlockM;
  rp->nq_pad = rp->n_qtiles * kBlockM;
  // shared memory: resident query tile + stages x gallery stage + barriers + the transpose buffers of 4 warps
  const size_t a_bytes = g.stream_a ? 0 : static_cast<size_t>(g.num_kb) * kATileBytes;
  const size_t b_tile = static_cast<size_t>(kBTileBytes) + (g.stream_a ? kATileBytes : 0);
  const size_t fixed = 1024 /*align slack*/ + 256 /*barriers*/ + 4 * kAccXposeWarpBytes;
  int stages = 2;
  DCR_REQUIRE(max_smem >= fixed + a_bytes + stages * b_tile, "sim_range: not enough shared memory (%zu B) for d=%d", max_smem, d);
  while (stages < 8 && max_smem >= fixed + a_bytes + (stages + 1) * b_tile) ++stages;
  rp->stages = stages;
  rp->smem_bytes = fixed + a_bytes + stages * b_tile;
  // every unit owns at least one tile of every chunk (the last chunk is the smallest): every slot the scan walks is written
  const int last = g.n_gtiles - (g.n_chunks - 1) * g.gchunk;
  rp->n_units = static_cast<int>(std::min<long long>(num_sms, static_cast<long long>(rp->n_qtiles) * last));
  rp->n_slots = g.n_chunks * (rp->n_units + rp->n_qtiles);
  rp->max_pieces = max_pairs / kRangePiece + nq;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  rp->off_qb = take(static_cast<size_t>(rp->nq_pad) * g.d_pad * 2);
  rp->off_gb = take(static_cast<size_t>(g.ng_pad) * g.d_pad * 2);
  rp->off_qnh = take(static_cast<size_t>(rp->nq_pad) * 4);
  rp->off_qnr = take(static_cast<size_t>(rp->nq_pad) * 4);
  rp->off_qnx = take(static_cast<size_t>(rp->nq_pad) * 4);
  rp->off_gmax = take(16);
  rp->off_colsum = take(static_cast<size_t>(d) * 16);
  rp->off_mu = take(static_cast<size_t>(d) * 4);
  rp->off_nu = take(static_cast<size_t>(d) * 4);
  rp->off_bias = take(static_cast<size_t>(g.ng_pad) * 4);
  rp->off_flag = take(16);
  rp->off_thr = take(static_cast<size_t>(nq) * 4);
  rp->off_seg = take(static_cast<size_t>(rp->n_slots) * kBlockM * 4);
  rp->off_row_cnt = take(static_cast<size_t>(nq) * 8);
  rp->off_row_cand = take((static_cast<size_t>(nq) + 1) * 8);
  rp->off_row_pcnt = take(static_cast<size_t>(nq) * 8);
  rp->off_row_piece = take((static_cast<size_t>(nq) + 1) * 8);
  rp->off_cand_idx = take(static_cast<size_t>(max_pairs) * 4);
  rp->off_cand_score = take(static_cast<size_t>(max_pairs) * 4);
  rp->off_piece_kept = take(static_cast<size_t>(rp->max_pieces) * 4);
  rp->off_piece_excl = take((static_cast<size_t>(rp->max_pieces) + 1) * 8);
  rp->total = off;
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
  DCR_CUDA_CHECK(cudaFuncSetAttribute(split_rescore_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  split_rescore_kernel<<<nq, 128, smem, stream>>>(q, g, d, n_chunks, cross, cand, n_cand, k, out_scores, out_idx);
  count_launch();
  DCR_CUDA_CHECK(cudaGetLastError());
  return 0;
}

size_t sim_topk_workspace_size(int nq, int ng, int d, int k) {
  const DeviceInfo* di = device_info();
  SimPlan pl;
  if (make_plan(nq, ng, d, k, di ? di->num_sms : 132, di ? di->max_smem_optin : 232448, &pl) != 0)
    return 0;
  return pl.total;
}

int sim_topk(const float* q, int nq, const float* g, int ng, int d, int k, long long g_index_base,
             long long g_index_stride, float* out_scores, long long* out_idx, void* ws, size_t ws_bytes,
             cudaStream_t stream, SimStats* stats) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  DCR_REQUIRE(di->cc_major == 9 && di->cc_minor == 0, "sim_topk: this build targets sm_90a; device reports sm_%d%d", di->cc_major,
              di->cc_minor);
  SimPlan pl;
  if (int rc = make_plan(nq, ng, d, k, di->num_sms, di->max_smem_optin, &pl)) return rc;
  DCR_REQUIRE(ws != nullptr && ws_bytes >= pl.total, "sim_topk: workspace too small (%zu < %zu)", ws_bytes, pl.total);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "sim_topk: workspace must be 256-byte aligned");
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0 && d % 4 == 0,
              "sim_topk: q/g must be 16-byte aligned with d %% 4 == 0 (d=%d)", d);
  uint8_t* w = static_cast<uint8_t*>(ws);
  auto* qb = reinterpret_cast<__nv_bfloat16*>(w + pl.off_qb);
  auto* qb1 = reinterpret_cast<__nv_bfloat16*>(w + pl.off_qb1);
  auto* gb = reinterpret_cast<__nv_bfloat16*>(w + pl.off_gb);
  auto* qnh = reinterpret_cast<float*>(w + pl.off_qnh);
  auto* qnr = reinterpret_cast<float*>(w + pl.off_qnr);
  auto* qnx = reinterpret_cast<float*>(w + pl.off_qnx);
  auto* gmax = reinterpret_cast<unsigned int*>(w + pl.off_gmax);
  auto* colsum = reinterpret_cast<double*>(w + pl.off_colsum);
  auto* mu = reinterpret_cast<float*>(w + pl.off_mu);
  auto* nu = reinterpret_cast<float*>(w + pl.off_nu);
  auto* bias = reinterpret_cast<float*>(w + pl.off_bias);
  PassBuffers pb;
  pb.cand = reinterpret_cast<uint2*>(w + pl.off_cand);
  pb.ccnt = reinterpret_cast<int*>(w + pl.off_cnt);
  pb.cthr = reinterpret_cast<float*>(w + pl.off_thr);
  auto* flag0 = reinterpret_cast<int*>(w + pl.off_flag0);
  auto* flag1 = reinterpret_cast<int*>(w + pl.off_flag1);
  auto* thr1 = reinterpret_cast<float*>(w + pl.off_thr1);
  auto* counts = reinterpret_cast<int*>(w + pl.off_counts);   // [0] flagged by pass 0, [1] flagged by pass 1
  auto* exact = reinterpret_cast<double*>(w + pl.off_exact);
  auto* clk = reinterpret_cast<unsigned long long*>(w + pl.off_clk);
  auto* gthr = reinterpret_cast<unsigned int*>(w + pl.off_gthr);

  DCR_CUDA_CHECK(cudaMemsetAsync(counts, 0, 16, stream));   // [0],[1] flagged counts, [2] query-centring flag
  int* qflag = counts + 2;   // device flag: query centring on/off
  const Operands ops = {qb, gb, qnh, qnr, qnx, gmax, colsum, mu, nu, bias, qflag};
  if (int rc = prepare_operands(q, nq, pl.p0.nq_pad, g, ng, d, pl, di, ops, stream)) return rc;

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
  if (int rc = launch_fused(pl, pl.p0, qb, gb, ng, pb, bias, qflag, nullptr, clk, gthr, stream)) return rc;
  DCR_CUDA_CHECK(cudaEventRecord(ev1, stream));

  auto rescore = [&](const PassPlan& pp, const int* qmap, int* flagged, int* n_flagged, float* thr_next) -> int {
    RescoreParams rp;
    rp.q = q, rp.g = g, rp.nq = pp.nq, rp.d = d, rp.d_pad = pl.d_pad, rp.k = k;
    rp.n_qtiles = pp.n_qtiles, rp.n_gtiles = pl.n_gtiles, rp.gchunk = pp.gchunk, rp.n_chunks = pp.n_chunks;
    rp.n_units = pp.n_units, rp.n_sets = pp.n_sets, rp.max_cand = pp.max_cand;
    rp.cand = pb.cand, rp.cand_cnt = pb.ccnt, rp.cand_thr = pb.cthr, rp.qmap = qmap;
    rp.mu = mu, rp.nu = nu, rp.nu_flag = qflag;
    rp.q_norm_hat = qnh, rp.q_norm_res = qnr, rp.q_norm_x = qnx, rp.g_max = gmax;
    rp.g_index_base = g_index_base, rp.g_index_stride = g_index_stride, rp.out_scores = out_scores, rp.out_idx = out_idx;
    rp.flagged = flagged, rp.n_flagged = n_flagged, rp.thr_next = thr_next;
    // one warp per query when a q-tile's candidate slots fit a lane each and four queries' rows fit a block's shared memory
    // (the block-wide form spends its time on barriers for such small candidate sets)
    const size_t per_query = RescoreSmem(d, pp.max_cand).bytes;
    const bool warp_form = pp.kp > 0 && pp.max_cand / pp.kp <= 32 && pp.n_chunks <= 32 && 4 * per_query <= 56 * 1024 &&
                           !tuning_flag("DCR_SIM_RESCORE_BLOCK");
    const int per_block = warp_form ? kRescoreThreads / 32 : 1;
    const size_t smem = per_block * per_query;
    auto kern = warp_form ? rescore_select_kernel<32> : rescore_select_kernel<kRescoreThreads>;
    DCR_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    kern<<<(pp.nq + per_block - 1) / per_block, kRescoreThreads, smem, stream>>>(rp);
    count_launch();
    DCR_CUDA_CHECK(cudaGetLastError());
    return 0;
  };
  if (int rc = rescore(pl.p0, nullptr, flag0, counts + 0, thr1)) return rc;

  int h_counts[2] = {0, 0};
  unsigned long long h_clk[4] = {0, 0, 0, 0};
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_counts, counts, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_clk, clk, 32, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  int n_second = 0;
  const int* exact_list = flag0;
  int n_exact = h_counts[0];
  if (h_counts[0] > 0 && pl.kp1) {
    // second chance: the flagged queries alone, 32 candidates per (query, segment)
    n_second = h_counts[0];
    PassPlan p1;
    if (int rc = plan_pass(n_second, pl.kp1, pl, di->num_sms, di->max_smem_optin, d, k, &p1)) return rc;
    gather_rows_kernel<<<std::min(di->num_sms * 8, (p1.nq_pad * (pl.d_pad / 8) + 255) / 256), 256, 0, stream>>>(
        qb, flag0, n_second, p1.nq_pad, pl.d_pad, qb1);
    count_launch();
    if (int rc = launch_fused(pl, p1, qb1, gb, ng, pb, bias, qflag, thr1, nullptr, gthr, stream)) return rc;
    if (int rc = rescore(p1, flag0, flag1, counts + 1, nullptr)) return rc;
    DCR_CUDA_CHECK(cudaMemcpyAsync(h_counts, counts, 8, cudaMemcpyDeviceToHost, stream));
    DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
    exact_list = flag1;
    n_exact = h_counts[1];
  }

  // brute-force fp64 path for the queries whose certificate still fails (ties beyond 32 candidates, NaNs, ...)
  if (n_exact > 0) {
    // queries per brute-force launch: as many as fit in shared memory next to each other (32 up to d = 1536)
    const int ex_batch = std::max(1, std::min<int>(kExactBatch, static_cast<int>(192 * 1024 / (static_cast<size_t>(d) * 4))));
    const size_t ex_smem = static_cast<size_t>(ex_batch) * d * 4;
    DCR_CUDA_CHECK(cudaFuncSetAttribute(exact_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(ex_smem)));
    const int* n_dev = (exact_list == flag0) ? counts + 0 : counts + 1;
    for (int done = 0; done < n_exact; done += ex_batch) {
      exact_scan_kernel<<<di->num_sms * 2, 256, ex_smem, stream>>>(q, g, ng, d, exact_list, done, n_dev, exact, ex_batch);
      count_launch();
      exact_select_kernel<<<ex_batch, 256, 0, stream>>>(exact, ng, k, exact_list, done, n_dev, g_index_base,
                                                           g_index_stride, out_scores, out_idx);
      count_launch();
    }
    DCR_CUDA_CHECK(cudaGetLastError());
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

size_t sim_range_workspace_size(int nq, int ng, int d, long long max_pairs) {
  const DeviceInfo* di = device_info();
  RangePlan rp;
  if (make_range_plan(nq, ng, d, max_pairs, di ? di->num_sms : 132, di ? di->max_smem_optin : 232448, &rp) != 0) return 0;
  return rp.total;
}

int sim_range(const float* q, int nq, const float* g, int ng, int d, float threshold, long long g_index_base,
              long long g_index_stride, long long* row_offsets, long long* out_idx, float* out_scores, long long max_pairs,
              long long* counts, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  DCR_REQUIRE(di->cc_major == 9 && di->cc_minor == 0, "sim_range: this build targets sm_90a; device reports sm_%d%d", di->cc_major,
              di->cc_minor);
  DCR_REQUIRE(!std::isnan(threshold), "sim_range: threshold is NaN");
  DCR_REQUIRE(g_index_stride >= 1, "sim_range: g_index_stride=%lld < 1", g_index_stride);
  RangePlan rp;
  if (int rc = make_range_plan(nq, ng, d, max_pairs, di->num_sms, di->max_smem_optin, &rp)) return rc;
  DCR_REQUIRE(ws != nullptr && ws_bytes >= rp.total, "sim_range: workspace too small (%zu < %zu)", ws_bytes, rp.total);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "sim_range: workspace must be 256-byte aligned");
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0,
              "sim_range: q/g must be 16-byte aligned");
  const SimPlan& geo = rp.geo;
  uint8_t* w = static_cast<uint8_t*>(ws);
  auto* qb = reinterpret_cast<__nv_bfloat16*>(w + rp.off_qb);
  auto* gb = reinterpret_cast<__nv_bfloat16*>(w + rp.off_gb);
  auto* qnh = reinterpret_cast<float*>(w + rp.off_qnh);
  auto* qnr = reinterpret_cast<float*>(w + rp.off_qnr);
  auto* qnx = reinterpret_cast<float*>(w + rp.off_qnx);
  auto* gmax = reinterpret_cast<unsigned int*>(w + rp.off_gmax);
  auto* mu = reinterpret_cast<float*>(w + rp.off_mu);
  auto* nu = reinterpret_cast<float*>(w + rp.off_nu);
  auto* bias = reinterpret_cast<float*>(w + rp.off_bias);
  auto* qflag = reinterpret_cast<int*>(w + rp.off_flag);
  auto* thr = reinterpret_cast<float*>(w + rp.off_thr);
  auto* seg = reinterpret_cast<int*>(w + rp.off_seg);
  auto* row_cnt = reinterpret_cast<long long*>(w + rp.off_row_cnt);
  auto* row_cand = reinterpret_cast<long long*>(w + rp.off_row_cand);
  auto* row_pcnt = reinterpret_cast<long long*>(w + rp.off_row_pcnt);
  auto* row_piece = reinterpret_cast<long long*>(w + rp.off_row_piece);
  auto* cand_idx = reinterpret_cast<int*>(w + rp.off_cand_idx);
  auto* cand_score = reinterpret_cast<float*>(w + rp.off_cand_score);
  auto* piece_kept = reinterpret_cast<int*>(w + rp.off_piece_kept);
  auto* piece_excl = reinterpret_cast<long long*>(w + rp.off_piece_excl);

  const Operands ops = {qb, gb, qnh, qnr, qnx, gmax, reinterpret_cast<double*>(w + rp.off_colsum), mu, nu, bias, qflag};
  if (int rc = prepare_operands(q, nq, rp.nq_pad, g, ng, d, geo, di, ops, stream)) return rc;
  range_threshold_kernel<<<(nq + 3) / 4, 128, 0, stream>>>(q, nq, d, geo.d_pad, threshold, qnh, qnr, qnx, gmax, mu, nu,
                                                           qflag, thr);
  count_launch();

  CUtensorMap tq, tg;
  if (int rc = make_tmap_2d_bf16(&tq, qb, rp.nq_pad, geo.d_pad, geo.d_pad, kBlockM, kBlockK)) return rc;
  if (int rc = make_tmap_2d_bf16(&tg, gb, geo.ng_pad, geo.d_pad, geo.d_pad, kBlockN, kBlockK)) return rc;
  RangeParams p;
  p.nq = nq;
  p.ng = ng;
  p.num_kb = geo.num_kb;
  p.stream_a = geo.stream_a;
  p.n_qtiles = rp.n_qtiles;
  p.n_gtiles = geo.n_gtiles;
  p.gchunk = geo.gchunk;
  p.n_chunks = geo.n_chunks;
  p.stages = rp.stages;
  p.bias_flag = qflag;
  p.col_bias = bias;
  p.thr = thr;
  p.seg = seg;
  p.row_cand = row_cand;
  p.cand_idx = cand_idx;
  auto launch = [&](auto kern) -> int {
    DCR_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(rp.smem_bytes)));
    kern<<<rp.n_units, 32 + 128, rp.smem_bytes, stream>>>(tq, tg, p);
    count_launch();
    DCR_CUDA_CHECK(cudaGetLastError());
    return 0;
  };
  // both centring variants are launched; the one that does not match the device flag returns at once
  if (int rc = launch(sim_range_kernel<false, false>)) return rc;
  if (int rc = launch(sim_range_kernel<true, false>)) return rc;
  range_slot_scan_kernel<<<(nq + 255) / 256, 256, 0, stream>>>(seg, nq, rp.n_qtiles, geo.n_gtiles, geo.gchunk,
                                                                geo.n_chunks, rp.n_units, row_cnt, row_pcnt);
  count_launch();
  exclusive_scan_kernel<long long><<<1, 1024, 0, stream>>>(row_cnt, nq, row_cand);
  count_launch();
  exclusive_scan_kernel<long long><<<1, 1024, 0, stream>>>(row_pcnt, nq, row_piece);
  count_launch();
  long long h_tot[2] = {0, 0};   // candidates, pieces
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_tot, row_cand + nq, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_tot + 1, row_piece + nq, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  const long long n_cand = h_tot[0], n_pieces = h_tot[1];
  counts[0] = 0;
  counts[1] = n_cand;
  if (n_cand > max_pairs)
    return set_error(DCR_ERR_CAPACITY, "sim_range: %lld candidate pairs exceed max_pairs=%lld (call again with that capacity)",
                     n_cand, max_pairs);

  if (n_pieces > 0) {
    if (int rc = launch(sim_range_kernel<false, true>)) return rc;
    if (int rc = launch(sim_range_kernel<true, true>)) return rc;
    const size_t smem = static_cast<size_t>(d) * 8;
    DCR_CUDA_CHECK(cudaFuncSetAttribute(range_rescore_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    range_rescore_kernel<<<static_cast<unsigned>(n_pieces), kRescoreThreads, smem, stream>>>(
        q, g, nq, d, threshold, row_cand, row_piece, cand_idx, cand_score, piece_kept);
    count_launch();
  }
  exclusive_scan_kernel<int><<<1, 1024, 0, stream>>>(piece_kept, n_pieces, piece_excl);
  count_launch();
  if (n_pieces > 0) {
    range_output_kernel<<<static_cast<unsigned>(n_pieces), 256, 0, stream>>>(row_cand, row_piece, nq, piece_excl, cand_idx,
                                                                             cand_score, g_index_base, g_index_stride,
                                                                             out_idx, out_scores);
    count_launch();
  }
  range_row_offsets_kernel<<<grid_for(nq + 1, 256, di->num_sms), 256, 0, stream>>>(row_piece, piece_excl, nq, row_offsets);
  count_launch();
  DCR_CUDA_CHECK(cudaGetLastError());
  long long h_pairs = 0;
  DCR_CUDA_CHECK(cudaMemcpyAsync(&h_pairs, piece_excl + n_pieces, 8, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  counts[0] = h_pairs;
  return 0;
}

}  // namespace dcr
