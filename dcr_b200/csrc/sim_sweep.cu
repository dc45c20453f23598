// Stage 1 of both similarity searches (sim_topk.cu, sim_range.cu) and the host side of their fused sweep
// (sim_sweep.cuh): the gallery and query centres, the decision whether to centre the queries, the bf16 operands with
// the norms of their rounding residuals, the operand buffers' place in the workspace, and the sweep geometry.
#include <cuda_bf16.h>

#include <algorithm>

#include "sim_sweep.cuh"

namespace dcr {

namespace {

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

// Stage 1 under the split score: part c of row r (p floats) -> bf16 at [r][c p_pad, c p_pad + p), zeros up to
// (c + 1) p_pad, and the norms of that part (as to_bf16_rows_kernel) at norm_*[r n_parts + c]; gmax[2c], gmax[2c + 1] =
// the maxima over the rows of part c.  A warp per (row, part), walked part-major: a warp's running maxima change part
// rarely, so it issues one pair of atomics per part it leaves instead of one per row.
__global__ void __launch_bounds__(256)
    to_bf16_parts_kernel(const float* __restrict__ x, int n, int n_pad, int n_parts, int p, int p_pad,
                         __nv_bfloat16* __restrict__ out, float* __restrict__ norm_hat, float* __restrict__ norm_res,
                         float* __restrict__ norm_x, unsigned int* __restrict__ gmax) {
  const int lane = threadIdx.x & 31;
  const long long warps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  const long long total = static_cast<long long>(n_parts) * n_pad;
  const size_t d = static_cast<size_t>(n_parts) * p, d_pad = static_cast<size_t>(n_parts) * p_pad;
  int cur = -1;
  unsigned int w_nx = 0u, w_nr = 0u;   // running maxima of part `cur` (lane 0)
  auto flush = [&]() {
    if (gmax && cur >= 0 && lane == 0) {
      atomicMax(gmax + 2 * cur, w_nx);
      atomicMax(gmax + 2 * cur + 1, w_nr);
    }
  };
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5); i < total; i += warps) {
    const int c = static_cast<int>(i / n_pad), row = static_cast<int>(i % n_pad);
    if (c != cur) {
      flush();
      cur = c;
      w_nx = w_nr = 0u;
    }
    const float* xr = x + static_cast<size_t>(row) * d + static_cast<size_t>(c) * p;
    __nv_bfloat16* o = out + static_cast<size_t>(row) * d_pad + static_cast<size_t>(c) * p_pad;
    float s_hat = 0.f, s_res = 0.f, s_x = 0.f;
    for (int e = lane * 4; e < p_pad; e += 128) {
      const float4 v = (row < n && e < p) ? *reinterpret_cast<const float4*>(xr + e) : make_float4(0.f, 0.f, 0.f, 0.f);   // p % 4 == 0
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y);
      const __nv_bfloat16 h2 = __float2bfloat16_rn(v.z), h3 = __float2bfloat16_rn(v.w);
      const float f0 = __bfloat162float(h0), f1 = __bfloat162float(h1), f2 = __bfloat162float(h2), f3 = __bfloat162float(h3);
      s_hat += f0 * f0 + f1 * f1 + f2 * f2 + f3 * f3;
      s_res += (v.x - f0) * (v.x - f0) + (v.y - f1) * (v.y - f1) + (v.z - f2) * (v.z - f2) + (v.w - f3) * (v.w - f3);
      s_x += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      uint2 pk;
      pk.x = static_cast<uint32_t>(__bfloat16_as_ushort(h0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h1)) << 16);
      pk.y = static_cast<uint32_t>(__bfloat16_as_ushort(h2)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h3)) << 16);
      *reinterpret_cast<uint2*>(o + e) = pk;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s_hat += __shfl_xor_sync(kFull, s_hat, off);
      s_res += __shfl_xor_sync(kFull, s_res, off);
      s_x += __shfl_xor_sync(kFull, s_x, off);
    }
    if (lane == 0 && row < n) {
      const float nh = sqrtf(s_hat) * 1.0001f, nr = sqrtf(s_res) * 1.0001f, nx = sqrtf(s_x) * 1.0001f;
      const size_t j = static_cast<size_t>(row) * n_parts + c;
      if (norm_hat) norm_hat[j] = nh;
      if (norm_res) norm_res[j] = nr;
      if (norm_x) norm_x[j] = nx;
      w_nx = max(w_nx, __float_as_uint(nx));
      w_nr = max(w_nr, __float_as_uint(nr));
    }
  }
  flush();
}

}  // namespace

void plan_split_geometry(int ng, int n_parts, int p, SweepGeometry* geo) {
  const int p_pad = (p + kBlockK - 1) / kBlockK * kBlockK;
  plan_geometry(ng, n_parts * p_pad, geo);   // the chunks of the dot product over the part-padded rows
  // always streamed: the consumer warpgroups need the shared memory of two column halves' lists (the running maximum of
  // a 128-column tile does not fit a thread's registers), and d_pad is far above 512 for per-token descriptors
  geo->stream_a = 1;
}

Operands carve_split_operands(Carve& w, int nq_pad, const SweepGeometry& geo, int n_parts) {
  Operands o = {};
  o.qb = w.take<__nv_bfloat16>(static_cast<size_t>(nq_pad) * geo.d_pad);
  o.gb = w.take<__nv_bfloat16>(static_cast<size_t>(geo.ng_pad) * geo.d_pad);
  o.qnh = w.take<float>(static_cast<size_t>(nq_pad) * n_parts);
  o.qnr = w.take<float>(static_cast<size_t>(nq_pad) * n_parts);
  o.qnx = w.take<float>(static_cast<size_t>(nq_pad) * n_parts);
  o.gmax = w.take<unsigned int>(2 * static_cast<size_t>(n_parts));
  return o;
}

int prepare_split_operands(const float* q, int nq, int nq_pad, const float* g, int ng, int n_parts, int p,
                           const SweepGeometry& geo, const DeviceInfo* di, const Operands& o, cudaStream_t stream) {
  DCR_CUDA_CHECK(cudaMemsetAsync(o.gmax, 0, 8 * static_cast<size_t>(n_parts), stream));
  const int p_pad = geo.d_pad / n_parts;
  const int blocks = di->num_sms * 8;
  if (int rc = launch(to_bf16_parts_kernel, blocks, 256, 0, stream, "sim_sweep", q, nq, nq_pad, n_parts, p, p_pad, o.qb,
                      o.qnh, o.qnr, o.qnx, nullptr))
    return rc;
  return launch(to_bf16_parts_kernel, blocks, 256, 0, stream, "sim_sweep", g, ng, geo.ng_pad, n_parts, p, p_pad, o.gb,
                nullptr, nullptr, nullptr, o.gmax);
}

void plan_geometry(int ng, int d, SweepGeometry* geo) {
  geo->d_pad = (d + kBlockK - 1) / kBlockK * kBlockK;
  geo->num_kb = geo->d_pad / kBlockK;
  geo->stream_a = geo->num_kb > kMaxKB ? 1 : 0;
  geo->rows_per_qtile = kBlockM;
  geo->n_gtiles = (ng + kBlockN - 1) / kBlockN;
  geo->ng_pad = geo->n_gtiles * kBlockN;
  // gallery chunks of ~40 MB of bf16 rows: the units sweep one chunk at a time so that it stays L2 resident
  const long long chunk_bytes = 40ll << 20;
  int gchunk = static_cast<int>(std::max<long long>(16, chunk_bytes / (static_cast<long long>(kBlockN) * geo->d_pad * 2)));
  int n_chunks = (geo->n_gtiles + gchunk - 1) / gchunk;
  if (n_chunks > 64) n_chunks = 64;
  gchunk = (geo->n_gtiles + n_chunks - 1) / n_chunks;   // equal chunks
  n_chunks = (geo->n_gtiles + gchunk - 1) / gchunk;
  geo->gchunk = gchunk;
  geo->n_chunks = n_chunks;
}

Operands carve_operands(Carve& w, int nq_pad, const SweepGeometry& geo, int d) {
  Operands o;
  o.qb = w.take<__nv_bfloat16>(static_cast<size_t>(nq_pad) * geo.d_pad);
  o.gb = w.take<__nv_bfloat16>(static_cast<size_t>(geo.ng_pad) * geo.d_pad);
  o.qnh = w.take<float>(nq_pad);
  o.qnr = w.take<float>(nq_pad);
  o.qnx = w.take<float>(nq_pad);
  o.gmax = w.take<unsigned int>(4);
  o.colsum = w.take<double>(2 * static_cast<size_t>(d));   // column sums + column sums of squares
  o.mu = w.take<float>(d);
  o.nu = w.take<float>(d);
  o.bias = w.take<float>(geo.ng_pad);
  o.qflag = nullptr;
  return o;
}

int prepare_operands(const float* q, int nq, int nq_pad, const float* g, int ng, int d, const SweepGeometry& geo,
                     const DeviceInfo* di, const Operands& o, cudaStream_t stream) {
  DCR_CUDA_CHECK(cudaMemsetAsync(o.gmax, 0, 16, stream));
  const int conv_blocks = di->num_sms * 8;
  auto sampled_mean = [&](const float* x, int n, float* out, bool decide) -> int {
    // any fixed vector works as a centre, so a strided sample of <= 8192 rows is enough
    DCR_CUDA_CHECK(cudaMemsetAsync(o.colsum, 0, static_cast<size_t>(d) * 16, stream));
    const int row_stride = std::max(1, n / 8192);
    const int n_sample = (n + row_stride - 1) / row_stride;
    if (int rc = launch(col_sum_kernel, std::max(1, std::min((n_sample + 63) / 64, di->num_sms)), kColSumThreads, 0, stream,
                        "sim_sweep", x, n_sample, row_stride, d, o.colsum, decide ? o.colsum + d : nullptr))
      return rc;
    if (int rc = launch(col_mean_finish_kernel, (d + 255) / 256, 256, 0, stream, "sim_sweep", o.colsum, n_sample, d, out))
      return rc;
    if (decide) return launch(centre_decision_kernel, 1, 256, 0, stream, "sim_sweep", o.colsum, o.colsum + d, n_sample, d, o.qflag);
    return 0;
  };
  if (int rc = sampled_mean(g, ng, o.mu, false)) return rc;    // gallery centre mu (always used)
  if (int rc = sampled_mean(q, nq, o.nu, true)) return rc;     // query centre nu + the decision whether to use it
  // q' = q - nu, g' = g - mu:  q.g = q'.g' + nu.g' + q.mu  -- the tensor cores see only the centred parts, nu.g' is a
  // per-gallery-row offset added to the accumulator columns, q.mu a per-query constant that cannot change the ranking
  // d_pad <= 256: 2 loads per lane cover the row; otherwise 4 per round (512 dims = one round)
  auto convert = (geo.d_pad <= 256) ? to_bf16_rows_kernel<2> : to_bf16_rows_kernel<4>;
  if (int rc = launch(convert, conv_blocks, 256, 0, stream, "sim_sweep", q, nq, d, nq_pad, geo.d_pad, o.nu, o.qb, o.qnh,
                      o.qnr, o.qnx, nullptr, nullptr, nullptr, o.qflag, nullptr))
    return rc;
  return launch(convert, conv_blocks, 256, 0, stream, "sim_sweep", g, ng, d, geo.ng_pad, geo.d_pad, o.mu, o.gb, nullptr,
                nullptr, nullptr, o.gmax, o.nu, o.bias, nullptr, o.qflag);
}

int sweep_setup(const SweepGeometry& geo, int nq, int n_qtiles, int ng, int gchunk, int n_chunks, const __nv_bfloat16* qb,
                const __nv_bfloat16* gb, SweepHead* head, CUtensorMap* tq, CUtensorMap* tg) {
  if (int rc = make_tmap_2d_bf16(tq, qb, static_cast<uint64_t>(n_qtiles) * kBlockM, geo.d_pad, geo.d_pad, kBlockM, kBlockK))
    return rc;
  if (int rc = make_tmap_2d_bf16(tg, gb, geo.ng_pad, geo.d_pad, geo.d_pad, kBlockN, kBlockK)) return rc;
  head->nq = nq;
  head->ng = ng;
  head->num_kb = geo.num_kb;
  head->stream_a = geo.stream_a;
  head->n_qtiles = n_qtiles;
  head->n_gtiles = geo.n_gtiles;
  head->gchunk = gchunk;
  head->n_chunks = n_chunks;
  return 0;
}

}  // namespace dcr
