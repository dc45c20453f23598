// Exact-arithmetic convolution / linear layer for the "exact" precision mode of the network executor.
//
// Same operands and the same epilogue as conv_gemm.cu (three bf16 planes per tensor: hi + mid + lo reconstruct the
// fp32 value exactly), but the products are accumulated in FLOAT64 on the CUDA cores instead of the tensor cores:
//     Y[m, n] = act( fmaf( fp32( sum_k  x[m, k] * w[n, k] ), scale[n], bias[n] ) (+ R[m, n]) )
// with x, w the exact fp32 values.  The double sum of fp32 products is exact to ~1e-16 relative, so every layer
// output is the correctly rounded fp32 result -- independent of summation order, tile shape or device.  This is the
// mode the parity tests use against the fp32 oracle / the golden vectors generated from the reference's own modules
// (metrics/inception.py, dino_vits.py): the tensor-core "parity" mode (6 bf16 cross terms, fp32 accumulation inside
// the MMA unit, which truncates) stays ~4e-6 relative per layer away from that, which compounds to ~3e-4 over the 94
// convolutions of the FID Inception network.
//
// It is a reference-quality path, not a fast one (fp64 FMA rate; ~30x slower than the bf16 tensor-core path).
#include <cuda_bf16.h>

#include <algorithm>

#include "dcr_internal.cuh"
#include "host_util.cuh"

namespace dcr {

namespace {

constexpr int kTM = 64, kTN = 64, kTK = 16, kThreadsExact = 256;

struct ExactParams {
  const __nv_bfloat16* in;
  long long in_plane_stride, sn, sh, sw;   // element strides of the (possibly overlapping-window) NHWC view
  int a_planes;
  int H, W, C;
  const __nv_bfloat16* weight;
  long long w_plane_stride;
  int w_planes;
  int N, kh, kw, stride, pad_h, pad_w, cblocks;
  int P, Q;
  long long M;
  const float* scale;
  const float* bias;
  const __nv_bfloat16* res;
  int ld_res, res_planes;
  long long res_plane_stride;
  __nv_bfloat16* out;
  int ld_out, out_col_off, out_planes;
  long long out_plane_stride;
  float* out_f32;
  int ld_out_f32;
  int act;
};

__device__ __forceinline__ float act_exact(float y, int act) {
  if (act == 1) return fmaxf(y, 0.f);
  if (act == 2) return 0.5f * y * (1.f + erff(y * 0.70710678118654752440f));
  if (act == 3) return y / (1.f + expf(-1.702f * y));   // QuickGELU
  return y;
}

// 4 consecutive bf16 of up to 3 planes -> their exact fp32 sums
__device__ __forceinline__ void load4_sum(const __nv_bfloat16* base, long long plane_stride, int planes, float (&v)[4]) {
  v[0] = v[1] = v[2] = v[3] = 0.f;
  for (int pl = 0; pl < planes; ++pl) {
    const uint2 r = *reinterpret_cast<const uint2*>(base + pl * plane_stride);
    v[0] += __uint_as_float(r.x << 16);
    v[1] += __uint_as_float(r.x & 0xffff0000u);
    v[2] += __uint_as_float(r.y << 16);
    v[3] += __uint_as_float(r.y & 0xffff0000u);
  }
}

__global__ void __launch_bounds__(kThreadsExact) conv_exact_kernel(const ExactParams p) {
  __shared__ float As[kTK][kTM + 4];
  __shared__ float Bs[kTK][kTN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = static_cast<long long>(blockIdx.x) * kTM;
  const int n0 = blockIdx.y * kTN;

  // loader role: row lr of the tile, 4 consecutive k
  const int lr = tid >> 2, lk = (tid & 3) * 4;
  const long long lm = m0 + lr;
  const bool lrow_ok = lm < p.M;
  int lb = 0, lp = 0, lq = 0;
  if (lrow_ok) {
    lb = static_cast<int>(lm / (static_cast<long long>(p.P) * p.Q));
    const int rem = static_cast<int>(lm % (static_cast<long long>(p.P) * p.Q));
    lp = rem / p.Q;
    lq = rem % p.Q;
  }
  const int ln = n0 + lr;
  const bool ln_ok = ln < p.N;
  const long long ktot = static_cast<long long>(p.kh) * p.kw * p.cblocks * 64;

  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;

  for (int tap = 0; tap < p.kh * p.kw; ++tap) {
    const int fr = tap / p.kw, fs = tap % p.kw;
    const int ih = lp * p.stride - p.pad_h + fr, iw = lq * p.stride - p.pad_w + fs;
    const bool pix_ok = lrow_ok && ih >= 0 && ih < p.H && iw >= 0 && iw < p.W;
    const __nv_bfloat16* arow = p.in + lb * p.sn + ih * p.sh + iw * p.sw;
    const __nv_bfloat16* wrow = p.weight + static_cast<long long>(ln) * ktot + static_cast<long long>(tap) * p.cblocks * 64;
    for (int c0 = 0; c0 < p.C; c0 += kTK) {
      float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f};
      const int c = c0 + lk;
      if (pix_ok && c < p.C) load4_sum(arow + c, p.in_plane_stride, p.a_planes, av);
      if (ln_ok && c < p.C) load4_sum(wrow + c, p.w_plane_stride, p.w_planes, bv);
      __syncthreads();   // previous chunk fully consumed
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        As[lk + e][lr] = av[e];
        Bs[lk + e][lr] = bv[e];
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < kTK; ++kk) {
        const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        const float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        const double a[4] = {a4.x, a4.y, a4.z, a4.w};
        const double b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
      }
    }
  }

  // epilogue: thread owns rows m0 + ty*4 + i, columns n0 + tx*4 + j (N % 8 == 0, so a group of 4 columns is all-in or all-out)
  const int nc = n0 + tx * 4;
  if (nc >= p.N) return;
  float sc[4], bi[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    sc[j] = p.scale ? p.scale[nc + j] : 1.f;
    bi[j] = p.bias ? p.bias[nc + j] : 0.f;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
    float y[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) y[j] = fmaf(static_cast<float>(acc[i][j]), sc[j], bi[j]);
    if (p.res) {
      float r[4];
      load4_sum(p.res + m * p.ld_res + nc, p.res_plane_stride, p.res_planes, r);
#pragma unroll
      for (int j = 0; j < 4; ++j) y[j] += r[j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) y[j] = act_exact(y[j], p.act);
    if (p.out_f32) *reinterpret_cast<float4*>(p.out_f32 + m * p.ld_out_f32 + nc) = make_float4(y[0], y[1], y[2], y[3]);
    if (p.out) {
      for (int pl = 0; pl < p.out_planes; ++pl) {
        __nv_bfloat16 h[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          h[j] = __float2bfloat16_rn(y[j]);
          y[j] -= __bfloat162float(h[j]);   // the next plane holds the rounding residual of this one
        }
        uint2 v;
        v.x = static_cast<uint32_t>(__bfloat16_as_ushort(h[0])) | (static_cast<uint32_t>(__bfloat16_as_ushort(h[1])) << 16);
        v.y = static_cast<uint32_t>(__bfloat16_as_ushort(h[2])) | (static_cast<uint32_t>(__bfloat16_as_ushort(h[3])) << 16);
        *reinterpret_cast<uint2*>(p.out + pl * p.out_plane_stride + m * p.ld_out + p.out_col_off + nc) = v;
      }
    }
  }
}

}  // namespace

int conv_exact(const ConvGemmDesc& d, cudaStream_t stream) {
  DCR_REQUIRE(d.C % 8 == 0 && d.N % 8 == 0, "conv_exact: C (%d) and N (%d) must be multiples of 8", d.C, d.N);
  DCR_REQUIRE(d.ld_out % 4 == 0 && d.out_col_off % 4 == 0 && d.ld_res % 4 == 0 && d.ld_out_f32 % 4 == 0,
              "conv_exact: leading dimensions / column offset must be multiples of 4");
  ExactParams p = {};
  const bool windowed = d.in_stride_w != 0;
  p.in = d.in;
  p.in_plane_stride = d.in_plane_stride;
  p.sw = windowed ? d.in_stride_w : d.ld_in;
  p.sh = windowed ? d.in_stride_h : static_cast<long long>(d.W) * d.ld_in;
  p.sn = windowed ? d.in_stride_n : static_cast<long long>(d.H) * d.W * d.ld_in;
  int a_planes = 0, w_planes = 0;
  for (int t = 0; t < d.n_terms; ++t) {
    a_planes = std::max(a_planes, d.term_a[t] + 1);
    w_planes = std::max(w_planes, d.term_w[t] + 1);
  }
  p.a_planes = a_planes;
  p.w_planes = w_planes;
  p.H = d.H; p.W = d.W; p.C = d.C;
  p.weight = d.weight;
  p.w_plane_stride = d.w_plane_stride;
  p.N = d.N; p.kh = d.kh; p.kw = d.kw; p.stride = d.stride; p.pad_h = d.pad_h; p.pad_w = d.pad_w;
  p.cblocks = (d.C + 63) / 64;
  p.P = (d.H + 2 * d.pad_h - d.kh) / d.stride + 1;
  p.Q = (d.W + 2 * d.pad_w - d.kw) / d.stride + 1;
  p.M = static_cast<long long>(d.B) * p.P * p.Q;
  DCR_REQUIRE(p.M > 0 && p.M < (1ll << 31), "conv_exact: M out of range");
  p.scale = d.scale;
  p.bias = d.bias;
  p.res = d.res;
  p.ld_res = d.ld_res;
  p.res_planes = d.res ? std::max(1, d.res_planes) : 0;
  p.res_plane_stride = d.res_plane_stride;
  p.out = d.out;
  p.ld_out = d.ld_out;
  p.out_col_off = d.out_col_off;
  p.out_planes = d.out ? std::max(1, d.out_planes) : 0;
  p.out_plane_stride = d.out_plane_stride;
  p.out_f32 = d.out_f32;
  p.ld_out_f32 = d.ld_out_f32;
  p.act = d.act;
  const dim3 grid(static_cast<unsigned>((p.M + kTM - 1) / kTM), static_cast<unsigned>((d.N + kTN - 1) / kTN));
  return launch(conv_exact_kernel, grid, kThreadsExact, 0, stream, "conv_exact", p);
}

}  // namespace dcr
