// Input kernels of the descriptor networks: the image batch -> the first layer's operand.  Each kernel owns only its
// output layout; every value comes from SourceRow::sample (image_in.cuh), which holds the transform.
#include <cuda_bf16.h>

#include <type_traits>

#include "dcr_internal.cuh"
#include "host_util.cuh"
#include "image_in.cuh"
#include "planes.cuh"

namespace dcr {
namespace {

// ---- im2col rows of the first (3-channel) convolution / patch embedding (ViT, CLIP, VGG, Inception) -------------
// out[m, k], m = (b, p, q) over the OHxOW output grid; K layout k = r * RP + s * 3 + c with RP = ceil8(3 * KW) (each
// filter row padded to a multiple of 8 elements so that a thread owns whole 16-byte groups and every (s, c) index is a
// compile-time constant), zero for k >= kh * RP and for taps in the zero padding.  One thread per (output pixel, filter
// row).
struct Im2colParams {
  ImageSource src;
  __nv_bfloat16* out;
  long long out_plane_stride;
  int planes;
  int B, kh, stride, pad, OH, OW, k_pad;
};

template <int KW, bool kF32, bool kResize>
__global__ void __launch_bounds__(256) im2col_u8_kernel(const Im2colParams p) {
  constexpr int RP = (3 * KW + 7) / 8 * 8;
  __shared__ float lut[3][256];
  p.src.fill_lut(lut);
  const int rows_k = (p.k_pad + RP - 1) / RP;   // kh filter rows + zero rows up to k_pad (the last one may be partial)
  const long long total = static_cast<long long>(p.B) * p.OH * p.OW * rows_k;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i % rows_k);
    const long long m = i / rows_k;
    const int q = static_cast<int>(m % p.OW);
    const int pp = static_cast<int>((m / p.OW) % p.OH);
    const int b = static_cast<int>(m / (static_cast<long long>(p.OW) * p.OH));
    const int y = pp * p.stride - p.pad + r;
    const int x0 = q * p.stride - p.pad;
    const bool row_ok = r < p.kh && y >= 0 && y < p.src.RH;
    const SourceRow<kF32, kResize> row(p.src, b, y);
    __nv_bfloat16* dst = p.out + static_cast<size_t>(m) * p.k_pad + r * RP;
#pragma unroll
    for (int g = 0; g < RP / 8; ++g) {
      if (r * RP + g * 8 >= p.k_pad) break;   // partial last zero row (k_pad is a multiple of 8, not always of RP)
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int j = g * 8 + e;          // compile-time after unrolling
        const int s = j / 3, c = j % 3;
        float val = 0.f;
        if (j < 3 * KW && row_ok && x0 + s >= 0 && x0 + s < p.src.RW) val = row.sample(lut, x0 + s, c);
        v[e] = val;
      }
      store8(dst, p.out_plane_stride, p.planes, g * 8, v);
    }
  }
}

// ---- space-to-depth input of the ResNet stem (7x7 / stride 2 / pad 3), parity modes and stem="s2d" ------------------
// Z[b, u, v, (i*2+j)*3 + c] = xn[2u + i - 3, 2v + j - 3, c]  (zero outside the image), channels 12..15 = 0, with xn the
// transformed network input.  A 7x7/2 convolution of xn equals a 4x4/1 convolution of Z (weights regrouped on the host),
// which the GEMM kernel reads through an overlapping-window tensor map -- no im2col matrix in HBM.
struct StemS2dParams {
  ImageSource src;
  int B, U, V;
  __nv_bfloat16* out;
  long long out_plane_stride;
  int planes;
};

// 6 blocks per SM (40 registers), the parent's occupancy for the common forms, without spills in any form
template <bool kF32, bool kResize>
__global__ void __launch_bounds__(256, 6) stem_s2d_u8_kernel(const StemS2dParams p) {
  __shared__ float lut[3][256];
  p.src.fill_lut(lut);
  const long long total = static_cast<long long>(p.B) * p.U * p.V;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(idx % p.V);
    const int u = static_cast<int>((idx / p.V) % p.U);
    const int b = static_cast<int>(idx / (static_cast<long long>(p.V) * p.U));
    float z[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) z[e] = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int y = 2 * u + i - 3;
      if (y < 0 || y >= p.src.RH) continue;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int x = 2 * v + j - 3;
        if (x < 0 || x >= p.src.RW) continue;
        const SourceRow<kF32, kResize> row(p.src, b, y);   // per tap: built per row, the resizing forms spill
#pragma unroll
        for (int c = 0; c < 3; ++c) z[(i * 2 + j) * 3 + c] = row.sample(lut, x, c);
      }
    }
    float lo[8], hi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      lo[e] = z[e];
      hi[e] = z[8 + e];
    }
    store8(p.out, p.out_plane_stride, p.planes, static_cast<size_t>(idx) * 16, lo);
    store8(p.out, p.out_plane_stride, p.planes, static_cast<size_t>(idx) * 16 + 8, hi);
  }
}

// ---- column-parity planes of the fused Toeplitz stem (stem_fused.cu), fast mode -------------------------------------
// With ip the zero-padded (3 pixels) network input: plane_e[P * PW + u] = { ip[2P + i][2u + e][c] : i in {0,1},
// c in {0,1,2} } + 2 zero channels, one 16-byte unit of 8 bf16.
struct StemRowsParams {
  ImageSource src;
  int B;
  __nv_bfloat16* out;
  long long img_stride, plane_stride;
  int PW, rows;     // units per pair-row, pair-rows written (OH + 3)
};

template <bool kF32, bool kResize>
__global__ void __launch_bounds__(256) stem_rows_kernel(const StemRowsParams p) {
  __shared__ float lut[3][256];
  p.src.fill_lut(lut);
  const long long per_img = 2ll * p.rows * p.PW;
  const long long total = per_img * p.B;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(idx / per_img);
    long long rem = idx - b * per_img;
    const int e = static_cast<int>(rem / (static_cast<long long>(p.rows) * p.PW));
    rem -= static_cast<long long>(e) * p.rows * p.PW;
    const int P = static_cast<int>(rem / p.PW), u = static_cast<int>(rem % p.PW);
    float z[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) z[k] = 0.f;
    const int x = 2 * u + e - 3;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int y = 2 * P + i - 3;
      if (y < 0 || y >= p.src.RH || x < 0 || x >= p.src.RW) continue;
      const SourceRow<kF32, kResize> row(p.src, b, y);
#pragma unroll
      for (int c = 0; c < 3; ++c) z[i * 3 + c] = row.sample(lut, x, c);
    }
    __nv_bfloat16* dst = p.out + static_cast<size_t>(b) * p.img_stride + static_cast<size_t>(e) * p.plane_stride +
                         (static_cast<size_t>(P) * p.PW + u) * 8;
    store8(dst, 0, 1, 0, z);   // one plane: the packed unit
  }
}

// Returns body(kF32, kResize), both std::bool_constant, for the form of the source.
template <class Body>
int with_source_form(const ImageSource& s, Body&& body) {
  if (s.img_f32) {
    if (s.rscale == 0.f) return body(std::true_type{}, std::false_type{});
    return body(std::true_type{}, std::true_type{});
  }
  if (s.rscale == 0.f) return body(std::false_type{}, std::false_type{});
  return body(std::false_type{}, std::true_type{});
}

template <int KW>
int launch_im2col(const Im2colParams& p, int grid, cudaStream_t stream) {
  return with_source_form(p.src, [&](auto f32, auto resize) {
    return launch(im2col_u8_kernel<KW, f32, resize>, grid, 256, 0, stream, "im2col_u8", p);
  });
}

}  // namespace

int im2col_u8(const ImageSource& src, int B, int kh, int kw, int stride, int pad, int k_pad, __nv_bfloat16* out,
              long long out_plane_stride, int planes, cudaStream_t stream) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  const int rp = (3 * kw + 7) / 8 * 8;
  DCR_REQUIRE(k_pad % 8 == 0 && k_pad >= kh * rp, "im2col_u8: k_pad %d must be a multiple of 8 and >= %d", k_pad, kh * rp);
  DCR_REQUIRE(kw == 3 || kw == 7 || kw == 8 || kw == 14 || kw == 16, "im2col_u8: filter width %d not instantiated (3, 7, 8, 14, 16)", kw);
  DCR_REQUIRE(src.RH >= kh && src.RW >= kw, "im2col_u8: network input %d x %d smaller than the filter", src.RH, src.RW);
  if (B == 0) return 0;
  Im2colParams p;
  p.src = src; p.B = B; p.kh = kh; p.stride = stride; p.pad = pad; p.k_pad = k_pad;
  p.OH = (src.RH + 2 * pad - kh) / stride + 1;
  p.OW = (src.RW + 2 * pad - kw) / stride + 1;
  p.out = out; p.out_plane_stride = out_plane_stride; p.planes = planes;
  const int grid = grid_for(static_cast<long long>(B) * p.OH * p.OW * ((k_pad + rp - 1) / rp), 256, di->num_sms);
  if (kw == 7) return launch_im2col<7>(p, grid, stream);
  if (kw == 3) return launch_im2col<3>(p, grid, stream);
  if (kw == 8) return launch_im2col<8>(p, grid, stream);
  if (kw == 14) return launch_im2col<14>(p, grid, stream);
  return launch_im2col<16>(p, grid, stream);
}

int stem_s2d_u8(const ImageSource& src, int B, __nv_bfloat16* out, long long out_plane_stride, int planes,
                cudaStream_t stream) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  DCR_REQUIRE(src.RH >= 2 && src.RW >= 2 && src.RH % 2 == 0 && src.RW % 2 == 0,
              "stem_s2d_u8: network input size must be even (%d x %d)", src.RH, src.RW);
  if (B == 0) return 0;
  StemS2dParams p;
  p.src = src; p.B = B;
  p.U = (src.RH + 6) / 2; p.V = (src.RW + 6) / 2;
  p.out = out; p.out_plane_stride = out_plane_stride; p.planes = planes;
  const int grid = grid_for(static_cast<long long>(B) * p.U * p.V, 256, di->num_sms);
  return with_source_form(src, [&](auto f32, auto resize) {
    return launch(stem_s2d_u8_kernel<f32, resize>, grid, 256, 0, stream, "stem_s2d_u8", p);
  });
}

int stem_rows(const ImageSource& src, int B, __nv_bfloat16* out, cudaStream_t stream) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  DCR_REQUIRE(src.RH >= 2 && src.RW >= 2 && src.RH % 2 == 0 && src.RW % 2 == 0,
              "stem_rows: network input size must be even (%d x %d)", src.RH, src.RW);
  if (B == 0) return 0;
  StemRowsParams p;
  p.src = src; p.B = B; p.out = out;
  const int OH = src.RH / 2, OW = src.RW / 2;
  p.PW = stem_fused_pitch(OW);
  p.rows = OH + 3;
  p.plane_stride = stem_fused_plane_units(OH, OW) * 8;
  p.img_stride = 2 * p.plane_stride;
  const int grid = grid_for(2ll * p.rows * p.PW * B, 256, di->num_sms);
  return with_source_form(src, [&](auto f32, auto resize) {
    return launch(stem_rows_kernel<f32, resize>, grid, 256, 0, stream, "stem_rows", p);
  });
}

}  // namespace dcr
