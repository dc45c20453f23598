// The input transform of the descriptor networks, shared by the three input kernels (image_in.cu): raw uint8 HWC
// pixels -> centre crop, ToTensor, Normalize, optional post affine -> optional bilinear resize, or an fp32 NCHW batch
// the caller has already transformed (then only the post affine is applied).
//
// Reference ops replaced:
//   diff_retrieval.py:325-330  Resize(256)/CenterCrop(224)/ToTensor/Normalize
//   embedding_search/utils.py:35-50 (ImageNet mean/std variant)
//   metrics/fid.py:104-110 + metrics/inception.py:152-153 (normalise twice: the post affine 2x-1)
//   utils_ret.py:676-698 `multi_scale`: F.interpolate(x, scale_factor=s, mode='bilinear', align_corners=False)
#pragma once
#include <cstddef>
#include <cstdint>
#include <type_traits>

namespace dcr {

// Trivially copyable, passed to the kernels inside their parameter structs.  Built and checked (crop inside the image,
// RH, RW resolved) by net.cu's input_source.
struct ImageSource {
  const uint8_t* img;     // uint8 HWC [B, IH, IW, 3], raw
  const float* img_f32;   // or fp32 NCHW [B, 3, IH, IW], already transformed (then img is unused)
  int IH, IW, crop_y, crop_x, H, W;   // H, W: size of the crop
  int RH, RW;                         // network input size: H, W, or the bilinearly resized crop (rscale != 0)
  float rscale;                       // float(1 / scale_factor), 0 = no resizing
  float mean[3], std[3], post_scale, post_shift;

  // u8 -> transformed value per channel, with the reference's arithmetic (ToTensor: u8/255, Normalize: (x-mean)/std, both
  // fp32 with IEEE division), then the post affine.  Called by every thread of the block; ends with __syncthreads().
  // (mean / std are selected, not indexed: an indexed mean[c] can make a local copy of the kernel parameters, and pointers
  // read from that copy lose their global address space.)
  __device__ __forceinline__ void fill_lut(float (&lut)[3][256]) const {
    for (int i = threadIdx.x; i < 768; i += blockDim.x) {
      const int c = i >> 8, u = i & 255;
      const float m = c == 0 ? mean[0] : (c == 1 ? mean[1] : mean[2]);
      const float s = c == 0 ? std[0] : (c == 1 ? std[1] : std[2]);
      const float val = (static_cast<float>(u) / 255.f - m) / s;
      lut[c][u] = post_scale * val + post_shift;
    }
    __syncthreads();
  }

  // transformed value of channel c of image b at crop coordinates (y, x)
  template <bool kF32>
  __device__ __forceinline__ float pixel(const float (&lut)[3][256], int b, int y, int x, int c) const {
    const size_t plane = static_cast<size_t>(IH) * IW;
    if constexpr (kF32) {
      const float* im = img_f32 + static_cast<size_t>(b) * 3 * plane;
      return fmaf(post_scale, im[c * plane + static_cast<size_t>(y + crop_y) * IW + (x + crop_x)], post_shift);
    } else {
      const uint8_t* im = img + static_cast<size_t>(b) * IH * IW * 3;
      return lut[c][im[(static_cast<size_t>(y + crop_y) * IW + (x + crop_x)) * 3 + c]];
    }
  }
};

// Bilinear source taps of output coordinate d along an axis of `size` source pixels, with torch's arithmetic: source
// index rscale * (d + 0.5) - 0.5 clamped to [0, size - 1]; value = h * v[i0] + l * v[i1].
struct Tap {
  int i0, i1;
  float l, h;
  __device__ __forceinline__ Tap(float rscale, int d, int size) {
    const float s = fmaxf(rscale * (static_cast<float>(d) + 0.5f) - 0.5f, 0.f);
    i0 = min(static_cast<int>(s), size - 1);
    i1 = i0 + (i0 < size - 1 ? 1 : 0);
    l = s - static_cast<float>(i0);
    h = 1.f - l;
  }
};

// Row y of image b of the network input (0 <= y < RH), set up once per row so that its samples share the vertical
// taps.  sample(lut, x, c) is the value the network sees at column x (0 <= x < RW), channel c.
template <bool kF32, bool kResize>
struct SourceRow {
  const ImageSource& src;
  int b, y;
  Tap ty;

  __device__ __forceinline__ SourceRow(const ImageSource& s, int b_, int y_) : src(s), b(b_), y(y_), ty(s.rscale, y_, s.H) {}

  __device__ __forceinline__ float sample(const float (&lut)[3][256], int x, int c) const {
    if constexpr (kResize) {
      // h * a + l * b as fmaf(h, a, l * b), written out: left to the compiler, which product it fuses depends on the
      // surrounding code, and the last bit of the result with it
      const auto lerp = [](float h, float a, float l, float b) { return fmaf(h, a, __fmul_rn(l, b)); };
      const Tap tx(src.rscale, x, src.W);
      return lerp(ty.h, lerp(tx.h, src.pixel<kF32>(lut, b, ty.i0, tx.i0, c), tx.l, src.pixel<kF32>(lut, b, ty.i0, tx.i1, c)),
                  ty.l, lerp(tx.h, src.pixel<kF32>(lut, b, ty.i1, tx.i0, c), tx.l, src.pixel<kF32>(lut, b, ty.i1, tx.i1, c)));
    } else {
      return src.pixel<kF32>(lut, b, y, x, c);
    }
  }
};

}  // namespace dcr
