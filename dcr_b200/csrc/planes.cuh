// 16-byte access to activation "planes": NHWC bf16 tensors stored as 1 plane (fast mode) or as a hi/mid/lo split whose
// sum carries fp32 precision (3 planes).  idx is an element index within a plane, a multiple of 8.
#pragma once
#include <cuda_bf16.h>

#include <cstddef>
#include <cstdint>

namespace dcr {

// v = sum of the planes at idx
__device__ __forceinline__ void load8(const __nv_bfloat16* base, long long plane_stride, int planes, size_t idx,
                                      float (&v)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = 0.f;
  for (int p = 0; p < planes; ++p) {
    const uint4 u = *reinterpret_cast<const uint4*>(base + p * plane_stride + idx);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[2 * j] += __uint_as_float(w[j] << 16);
      v[2 * j + 1] += __uint_as_float(w[j] & 0xffff0000u);
    }
  }
}

// splits v over the planes: each plane stores the bf16 rounding of what the previous ones left (v is consumed)
__device__ __forceinline__ void store8(__nv_bfloat16* base, long long plane_stride, int planes, size_t idx,
                                       float (&v)[8]) {
  for (int p = 0; p < planes; ++p) {
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat16 a = __float2bfloat16_rn(v[2 * j]), b = __float2bfloat16_rn(v[2 * j + 1]);
      w[j] = static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
      v[2 * j] -= __bfloat162float(a);
      v[2 * j + 1] -= __bfloat162float(b);
    }
    *reinterpret_cast<uint4*>(base + p * plane_stride + idx) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

}  // namespace dcr
