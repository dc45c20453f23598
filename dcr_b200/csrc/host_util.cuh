// Host-side helpers shared by the .cu translation units: error capture for the C ABI, the driver entry point
// for tensor-map encoding (no link-time dependency on libcuda), SM count cache, kernel launches.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>
#include <utility>

namespace dcr {

// last error message, per host thread (returned by dcr_last_error()).
std::string& last_error_storage();
int set_error(int code, const char* fmt, ...);

#define DCR_CUDA_CHECK(expr)                                                                           \
  do {                                                                                                 \
    cudaError_t _e = (expr);                                                                           \
    if (_e != cudaSuccess)                                                                             \
      return ::dcr::set_error(-2, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define DCR_REQUIRE(cond, ...)                        \
  do {                                                \
    if (!(cond)) return ::dcr::set_error(-1, __VA_ARGS__); \
  } while (0)

struct DeviceInfo {
  int device = -1;
  int num_sms = 0;
  int cc_major = 0, cc_minor = 0;
  size_t max_smem_optin = 0;
};
// cumulative number of kernels this library has launched (all threads)
void count_launch(int n = 1);
long long launch_count();

// Test switches: they exist so that the tests can run a second path on the same input and compare it with the one the
// library picks.  They are DCR_ATTN_FP32, DCR_LN_GENERIC, DCR_POOL_GENERIC, DCR_NO_BLOCK_FUSION, DCR_SIM_RESCORE_BLOCK,
// DCR_CONV_NO_HALO, DCR_GEMM_DIRECT_EPILOGUE and DCR_GEMM_TILE_ORDER, and they are honoured ONLY when DCR_B200_TUNING=1
// is set in the environment: a stray variable cannot change what a benchmark or a user's run computes.  Every other
// choice of path is made from the problem and the device.
bool tuning_enabled();
int tuning_int(const char* name, int dflt);
bool tuning_flag(const char* name);   // true when tuning is enabled and the variable is set (to anything)

// cached per current device; returns nullptr and sets the error on failure
const DeviceInfo* device_info();

// 0 on an sm_90 device, else -1 with an error naming `who`: the tensor-core kernels are built for sm_90a only
int require_sm90a(const DeviceInfo* di, const char* who);

// Lets `func` be launched with `bytes` of dynamic shared memory on the current device.  Above 32 KB (the default 48 KB
// counts static shared memory too) the kernel's limit is raised to the most the device allows it (the opt-in maximum less its static shared memory), once per
// (kernel, device), so every later size is covered; more than that is refused (-1, naming `who`).
int allow_dynamic_smem(const void* func, size_t bytes, const char* who);

// kern<<<grid, block, smem, stream>>>(args...) after allow_dynamic_smem, counted, with a launch error named after `who`
template <class... Params, class... Args>
int launch(void (*kern)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, const char* who,
           Args&&... args) {
  if (int rc = allow_dynamic_smem(reinterpret_cast<const void*>(kern), smem, who)) return rc;
  kern<<<grid, block, smem, stream>>>(std::forward<Args>(args)...);
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(-2, "%s: kernel launch failed: %s", who, cudaGetErrorString(e));
  return 0;
}

// Cuts a workspace into buffers, each 256-byte aligned on its own, so the size does not depend on their order.  A
// planner runs the same code as its entry point on a null base: `bytes` is then the workspace size it reports.
struct Carve {
  uint8_t* base = nullptr;
  size_t bytes = 0;
  template <class T>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += (count * sizeof(T) + 255) / 256 * 256;
    return p;
  }
};

// blocks for a grid-stride loop over work_items: one item per thread, at most 16 blocks per SM
inline int grid_for(long long work_items, int block, int num_sms) {
  const long long blocks = (work_items + block - 1) / block;
  return static_cast<int>(blocks < 16ll * num_sms ? blocks : 16ll * num_sms);
}

// 2-D row-major bf16 tensor [rows, cols] (cols contiguous), box = [box_rows, box_cols], 128-byte swizzle.
// box_cols * 2 bytes must be 128.
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_elems,
                      uint32_t box_rows, uint32_t box_cols);

// im2col tensor map over an NHWC bf16 activation tensor (see conv_gemm.cu)
// stride_w/h/n: element strides of the (possibly overlapping-window) NHWC view; 0 = dense
// 4-D tiled map over an NHWC bf16 tensor (dims C, W, H, N; `pixel_stride` elements between pixels), box = 64 channels x
// box_w x box_h x 1 image, 128B swizzle, out-of-bounds elements read as zero / are not written.
int make_tmap_nhwc_box_bf16(CUtensorMap* out, const void* base, int n, int h, int w, int c, long long pixel_stride,
                            uint32_t box_w, uint32_t box_h);
int make_tmap_im2col_bf16(CUtensorMap* out, const void* base, int n, int h, int w, int c, int pad_h, int pad_w,
                          int kh, int kw, int stride, int channels_per_pixel, int pixels_per_column,
                          long long stride_w = 0, long long stride_h = 0, long long stride_n = 0);

}  // namespace dcr
