#include "host_util.cuh"

#include <cstdlib>
#include <cstring>
#include <atomic>
#include <mutex>
#include <map>
#include <utility>

namespace dcr {

std::string& last_error_storage() {
  static thread_local std::string s;
  return s;
}

int set_error(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error_storage() = buf;
  return code;
}

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }

bool tuning_enabled() {
  const char* e = getenv("DCR_B200_TUNING");   // read per call: the tests switch it on and off inside one process
  return e != nullptr && e[0] == '1';
}
int tuning_int(const char* name, int dflt) {
  if (!tuning_enabled()) return dflt;
  const char* e = getenv(name);
  return (e && *e) ? atoi(e) : dflt;
}
bool tuning_flag(const char* name) { return tuning_enabled() && getenv(name) != nullptr; }

const DeviceInfo* device_info() {
  static DeviceInfo cache[64];
  static std::mutex mu;
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    set_error(-2, "cudaGetDevice failed (no CUDA device visible)");
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(mu);
  DeviceInfo& d = cache[dev];
  if (d.device != dev) {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
      set_error(-2, "cudaGetDeviceProperties failed");
      return nullptr;
    }
    d.device = dev;
    d.num_sms = prop.multiProcessorCount;
    d.cc_major = prop.major;
    d.cc_minor = prop.minor;
    d.max_smem_optin = prop.sharedMemPerBlockOptin;
  }
  return &d;
}

int require_sm90a(const DeviceInfo* di, const char* who) {
  DCR_REQUIRE(di->cc_major == 9 && di->cc_minor == 0, "%s: this build targets sm_90a; device reports sm_%d%d", who,
              di->cc_major, di->cc_minor);
  return 0;
}

int allow_dynamic_smem(const void* func, size_t bytes, const char* who) {
  // within the default 48 KB even next to 16 KB of static shared memory (the default counts both; no kernel here has more)
  if (bytes <= 32 * 1024) return 0;
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  static std::map<std::pair<const void*, int>, size_t> limits;   // (kernel, device) -> dynamic shared memory allowed
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  auto it = limits.find({func, di->device});
  if (it == limits.end()) {
    // the kernel's static shared memory counts against the device's opt-in maximum too
    cudaFuncAttributes fa;
    DCR_CUDA_CHECK(cudaFuncGetAttributes(&fa, func));
    const size_t limit = di->max_smem_optin - fa.sharedSizeBytes;
    DCR_CUDA_CHECK(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(limit)));
    it = limits.emplace(std::make_pair(func, di->device), limit).first;
  }
  DCR_REQUIRE(bytes <= it->second, "%s: %zu bytes of dynamic shared memory exceed the %zu the device allows this kernel", who,
              bytes, it->second);
  return 0;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                     const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static void* driver_fn(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_elems,
                      uint32_t box_rows, uint32_t box_cols) {
  static PFN_encodeTiled fn = reinterpret_cast<PFN_encodeTiled>(driver_fn("cuTensorMapEncodeTiled"));
  DCR_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  DCR_REQUIRE(box_cols * 2 == 128, "tensor-map box inner extent must be 128 bytes (got %u)", box_cols * 2);
  DCR_REQUIRE(box_rows >= 1 && box_rows <= 256, "tensor-map box rows out of range: %u", box_rows);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor-map base must be 16-byte aligned");
  DCR_REQUIRE((row_stride_elems * 2) % 16 == 0, "tensor-map row stride must be a multiple of 16 bytes");
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {row_stride_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DCR_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (rows=%llu cols=%llu box=%ux%u)",
              static_cast<int>(r), (unsigned long long)rows, (unsigned long long)cols, box_rows, box_cols);
  return 0;
}

int make_tmap_nhwc_box_bf16(CUtensorMap* out, const void* base, int n, int h, int w, int c, long long pixel_stride,
                            uint32_t box_w, uint32_t box_h) {
  static PFN_encodeTiled fn = reinterpret_cast<PFN_encodeTiled>(driver_fn("cuTensorMapEncodeTiled"));
  DCR_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor-map base must be 16-byte aligned");
  DCR_REQUIRE(box_w >= 1 && box_w <= 256 && box_h >= 1 && box_h <= 256, "tensor-map box out of range: %u x %u", box_w, box_h);
  DCR_REQUIRE((pixel_stride * 2) % 16 == 0, "tensor-map pixel stride must be a multiple of 16 bytes");
  cuuint64_t gdim[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t gstride[3] = {(cuuint64_t)pixel_stride * 2, (cuuint64_t)pixel_stride * 2 * w, (cuuint64_t)pixel_stride * 2 * w * h};
  cuuint32_t box[4] = {64, box_w, box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DCR_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (NHWC box) failed with CUresult %d (n=%d h=%d w=%d c=%d box=%ux%u)",
              static_cast<int>(r), n, h, w, c, box_w, box_h);
  return 0;
}

int make_tmap_im2col_bf16(CUtensorMap* out, const void* base, int n, int h, int w, int c, int pad_h, int pad_w,
                          int kh, int kw, int stride, int channels_per_pixel, int pixels_per_column,
                          long long stride_w, long long stride_h, long long stride_n) {
  static PFN_encodeIm2col fn = reinterpret_cast<PFN_encodeIm2col>(driver_fn("cuTensorMapEncodeIm2col"));
  DCR_REQUIRE(fn != nullptr, "cuTensorMapEncodeIm2col driver entry point not available");
  DCR_REQUIRE(channels_per_pixel * 2 == 128, "im2col box inner extent must be 128 bytes");
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor-map base must be 16-byte aligned");
  cuuint64_t gdim[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  if (stride_w == 0) stride_w = c;
  if (stride_h == 0) stride_h = static_cast<long long>(w) * c;
  if (stride_n == 0) stride_n = static_cast<long long>(h) * w * c;
  DCR_REQUIRE((stride_w * 2) % 16 == 0 && (stride_h * 2) % 16 == 0 && (stride_n * 2) % 16 == 0,
              "im2col tensor map: strides must be multiples of 16 bytes");
  cuuint64_t gstride[3] = {(cuuint64_t)stride_w * 2, (cuuint64_t)stride_h * 2, (cuuint64_t)stride_n * 2};
  // base-pixel bounding box: lower corner = -pad, upper corner = pad - (filter - 1)   {W, H} order
  int lower[2] = {-pad_w, -pad_h};
  int upper[2] = {pad_w - (kw - 1), pad_h - (kh - 1)};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstride, lower, upper,
                  (cuuint32_t)channels_per_pixel, (cuuint32_t)pixels_per_column, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DCR_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeIm2col failed with CUresult %d (nhwc=%d,%d,%d,%d k=%dx%d s=%d)",
              static_cast<int>(r), n, h, w, c, kh, kw, stride);
  return 0;
}

}  // namespace dcr
