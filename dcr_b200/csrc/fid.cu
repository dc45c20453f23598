// Streaming FID activation statistics on the device (float64).
// Replaces   pred_arr[...] = pred  (float64 [N,2048] on the host, metrics/fid.py:118,135) followed by
//            mu = np.mean(act, axis=0); sigma = np.cov(act, rowvar=False)      metrics/fid.py:219-220
// The [N, d] activation matrix is never kept: every batch is folded into  s = sum(x - c)  and  S = (x-c)^T (x-c)
// (c = mean of the first batch, a fixed shift that removes the cancellation of the one-pass formula), and
//   mu = c + s/n,   sigma = (S - s s^T / n) / (n - 1)        (unbiased, as np.cov)
// Roofline: 2*n*d^2 fp64 FLOP (0.42 TFLOP per 50k x 2048 set) on the fp64 pipe; the upper triangle only is computed.
#include <vector>

#include "dcr_internal.cuh"
#include "host_util.cuh"

namespace dcr {

struct FidState {
  int d = 0;
  long long n = 0;
  double* shift = nullptr;   // [d]
  double* sum = nullptr;     // [d]
  double* xtx = nullptr;     // [d, d], upper-triangular tiles valid
};

namespace {
constexpr int kTile = 64;
constexpr int kRows = 32;

__global__ void fid_shift_kernel(const float* __restrict__ x, int n, int d, double* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= d) return;
  double s = 0.0;
  for (int r = 0; r < n; ++r) s += static_cast<double>(x[static_cast<size_t>(r) * d + c]);
  shift[c] = s / n;
}

// grid (d/64, d/64) upper triangle, 256 threads, each thread a 4x4 block of the 64x64 tile
__global__ void __launch_bounds__(256)
    fid_accumulate_kernel(const float* __restrict__ x, int n, int d, const double* __restrict__ shift,
                          double* __restrict__ sum, double* __restrict__ xtx) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (tj < ti) return;
  __shared__ double a[kRows][kTile + 1];
  __shared__ double b[kRows][kTile + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4] = {};
  double colsum = 0.0;   // diagonal tiles, threads 0..63: column sums
  for (int r0 = 0; r0 < n; r0 += kRows) {
    for (int i = threadIdx.x; i < kRows * kTile; i += 256) {
      const int r = i / kTile, c = i % kTile;
      const bool ok = r0 + r < n;
      const int ca = ti * kTile + c, cb = tj * kTile + c;
      a[r][c] = (ok && ca < d) ? static_cast<double>(x[static_cast<size_t>(r0 + r) * d + ca]) - shift[ca] : 0.0;
      b[r][c] = (ok && cb < d) ? static_cast<double>(x[static_cast<size_t>(r0 + r) * d + cb]) - shift[cb] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < kRows; ++r) {
      double av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        av[i] = a[r][ty * 4 + i];
        bv[i] = b[r][tx * 4 + i];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(av[i], bv[j], acc[i][j]);
    }
    if (ti == tj && threadIdx.x < kTile)
      for (int r = 0; r < kRows; ++r) colsum += a[r][threadIdx.x];
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int row = ti * kTile + ty * 4 + i, col = tj * kTile + tx * 4 + j;
      if (row < d && col < d) xtx[static_cast<size_t>(row) * d + col] += acc[i][j];   // one block owns the tile
    }
  if (ti == tj && threadIdx.x < kTile && ti * kTile + threadIdx.x < d) sum[ti * kTile + threadIdx.x] += colsum;
}

// Packed state (include/dcr_b200.h): int64 header {kPackedMagic, d, n, 0}, then double shift[d], sum[d], xtx[d*d].
constexpr long long kPackedMagic = 0x31444946524344LL;   // "DCRFID1"
constexpr int kHeaderWords = 4;

__host__ __device__ inline const double* packed_shift(const unsigned char* p) {
  return reinterpret_cast<const double*>(p + kHeaderWords * sizeof(long long));
}

// Folds `count` packed states into (shift, sum, xtx) in order, one thread per element (i, j >= i) of the triangle.
// n_state: the state's count before the fold.  When it is 0, the first non-empty peer is copied (its shift included)
// and later peers are rebased onto that shift, so no thread reads `shift` then and the diagonal threads may write it.
// Every element sees the peers in the same fixed order: the result does not depend on scheduling.
__global__ void fid_merge_kernel(const unsigned char* __restrict__ packed, size_t stride, int count, int d,
                                 long long n_state, double* __restrict__ shift, double* __restrict__ sum,
                                 double* __restrict__ xtx) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<size_t>(d) * d) return;
  const int i = static_cast<int>(e / d), j = static_cast<int>(e % d);
  if (j < i) return;
  long long na = n_state;
  double ci = 0.0, cj = 0.0, si = 0.0, sij = 0.0;
  if (na > 0) {
    ci = shift[i];
    cj = shift[j];
    si = sum[i];
    sij = xtx[e];
  }
  for (int p = 0; p < count; ++p) {
    const unsigned char* b = packed + static_cast<size_t>(p) * stride;
    const long long nb = reinterpret_cast<const long long*>(b)[2];
    if (nb == 0) continue;
    const double* cb = packed_shift(b);
    const double* sb = cb + d;
    const double* xb = sb + d;
    if (na == 0) {
      ci = cb[i];
      cj = cb[j];
      si = sb[i];
      sij = xb[e];
    } else {
      // delta = c_a - c_b:  S_a += S_b - s_b delta^T - delta s_b^T + n_b delta delta^T,  s_a += s_b - n_b delta
      const double di = ci - cb[i], dj = cj - cb[j], sbi = sb[i], sbj = sb[j], fn = static_cast<double>(nb);
      sij += xb[e] - sbi * dj - di * sbj + fn * di * dj;
      si += sbi - fn * di;
    }
    na += nb;
  }
  xtx[e] = sij;
  if (i == j) {
    sum[i] = si;
    if (n_state == 0) shift[i] = ci;
  }
}
}  // namespace

size_t fid_packed_size(int d) {
  if (d < 1 || d > 16384) return 0;
  return kHeaderWords * sizeof(long long) + sizeof(double) * (2 * static_cast<size_t>(d) + static_cast<size_t>(d) * d);
}

int fid_export(const FidState* s, void* packed, cudaStream_t stream) {
  DCR_REQUIRE(s && packed, "fid_export: null argument");
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 7) == 0, "fid_export: packed buffer must be 8-byte aligned");
  const int d = s->d;
  const long long hdr[kHeaderWords] = {kPackedMagic, d, s->n, 0};
  unsigned char* p = static_cast<unsigned char*>(packed);
  double* shift = reinterpret_cast<double*>(p + kHeaderWords * sizeof(long long));
  // pageable source: the copy has been staged when the call returns, so `hdr` may go out of scope
  DCR_CUDA_CHECK(cudaMemcpyAsync(p, hdr, sizeof(hdr), cudaMemcpyHostToDevice, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(shift, s->shift, sizeof(double) * d, cudaMemcpyDeviceToDevice, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(shift + d, s->sum, sizeof(double) * d, cudaMemcpyDeviceToDevice, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(shift + 2 * d, s->xtx, sizeof(double) * d * d, cudaMemcpyDeviceToDevice, stream));
  return 0;
}

int fid_merge(FidState* s, const void* packed, int count, cudaStream_t stream) {
  DCR_REQUIRE(s && (packed || count == 0), "fid_merge: null argument");
  DCR_REQUIRE(count >= 0, "fid_merge: bad count %d", count);
  if (count == 0) return 0;
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 7) == 0, "fid_merge: packed buffer must be 8-byte aligned");
  const int d = s->d;
  const size_t stride = fid_packed_size(d);
  // the headers: one strided device-to-host copy, so that the state's host-side count is right on return
  std::vector<long long> hdr(static_cast<size_t>(count) * kHeaderWords);
  DCR_CUDA_CHECK(cudaMemcpy2DAsync(hdr.data(), kHeaderWords * sizeof(long long), packed, stride,
                                   kHeaderWords * sizeof(long long), count, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  long long n = s->n;
  for (int p = 0; p < count; ++p) {
    const long long* h = &hdr[static_cast<size_t>(p) * kHeaderWords];
    DCR_REQUIRE(h[0] == kPackedMagic, "fid_merge: packed state %d is not an exported dcr_fid state", p);
    DCR_REQUIRE(h[1] == d, "fid_merge: packed state %d has d = %lld, this state has d = %d", p, h[1], d);
    DCR_REQUIRE(h[2] >= 0, "fid_merge: packed state %d has a negative count %lld", p, h[2]);
    n += h[2];
  }
  if (n == s->n) return 0;   // only empty states
  const size_t elems = static_cast<size_t>(d) * d;
  fid_merge_kernel<<<static_cast<unsigned>((elems + 255) / 256), 256, 0, stream>>>(
      static_cast<const unsigned char*>(packed), stride, count, d, s->n, s->shift, s->sum, s->xtx);
  count_launch();
  DCR_CUDA_CHECK(cudaGetLastError());
  s->n = n;
  return 0;
}

int fid_create(int d, FidState** out) {
  DCR_REQUIRE(d >= 1 && d <= 16384, "fid_create: bad dim %d", d);
  if (!device_info()) return -2;
  FidState* s = new FidState();
  s->d = d;
  DCR_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&s->shift), sizeof(double) * d));
  DCR_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&s->sum), sizeof(double) * d));
  DCR_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&s->xtx), sizeof(double) * d * d));
  DCR_CUDA_CHECK(cudaMemset(s->sum, 0, sizeof(double) * d));
  DCR_CUDA_CHECK(cudaMemset(s->xtx, 0, sizeof(double) * d * d));
  *out = s;
  return 0;
}

void fid_destroy(FidState* s) {
  if (!s) return;
  cudaFree(s->shift);
  cudaFree(s->sum);
  cudaFree(s->xtx);
  delete s;
}

int fid_accumulate(FidState* s, const float* act, int n, cudaStream_t stream) {
  DCR_REQUIRE(s && act, "fid_accumulate: null argument");
  if (n <= 0) return 0;
  if (s->n == 0) {
    fid_shift_kernel<<<(s->d + 127) / 128, 128, 0, stream>>>(act, n, s->d, s->shift);
    count_launch();
  }
  const int t = (s->d + kTile - 1) / kTile;
  fid_accumulate_kernel<<<dim3(t, t), 256, 0, stream>>>(act, n, s->d, s->shift, s->sum, s->xtx);
  count_launch();
  DCR_CUDA_CHECK(cudaGetLastError());
  s->n += n;
  return 0;
}

int fid_finalize(FidState* s, double* mu_host, double* sigma_host, long long* n_out, cudaStream_t stream) {
  DCR_REQUIRE(s && mu_host && sigma_host, "fid_finalize: null argument");
  DCR_REQUIRE(s->n >= 2, "fid_finalize: need at least 2 samples (have %lld)", s->n);
  const int d = s->d;
  std::vector<double> shift(d), sum(d);
  DCR_CUDA_CHECK(cudaMemcpyAsync(shift.data(), s->shift, sizeof(double) * d, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(sum.data(), s->sum, sizeof(double) * d, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaMemcpyAsync(sigma_host, s->xtx, sizeof(double) * d * d, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  const double n = static_cast<double>(s->n);
  for (int i = 0; i < d; ++i) mu_host[i] = shift[i] + sum[i] / n;
  for (int i = 0; i < d; ++i)
    for (int j = i; j < d; ++j) {
      const double v = (sigma_host[static_cast<size_t>(i) * d + j] - sum[i] * sum[j] / n) / (n - 1.0);
      sigma_host[static_cast<size_t>(i) * d + j] = v;
      sigma_host[static_cast<size_t>(j) * d + i] = v;
    }
  if (n_out) *n_out = s->n;
  return 0;
}

}  // namespace dcr
