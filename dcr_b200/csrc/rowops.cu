// Small HBM-bound row kernels around the similarity step.
//   l2_normalize : nn.functional.normalize(x, dim=1, p=2)            reference diff_retrieval.py:388-389
//   topk_merge   : merge per-shard top-k lists (score desc, index asc) reference-equivalent of running topk over
//                  the concatenated gallery; used after the all-gather of per-shard results (SURVEY 8e) and by the
//                  chunked search of embedding_search/similarity_search.py:70-74
#include "dcr_internal.cuh"
#include "host_util.cuh"

namespace dcr {

namespace {
constexpr uint32_t kFull = 0xffffffffu;

// one warp per row, float4 loads when d % 4 == 0
__global__ void l2_normalize_kernel(float* __restrict__ x, int n, int d, float eps) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < n; row += gridDim.x * wpb) {
    float* xr = x + static_cast<size_t>(row) * d;
    float s = 0.f;
    if ((d & 3) == 0) {
      for (int c = lane * 4; c < d; c += 128) {
        const float4 v = *reinterpret_cast<const float4*>(xr + c);
        s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      }
    } else {
      for (int c = lane; c < d; c += 32) s += xr[c] * xr[c];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(kFull, s, off);
    const float denom = fmaxf(sqrtf(s), eps);   // torch: x / max(||x||_2, eps)
    if ((d & 3) == 0) {
      for (int c = lane * 4; c < d; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(xr + c);
        v.x /= denom;
        v.y /= denom;
        v.z /= denom;
        v.w /= denom;
        *reinterpret_cast<float4*>(xr + c) = v;
      }
    } else {
      for (int c = lane; c < d; c += 32) xr[c] /= denom;
    }
  }
}

// one warp per query; nlists*k_in <= 1024 entries are ranked by counting (score desc, idx asc); idx < 0 = empty
__global__ void topk_merge_kernel(const float* __restrict__ scores, const long long* __restrict__ idx, int nq,
                                  int nlists, int k_in, int k_out, float* __restrict__ out_scores,
                                  long long* __restrict__ out_idx) {
  extern __shared__ __align__(16) uint8_t sm[];
  const int wpb = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = nlists * k_in;
  float* s_s = reinterpret_cast<float*>(sm) + static_cast<size_t>(warp) * m;
  long long* s_i = reinterpret_cast<long long*>(sm + ((static_cast<size_t>(wpb) * m * 4 + 15) & ~size_t(15))) +
                   static_cast<size_t>(warp) * m;
  for (int q = blockIdx.x * wpb + warp; q < nq; q += gridDim.x * wpb) {
    for (int e = lane; e < m; e += 32) {
      const int l = e / k_in, j = e % k_in;
      const size_t src = (static_cast<size_t>(l) * nq + q) * k_in + j;   // layout [nlists][nq][k_in]
      s_s[e] = scores[src];
      s_i[e] = idx[src];
    }
    // fewer than k_out valid entries (a total gallery smaller than k): the remaining slots are (-inf, -1)
    for (int r = lane; r < k_out; r += 32) {
      out_scores[static_cast<size_t>(q) * k_out + r] = -INFINITY;
      out_idx[static_cast<size_t>(q) * k_out + r] = -1;
    }
    __syncwarp();
    for (int e = lane; e < m; e += 32) {
      const float se_raw = s_s[e];
      const float se = (se_raw != se_raw) ? -INFINITY : se_raw;   // NaN orders last; ranks stay a permutation
      const long long ie = s_i[e];
      if (ie < 0) continue;
      int rank = 0;
      for (int o = 0; o < m; ++o) {
        const float so_raw = s_s[o];
        const float so = (so_raw != so_raw) ? -INFINITY : so_raw;
        const long long io = s_i[o];
        // total order: score desc, index asc, list position asc (duplicate (score, index) pairs do not collide)
        rank += (io >= 0) && ((so > se) || (so == se && (io < ie || (io == ie && o < e))));
      }
      if (rank < k_out) {
        out_scores[static_cast<size_t>(q) * k_out + rank] = se_raw;
        out_idx[static_cast<size_t>(q) * k_out + rank] = ie;
      }
    }
    __syncwarp();
  }
}
__global__ void pad_topk_lists_kernel(const float* __restrict__ s_in, const long long* __restrict__ i_in, int nq, int k_in, int k_out,
                                      float* __restrict__ s_out, long long* __restrict__ i_out) {
  const long long total = static_cast<long long>(nq) * k_out;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(t / k_out), j = static_cast<int>(t % k_out);
    s_out[t] = j < k_in ? s_in[static_cast<size_t>(q) * k_in + j] : -INFINITY;
    i_out[t] = j < k_in ? i_in[static_cast<size_t>(q) * k_in + j] : -1;
  }
}
}  // namespace

int pad_topk_lists(const float* s_in, const long long* i_in, int nq, int k_in, int k_out, float* s_out, long long* i_out,
                   cudaStream_t stream) {
  DCR_REQUIRE(nq >= 1 && k_in >= 1 && k_out >= k_in, "pad_topk_lists: bad arguments");
  const long long total = static_cast<long long>(nq) * k_out;
  return launch(pad_topk_lists_kernel, static_cast<int>(std::min<long long>((total + 255) / 256, 1184)), 256, 0, stream,
                "pad_topk_lists", s_in, i_in, nq, k_in, k_out, s_out, i_out);
}

int l2_normalize(float* x, int n, int d, float eps, cudaStream_t stream) {
  DCR_REQUIRE(n >= 0 && d >= 1, "l2_normalize: bad shape (%d,%d)", n, d);
  if (n == 0) return 0;
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  const int blocks = std::min((n + 7) / 8, di->num_sms * 8);
  return launch(l2_normalize_kernel, blocks, 256, 0, stream, "l2_normalize", x, n, d, eps);
}

int topk_merge(const float* scores, const long long* idx, int nq, int nlists, int k_in, int k_out, float* out_scores,
               long long* out_idx, cudaStream_t stream) {
  DCR_REQUIRE(nq >= 0 && nlists >= 1 && k_in >= 1 && k_out >= 1, "topk_merge: bad arguments");
  DCR_REQUIRE(k_out <= nlists * k_in, "topk_merge: k_out=%d > %d available", k_out, nlists * k_in);
  DCR_REQUIRE(nlists * k_in <= 1024, "topk_merge: nlists*k_in=%d > 1024", nlists * k_in);
  if (nq == 0) return 0;
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  const int wpb = 4;
  const int m = nlists * k_in;
  const size_t smem = ((static_cast<size_t>(wpb) * m * 4 + 15) & ~size_t(15)) + static_cast<size_t>(wpb) * m * 8;
  const int blocks = std::min((nq + wpb - 1) / wpb, di->num_sms * 8);
  return launch(topk_merge_kernel, blocks, wpb * 32, smem, stream, "topk_merge", scores, idx, nq, nlists, k_in, k_out,
                out_scores, out_idx);
}

}  // namespace dcr
