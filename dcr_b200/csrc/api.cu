// C-ABI entry points (include/dcr_b200.h).  Thin: argument checks + dispatch into the dcr:: functions.
#include <cstring>

#include "../../include/dcr_b200.h"
#include "dcr_internal.cuh"
#include "host_util.cuh"

namespace {
thread_local dcr::SimStats g_last_stats = {};
inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }
}  // namespace

extern "C" {

int dcr_version(void) { return DCR_B200_VERSION; }

const char* dcr_last_error(void) { return dcr::last_error_storage().c_str(); }

int dcr_device_sm_count(void) {
  const dcr::DeviceInfo* di = dcr::device_info();
  return di ? di->num_sms : -2;
}

int dcr_l2_normalize(float* x, int n, int d, float eps, void* stream) {
  DCR_REQUIRE(x != nullptr || n == 0, "dcr_l2_normalize: null pointer");
  return dcr::l2_normalize(x, n, d, eps, as_stream(stream));
}

size_t dcr_sim_topk_workspace_size(int nq, int ng, int d, int k) { return dcr::sim_topk_workspace_size(nq, ng, d, k); }

int dcr_sim_topk(const float* q, int nq, const float* g, int ng, int d, int k, int64_t g_index_base,
                 int64_t g_index_stride, float* out_scores, int64_t* out_idx, void* workspace, size_t workspace_bytes,
                 void* stream) {
  DCR_REQUIRE(q && g && out_scores && out_idx, "dcr_sim_topk: null pointer argument");
  static_assert(sizeof(long long) == sizeof(int64_t), "int64 layout");
  return dcr::sim_topk(q, nq, g, ng, d, k, g_index_base, g_index_stride, out_scores,
                       reinterpret_cast<long long*>(out_idx), workspace, workspace_bytes, as_stream(stream),
                       &g_last_stats);
}

int dcr_sim_topk_host(const float* q, int nq, const float* g, int ng, int d, int k, float* out_scores,
                      int64_t* out_idx) {
  DCR_REQUIRE(q && g && out_scores && out_idx, "dcr_sim_topk_host: null pointer argument");
  const size_t ws_bytes = dcr::sim_topk_workspace_size(nq, ng, d, k);
  if (ws_bytes == 0) return -1;
  float *dq = nullptr, *dg = nullptr, *ds = nullptr;
  long long* di = nullptr;
  void* ws = nullptr;
  cudaStream_t st = nullptr;
  int rc = 0;
  auto cleanup = [&]() {
    if (dq) cudaFree(dq);
    if (dg) cudaFree(dg);
    if (ds) cudaFree(ds);
    if (di) cudaFree(di);
    if (ws) cudaFree(ws);
    if (st) cudaStreamDestroy(st);
  };
#define DCR_TRY(expr)                                                                                    \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) {                                                                             \
      rc = dcr::set_error(-2, "%s failed: %s", #expr, cudaGetErrorString(_e));                           \
      cleanup();                                                                                         \
      return rc;                                                                                         \
    }                                                                                                    \
  } while (0)
  DCR_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  DCR_TRY(cudaMalloc(&dq, static_cast<size_t>(nq) * d * 4));
  DCR_TRY(cudaMalloc(&dg, static_cast<size_t>(ng) * d * 4));
  DCR_TRY(cudaMalloc(&ds, static_cast<size_t>(nq) * k * 4));
  DCR_TRY(cudaMalloc(&di, static_cast<size_t>(nq) * k * 8));
  DCR_TRY(cudaMalloc(&ws, ws_bytes));
  DCR_TRY(cudaMemcpyAsync(dq, q, static_cast<size_t>(nq) * d * 4, cudaMemcpyHostToDevice, st));
  DCR_TRY(cudaMemcpyAsync(dg, g, static_cast<size_t>(ng) * d * 4, cudaMemcpyHostToDevice, st));
  rc = dcr::sim_topk(dq, nq, dg, ng, d, k, 0, 1, ds, di, ws, ws_bytes, st, &g_last_stats);
  if (rc == 0) {
    DCR_TRY(cudaMemcpyAsync(out_scores, ds, static_cast<size_t>(nq) * k * 4, cudaMemcpyDeviceToHost, st));
    DCR_TRY(cudaMemcpyAsync(out_idx, di, static_cast<size_t>(nq) * k * 8, cudaMemcpyDeviceToHost, st));
    DCR_TRY(cudaStreamSynchronize(st));
  }
#undef DCR_TRY
  cleanup();
  return rc;
}

namespace {
inline size_t up256(size_t x) { return (x + 255) / 256 * 256; }
}  // namespace

size_t dcr_sim_topk_sharded_workspace_size(int nq, int ng_local, int d, int k, int world) {
  if (world < 1 || k < 1 || nq < 1) return 0;
  const int kk = k < ng_local ? k : ng_local;
  const size_t inner = dcr::sim_topk_workspace_size(nq, ng_local, d, kk < 1 ? 1 : kk);
  if (inner == 0) return 0;
  const size_t list = static_cast<size_t>(nq) * k;
  // local scores + indices, gathered scores + indices (each rank's block: [scores f32 | indices i64])
  return up256(inner) + up256(list * 12) + up256(list * 12 * world) + up256(list * 4 * world) + up256(list * 8 * world);
}

int dcr_sim_topk_sharded(const float* q, int nq, const float* g, int ng_local, int d, int k, int64_t g_index_base,
                         int64_t g_index_stride, int world, dcr_allgather_fn allgather, void* allgather_ctx,
                         float* out_scores, int64_t* out_idx, void* workspace, size_t workspace_bytes, void* stream) {
  DCR_REQUIRE(q && g && out_scores && out_idx && workspace, "dcr_sim_topk_sharded: null pointer argument");
  DCR_REQUIRE(world >= 1 && (world == 1 || allgather != nullptr), "dcr_sim_topk_sharded: world=%d needs an all-gather callback", world);
  DCR_REQUIRE(static_cast<long long>(world) * k <= 1024, "dcr_sim_topk_sharded: world * k = %d > 1024", world * k);
  const size_t need = dcr_sim_topk_sharded_workspace_size(nq, ng_local, d, k, world);
  DCR_REQUIRE(need != 0 && workspace_bytes >= need, "dcr_sim_topk_sharded: workspace too small (%zu < %zu)", workspace_bytes, need);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "dcr_sim_topk_sharded: workspace must be 256-byte aligned");
  cudaStream_t st = as_stream(stream);
  const int kk = k < ng_local ? k : ng_local;       // a shard smaller than k contributes empty (-inf, -1) entries
  const size_t list = static_cast<size_t>(nq) * k;
  uint8_t* w = static_cast<uint8_t*>(workspace);
  const size_t inner = dcr::sim_topk_workspace_size(nq, ng_local, d, kk);
  uint8_t* send = w + up256(inner);                                  // [scores f32 [nq,k] | indices i64 [nq,k]]
  uint8_t* recv = send + up256(list * 12);                           // world x the same block
  float* all_s = reinterpret_cast<float*>(recv + up256(list * 12 * world));        // [world][nq][k]
  long long* all_i = reinterpret_cast<long long*>(reinterpret_cast<uint8_t*>(all_s) + up256(list * 4 * world));
  float* loc_s = reinterpret_cast<float*>(send);
  long long* loc_i = reinterpret_cast<long long*>(send + list * 4);
  if (kk == k) {
    if (int rc = dcr::sim_topk(q, nq, g, ng_local, d, k, g_index_base, g_index_stride, loc_s, loc_i, w, inner, st, &g_last_stats))
      return rc;
  } else {
    // fewer gallery rows than k on this rank: top-kk into a compact list, spread into the k-wide slots, the rest empty
    float* tmp_s = all_s;                      // scratch (not yet in use)
    long long* tmp_i = all_i;
    if (int rc = dcr::sim_topk(q, nq, g, ng_local, d, kk, g_index_base, g_index_stride, tmp_s, tmp_i, w, inner, st, &g_last_stats))
      return rc;
    if (int rc = dcr::pad_topk_lists(tmp_s, tmp_i, nq, kk, k, loc_s, loc_i, st)) return rc;
  }
  if (world == 1) {
    DCR_CUDA_CHECK(cudaMemcpyAsync(out_scores, loc_s, list * 4, cudaMemcpyDeviceToDevice, st));
    DCR_CUDA_CHECK(cudaMemcpyAsync(out_idx, loc_i, list * 8, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  const int arc = allgather(send, recv, list * 12, allgather_ctx, stream);
  DCR_REQUIRE(arc == 0, "dcr_sim_topk_sharded: the all-gather callback failed (%d)", arc);
  // un-interleave the gathered blocks into [world][nq][k] score and index arrays, then merge
  for (int r = 0; r < world; ++r) {
    DCR_CUDA_CHECK(cudaMemcpyAsync(all_s + static_cast<size_t>(r) * list, recv + static_cast<size_t>(r) * list * 12, list * 4,
                                   cudaMemcpyDeviceToDevice, st));
    DCR_CUDA_CHECK(cudaMemcpyAsync(all_i + static_cast<size_t>(r) * list, recv + static_cast<size_t>(r) * list * 12 + list * 4, list * 8,
                                   cudaMemcpyDeviceToDevice, st));
  }
  return dcr::topk_merge(all_s, all_i, nq, world, k, k, out_scores, reinterpret_cast<long long*>(out_idx), st);
}

size_t dcr_sim_range_workspace_size(int nq, int ng, int d, int64_t max_pairs) {
  return dcr::sim_range_workspace_size(nq, ng, d, max_pairs);
}

int dcr_sim_range(const float* q, int nq, const float* g, int ng, int d, float threshold, int64_t g_index_base,
                  int64_t g_index_stride, int64_t* row_offsets, int64_t* out_idx, float* out_scores, int64_t max_pairs,
                  int64_t* counts, void* workspace, size_t workspace_bytes, void* stream) {
  DCR_REQUIRE(q && g && row_offsets && counts && (max_pairs == 0 || (out_idx && out_scores)),
              "dcr_sim_range: null pointer argument");
  return dcr::sim_range(q, nq, g, ng, d, threshold, g_index_base, g_index_stride, reinterpret_cast<long long*>(row_offsets),
                        reinterpret_cast<long long*>(out_idx), out_scores, max_pairs, reinterpret_cast<long long*>(counts),
                        workspace, workspace_bytes, as_stream(stream));
}

int dcr_sim_topk_last_stats(int* out8) {
  DCR_REQUIRE(out8 != nullptr, "dcr_sim_topk_last_stats: null pointer");
  out8[0] = g_last_stats.cta_group;
  out8[1] = g_last_stats.grid;
  out8[2] = g_last_stats.smem_bytes;
  out8[3] = g_last_stats.stages;
  out8[4] = g_last_stats.kp;
  out8[5] = g_last_stats.cap;
  out8[6] = g_last_stats.n_flagged;
  out8[7] = g_last_stats.d_pad;
  return 0;
}

float dcr_sim_topk_last_kernel_ms(void) { return g_last_stats.kernel_ms; }
float dcr_sim_topk_last_sm_mhz(void) { return g_last_stats.sm_mhz; }
int dcr_sim_topk_last_epilogue_sets(void) { return g_last_stats.n_sets; }
int dcr_sim_topk_last_second_pass(void) { return g_last_stats.n_second; }

long long dcr_kernel_launch_count(void) { return dcr::launch_count(); }

int dcr_topk_merge(const float* scores, const int64_t* idx, int nq, int nlists, int k_in, int k_out,
                   float* out_scores, int64_t* out_idx, void* stream) {
  DCR_REQUIRE(scores && idx && out_scores && out_idx, "dcr_topk_merge: null pointer argument");
  return dcr::topk_merge(scores, reinterpret_cast<const long long*>(idx), nq, nlists, k_in, k_out, out_scores,
                         reinterpret_cast<long long*>(out_idx), as_stream(stream));
}

int dcr_split_rescore(const float* q, const float* g, int nq, int d, int n_chunks, int cross, const int64_t* cand,
                      int n_cand, int k, float* out_scores, int64_t* out_idx, void* stream) {
  DCR_REQUIRE(q && g && cand && out_scores && out_idx, "dcr_split_rescore: null pointer argument");
  return dcr::split_rescore(q, g, nq, d, n_chunks, cross, reinterpret_cast<const long long*>(cand), n_cand, k, out_scores,
                            reinterpret_cast<long long*>(out_idx), as_stream(stream));
}

int dcr_conv2d_bf16(const void* x, int x_planes, int64_t x_plane_stride, int B, int H, int W, int C, const void* w,
                    int w_planes, int64_t w_plane_stride, int N, int kh, int kw, int stride, int pad_h, int pad_w,
                    int terms, const float* scale, const float* bias, const void* residual, int res_planes,
                    int64_t res_plane_stride, int act, void* out, int out_planes, int64_t out_plane_stride, int ld_out,
                    int out_col_off, float* out_f32, void* stream) {
  DCR_REQUIRE(x && w, "dcr_conv2d_bf16: null input");
  DCR_REQUIRE(out || out_f32, "dcr_conv2d_bf16: no output requested");
  DCR_REQUIRE(terms == 1 || terms == 3 || terms == 6, "dcr_conv2d_bf16: terms must be 1, 3 or 6 (got %d)", terms);
  const int need = terms == 1 ? 1 : (terms == 3 ? 2 : 3);
  DCR_REQUIRE(x_planes >= need && w_planes >= need, "dcr_conv2d_bf16: terms=%d needs %d planes (x has %d, w has %d)",
              terms, need, x_planes, w_planes);
  dcr::ConvGemmDesc d;
  d.in = static_cast<const __nv_bfloat16*>(x);
  d.in_plane_stride = x_plane_stride;
  d.B = B; d.H = H; d.W = W; d.C = C; d.ld_in = C;
  d.weight = static_cast<const __nv_bfloat16*>(w);
  d.w_plane_stride = w_plane_stride;
  d.N = N; d.kh = kh; d.kw = kw; d.stride = stride; d.pad_h = pad_h; d.pad_w = pad_w;
  static const int ta[6] = {0, 0, 1, 1, 0, 2}, tw[6] = {0, 1, 0, 1, 2, 0};
  d.n_terms = terms;
  for (int t = 0; t < terms; ++t) { d.term_a[t] = ta[t]; d.term_w[t] = tw[t]; }
  d.scale = scale; d.bias = bias;
  d.res = static_cast<const __nv_bfloat16*>(residual);
  d.ld_res = N; d.res_planes = res_planes; d.res_plane_stride = res_plane_stride;
  d.out = static_cast<__nv_bfloat16*>(out);
  d.ld_out = ld_out; d.out_col_off = out_col_off; d.out_planes = out_planes; d.out_plane_stride = out_plane_stride;
  d.out_f32 = out_f32; d.ld_out_f32 = N;
  d.act = act;
  return dcr::conv_gemm(d, as_stream(stream));
}

struct dcr_net;   // opaque alias of dcr::Net

int dcr_net_create(int max_batch, int planes, dcr_net** out) {
  DCR_REQUIRE(out != nullptr, "dcr_net_create: null out pointer");
  return dcr::net_create(max_batch, planes, reinterpret_cast<dcr::Net**>(out));
}
int dcr_net_set_exact(dcr_net* net, int on) { return dcr::net_set_exact(reinterpret_cast<dcr::Net*>(net), on); }
void dcr_net_destroy(dcr_net* net) { dcr::net_destroy(reinterpret_cast<dcr::Net*>(net)); }
int dcr_net_fork(const dcr_net* net, dcr_net** out) {
  DCR_REQUIRE(net != nullptr && out != nullptr, "dcr_net_fork: null argument");
  return dcr::net_fork(reinterpret_cast<const dcr::Net*>(net), reinterpret_cast<dcr::Net**>(out));
}
int dcr_net_add_tensor(dcr_net* net, int64_t rows_per_image, int channels) {
  return dcr::net_add_tensor(reinterpret_cast<dcr::Net*>(net), rows_per_image, channels);
}
int dcr_net_alias_tensor(dcr_net* net, int src_tensor, int64_t rows_per_image, int channels) {
  return dcr::net_alias_tensor(reinterpret_cast<dcr::Net*>(net), src_tensor, rows_per_image, channels);
}
int dcr_net_add_param(dcr_net* net, const void* host_data, size_t bytes) {
  return dcr::net_add_param(reinterpret_cast<dcr::Net*>(net), host_data, bytes);
}
int dcr_net_set_output(dcr_net* net, int dim) { return dcr::net_set_output(reinterpret_cast<dcr::Net*>(net), dim); }
int dcr_net_add_op(dcr_net* net, int kind, const int* iargs, int n_iargs, const float* fargs, int n_fargs) {
  return dcr::net_add_op(reinterpret_cast<dcr::Net*>(net), kind, iargs, n_iargs, fargs, n_fargs);
}
int dcr_net_forward(dcr_net* net, const uint8_t* images, int n, float* out, void* stream) {
  return dcr::net_forward(reinterpret_cast<dcr::Net*>(net), images, n, out, as_stream(stream));
}

int dcr_net_tensor(const dcr_net* net, int t, void** ptr, int64_t* plane_stride) {
  DCR_REQUIRE(ptr != nullptr && plane_stride != nullptr, "dcr_net_tensor: null out pointer");
  long long ps = 0;
  const int rc = dcr::net_tensor(reinterpret_cast<const dcr::Net*>(net), t, ptr, &ps);
  *plane_stride = ps;
  return rc;
}

int64_t dcr_stem_plane_units(int out_h, int out_w) { return dcr::stem_fused_plane_units(out_h, out_w); }
int dcr_net_forward_f32(dcr_net* net, const float* x_nchw, int n, float* out, void* stream) {
  DCR_REQUIRE(x_nchw != nullptr, "dcr_net_forward_f32: null input");
  return dcr::net_forward(reinterpret_cast<dcr::Net*>(net), nullptr, n, out, as_stream(stream), x_nchw);
}

struct dcr_fid;   // opaque alias of dcr::FidState
int dcr_fid_create(int d, dcr_fid** out) {
  DCR_REQUIRE(out != nullptr, "dcr_fid_create: null out pointer");
  return dcr::fid_create(d, reinterpret_cast<dcr::FidState**>(out));
}
void dcr_fid_destroy(dcr_fid* st) { dcr::fid_destroy(reinterpret_cast<dcr::FidState*>(st)); }
int dcr_fid_accumulate(dcr_fid* st, const float* act, int n, void* stream) {
  return dcr::fid_accumulate(reinterpret_cast<dcr::FidState*>(st), act, n, as_stream(stream));
}
int dcr_fid_finalize(dcr_fid* st, double* mu, double* sigma, int64_t* n_out, void* stream) {
  long long n = 0;
  const int rc = dcr::fid_finalize(reinterpret_cast<dcr::FidState*>(st), mu, sigma, &n, as_stream(stream));
  if (n_out) *n_out = n;
  return rc;
}
size_t dcr_fid_packed_size(int d) {
  const size_t bytes = dcr::fid_packed_size(d);
  if (bytes == 0) dcr::set_error(-1, "dcr_fid_packed_size: bad dim %d", d);
  return bytes;
}
int dcr_fid_export(const dcr_fid* st, void* packed, void* stream) {
  return dcr::fid_export(reinterpret_cast<const dcr::FidState*>(st), packed, as_stream(stream));
}
int dcr_fid_merge(dcr_fid* st, const void* packed, int count, void* stream) {
  return dcr::fid_merge(reinterpret_cast<dcr::FidState*>(st), packed, count, as_stream(stream));
}

}  // extern "C"
