/*
 * dcr_b200.h -- C ABI of libdcr_b200.so: the H100 (sm_90a) replacement for DCR's embed -> match -> top-k (+FID)
 * hot path.  Plain pointers and sizes only; no torch / CUDA types in any signature.
 *
 * The reference (somepago/DCR) is pure Python and has no FFI layer; each entry point below names
 * the reference call site it replaces (file:line).  A Python maintainer binds these with ctypes (INTEGRATION.md).
 *
 * Conventions
 *   - every function returning int: 0 = ok, < 0 = error; the message is available from dcr_last_error() (per host
 *     thread).  Nothing throws, nothing aborts.
 *   - "device pointer" arguments are raw CUDA device addresses on the CURRENT device; `stream` is a cudaStream_t
 *     passed as void* (NULL = legacy default stream).  Work is enqueued on that stream; functions that must read a
 *     result back (dcr_sim_topk: the count of queries that needed the exact fallback) synchronise that stream
 *     before returning.
 *   - workspaces are caller-owned device buffers, 256-byte aligned, sized by the matching *_workspace_size().
 *   - the library never falls back to the CPU: on a machine without an sm_90 device every compute call fails with
 *     a message.
 */
#ifndef DCR_B200_H_
#define DCR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DCR_B200_VERSION 100 /* 0.1.0 */

/* ---- library ------------------------------------------------------------------------------------------------ */
int dcr_version(void);
const char* dcr_last_error(void);
/* number of SMs of the current device, or < 0 when no usable device is visible */
int dcr_device_sm_count(void);

/* ---- descriptor post-processing ------------------------------------------------------------------------------- */
/* x[n,d] (device, fp32, row-major) <- x / max(||x||_2, eps) per row.
 * Replaces nn.functional.normalize(features, dim=1, p=2)          diff_retrieval.py:388-389 */
int dcr_l2_normalize(float* x, int n, int d, float eps, void* stream);

/* ---- similarity + top-k ------------------------------------------------------------------------------------- */
/* Bytes of device workspace dcr_sim_topk needs for this problem size (0 on invalid arguments, see last error). */
size_t dcr_sim_topk_workspace_size(int nq, int ng, int d, int k);

/* For every query row q[i,:] the k gallery rows with the largest dot product, ordered by (score descending,
 * gallery index ascending).  q[nq,d], g[ng,d]: device, fp32, row-major, 16-byte aligned, d % 4 == 0, d <= 8192 (the query tile is
 * shared-memory resident up to d = 512 and streamed with the gallery tiles beyond),
 * 1 <= k <= 16, k <= ng.  out_scores[nq,k] fp32, out_idx[nq,k] int64 (device); reported index =
 * g_index_base + g_index_stride * row (lets a rank that holds a contiguous or strided gallery shard report global
 * indices).  Scores are the fp64-accumulated dot products of the fp32 inputs rounded to fp32; the [nq,ng] matrix
 * is never materialised.
 * Replaces   sim = torch.mm(values_features, query_features.T)         diff_retrieval.py:402
 *            simscores.topk(k, axis=1, largest=True)                   diff_retrieval.py:417, 613, 621
 *            sim2 = mm(values, values.T); bg.topk(2)                   diff_retrieval.py:403, 418-419 (q = g, k = 2)
 *            features @ batch.T ; .max(dim=0)                          embedding_search/similarity_search.py:62-63 */
int dcr_sim_topk(const float* q, int nq, const float* g, int ng, int d, int k, int64_t g_index_base,
                 int64_t g_index_stride, float* out_scores, int64_t* out_idx, void* workspace,
                 size_t workspace_bytes, void* stream);

/* Same computation with HOST buffers (pageable or pinned): allocates device memory, copies in, runs, copies the
 * results back, frees.  The zero-setup entry for a caller that holds numpy arrays (what diff_retrieval.py:386-417 has
 * when use_cuda is falsy); tests/test_sim_topk_gpu.py drives it through ctypes with numpy buffers. */
int dcr_sim_topk_host(const float* q, int nq, const float* g, int ng, int d, int k, float* out_scores,
                      int64_t* out_idx);

/* Launch facts of the most recent dcr_sim_topk on this host thread:
 * out[0]=cta_group out[1]=grid out[2]=dynamic smem bytes out[3]=pipeline stages out[4]=candidates kept per segment
 * out[5]=list capacity out[6]=queries recomputed by the exact fallback out[7]=padded descriptor dim */
int dcr_sim_topk_last_stats(int* out8);

/* Device time (ms, CUDA events on the call's stream) of the fused similarity+top-k kernel alone in the most recent
 * dcr_sim_topk on this host thread; the conversion / re-score kernels are excluded. */
float dcr_sim_topk_last_kernel_ms(void);
/* SM clock (MHz) while that kernel ran, from clock64 / %globaltimer read by its first CTA (0 if not measured), and
 * the number of epilogue warp sets (4 warps each) it ran with. */
float dcr_sim_topk_last_sm_mhz(void);
int dcr_sim_topk_last_epilogue_sets(void);
/* number of queries that went through the second-chance pass (32 candidates) in that call */
int dcr_sim_topk_last_second_pass(void);

/* Cumulative number of CUDA kernels this library has launched in this process (all entry points). */
long long dcr_kernel_launch_count(void);

/* Merge nlists per-shard results.  scores/idx: device, layout [nlists][nq][k_in]; entries with idx < 0 are empty.
 * Output [nq][k_out] ordered by (score desc, idx asc).  nlists*k_in <= 1024.
 * Replaces the running cross-folder merge                        embedding_search/similarity_search.py:70-74
 * and is the reduction after the per-shard top-k all-gather (SURVEY.md 8e). */
int dcr_topk_merge(const float* scores, const int64_t* idx, int nq, int nlists, int k_in, int k_out,
                   float* out_scores, int64_t* out_idx, void* stream);

/* Gallery-sharded form (SURVEY.md 8e; replaces the per-batch all_gather pair of utils_ret.py:763-779 and the rank-0-only
 * mm/topk of diff_retrieval.py:402-417): this rank scores ALL queries q[nq,d] against ITS gallery shard g[ng_local,d] (global
 * index of local row r = g_index_base + g_index_stride * r), the per-shard (score, index) lists are exchanged by ONE
 * all-gather and merged, and out_scores / out_idx [nq,k] receive the global top-k on every rank.
 * The library does not link a communication library: the caller supplies the all-gather as a callback that must enqueue,
 * on `stream`, an all-gather of `bytes_per_rank` bytes from device buffer `send` into device buffer `recv`
 * (world * bytes_per_rank bytes, rank-major) -- one ncclAllGather(send, recv, bytes_per_rank, ncclUint8, comm, stream)
 * call, or torch.distributed.all_gather_into_tensor from Python (dcr_b200/dist.py).  Returns non-zero to abort.
 * workspace: dcr_sim_topk_sharded_workspace_size(nq, ng_local, d, k, world) bytes. */
typedef int (*dcr_allgather_fn)(const void* send, void* recv, size_t bytes_per_rank, void* ctx, void* stream);
size_t dcr_sim_topk_sharded_workspace_size(int nq, int ng_local, int d, int k, int world);
int dcr_sim_topk_sharded(const float* q, int nq, const float* g, int ng_local, int d, int k, int64_t g_index_base,
                         int64_t g_index_stride, int world, dcr_allgather_fn allgather, void* allgather_ctx,
                         float* out_scores, int64_t* out_idx, void* workspace, size_t workspace_bytes, void* stream);

/* Final step of the 'splitloss' similarity (diff_retrieval.py:393-400: descriptors cut into n_chunks equal parts, pair
 * score = max over the parts of the per-part dot products).  The caller runs dcr_sim_topk once per part and passes
 * the union of the per-part top-k rows as cand [nq][n_cand] (duplicates allowed); this evaluates the exact split
 * score of every candidate (float64 accumulation, reported as fp32) and writes the k best per query ordered by
 * (score desc, row asc).  d %% n_chunks == 0, (d / n_chunks) %% 4 == 0, k <= n_cand <= 4096; negative entries of
 * cand are empty slots.
 * cross != 0: the 'cross' form (--stype cross, einsum_in_chunks diff_retrieval.py:643-662): score = max over EVERY pair
 * (gallery part, query part); the caller then collects candidates by running dcr_sim_topk on the part matrices
 * [nq * n_chunks, d / n_chunks] x [ng * n_chunks, d / n_chunks] with k' = (k - 1) * n_chunks + 1 (when k' <= 16), or once
 * per gallery part [nq * n_chunks, d / n_chunks] x [ng, d / n_chunks] with k' = k (any n_chunks; dcr_b200/similarity.py). */
int dcr_split_rescore(const float* q, const float* g, int nq, int d, int n_chunks, int cross, const int64_t* cand,
                      int n_cand, int k, float* out_scores, int64_t* out_idx, void* stream);

/* ---- threshold search ----------------------------------------------------------------------------------------- */
#define DCR_ERR_CAPACITY (-3) /* more result candidates than the caller's max_pairs; counts[1] says how many */

/* Bytes of device workspace dcr_sim_range needs (host-only planning; 0 on invalid arguments, see last error).  It grows
 * with nq, ng, d and max_pairs, never with nq * ng. */
size_t dcr_sim_range_workspace_size(int nq, int ng, int d, int64_t max_pairs);

/* For every query row i, every gallery row j whose score s_ij >= threshold.  s_ij is the score dcr_sim_topk reports for
 * the same pair, bit for bit: the fp64 sum of the fp32 products (the association of its exact re-score) rounded to
 * fp32.  A NaN score is never reported; threshold = -inf reports all nq * ng pairs; a NaN threshold is an error.
 * The answer is exact (no qualifying pair is missed, no other pair reported) and the same bits on every call.
 * q[nq,d], g[ng,d]: as dcr_sim_topk (device, fp32, 16-byte aligned, d % 4 == 0, d <= 8192).  Output, CSR (device):
 *   row_offsets[nq + 1]  int64, row i's pairs are entries row_offsets[i] .. row_offsets[i + 1] - 1
 *   out_idx[max_pairs]   int64, g_index_base + g_index_stride * j, ascending j within a row (g_index_stride >= 1)
 *   out_scores[max_pairs] fp32
 * counts (HOST [2]): [0] pairs returned, [1] candidate pairs examined = the capacity this call needs.  When the
 * candidates exceed max_pairs the call returns DCR_ERR_CAPACITY after the counting pass, with counts[1] set and the
 * outputs undefined; the same call with max_pairs = counts[1] then succeeds.  Synchronises `stream` before returning.
 * Replaces   sim = torch.mm(values, query.T); sim2 = mm(values, values.T)    diff_retrieval.py:402-403
 *            torch.save(sim / sim2, 'similarity*.pth')                       diff_retrieval.py:414-415
 *            the fraction of scores above 0.5 (sim_gt_05pc)                  diff_retrieval.py:454 */
int dcr_sim_range(const float* q, int nq, const float* g, int ng, int d, float threshold, int64_t g_index_base,
                  int64_t g_index_stride, int64_t* row_offsets, int64_t* out_idx, float* out_scores, int64_t max_pairs,
                  int64_t* counts, void* workspace, size_t workspace_bytes, void* stream);

/* ---- dense contraction of the descriptor networks ------------------------------------------------------------- */
/* y = act(scale[n] * conv2d(x, w)[.., n] + bias[n] (+ residual)) as a wgmma implicit GEMM.
 *   x        NHWC bf16, `x_planes` planes of B*H*W*C elements each (plane p at x + p*x_plane_stride elements);
 *            C % 8 == 0.  A Linear layer is the case H = W = kh = kw = 1, B = rows.
 *   w        prepared weights: bf16 [w_planes][N][kh*kw*ceil64(C)], tap-major, channels zero-padded to 64
 *            (dcr_b200.ops.prepare_conv_weight); N % 8 == 0.
 *   terms    1 = bf16 x bf16 (fast); 3 or 6 = split-bf16 cross terms hi*hi, hi*mid, mid*hi[, mid*mid, hi*lo, lo*hi]
 *            which need x_planes/w_planes >= 2 (3 terms) or 3 (6 terms) and reproduce fp32 accuracy.
 *   scale/bias  fp32 [N] or NULL; residual: bf16 planes [res_planes][M][N] or NULL; act: 0 none, 1 ReLU, 2 GELU, 3 QuickGELU
 *            (GELU: the erf form, |error| <= 2e-7, with split planes; with ONE plane -- bf16 activations -- its tanh form through
 *            tanh.approx, within 1.5e-3 absolute of the erf form, i.e. below the bf16 rounding of the stored value)
 *   out      bf16 planes [out_planes][M][ld_out] written at column offset out_col_off (concat by offset), or NULL;
 *   out_f32  fp32 [M][N] or NULL.   M = B * Hout * Wout.
 * Replaces the cuDNN / cuBLAS calls behind `model(samples)`        utils_ret.py:751 (nn.Conv2d+BatchNorm2d+ReLU of the
 * SSCD trunk; nn.Linear of dino_vits.py:96-102,119,127; BasicConv2d of metrics/inception.py). */
int dcr_conv2d_bf16(const void* x, int x_planes, int64_t x_plane_stride, int B, int H, int W, int C,
                    const void* w, int w_planes, int64_t w_plane_stride, int N, int kh, int kw, int stride,
                    int pad_h, int pad_w, int terms, const float* scale, const float* bias, const void* residual,
                    int res_planes, int64_t res_plane_stride, int act, void* out, int out_planes,
                    int64_t out_plane_stride, int ld_out, int out_col_off, float* out_f32, void* stream);

/* ---- descriptor networks ---------------------------------------------------------------------------------------- */
/* A dcr_net is an op list over numbered activation tensors, built once by the host from a model's weights
 * (dcr_b200/nets.py mirrors torchvision ResNet-50 + SSCD head, dino_vits.VisionTransformer and
 * metrics/inception.InceptionV3) and run per batch.  dcr_net_forward replaces `model(samples)`:
 *   utils_ret.py:751 (extract_features), embedding_search/utils.py:101, metrics/fid.py:126.
 *
 * planes: 1 = bf16 activations/weights (fast); 3 = split-bf16 planes carrying fp32 precision (parity mode).
 * Tensor ids / param ids / op ids are the non-negative return values; negative = error.
 * Op kinds and their integer / float argument vectors (all sizes per image; the batch is given at forward time):
 *   0 IM2COL_U8  i: out_t, IH, IW, crop_y, crop_x, H, W, kh, kw, stride, pad, k_pad [, RH, RW]     f: mean[3], std[3], post_scale, post_shift [, rscale]
 *                (optional RH, RW, rscale as for STEM_S2D: bilinear resize of the transformed crop, utils_ret.py:676-698)
 *                uint8 HWC input -> normalised im2col rows of the first (3-channel) convolution / patch embedding
 *   1 CONV       i: in_t, out_t|-1, H, W, C, w_param, N, kh, kw, stride, pad_h, pad_w, scale_param|-1, bias_param|-1,
 *                   residual_t|-1, act(0 none,1 relu,2 gelu), out_col_off, to_output(0/1)
 *   2 MAXPOOL / 3 AVGPOOL(count_include_pad=False)  i: in_t, out_t, H, W, C, k, stride, pad, out_col_off
 *   4 GEM        i: in_t, out_t|-1, HW, C, to_output     f: p, eps
 *   5 GAP        i: in_t, out_t|-1, HW, C, to_output     (global average pool)
 *   6 LAYERNORM  i: in_t, out_t|-1, rows_out_per_image, C, gamma_param, beta_param, in_row_stride(rows), to_output   f: eps
 *   7 VIT_TOKENS i: patch_t, out_t, n_patches, C, cls_param, pos_param
 *   8 ATTENTION  i: qkv_t, out_t, T, heads, head_dim [, causal(0/1)]      f: scale
 *   9 L2NORM_OUT f: eps        (row-normalise the fp32 output buffer in place)
 *  10 STEM_S2D   i: out_t, IH, IW, crop_y, crop_x, H, W [, RH, RW]     f: mean[3], std[3], post_scale, post_shift [, rscale]
 *                (optional RH, RW, rscale: the normalised crop is first resized to RH x RW with torch's bilinear
 *                 F.interpolate(scale_factor=s, align_corners=False) arithmetic, rscale = float(1/s); utils_ret.py:676-698)
 *                uint8 HWC input -> normalised, zero-padded 2x2 space-to-depth tensor [(H+6)/2, (W+6)/2, 16] of the
 *                7x7/2/pad-3 stem; the following CONV passes two extra ints (elements per stored pixel, stored pixels
 *                per row) to read 4 adjacent stored pixels as one 64-channel pixel (kh = 4, kw = 1).
 *  11 EMBED      i: out_t, T, C, table_param, pos_param, vocab
 *                the network input is DEVICE int32 token ids [n, T] (pass them as the `images` pointer of dcr_net_forward):
 *                rows table[id] + pos[t]  (CLIP text tower; utils_ret.py:1046-1066 `model.encode_text`)
 *  12 STEM_ROWS  i: out_t, IH, IW, crop_y, crop_x, H, W [, RH, RW]     f: as STEM_S2D
 *                uint8 HWC (or fp32 NCHW) input -> the two column-parity planes of 16-byte pixel units the fused stem
 *                kernel reads through overlapping-window descriptors (csrc/stem_fused.cu); out_t has
 *                2 * dcr_stem_plane_units(H/2, W/2) rows of 8 channels per image.  One-plane (fast) networks only.
 *  13 STEM_CONV  i: planes_t, out_t, OH, OW, w_param ([64][256] bf16, k = ((a*2+e)*4+b)*8 + i*3+c), scale_param|-1, bias_param|-1 [, pool]
 *                7x7/2/pad-3 convolution + BN + ReLU -> NHWC [OH*OW, 64]; pool = 1: the following 3x3/2/pad-1 max pool is
 *                taken in the epilogue and out_t is [((OH-1)/2+1) * ((OW-1)/2+1), 64]
 * CONV act: 0 none, 1 ReLU, 2 GELU (erf form; tanh form in one-plane mode, see dcr_conv2d_bf16), 3 QuickGELU x*sigmoid(1.702x). */
typedef struct dcr_net dcr_net;
int dcr_net_create(int max_batch, int planes, dcr_net** out);
/* on != 0: every CONV op accumulates its products in float64 on the CUDA cores (correctly rounded fp32 layer outputs,
 * the mode the parity tests use against the fp32 oracle); needs planes == 3.  Default 0: wgmma tensor cores. */
int dcr_net_set_exact(dcr_net* net, int on);
void dcr_net_destroy(dcr_net* net);
/* A second executor of a fully described network: its own activation buffers, the same uploaded parameters (reference
 * counted: either handle may be destroyed first).  Lets two batches be in flight on two streams, which is how
 * extract_features (utils_ret.py:704-787 replacement) keeps all SMs busy across the kernels' wave tails. */
int dcr_net_fork(const dcr_net* net, dcr_net** out);
int dcr_net_add_tensor(dcr_net* net, int64_t rows_per_image, int channels);
/* another (rows_per_image, channels) factorisation of an existing tensor's buffer (flatten in front of a Linear layer) */
int dcr_net_alias_tensor(dcr_net* net, int src_tensor, int64_t rows_per_image, int channels);
/* copies `bytes` from HOST memory to a new device buffer */
int dcr_net_add_param(dcr_net* net, const void* host_data, size_t bytes);
int dcr_net_set_output(dcr_net* net, int dim);
int dcr_net_add_op(dcr_net* net, int kind, const int* iargs, int n_iargs, const float* fargs, int n_fargs);
/* images: DEVICE uint8 [n, IH, IW, 3]; out: DEVICE fp32 [n, dim]; n <= max_batch */
int dcr_net_forward(dcr_net* net, const uint8_t* images, int n, float* out, void* stream);
/* device address and plane stride (elements) of activation tensor t: read/write, for tests and tools.  The buffer holds
 * `planes` planes of [max_batch, rows_per_image, channels] bf16, plane p at *ptr + p * plane_stride elements. */
int dcr_net_tensor(const dcr_net* net, int t, void** ptr, int64_t* plane_stride);
/* units (16-byte pixels) per image and plane of the STEM_ROWS tensor for an OH x OW stem output (includes read slack) */
int64_t dcr_stem_plane_units(int out_h, int out_w);
/* Same network, fed with what the reference's own loop feeds `model(samples)` (utils_ret.py:751; embedding_search/
 * utils.py:101; metrics/fid.py:126 `model(batch)[0]`): x_nchw DEVICE fp32 [n, 3, H, W], already transformed by the
 * caller's torchvision pipeline (H x W = the network's input size after the centre crop, e.g. 224 x 224 / 299 x 299).
 * Only the network's own input affine is applied (FID's internal 2x-1, metrics/inception.py:152-153). */
int dcr_net_forward_f32(dcr_net* net, const float* x_nchw, int n, float* out, void* stream);

/* ---- FID statistics ---------------------------------------------------------------------------------------------- */
/* Streaming mean / unbiased covariance (float64) of activation rows, accumulated on the device batch by batch.
 * Replaces  pred_arr (float64 [N,2048] host buffer, metrics/fid.py:118,135) + np.mean / np.cov   (metrics/fid.py:219-220).
 * act: DEVICE fp32 [n, d].  finalize writes HOST buffers mu[d], sigma[d*d] (row-major) and the sample count. */
typedef struct dcr_fid dcr_fid;
int dcr_fid_create(int d, dcr_fid** out);
void dcr_fid_destroy(dcr_fid* st);
int dcr_fid_accumulate(dcr_fid* st, const float* act, int n, void* stream);
int dcr_fid_finalize(dcr_fid* st, double* mu, double* sigma, int64_t* n_out, void* stream);

/* Statistics of one image set computed on several devices (each rank accumulates its shard): export every state, exchange
 * the packed states (an all-gather), and fold them into one state.  A state keeps a shift c (the mean of its first batch),
 * s = sum(x - c), S = sum((x - c)(x - c)^T) (upper triangle) and n; folding peer b into a rebases b onto a's shift,
 * delta = c_a - c_b:
 *     s_a += s_b - n_b delta,   S_a += S_b - s_b delta^T - delta s_b^T + n_b delta delta^T,   n_a += n_b
 * (an empty a takes b as it is, shift included).
 * Packed layout, dcr_fid_packed_size(d) bytes, 8-byte aligned (DEVICE memory):
 *     int64 header[4] = {0x31444946524344 ("DCRFID1" in memory), d, n, 0}
 *     double shift[d], sum[d], xtx[d*d]   (row-major; only the upper triangle i <= j is meaningful; shift is undefined
 *                                          when n = 0)
 * dcr_fid_packed_size returns 0 for a bad d.  dcr_fid_export enqueues device-to-device copies on `stream`.
 * dcr_fid_merge folds `count` packed states laid out back to back (state p at packed + p * dcr_fid_packed_size(d)) into
 * `st`, in order p = 0, 1, ...: one float64 kernel, each element of the triangle loops over the peers in that order, so
 * the result is the same on every run and every rank that folds the same states.  States with n = 0 are skipped; a
 * state of another d (or not produced by dcr_fid_export) is an error and nothing is merged.  It reads the headers with
 * one synchronous device-to-host copy on `stream`.  dcr_fid_accumulate and dcr_fid_finalize work on the merged state. */
size_t dcr_fid_packed_size(int d);
int dcr_fid_export(const dcr_fid* st, void* packed, void* stream);
int dcr_fid_merge(dcr_fid* st, const void* packed, int count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DCR_B200_H_ */
