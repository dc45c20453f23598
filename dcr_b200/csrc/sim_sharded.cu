// Gallery-sharded search: every rank searches ALL queries against its own gallery shard, the per-rank results are
// exchanged through the caller's all-gather, and a merge on the device turns them into the result of the whole gallery
// on every rank.
//
// Top-k (dcr_sim_topk_sharded): sim_topk into this rank's list (a shard smaller than k padded with empty entries), one
// all-gather of the lists, topk_merge of the world lists.
//
// Threshold search (dcr_sim_range_sharded):
//   1. local search     sim_range into this rank's message: offsets, global indices, scores
//   2. header exchange  a fixed-size header per rank (status, pair count, candidate need, capacities, nq, d, threshold
//                       bits); every rank decides the outcome from the same gathered headers, so every rank returns the
//                       same code and no rank is left waiting in a collective its peers skipped
//   3. payload exchange each rank's message padded to the largest one (known from the headers)
//   4. merge            merged row counts summed in rank order and scanned (exclusive_scan_i64); every entry finds its
//                       place in its row by binary search in the other ranks' pieces of that row.  No atomic decides an
//                       order; a check pass before it refuses overlapping shards and malformed messages.
// Every score is a function of its pair alone and the pieces are complete, so the merged rows are the rows sim_range
// returns for the union of the shards.  The split forms (dcr_sim_range_split_sharded, dcr_sim_range_cross_sharded) run
// sim_range_split, aligned or cross, as the local search; the exchange and the merge are the same, and header word [9]
// carries the score (0 the dot product, n_parts aligned, -n_parts cross) so that ranks running different searches
// disagree instead of merging.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/dcr_b200.h"
#include "dcr_internal.cuh"
#include "host_util.cuh"
#include "ptx.cuh"

namespace dcr {

namespace {

constexpr int kHdrWords = 10;                               // int64 words of a header (layout in dcr_b200.h)
constexpr long long kHdrMagic = 0x31474E52524344ll;         // "DCRRNG1" in memory
constexpr int kMaxWorld = 65535;                            // ranks: the merge grid's y extent
constexpr long long kMaxLocalPairs = 1ll << 40;             // as sim_range's max_pairs
enum { H_MAGIC, H_STATUS, H_PAIRS, H_CAND, H_CAND_CAP, H_MAX_PAIRS, H_NQ, H_D, H_THR, H_PARTS };

// bytes of a message holding `pairs` pairs: int64 offsets[nq + 1], int64 idx[pairs], fp32 scores[pairs], 16-byte multiple
inline size_t msg_bytes(int nq, long long pairs) {
  return (8 * (static_cast<size_t>(nq) + 1) + 12 * static_cast<size_t>(pairs) + 15) / 16 * 16;
}

// the header buffers [send | world receive slots] at the head of the workspace
inline size_t header_bytes(int world) { return kHdrWords * sizeof(long long) * (static_cast<size_t>(world) + 1); }

// The workspace: the header buffers, the local search's workspace, the send and receive buffers, the merged row counts
// and a flag.  With a null base only L->total is meaningful.
struct ShardLayout {
  size_t inner;                      // sim_range workspace of the local search
  uint8_t *inner_ws, *send, *recv;
  long long* row_cnt;
  int* flag;
  size_t total;
};

// The score a sharded threshold search computes.  One part of either split score is the dot product: such a rank plans,
// searches and writes header word [9] as kDot, so it agrees with a dot-product peer.
enum class Score { kDot, kAligned, kCross };

const char* sharded_name(Score s) {
  return s == Score::kDot ? "sim_range_sharded" : s == Score::kCross ? "sim_range_cross_sharded" : "sim_range_split_sharded";
}

// header word [9]: 0 the dot product, n_parts the aligned split score, -n_parts the cross split score (n_parts >= 2), so
// that no two forms write the same word
long long score_word(Score s, int n_parts) {
  return s == Score::kDot ? 0 : s == Score::kCross ? -static_cast<long long>(n_parts) : n_parts;
}

// the form a header word names, for the disagreement message
std::string score_of_word(long long w) {
  if (w == 0) return "the dot product";
  const unsigned long long parts = w < 0 ? 0ull - static_cast<unsigned long long>(w) : static_cast<unsigned long long>(w);
  return std::string(w < 0 ? "the cross score over " : "the aligned score over ") + std::to_string(parts) + " parts";
}

// kDot: the local search is sim_range (n_parts unused); kAligned / kCross: sim_range_split over n_parts >= 2 parts
int shard_layout(int nq, int ng_local, int d, Score score, int n_parts, int world, long long cap, void* base,
                 ShardLayout* L) {
  const char* who = sharded_name(score);
  DCR_REQUIRE(world >= 1 && world <= kMaxWorld, "%s: world=%d outside [1, %d]", who, world, kMaxWorld);
  DCR_REQUIRE(nq >= 1 && ng_local >= 0, "%s: bad problem (nq=%d ng_local=%d)", who, nq, ng_local);
  DCR_REQUIRE(cap >= 0 && cap <= kMaxLocalPairs, "%s: max_local_pairs=%lld outside [0, 2^40]", who, cap);
  // an empty shard runs no search, but its d is still checked by the same planner
  const int ng_plan = ng_local > 0 ? ng_local : 1;
  L->inner = score == Score::kDot ? sim_range_workspace_size(nq, ng_plan, d, cap)
                                  : sim_range_split_workspace_size(nq, ng_plan, d, n_parts, cap, score == Score::kCross);
  if (L->inner == 0) return -1;
  if (ng_local == 0) L->inner = 0;
  const size_t msg = msg_bytes(nq, cap);
  Carve w{static_cast<uint8_t*>(base)};
  w.take<uint8_t>(header_bytes(world));
  L->inner_ws = w.take<uint8_t>(L->inner);
  L->send = w.take<uint8_t>(msg);
  L->recv = w.take<uint8_t>(msg * static_cast<size_t>(world));
  L->row_cnt = w.take<long long>(nq);
  L->flag = w.take<int>(1);
  L->total = w.bytes;
  return 0;
}

// the gathered messages, rank-major, `stride` bytes apart; pairs of rank r = hdr[r][H_PAIRS]
struct ShardMsgs {
  const uint8_t* base;
  size_t stride;
  const long long* hdr;
  int nq, world;
  DCR_DEVICE const long long* off(int r) const { return reinterpret_cast<const long long*>(base + r * stride); }
  DCR_DEVICE const long long* idx(int r) const { return off(r) + nq + 1; }
  DCR_DEVICE const float* scores(int r) const { return reinterpret_cast<const float*>(idx(r) + pairs(r)); }
  DCR_DEVICE long long pairs(int r) const { return hdr[static_cast<size_t>(r) * kHdrWords + H_PAIRS]; }
};

// merged count of every row, summed in rank order; bad = 1 when a message's offsets are not a CSR of its pair count
__global__ void __launch_bounds__(256) shard_row_count_kernel(const ShardMsgs m, long long* __restrict__ row_cnt,
                                                              int* __restrict__ bad) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m.nq; i += gridDim.x * blockDim.x) {
    long long c = 0;
    bool ok = true;
    for (int r = 0; r < m.world; ++r) {
      const long long* o = m.off(r);
      const long long p = m.pairs(r), lo = o[i], hi = o[i + 1];
      ok = ok && lo >= 0 && lo <= hi && hi <= p && (i > 0 || lo == 0) && (i < m.nq - 1 || hi == p);
      c += hi - lo;
    }
    row_cnt[i] = c;
    if (!ok) *bad = 1;
  }
}

// Entry e of rank blockIdx.y: its row i (binary search in the rank's offsets) and its place in the merged row, the
// entries of row i before it in its own piece plus, for every other rank, the entries of that rank's piece of row i
// with a smaller index (lower bound).  kPlace = 0 only checks: indices strictly ascending within a piece and no index
// in two ranks' pieces of a row.  kPlace = 1 writes the entry; it runs only after the check passed.  Reads are clamped
// to each message's pairs, so a malformed message is found without reading past it.
template <bool kPlace>
__global__ void __launch_bounds__(256)
    shard_merge_kernel(const ShardMsgs m, const long long* __restrict__ row_offsets, long long* __restrict__ out_idx,
                       float* __restrict__ out_scores, int* __restrict__ bad) {
  const int r = blockIdx.y;
  const long long pr = m.pairs(r);
  const long long* o = m.off(r);
  const long long* ix = m.idx(r);
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < pr;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    int lo = 0, hi = m.nq;   // o[lo] <= e < o[hi]
    while (hi - lo > 1) {
      const int mid = lo + (hi - lo) / 2;
      if (o[mid] <= e) lo = mid;
      else hi = mid;
    }
    const int i = lo;
    const long long v = ix[e];
    bool dup = e > 0 && e > o[i] && ix[e - 1] >= v;
    long long pos = e - o[i];
    for (int s = 0; s < m.world; ++s) {
      if (s == r) continue;
      const long long ps = m.pairs(s);
      const long long* os = m.off(s);
      const long long* xs = m.idx(s);
      const long long b = min(max(os[i], 0ll), ps);
      long long a = b, z = min(max(os[i + 1], b), ps);   // lower bound of v in xs[b, z)
      while (a < z) {
        const long long mid = a + (z - a) / 2;
        if (xs[mid] < v) a = mid + 1;
        else z = mid;
      }
      pos += a - b;
      dup = dup || (a < min(max(os[i + 1], b), ps) && xs[a] == v);
    }
    if constexpr (kPlace) {
      const long long at = row_offsets[i] + pos;
      out_idx[at] = v;
      out_scores[at] = m.scores(r)[e];
    } else {
      if (dup) *bad = 1;
    }
  }
}

// Gathers `bytes` from every rank's `send` into `recv`, rank-major: a copy when world = 1, else the caller's callback.
int allgather_step(const char* who, int world, AllgatherFn allgather, void* ctx, const void* send, void* recv, size_t bytes,
                   cudaStream_t stream) {
  if (world == 1) {
    DCR_CUDA_CHECK(cudaMemcpyAsync(recv, send, bytes, cudaMemcpyDeviceToDevice, stream));
    return 0;
  }
  const int arc = allgather(send, recv, bytes, ctx, static_cast<void*>(stream));
  DCR_REQUIRE(arc == 0, "%s: the all-gather callback failed (%d)", who, arc);
  return 0;
}

// The top-k workspace: the local search's, this rank's list [scores f32 [nq,k] | indices i64 [nq,k]], world such lists
// gathered, and those un-interleaved into [world][nq][k] scores and indices.  With a null base only inner and total are
// meaningful; total is 0 for a problem the local planner refuses.
struct TopkShardLayout {
  size_t inner;                      // sim_topk workspace of the local search
  uint8_t *inner_ws, *send, *recv;
  float* all_s;
  long long* all_i;
  size_t total;
};

TopkShardLayout topk_shard_layout(int nq, int ng_local, int d, int k, int world, void* base) {
  TopkShardLayout L{};
  if (world < 1 || k < 1 || nq < 1) return L;
  const int kk = std::min(k, ng_local);
  L.inner = sim_topk_workspace_size(nq, ng_local, d, std::max(kk, 1));
  if (L.inner == 0) return L;
  const size_t list = static_cast<size_t>(nq) * k;
  Carve w{static_cast<uint8_t*>(base)};
  L.inner_ws = w.take<uint8_t>(L.inner);
  L.send = w.take<uint8_t>(list * 12);
  L.recv = w.take<uint8_t>(list * 12 * world);
  L.all_s = w.take<float>(list * world);
  L.all_i = w.take<long long>(list * world);
  L.total = w.bytes;
  return L;
}

// the header buffers of one call: at the head of the workspace, or -- when the caller's workspace cannot hold even them
// -- allocated on the stream, so that such a rank still takes part in the header exchange
struct HeaderBuf {
  long long* p = nullptr;
  bool owned = false;
  cudaStream_t st;
  explicit HeaderBuf(cudaStream_t s) : st(s) {}
  ~HeaderBuf() {
    if (owned) cudaFreeAsync(p, st);
  }
};

}  // namespace

size_t sim_topk_sharded_workspace_size(int nq, int ng_local, int d, int k, int world) {
  return topk_shard_layout(nq, ng_local, d, k, world, nullptr).total;
}

int sim_topk_sharded(const float* q, int nq, const float* g, int ng_local, int d, int k, long long g_index_base,
                     long long g_index_stride, int world, AllgatherFn allgather, void* allgather_ctx, float* out_scores,
                     long long* out_idx, void* ws, size_t ws_bytes, cudaStream_t stream, SimStats* stats) {
  DCR_REQUIRE(q && g && out_scores && out_idx && ws, "dcr_sim_topk_sharded: null pointer argument");
  DCR_REQUIRE(world >= 1 && (world == 1 || allgather != nullptr), "dcr_sim_topk_sharded: world=%d needs an all-gather callback", world);
  DCR_REQUIRE(static_cast<long long>(world) * k <= 1024, "dcr_sim_topk_sharded: world * k = %d > 1024", world * k);
  const TopkShardLayout L = topk_shard_layout(nq, ng_local, d, k, world, ws);
  DCR_REQUIRE(L.total != 0 && ws_bytes >= L.total, "dcr_sim_topk_sharded: workspace too small (%zu < %zu)", ws_bytes, L.total);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "dcr_sim_topk_sharded: workspace must be 256-byte aligned");
  const size_t list = static_cast<size_t>(nq) * k;
  float* loc_s = reinterpret_cast<float*>(L.send);
  long long* loc_i = reinterpret_cast<long long*>(L.send + list * 4);
  // fewer gallery rows than k on this rank: top-kk into a compact list in all_s/all_i (not yet in use), then spread into
  // the k-wide slots with empty (-inf, -1) entries in the rest
  const int kk = std::min(k, ng_local);
  if (int rc = sim_topk(q, nq, g, ng_local, d, kk, g_index_base, g_index_stride, kk < k ? L.all_s : loc_s,
                        kk < k ? L.all_i : loc_i, L.inner_ws, L.inner, stream, stats))
    return rc;
  if (kk < k) {
    if (int rc = pad_topk_lists(L.all_s, L.all_i, nq, kk, k, loc_s, loc_i, stream)) return rc;
  }
  if (world == 1) {
    DCR_CUDA_CHECK(cudaMemcpyAsync(out_scores, loc_s, list * 4, cudaMemcpyDeviceToDevice, stream));
    DCR_CUDA_CHECK(cudaMemcpyAsync(out_idx, loc_i, list * 8, cudaMemcpyDeviceToDevice, stream));
    return 0;
  }
  if (int rc = allgather_step("dcr_sim_topk_sharded", world, allgather, allgather_ctx, L.send, L.recv, list * 12, stream))
    return rc;
  // un-interleave the gathered lists into [world][nq][k] score and index arrays, then merge
  for (int r = 0; r < world; ++r) {
    const uint8_t* block = L.recv + static_cast<size_t>(r) * list * 12;
    DCR_CUDA_CHECK(cudaMemcpyAsync(L.all_s + static_cast<size_t>(r) * list, block, list * 4, cudaMemcpyDeviceToDevice, stream));
    DCR_CUDA_CHECK(cudaMemcpyAsync(L.all_i + static_cast<size_t>(r) * list, block + list * 4, list * 8, cudaMemcpyDeviceToDevice,
                                   stream));
  }
  return topk_merge(L.all_s, L.all_i, nq, world, k, k, out_scores, out_idx, stream);
}

namespace {

// The sharded threshold search.  score = kDot: the dot product (n_parts unused); kAligned / kCross: that split score over
// n_parts parts, one part being the dot product itself (the search, and header word [9], of kDot then).
int range_sharded(const float* q, int nq, const float* g, int ng_local, int d, Score score, int n_parts, float threshold,
                  long long g_index_base, long long g_index_stride, int world, AllgatherFn allgather, void* allgather_ctx,
                  long long* row_offsets, long long* out_idx, float* out_scores, long long max_pairs,
                  long long max_local_pairs, long long* counts, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const char* who = sharded_name(score);
  const Score form = n_parts > 1 ? score : Score::kDot;   // one part is the dot product; n_parts < 1 is refused below
  // the only outcomes decided before the first exchange: without these there is nobody to agree with
  DCR_REQUIRE(world >= 1 && world <= kMaxWorld, "%s: world=%d outside [1, %d]", who, world, kMaxWorld);
  DCR_REQUIRE(world == 1 || allgather != nullptr, "%s: world=%d needs an all-gather callback", who, world);

  // 1. the local search; its outcome goes into the header, whatever it is
  uint32_t thr_bits;
  std::memcpy(&thr_bits, &threshold, 4);
  long long hdr[kHdrWords] = {kHdrMagic, 0, 0, 0, max_local_pairs, max_pairs, nq, d, static_cast<long long>(thr_bits),
                             score_word(form, n_parts)};
  ShardLayout L{};
  uint8_t* w = static_cast<uint8_t*>(ws);
  auto local = [&]() -> int {
    DCR_REQUIRE(q && (g || ng_local == 0) && row_offsets && counts && (max_pairs == 0 || (out_idx && out_scores)),
                "%s: null pointer argument", who);
    DCR_REQUIRE(score == Score::kDot || n_parts >= 1, "%s: n_parts=%d < 1", who, n_parts);
    DCR_REQUIRE(!std::isnan(threshold), "%s: threshold is NaN", who);
    DCR_REQUIRE(g_index_stride >= 1, "%s: g_index_stride=%lld < 1", who, g_index_stride);
    DCR_REQUIRE(max_pairs >= 0, "%s: max_pairs=%lld < 0", who, max_pairs);
    if (int rc = shard_layout(nq, ng_local, d, form, n_parts, world, max_local_pairs, w, &L)) return rc;
    DCR_REQUIRE(w != nullptr && ws_bytes >= L.total, "%s: workspace too small (%zu < %zu)", who, ws_bytes, L.total);
    DCR_REQUIRE((reinterpret_cast<uintptr_t>(w) & 255) == 0, "%s: workspace must be 256-byte aligned", who);
    long long* send_off = reinterpret_cast<long long*>(L.send);
    if (ng_local == 0) {
      DCR_CUDA_CHECK(cudaMemsetAsync(send_off, 0, 8 * (static_cast<size_t>(nq) + 1), stream));
      return 0;
    }
    // indices go straight into the message; the scores wait in the (not yet used) receive buffer and follow the
    // indices once their count is known
    long long* send_idx = send_off + nq + 1;
    float* tmp_scores = reinterpret_cast<float*>(L.recv);
    long long c[2] = {0, 0};
    const int rc = form == Score::kDot
                       ? sim_range(q, nq, g, ng_local, d, threshold, g_index_base, g_index_stride, send_off, send_idx,
                                   tmp_scores, max_local_pairs, c, L.inner_ws, L.inner, stream)
                       : sim_range_split(q, nq, g, ng_local, d, n_parts, threshold, g_index_base, g_index_stride, send_off,
                                         send_idx, tmp_scores, max_local_pairs, c, L.inner_ws, L.inner, stream,
                                         form == Score::kCross);
    hdr[H_CAND] = c[1];
    if (rc) return rc;
    hdr[H_PAIRS] = c[0];
    if (c[0] > 0)
      DCR_CUDA_CHECK(cudaMemcpyAsync(send_idx + c[0], tmp_scores, 4 * static_cast<size_t>(c[0]), cudaMemcpyDeviceToDevice,
                                     stream));
    return 0;
  };
  const int local_rc = local();
  const std::string local_msg = local_rc ? last_error_storage() : std::string();
  hdr[H_STATUS] = local_rc;

  // 2. the headers: every rank decides from the same gathered words
  HeaderBuf hb(stream);
  const size_t hbytes = kHdrWords * sizeof(long long);
  if (w != nullptr && (reinterpret_cast<uintptr_t>(w) & 255) == 0 && ws_bytes >= header_bytes(world)) {
    hb.p = reinterpret_cast<long long*>(w);
  } else {
    DCR_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&hb.p), header_bytes(world), stream));
    hb.owned = true;
  }
  long long* h_send = hb.p;
  long long* h_recv = hb.p + kHdrWords;
  DCR_CUDA_CHECK(cudaMemcpyAsync(h_send, hdr, hbytes, cudaMemcpyHostToDevice, stream));
  if (int rc = allgather_step(who, world, allgather, allgather_ctx, h_send, h_recv, hbytes, stream)) return rc;
  std::vector<long long> H(static_cast<size_t>(world) * kHdrWords);
  DCR_CUDA_CHECK(cudaMemcpyAsync(H.data(), h_recv, hbytes * world, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  auto h = [&](int r, int f) { return H[static_cast<size_t>(r) * kHdrWords + f]; };
  if (counts) counts[0] = counts[1] = counts[2] = 0;
  for (int r = 0; r < world; ++r)
    DCR_REQUIRE(h(r, H_MAGIC) == kHdrMagic, "%s: rank %d sent a malformed header", who, r);
  for (int r = 0; r < world; ++r) {
    const long long st = h(r, H_STATUS);
    if (st != 0 && st != DCR_ERR_CAPACITY)
      return set_error(static_cast<int>(st), "%s: rank %d failed (%lld)%s%s", who, r, st,
                       local_rc ? "; this rank: " : "", local_msg.c_str());
  }
  for (int r = 1; r < world; ++r)
    DCR_REQUIRE(h(r, H_NQ) == h(0, H_NQ) && h(r, H_D) == h(0, H_D) && h(r, H_THR) == h(0, H_THR),
                "%s: ranks disagree on the problem: rank 0 has nq=%lld d=%lld threshold bits 0x%llx, rank %d "
                "has nq=%lld d=%lld threshold bits 0x%llx",
                who, h(0, H_NQ), h(0, H_D), h(0, H_THR), r, h(r, H_NQ), h(r, H_D), h(r, H_THR));
  for (int r = 1; r < world; ++r)
    DCR_REQUIRE(h(r, H_PARTS) == h(0, H_PARTS), "%s: ranks disagree on the score: rank 0 computes %s, rank %d %s", who,
                score_of_word(h(0, H_PARTS)).c_str(), r, score_of_word(h(r, H_PARTS)).c_str());
  // capacities: every local search finished, every receive buffer holds the largest message, every output the total
  bool finished = true;
  long long cand_need = 0, p_max = 0, total = 0, min_cap = h(0, H_CAND_CAP), min_out = h(0, H_MAX_PAIRS);
  for (int r = 0; r < world; ++r) {
    const bool ok = h(r, H_STATUS) == 0;
    finished = finished && ok;
    cand_need = std::max(cand_need, h(r, H_CAND));
    if (ok) p_max = std::max(p_max, h(r, H_PAIRS));
    total += ok ? h(r, H_PAIRS) : h(r, H_CAND);   // an unfinished search: its candidates bound its pairs
    min_cap = std::min(min_cap, h(r, H_CAND_CAP));
    min_out = std::min(min_out, h(r, H_MAX_PAIRS));
  }
  counts[1] = cand_need;
  counts[2] = total;
  if (!finished || p_max > min_cap || total > min_out)
    return set_error(DCR_ERR_CAPACITY,
                     "%s: capacity too small on some rank (call again with max_local_pairs=%lld, "
                     "max_pairs=%lld on every rank)", who, cand_need, total);

  // 3. the messages, each padded to the largest
  const size_t msg = msg_bytes(nq, p_max);
  if (int rc = allgather_step(who, world, allgather, allgather_ctx, L.send, L.recv, msg, stream)) return rc;

  // 4. the merge
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  long long* row_cnt = L.row_cnt;
  int* bad = L.flag;
  const ShardMsgs m = {L.recv, msg, h_recv, nq, world};
  const dim3 grid(static_cast<unsigned>(std::max(1, grid_for(std::max(p_max, 1ll), 256, di->num_sms) / world)),
                  static_cast<unsigned>(world));
  DCR_CUDA_CHECK(cudaMemsetAsync(bad, 0, 4, stream));
  if (int rc = launch(shard_row_count_kernel, grid_for(nq, 256, di->num_sms), 256, 0, stream, who, m, row_cnt, bad))
    return rc;
  if (p_max > 0) {
    if (int rc = launch(shard_merge_kernel<false>, grid, 256, 0, stream, who, m, nullptr, nullptr, nullptr, bad))
      return rc;
  }
  int h_bad = 0;
  DCR_CUDA_CHECK(cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, stream));
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  DCR_REQUIRE(h_bad == 0,
              "%s: two ranks report the same gallery index (the shards overlap), or a rank's message is "
              "not an ascending CSR of its pairs", who);
  if (int rc = exclusive_scan_i64(row_cnt, nq, row_offsets, stream)) return rc;
  if (p_max > 0) {
    if (int rc = launch(shard_merge_kernel<true>, grid, 256, 0, stream, who, m, row_offsets, out_idx, out_scores, bad))
      return rc;
  }
  DCR_CUDA_CHECK(cudaStreamSynchronize(stream));
  counts[0] = total;
  return 0;
}

}  // namespace

size_t sim_range_sharded_workspace_size(int nq, int ng_local, int d, int world, long long max_local_pairs) {
  ShardLayout L;
  if (shard_layout(nq, ng_local, d, Score::kDot, 0, world, max_local_pairs, nullptr, &L) != 0) return 0;
  return L.total;
}

int sim_range_sharded(const float* q, int nq, const float* g, int ng_local, int d, float threshold, long long g_index_base,
                      long long g_index_stride, int world, AllgatherFn allgather, void* allgather_ctx, long long* row_offsets,
                      long long* out_idx, float* out_scores, long long max_pairs, long long max_local_pairs,
                      long long* counts, void* ws, size_t ws_bytes, cudaStream_t stream) {
  return range_sharded(q, nq, g, ng_local, d, Score::kDot, 0, threshold, g_index_base, g_index_stride, world, allgather,
                       allgather_ctx, row_offsets, out_idx, out_scores, max_pairs, max_local_pairs, counts, ws, ws_bytes,
                       stream);
}

size_t sim_range_split_sharded_workspace_size(int nq, int ng_local, int d, int n_parts, int world, long long max_local_pairs,
                                              bool cross) {
  const Score score = cross ? Score::kCross : Score::kAligned;
  if (n_parts < 1) {
    set_error(-1, "%s: n_parts=%d < 1", sharded_name(score), n_parts);
    return 0;
  }
  ShardLayout L;
  if (shard_layout(nq, ng_local, d, n_parts == 1 ? Score::kDot : score, n_parts, world, max_local_pairs, nullptr, &L) != 0)
    return 0;
  return L.total;
}

int sim_range_split_sharded(const float* q, int nq, const float* g, int ng_local, int d, int n_parts, float threshold,
                            long long g_index_base, long long g_index_stride, int world, AllgatherFn allgather,
                            void* allgather_ctx, long long* row_offsets, long long* out_idx, float* out_scores,
                            long long max_pairs, long long max_local_pairs, long long* counts, void* ws, size_t ws_bytes,
                            cudaStream_t stream, bool cross) {
  return range_sharded(q, nq, g, ng_local, d, cross ? Score::kCross : Score::kAligned, n_parts, threshold, g_index_base,
                       g_index_stride, world, allgather, allgather_ctx, row_offsets, out_idx, out_scores, max_pairs,
                       max_local_pairs, counts, ws, ws_bytes, stream);
}

}  // namespace dcr
