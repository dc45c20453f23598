// 3x3 / stride 1 / pad 1 convolution as an implicit GEMM whose A operand is loaded ONCE per tile.
//
// The generic kernel (conv_gemm.cu) gathers one [128 pixels x 64 channels] A tile per filter tap, i.e. every input
// pixel travels L2 -> shared memory nine times; for the convolutions with few output channels that ingest is the
// bound (DESIGN.md section 5: load-only timing mode = 96 % of the layer time).  Here a tile is R whole output rows of
// one image and the producer loads, per 64-channel block, ONE halo block
//       [(R + 2) input rows] x [(W + 2) pixels, the two extra ones zero-filled by the TMA unit] x [64 channels]
// as a single 4-D tiled TMA box.  In shared memory that is a width-padded raster of 128-byte rows, so the A operand of
// filter tap (r, s) is the SAME buffer read from a start address shifted by (r * (W + 2) + s) rows: nine wgmma descriptor
// start addresses instead of nine loads.  (The 128-byte swizzle is a function of the absolute shared-memory address
// on both the TMA write and the wgmma read side, so a start address that is a multiple of 128 B but not of 1024 B is
// fine.)  MMA row m of the tile is padded-raster position m = pl * (W + 2) + ql; positions with ql >= W (2 per row)
// and the rows past R * (W + 2) are junk that the epilogue drops when it compacts the tile into the [R x W] staging
// box of the TMA store.  W + 2 <= 64 and R = 128 / (W + 2) rows: 2 rows at 56 wide (87.5 % useful MMA rows), 4 at 28,
// 8 at 14.  Used for N <= 128 (at N = 256 only two 32 KB weight stages fit beside the halo buffers).
//
// Weights are streamed per (tap, channel block) exactly as in the generic kernel (all SMs read the same tiles; that
// traffic is served at several times the rate of per-SM-unique data).  Fast (single-plane bf16) mode only, no residual:
// what the 3x3 convolutions of the ResNet / ResNeXt bottlenecks need.
//
// Ping-pong schedule (as in conv_gemm.cu): the CTA's tiles are dealt alternately to the two consumer
// warpgroups, each accumulates whole 128 x BN tiles, and a warpgroup starts its k-loop only once the other one has issued
// its last wgmma, so one tile's epilogue runs under the next tile's k-loop.  The halo ring and the weight ring (or the
// resident taps) are shared in tile order; each warpgroup has its own output staging box, which its epilogue fills
// straight from the accumulator layout (no transpose buffers: that shared memory keeps a third halo buffer at W = 56).
#include <cuda_bf16.h>

#include <algorithm>
#include <cstring>

#include "dcr_internal.cuh"
#include "host_util.cuh"
#include "ptx.cuh"

namespace dcr {

namespace {

constexpr int kHM = 128;                    // MMA rows (padded-raster positions) per tile
constexpr int kHK = 64;                     // channels per block = one 128-byte swizzled row
constexpr int kSlabBytes = kHM * 128;       // one 64-channel slab of the output staging tile
// warps 0-7 two consumer warpgroups (MMA + epilogue), warp 8 producer, warps 9-11 idle: the producer warpgroup's
// registers go to the consumers (8 x 224 + 4 x 56 per lane = the 384 x 168 the CTA is launched with)
constexpr int kHThreads = 384;
constexpr int kHConsumerRegs = 224, kHProducerRegs = 56;

struct HaloMaps {
  CUtensorMap a;     // input  [B][H][W][C]   box 64 x (W+2) x (R+2) x 1
  CUtensorMap w;     // weights [N][9 * cblocks * 64] box 64 x BN
  CUtensorMap out;   // output [B][H][W][ld_out] box 64 x W x R x 1
};

struct HaloParams {
  int H, W, Wp, R, N, cblocks;
  int tiles_per_img, num_tiles;
  int a_bufs, w_stages;
  uint32_t halo_bytes;     // bytes one halo box delivers
  uint32_t a_buf_bytes;    // bytes reserved per halo buffer: the box and the last tap's 128-row window stay inside (1024-aligned)
  const float* scale;
  const float* bias;
  int act, out_col_off;
};

// kRW: ALL filter taps stay resident in shared memory (9 * cblocks tiles of [BN x 64]; fits for the 64 -> 64 convolutions of
// ResNet layer1: 72 KB): no weight ring, the producer only streams halo boxes.
template <int BN, bool kRW>
__global__ void __launch_bounds__(kHThreads, 1)
    conv3x3_halo_kernel(const __grid_constant__ HaloMaps maps, const HaloParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  constexpr int kWStage = BN * 128;
  constexpr int kStageBytes = (BN / 64) * kSlabBytes;                       // one output staging box
  uint8_t* a_ring = smem;
  uint8_t* w_ring = a_ring + p.a_bufs * p.a_buf_bytes;                // kRW: 9 * cblocks resident tiles, tap-major
  uint8_t* out_stage = w_ring + (kRW ? 9 * p.cblocks : p.w_stages) * kWStage;   // [2 warpgroups] BN/64 slabs
  float* sb = reinterpret_cast<float*>(out_stage + 2 * kStageBytes);      // [scale | bias][BN]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sb + 2 * BN);
  uint64_t* a_full = bars;          // [4]
  uint64_t* a_empty = bars + 4;     // [4]
  uint64_t* w_full = bars + 8;      // [8]
  uint64_t* w_empty = bars + 16;    // [8]
  uint64_t* turn = bars + 24;       // [2] PingPong::turn

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&maps.a);
    tma_prefetch_desc(&maps.w);
    tma_prefetch_desc(&maps.out);
  }
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < p.a_bufs; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 4);   // one arrive per warp of the warpgroup that consumes it
    }
    for (int s = 0; s < (kRW ? 1 : p.w_stages); ++s) {
      mbar_init(&w_full[s], 1);
      mbar_init(&w_empty[s], 4);
    }
    for (int g = 0; g < 2; ++g) mbar_init(&turn[g], 4);   // the other warpgroup's four warps
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================================== TMA producer =====================================
    // (whole warp walks the loop, one elected lane issues: see conv_gemm.cu)
    wg_regs_dec<kHProducerRegs>();
    if (warp == 8) {
      PipeState as(p.a_bufs), ws(kRW ? 1 : p.w_stages);
      if constexpr (kRW) {   // every filter tap once
        if (elect_one()) {
          mbar_arrive_expect_tx(&w_full[0], 9 * p.cblocks * kWStage);
          for (int t = 0; t < 9 * p.cblocks; ++t)
            tma_load_2d(w_ring + t * kWStage, &maps.w, &w_full[0], t * kHK, 0, kEvictLast);
        }
        __syncwarp();
      }
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int b = tile / p.tiles_per_img;
        const int p0 = (tile - b * p.tiles_per_img) * p.R;
        for (int cb = 0; cb < p.cblocks; ++cb, as.next()) {
          const uint32_t sa = as.s, pha = as.ph;
          mbar_wait(&a_empty[sa], pha ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&a_full[sa], p.halo_bytes);
            // rows p0-1 .. p0+R, columns -1 .. W: everything outside the image arrives as zeros (the padding)
            tma_load_4d(a_ring + sa * p.a_buf_bytes, &maps.a, &a_full[sa], cb * kHK, -1, p0 - 1, b, kEvictNormal);
          }
          __syncwarp();
          if constexpr (kRW) continue;
          for (int tap = 0; tap < 9; ++tap, ws.next()) {
            const uint32_t sw = ws.s, phw = ws.ph;
            mbar_wait(&w_empty[sw], phw ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&w_full[sw], kWStage);
              tma_load_2d(w_ring + sw * kWStage, &maps.w, &w_full[sw], (tap * p.cblocks + cb) * kHK, 0, kEvictLast);
            }
            __syncwarp();
          }
        }
      }
    }
  } else {
    // ===================================== consumer warpgroups =====================================
    wg_regs_inc<kHConsumerRegs>();
    const uint32_t quad = warp & 3;
    const uint32_t wg = warp >> 2;
    const uint32_t gtid = (warp & 3) * 32 + lane;       // 0..127 within the warpgroup
    const uint32_t a_base = smem_u32(a_ring);
    const uint32_t w_base = smem_u32(w_ring);
    const uint32_t row_bytes = static_cast<uint32_t>(p.Wp) * 128u;   // one padded image row (128 B per pixel)
    const int k_groups = 9 * p.cblocks;                 // one wgmma group (4 x k16) per (channel block, tap)
    PipeState as(p.a_bufs), ws(kRW ? 1 : p.w_stages);
    if constexpr (kRW) mbar_wait(&w_full[0], 0);
    // this thread's accumulator rows (WgAcc layout: rows r0 + 8 g of its warp's 32-row block, g = 0..3) -> rows of the
    // compact [R x W] staging box; junk positions (the two pad columns per padded row, rows past R) are dropped
    const uint32_t r0 = lane >> 2, c0 = 2 * (lane & 3);
    uint32_t srow[4];
    bool valid[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int m = static_cast<int>(quad * 32 + r0 + 8 * g);   // padded-raster position
      const int pl = m / p.Wp, ql = m - pl * p.Wp;
      valid[g] = ql < p.W && pl < p.R;
      srow[g] = static_cast<uint32_t>(pl * p.W + ql);
    }
    const uint32_t sb_addr = smem_u32(sb), stage_addr = smem_u32(out_stage) + wg * kStageBytes;
    uint8_t* ostage = out_stage + wg * kStageBytes;
    for (int c = warp * 32 + lane; c < BN; c += 256) {
      st_shared_f32(sb_addr + c * 4, p.scale ? p.scale[c] : 1.f);
      st_shared_f32(sb_addr + (BN + c) * 4, p.bias ? p.bias[c] : 0.f);
    }
    named_bar_sync(5, 256);
    if (wg == 1) {                                      // the CTA's first tile is warpgroup 0's
      as.skip(p.cblocks);
      if constexpr (!kRW) ws.skip(k_groups);
    }
    const PingPong pingpong{turn};
    uint32_t tc = 0;
    for (int tile = blockIdx.x + wg * gridDim.x; tile < p.num_tiles; tile += 2 * gridDim.x, ++tc) {
      const int b = tile / p.tiles_per_img;
      const int p0 = (tile - b * p.tiles_per_img) * p.R;
      if (gtid == 0) tma_store_wait_read<0>();     // this warpgroup's previous store has finished reading its staging box
      named_bar_sync(1 + 2 * wg, 128);
      pingpong.wait(wg, tc);
      // main loop: per channel block one halo box, nine taps = nine start addresses into it.  Group (cb, tap)'s operands
      // are released once wgmma_wait<1> after the next group has seen it complete.
      WgAcc<BN> acc;
      uint32_t prev_w = 0, prev_a = 0;
      bool prev_a_last = false;
      for (int cb = 0; cb < p.cblocks; ++cb, as.next()) {
        const uint32_t sa = as.s;
        mbar_wait(&a_full[sa], as.ph);
        const uint32_t a_buf = a_base + sa * p.a_buf_bytes;
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
          const int r = tap / 3, s = tap - 3 * r;
          uint32_t sw = 0;
          if constexpr (!kRW) {
            sw = ws.s;
            mbar_wait(&w_full[sw], ws.ph);
          } else {
            sw = static_cast<uint32_t>(tap * p.cblocks + cb);   // resident tile of this (tap, channel block)
          }
          // the tap's view of the halo block: same buffer, start shifted by r padded rows + s pixels (128 B each)
          const uint32_t a_addr = a_buf + r * row_bytes + s * 128u;
          const uint32_t b_addr = w_base + sw * kWStage;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kHK / 16; ++k) acc.mma(a_addr + 32 * k, wgmma_desc_sw128(b_addr + 32 * k), (cb | tap | k) != 0);
          wgmma_commit();
          const bool last = cb == p.cblocks - 1 && tap == 8;
          if (last && lane == 0) pingpong.hand_over(wg);
          wgmma_wait<1>();
          if ((cb | tap) != 0 && lane == 0) {
            if constexpr (!kRW) mbar_arrive(&w_empty[prev_w]);
            if (prev_a_last) mbar_arrive(&a_empty[prev_a]);
          }
          prev_w = sw;
          prev_a = sa;
          prev_a_last = tap == 8;
          if constexpr (!kRW) ws.next();
        }
      }
      wgmma_wait<0>();
      acc.fence_regs();
      if (lane == 0) {
        if constexpr (!kRW) mbar_arrive(&w_empty[prev_w]);
        mbar_arrive(&a_empty[prev_a]);
      }
      as.skip(p.cblocks);                                // the other warpgroup's next tile
      if constexpr (!kRW) ws.skip(k_groups);
      // epilogue: straight from the accumulator layout into the 128B-swizzled staging box, one bf16 pair per store (a
      // warp's 8 rows x 16 B per store land in 8 different 16-byte bank groups)
      acc.for_each_pair(lane, [&](uint32_t row, uint32_t col, float v0, float v1) {
        const uint32_t g = (row - r0) >> 3;
        const float2 sc = ld_shared_f2(sb_addr + col * 4);
        const float2 bi = ld_shared_f2(sb_addr + (BN + col) * 4);
        float y0 = fmaf(v0, sc.x, bi.x), y1 = fmaf(v1, sc.y, bi.y);
        if (p.act == 1) {
          y0 = fmaxf(y0, 0.f);
          y1 = fmaxf(y1, 0.f);
        }
        const uint32_t chunk = (col & 63) >> 3;
        if (valid[g])
          st_shared_u32(stage_addr + (col >> 6) * kSlabBytes + srow[g] * 128 + ((chunk ^ (srow[g] & 7)) << 4) + c0 * 2,
                        pack_bf16x2(y0, y1));
      });
      fence_proxy_async();
      named_bar_sync(2 + 2 * wg, 128);
      if (gtid == 0) {
        for (int sl = 0; sl < BN / 64; ++sl) tma_store_4d(&maps.out, smem_u32(ostage + sl * kSlabBytes), p.out_col_off + sl * 64, 0, p0, b);
        tma_store_commit();
      }
    }
    if (gtid == 0) tma_store_wait_all();
  }
}

template <int BN, bool kRW>
int launch_halo(const HaloMaps& maps, HaloParams& p, int num_sms, size_t max_smem, cudaStream_t stream) {
  constexpr size_t kWStage = static_cast<size_t>(BN) * 128;
  const size_t fixed = 1024 + static_cast<size_t>(2) * (BN / 64) * kSlabBytes + 2 * BN * 4 + 256;   // 2 staging boxes
  const size_t abuf = p.a_buf_bytes;
  size_t smem = 0;
  if constexpr (kRW) {
    const size_t wres = static_cast<size_t>(9) * p.cblocks * kWStage;
    DCR_REQUIRE(max_smem >= fixed + wres + 2 * abuf, "conv3x3_halo: resident weights do not fit");
    p.a_bufs = static_cast<int>(std::min<size_t>(4, (max_smem - fixed - wres) / abuf));
    p.w_stages = 0;
    smem = fixed + wres + static_cast<size_t>(p.a_bufs) * abuf;
  } else {
    // two halo buffers and 3..8 weight stages; a third halo buffer if 6 weight stages still fit beside it
    p.a_bufs = 2;
    DCR_REQUIRE(max_smem >= fixed + 2 * abuf + 3 * kWStage, "conv3x3_halo: not enough shared memory");
    p.w_stages = static_cast<int>(std::min<size_t>(8, (max_smem - fixed - 2 * abuf) / kWStage));
    if (max_smem >= fixed + 3 * abuf + 6 * kWStage) {
      p.a_bufs = 3;
      p.w_stages = static_cast<int>(std::min<size_t>(8, (max_smem - fixed - 3 * abuf) / kWStage));
    }
    smem = fixed + static_cast<size_t>(p.a_bufs) * abuf + static_cast<size_t>(p.w_stages) * kWStage;
  }
  return launch(conv3x3_halo_kernel<BN, kRW>, std::min(p.num_tiles, num_sms), kHThreads, smem, stream, "conv3x3_halo",
                maps, p);
}

}  // namespace

bool conv3x3_halo_eligible(const ConvGemmDesc& d) {
  if (tuning_flag("DCR_CONV_NO_HALO")) return false;
  const bool shape = d.kh == 3 && d.kw == 3 && d.stride == 1 && d.pad_h == 1 && d.pad_w == 1 && d.in_stride_w == 0;
  const bool fast = d.n_terms == 1 && d.term_a[0] == 0 && d.term_w[0] == 0 && !d.exact && d.out != nullptr &&
                    d.out_planes <= 1 && d.out_f32 == nullptr && d.res == nullptr && (d.act == 0 || d.act == 1);
  const bool dims = d.C % 64 == 0 && d.ld_in == d.C && d.N % 64 == 0 && d.N <= 128 && d.ld_out % 8 == 0 &&
                    d.out_col_off % 8 == 0 && d.W + 2 <= 64 && d.W >= 8 && d.H >= 2 && d.B >= 1;
  return shape && fast && dims;
}

int conv3x3_halo(const ConvGemmDesc& d, cudaStream_t stream) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  HaloParams p;
  memset(&p, 0, sizeof(p));
  p.H = d.H; p.W = d.W; p.Wp = d.W + 2;
  p.R = std::min(kHM / p.Wp, d.H);
  p.N = d.N;
  p.cblocks = d.C / 64;
  p.tiles_per_img = (d.H + p.R - 1) / p.R;
  p.num_tiles = d.B * p.tiles_per_img;
  p.halo_bytes = static_cast<uint32_t>(128) * p.Wp * (p.R + 2);
  p.scale = d.scale; p.bias = d.bias; p.act = d.act; p.out_col_off = d.out_col_off;
  // the loaded block and the last tap's 128-row window (start row 2 * Wp + 2) must stay inside the buffer
  p.a_buf_bytes = (std::max<uint32_t>(p.halo_bytes, static_cast<uint32_t>(2 * p.Wp + 2 + kHM) * 128u) + 1023u) & ~1023u;
  HaloMaps maps;
  memset(&maps, 0, sizeof(maps));
  if (int rc = make_tmap_nhwc_box_bf16(&maps.a, d.in, d.B, d.H, d.W, d.C, d.C, p.Wp, p.R + 2)) return rc;
  const int BN = d.N <= 64 ? 64 : 128;
  const int ktot = 9 * p.cblocks * 64;
  if (int rc = make_tmap_2d_bf16(&maps.w, d.weight, d.N, ktot, ktot, BN, 64)) return rc;
  if (int rc = make_tmap_nhwc_box_bf16(&maps.out, d.out, d.B, d.H, d.W, d.ld_out, d.ld_out, d.W, p.R)) return rc;
  // all taps resident when the weights are small (ResNet layer1: 9 x [64 x 64] = 72 KB)
  const bool resident = BN == 64 && static_cast<size_t>(9) * p.cblocks * BN * 128 <= 80 * 1024;
  if (BN == 64) return resident ? launch_halo<64, true>(maps, p, di->num_sms, di->max_smem_optin, stream)
                                : launch_halo<64, false>(maps, p, di->num_sms, di->max_smem_optin, stream);
  return launch_halo<128, false>(maps, p, di->num_sms, di->max_smem_optin, stream);
}

}  // namespace dcr
