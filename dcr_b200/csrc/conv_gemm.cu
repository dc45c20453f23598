// wgmma GEMM / implicit-GEMM convolution with fused epilogue (sm_90a).
//
// One kernel family computes   Y[m, n] = act( scale[n] * sum_k A[m, k] * W[n, k] + bias[n] (+ R[m, n]) )
// for every dense contraction of the descriptor networks:
//   - 1x1 stride-1 convolutions and Linear layers: A is the NHWC activation matrix [M = B*H*W, K = C]   (TILED)
//   - kxk / strided convolutions: A rows are gathered on the fly by TMA im2col loads from the NHWC tensor,
//     one (filter tap, 64-channel block) per pipeline stage -- the im2col matrix never exists in HBM   (IM2COL)
// Reference call sites this replaces (all reached through `model(samples)`, utils_ret.py:751):
//   SSCD ResNet-50 trunk convs + BN + ReLU (+ residual)            (torchvision resnet50; SURVEY.md 8a4)
//   DINO ViT-S qkv / proj / fc1(+GELU) / fc2 Linear layers          dino_vits.py:96-102,119,127
//   FID Inception BasicConv2d (conv + BN eps=1e-3 + ReLU)           metrics/inception.py:197-341
//
// Precision: operands are bf16 "planes".  Fast mode uses one plane (plain bf16 x bf16 -> fp32).  Parity mode
// stores every activation / weight as 2-3 bf16 planes (hi, mid, lo with x = hi + mid + lo to ~2^-24) and
// accumulates the listed cross terms into the same register accumulator, which reproduces fp32 arithmetic on the
// tensor cores (DESIGN.md section 5).
//
// Structure per CTA (384 threads, persistent over output tiles of 128 x BN, BN = 64 or 128):
//   warps 0-7 : two consumer warpgroups in a ping-pong schedule.  The CTA's tiles are dealt alternately to warpgroup 0
//               and 1; each owns whole tiles (two m64 x BN x k16 wgmma per k16 step, fp32 accumulators in registers)
//               and runs their epilogue (scale/bias/residual/activation -> bf16 planes / fp32 -> global).  A warpgroup
//               starts its k-loop only once the other one has issued its last k-block, so the tensor core sees
//               back-to-back k-loops and each epilogue runs under the other warpgroup's k-loop.
//   warp 8    : TMA producer (A tile 128x64, W tile BNx64 per stage, 128B swizzle), one stage ring in tile order
//   warps 9-11: idle (they complete the producer warpgroup for the register reallocation)
#include <cuda_bf16.h>

#include <algorithm>
#include <cstring>

#include "dcr_internal.cuh"
#include "host_util.cuh"
#include "ptx.cuh"

namespace dcr {

namespace {

constexpr int kBM = 128;
constexpr int kBK = 64;
// warps 0-7 MMA + epilogue (two warpgroups), warp 8 TMA; warps 9-11 only complete the producer warpgroup, whose
// registers (setmaxnreg) go to the consumers: 8 x 224 + 4 x 56 per lane = the 384 x 168 the CTA is launched with.  The
// direct epilogue (run-time activation, up to three output planes, fp32 output) needs more: 8 x 240 + 4 x 24.  These
// are the splits at which ptxas reports no spills for any instantiation (DESIGN.md section 6).
constexpr int kThreads = 384;
constexpr int consumer_regs(int epi) { return epi == 0 ? 240 : 224; }
constexpr int producer_regs(int epi) { return epi == 0 ? 24 : 56; }
constexpr int kAccXposeBytes = 8 * kAccXposeWarpBytes;
constexpr int kAStage = kBM * kBK * 2;   // 16 KB
// direct epilogue: per epilogue warp a [32 rows][64 B + 16 B pad] buffer through which the bf16 planes are transposed, so that
// one warp instruction touches 8 rows x 64 contiguous bytes of global memory instead of 32 rows x 16 bytes
constexpr int kXposePitch = 80;
constexpr int kXposeWarpBytes = 32 * kXposePitch;
constexpr int kXposeBytes = 8 * kXposeWarpBytes;

struct GemmMaps {
  CUtensorMap a[3];
  CUtensorMap w[3];
  CUtensorMap out;   // TMA-store epilogue (single-plane bf16 output)
  CUtensorMap res;   // residual tile loads for that epilogue
};

struct GemmParams {
  int M, N;
  int taps, kw, cblocks;      // filter taps (kh*kw), filter width, 64-channel blocks per tap
  int n_terms;
  int term_a[kMaxGemmTerms], term_w[kMaxGemmTerms];
  int P, Q, stride, pad_h, pad_w;   // im2col geometry (output H, W)
  int num_m_tiles, num_n_tiles, stages;
  const float* scale;         // [N] or null (= 1)
  const float* bias;          // [N] or null (= 0)
  const __nv_bfloat16* res;   // residual planes [res_planes][M][ld_res] or null
  int ld_res, res_planes;
  long long res_plane_stride;
  __nv_bfloat16* out;         // [out_planes][M][ld_out] (+ out_col_off) or null
  int ld_out, out_col_off, out_planes;
  long long out_plane_stride;
  float* out_f32;             // [M][ld_out_f32] or null
  int ld_out_f32;
  int act;                    // 0 none, 1 relu, 2 gelu (erf)
  int tma_epi;                // 1: stage the bf16 output tile in shared memory and write it with TMA stores
  int fast_gelu;              // 1: single-plane bf16 mode: act 2 is the tanh-form GELU (gelu_tanh_fast); 0: erf form
  int n_fastest;              // 1: consecutive tiles are the column blocks of one m-tile (round robin over the CTAs: the CTAs that
                              //    share an m-tile's A rows read them at the same time, one HBM read + L2 hits).  Default order is
                              //    m-fastest (a CTA keeps its column block, W tile and affine for many tiles): right while A fits L2
  int a_resident;             // 1: the A rows of an m-tile (all of K) stay in shared memory while the CTA walks that m-tile's
                              //    column blocks (tiles n-fastest, contiguous tile range per CTA); stages carry only W tiles
};

// exact-erf GELU of the tensor-core epilogues: erf by Abramowitz-Stegun 7.1.26 (|error| <= 2e-7 absolute: below the bf16
// rounding of a stored activation and at the level of the split-bf16 modes' own accumulation error) -- about half the instructions of erff(), whose two-branch evaluation makes
// the fc1 + GELU layers of the ViTs ALU bound in their epilogue.
DCR_DEVICE float gelu_erf_fast(float y) {
  const float ax = fabsf(y) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, ax, 1.f)));
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * ax * ax));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float erf_abs = fmaf(-poly * t, e, 1.f);               // erf(|y| / sqrt 2)
  return 0.5f * y + 0.5f * fabsf(y) * erf_abs;                 // 0.5 y (1 + erf(y / sqrt 2)),  y erf(..) = |y| erf(|..|)
}

// GELU of the single-plane bf16 ("fast") mode: the tanh form with the hardware tanh -- 0.5 y (1 + tanh(0.79788 (y + 0.044715 y^3))),
// five FMA-pipe instructions and one MUFU per element.  It differs from the erf form by <= 4.7e-4 absolute (the form itself) plus
// <= 5e-4 |y| / 2 (tanh.approx.f32), below the bf16 rounding of the stored activation (2^-9 relative) for every |y| >= 0.1 and
// within two bf16 ulps below that.  The erf polynomial above costs 16 instructions and TWO MUFU ops per element: over a 128 x 256
// tile that is 4096 MUFU cycles against 3072 MMA cycles, which makes fc1 + GELU epilogue bound.
// The split-bf16 (fp32-level) modes and the float64 mode keep the erf forms.
DCR_DEVICE float gelu_tanh_fast(float y) {
  const float u = y * y;
  const float inner = y * fmaf(0.0356774081f, u, 0.7978845608f);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(inner));
  const float h = 0.5f * y;
  return fmaf(h, t, h);
}

DCR_DEVICE float apply_act(float y, int act) {
  if (act == 1) return fmaxf(y, 0.f);
  if (act == 2) return gelu_erf_fast(y);                 // every tensor-core epilogue; the float64 mode (conv_exact.cu) keeps erff
  if (act == 3) return y / (1.f + expf(-1.702f * y));   // QuickGELU: x * sigmoid(1.702 x)  (CLIP, clip/model.py)
  return y;
}

// kEpi: 0 = direct epilogue (any number of planes, optional fp32 output, runtime activation; parity mode and final
//           layers), 1/2/3/4 = TMA-store epilogue with compile-time activation none / ReLU / GELU / QuickGELU (fast mode hot path).
// Eight MMA + epilogue warps: warp w of a warpgroup owns rows 32w .. 32w+31 of the warpgroup's accumulator tile.
template <int BN, bool kIm2col, int kEpi>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_bf16_kernel(const __grid_constant__ GemmMaps maps, const GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  constexpr bool kTma = kEpi != 0;
  constexpr int kBStage = BN * kBK * 2;
  constexpr int kStageBytes = kAStage + kBStage;
  constexpr int kStagingBytes = (BN / 64) * kBM * 128;   // BN/64 slabs of [128 rows x 64 bf16], 128B swizzle
  constexpr int kChunksPerWarp = BN / 32;                // 32-column chunks each epilogue warp handles per tile
  // wgmma groups (k-iterations) a warpgroup keeps in flight before it waits: one k-block of a 64-column tile is half the
  // tensor-core work of a 128-column one, too little to cover the wgmma latency with a single group behind it
  constexpr int kPend = BN <= 64 ? 2 : 1;
  const int stages = p.stages;
  const int k_iters = p.n_terms * p.taps * p.cblocks;
  // A-resident mode (wide 1x1 convolutions / Linear layers with small K): [k_iters x 16 KB A rows of the current m-tile]
  // first, then stages that carry only the W tile; the per-channel affine of ALL column blocks is staged once.
  const bool a_res = p.a_resident != 0;
  const int stage_bytes = a_res ? kBStage : kStageBytes;
  const int num_n_tiles = p.num_n_tiles;
  uint8_t* smem_ares = smem;
  uint8_t* smem_ab = smem + (a_res ? k_iters * kAStage : 0);
  uint8_t* out_stage = smem_ab + stages * stage_bytes;                      // 1024-aligned
  // TMA-store epilogue: one staging tile per warpgroup (the residual lands in it by TMA and is overwritten in place by
  // the output); direct epilogue: a 32-row transpose buffer per warp instead
  uint8_t* acc_xpose = out_stage + (kTma ? 2 * kStagingBytes : kXposeBytes);   // [8 warps] accumulator transposes
  // [2 warpgroups][2 bufs][2 (scale,bias)][BN] | a_res: [2][n_tiles*BN]
  float* sb = reinterpret_cast<float*>(acc_xpose + kAccXposeBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sb + (a_res ? 2 * num_n_tiles * BN : 8 * BN));
  uint64_t* full = bars;          // [stages] (<= 12)
  uint64_t* empty = bars + 12;    // [stages]
  uint64_t* res_full = bars + 28;   // [2]  one per warpgroup
  uint64_t* turn = bars + 30;       // [2]  PingPong::turn
  // A-resident mode (stages <= 8, so full[9..11] are free): a_full[j & 1] completes when the rows of the CTA's j-th
  // m-tile have landed.  Two barriers, because a ping-pong warpgroup may have no tile in the CTA's first m-tile and then
  // waits for the second one: on a single barrier that parity would also match the not-yet-completed first phase.  Only
  // the first and the last m-tile of the CTA can lack a tile of one warpgroup: the CTA's tiles are a contiguous range of
  // the n-fastest order and A-resident layers have num_n_tiles >= 2, so every other m-tile contributes two or more
  // consecutive tiles, which the alternation deals to both warpgroups.  A warpgroup therefore never waits on a barrier
  // more than one phase ahead of the last phase it has seen complete, or could have seen (the CTA's first m-tile).
  uint64_t* a_full = bars + 9;     // [2]
  uint64_t* a_empty = bars + 11;

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // hoist everything the tile loops need out of the constant bank once
  const int M = p.M, N = p.N, num_m_tiles = p.num_m_tiles;
  const bool has_res = p.res != nullptr;
  const int num_tiles = num_m_tiles * p.num_n_tiles;
  const int unit = static_cast<int>(blockIdx.x), n_units = static_cast<int>(gridDim.x);
  // tile sequence of this CTA: m-fastest round robin (default) or a contiguous range of the n-fastest order (A-resident)
  const int t_first = a_res ? static_cast<int>(static_cast<long long>(num_tiles) * blockIdx.x / gridDim.x) : unit;
  const int t_end = a_res ? static_cast<int>(static_cast<long long>(num_tiles) * (blockIdx.x + 1) / gridDim.x) : num_tiles;
  const int t_step = a_res ? 1 : n_units;
  const bool n_fast = p.n_fastest != 0;
  auto tile_m = [&](int t) {
    return a_res ? t / num_n_tiles : (n_fast ? t / num_n_tiles : t % num_m_tiles);
  };
  auto tile_n = [&](int t) { return (a_res || n_fast) ? t % num_n_tiles : t / num_m_tiles; };

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&maps.out);
    tma_prefetch_desc(&maps.res);
    for (int i = 0; i < 3; ++i) {
      tma_prefetch_desc(&maps.a[i]);
      tma_prefetch_desc(&maps.w[i]);
    }
  }
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);           // one arrive per warp of the consuming warpgroup once its wgmma on the stage completed
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&res_full[b], 1);
      mbar_init(&turn[b], 4);            // the four warps of the other warpgroup, after their last k-block's wgmma
    }
    mbar_init(&a_full[0], 1);
    mbar_init(&a_full[1], 1);
    mbar_init(a_empty, 8);               // 8 warp arrivals per m-tile (see the release below)
    fence_mbar_init();
  }
  __syncthreads();

  // Producer: the WHOLE warp walks the loops (so that every value is provably warp-uniform and lives in uniform
  // registers) and one elected lane issues the TMA instructions.
  if (warp >= 8) {
    wg_regs_dec<producer_regs(kEpi)>();
    if (warp == 8) {
      const int n_terms = p.n_terms, taps = p.taps, kw = p.kw, cblocks = p.cblocks;
      PipeState st(stages);
      int res_m = -1;
      uint32_t a_seg = 0;
      for (int tile = t_first; tile < t_end; tile += t_step) {
        const int m0 = tile_m(tile) * kBM;
        const int n0 = tile_n(tile) * BN;
        if (a_res) {
          if (m0 != res_m) {   // new m-tile: its A rows (all of K) once, after the MMAs on the previous rows have retired
            res_m = m0;
            mbar_wait(a_empty, (a_seg & 1) ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&a_full[a_seg & 1], k_iters * kAStage);
              for (int ki = 0; ki < k_iters; ++ki)
                tma_load_2d(smem_ares + ki * kAStage, &maps.a[p.term_a[0]], &a_full[a_seg & 1], ki * kBK, m0, kEvictFirst);
            }
            __syncwarp();
            ++a_seg;
          }
          for (int ki = 0; ki < k_iters; ++ki, st.next()) {
            const uint32_t s = st.s;
            mbar_wait(&empty[s], st.ph ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&full[s], kBStage);
              tma_load_2d(smem_ab + s * kBStage, &maps.w[p.term_w[0]], &full[s], ki * kBK, n0, kEvictLast);
            }
            __syncwarp();
          }
          continue;
        }
        int img = 0, h0 = 0, w0 = 0;
        if constexpr (kIm2col) {
          const int pq = p.P * p.Q;
          img = m0 / pq;
          const int rem = m0 - img * pq;
          const int p0 = rem / p.Q, q0 = rem - p0 * p.Q;
          h0 = p0 * p.stride - p.pad_h;
          w0 = q0 * p.stride - p.pad_w;
        }
        for (int t = 0; t < n_terms; ++t) {
          const CUtensorMap* ma = &maps.a[p.term_a[t]];
          const CUtensorMap* mw = &maps.w[p.term_w[t]];
          for (int tap = 0; tap < taps; ++tap) {
            const int r = tap / kw, sx = tap - r * kw;
            for (int cb = 0; cb < cblocks; ++cb, st.next()) {
              const uint32_t s = st.s, ph = st.ph;
              mbar_wait(&empty[s], ph ^ 1);
              if (elect_one()) {
                mbar_arrive_expect_tx(&full[s], kStageBytes);
                uint8_t* sa = smem_ab + s * kStageBytes;
                if constexpr (kIm2col) {
                  tma_load_im2col_4d(sa, ma, &full[s], cb * kBK, w0, h0, img, static_cast<uint16_t>(sx),
                                          static_cast<uint16_t>(r));
                } else
                  tma_load_2d(sa, ma, &full[s], cb * kBK, m0, kEvictNormal);
                tma_load_2d(sa + kAStage, mw, &full[s], (tap * cblocks + cb) * kBK, n0, kEvictNormal);
              }
              __syncwarp();
            }
          }
        }
      }
    }
  } else {
    wg_regs_inc<consumer_regs(kEpi)>();
    const uint32_t ewarp = warp;                   // 0..7
    const uint32_t quad = warp & 3;                // rows quad*32 .. +31 of the tile
    const uint32_t wg = ewarp >> 2;                // consumer warpgroup
    const uint32_t row = quad * 32 + lane;
    const uint32_t etid = ewarp * 32 + lane;       // 0..255 among the consumer threads
    const uint32_t gtid = etid & 127;              // 0..127 within the warpgroup
    const uint32_t bar_top = 1 + 2 * wg, bar_end = bar_top + 1;   // the warpgroup's named barriers
    const uint32_t xacc = smem_u32(acc_xpose) + warp * kAccXposeWarpBytes;
    const int act = p.act;
    uint32_t tc = 0;                               // tiles this thread's warpgroup has run
    const PingPong pingpong{turn};
    PipeState st(stages);
    const uint32_t a_base = smem_u32(a_res ? smem_ares : smem_ab);
    const uint32_t b_base = smem_u32(a_res ? smem_ab : smem_ab + kAStage);
    int res_m_c = -1;
    const int m_first = t_first < t_end ? tile_m(t_first) : 0;
    auto load_residual = [&](int tile_idx, uint8_t* dst, uint64_t* bar) {   // one thread: residual tile -> dst
      const int rm0 = tile_m(tile_idx) * kBM;
      const int rn0 = tile_n(tile_idx) * BN;
      int slabs = 0;
      for (int sl = 0; sl < BN / 64; ++sl)
        if (rn0 + sl * 64 < N) ++slabs;
      mbar_arrive_expect_tx(bar, slabs * kBM * 128);
      for (int sl = 0; sl < BN / 64; ++sl)
        if (rn0 + sl * 64 < N) tma_load_2d(dst + sl * kBM * 128, &maps.res, bar, rn0 + sl * 64, rm0, kEvictFirst);
    };
    const uint32_t sb_addr = smem_u32(sb) + (a_res ? 0 : wg * 4 * BN * 4);
    int staged_n0 = -1;
    uint32_t sbsel = 1;
    if (a_res) {   // per-channel affine of every column block, once
      const int npad = num_n_tiles * BN;
      for (int c = etid; c < npad; c += 256) {
        st_shared_f32(sb_addr + c * 4, (p.scale && c < N) ? p.scale[c] : 1.f);
        st_shared_f32(sb_addr + (npad + c) * 4, (p.bias && c < N) ? p.bias[c] : 0.f);
      }
      named_bar_sync(5, 256);
    }
    if (wg == 1) st.skip(k_iters);                 // the CTA's first tile is warpgroup 0's
    for (int tile = t_first + static_cast<int>(wg) * t_step; tile < t_end; tile += 2 * t_step, ++tc) {
      const int m0 = tile_m(tile) * kBM;
      const int n0 = tile_n(tile) * BN;
      uint8_t* ostage = out_stage + wg * kStagingBytes;
      const uint32_t ostage_addr = smem_u32(ostage);
      if (kTma && gtid == 0) {
        // the warpgroup's staging tile is free once its previous store has finished READING it; the residual then lands
        // in it (the other warpgroup's k-loop hides the load)
        tma_store_wait_read<0>();
        if (has_res) load_residual(tile, ostage, &res_full[wg]);
      }
      // Per-channel affine: staged only when the column block changes (tiles are walked m-fastest, so a CTA keeps its
      // column block for many tiles) into the warpgroup's buffer the previous block did not use -- warps still finishing
      // the previous tile read the other one.  The barrier also orders the staging tile's reuse after the wait above.
      const bool restage = !a_res && n0 != staged_n0;
      if (restage) {
        sbsel ^= 1;
        staged_n0 = n0;
        for (int c = gtid; c < BN; c += 128) {
          const int n = n0 + c;
          st_shared_f32(sb_addr + (sbsel * 2 * BN + c) * 4, (p.scale && n < N) ? p.scale[n] : 1.f);
          st_shared_f32(sb_addr + (sbsel * 2 * BN + BN + c) * 4, (p.bias && n < N) ? p.bias[n] : 0.f);
        }
      }
      if (restage || kTma) named_bar_sync(bar_top, 128);
      const uint32_t s_scale = a_res ? sb_addr + n0 * 4 : sb_addr + sbsel * 2 * BN * 4;
      const uint32_t s_bias = s_scale + (a_res ? num_n_tiles * BN : BN) * 4;
      // ---- main loop: this warpgroup's 128 x BN accumulator over all k-iterations.  The stage of k-iteration i is
      // released once wgmma_wait<1> in iteration i+1 has seen its MMAs complete.
      bool a_release = false;
      uint32_t a_release_cnt = 1;
      if (a_res) {
        const int mt = tile_m(tile);
        if (mt != res_m_c) {
          res_m_c = mt;
          const int seg = mt - m_first;             // the CTA's seg-th m-tile
          mbar_wait(&a_full[seg & 1], (seg >> 1) & 1);
        }
        // The resident rows are released by the last MMAs on them: 8 warp arrivals per m-tile, each warpgroup's 4
        // warps after its own last tile of the m-tile, or 2 each when the m-tile has no tile of the other warpgroup
        // (tiles are a contiguous range, so the other warpgroup's tiles of this m-tile include a neighbour).
        const int next = tile + 2 * t_step;
        a_release = next >= t_end || tile_m(next) != mt;
        const bool alone = (tile - t_step < t_first || tile_m(tile - t_step) != mt) &&
                           (tile + t_step >= t_end || tile_m(tile + t_step) != mt);
        a_release_cnt = alone ? 2 : 1;
      }
      pingpong.wait(wg, tc);
      WgAcc<BN> acc;
      // pend[]: the stages of the last kPend k-iterations, oldest first (their wgmma groups may still be in flight)
      uint32_t pend[kPend] = {};
      for (int ki = 0; ki < k_iters; ++ki, st.next()) {
        const uint32_t s = st.s;
        mbar_wait(&full[s], st.ph);
        const uint32_t a_addr = a_base + (a_res ? static_cast<uint32_t>(ki) * kAStage : s * kStageBytes);
        const uint32_t b_addr = b_base + s * static_cast<uint32_t>(stage_bytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k) acc.mma(a_addr + 32 * k, wgmma_desc_sw128(b_addr + 32 * k), (ki | k) != 0);
        wgmma_commit();
        if (ki == k_iters - 1 && lane == 0) pingpong.hand_over(wg);
        wgmma_wait<kPend>();
        if (ki >= kPend && lane == 0) mbar_arrive(&empty[pend[0]]);
#pragma unroll
        for (int j = 0; j + 1 < kPend; ++j) pend[j] = pend[j + 1];
        pend[kPend - 1] = s;
      }
      wgmma_wait<0>();
      acc.fence_regs();
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < kPend; ++j)
          if (k_iters - kPend + j >= 0) mbar_arrive(&empty[pend[j]]);
        if (a_release) mbar_arrive_cnt(a_empty, a_release_cnt);
      }
      st.skip(k_iters);                            // the other warpgroup's next tile
      if (kTma && has_res) mbar_wait(&res_full[wg], tc & 1);
      const int m = m0 + static_cast<int>(row);
      const bool row_ok = m < M;
#pragma unroll
      for (int ci = 0; ci < kChunksPerWarp; ++ci) {
        const int ch = ci;
        uint32_t r[32];
        acc.rows32(ci, r, xacc, lane);
        const int nc = n0 + ch * 32;
        if (nc >= N) continue;
        float y[32];
#pragma unroll
        for (int c = 0; c < 32; c += 4) {
          const float4 sc = ld_shared_f4(s_scale + (ch * 32 + c) * 4);
          const float4 bi = ld_shared_f4(s_bias + (ch * 32 + c) * 4);
          y[c + 0] = fmaf(__uint_as_float(r[c + 0]), sc.x, bi.x);
          y[c + 1] = fmaf(__uint_as_float(r[c + 1]), sc.y, bi.y);
          y[c + 2] = fmaf(__uint_as_float(r[c + 2]), sc.z, bi.z);
          y[c + 3] = fmaf(__uint_as_float(r[c + 3]), sc.w, bi.w);
        }
        if constexpr (kTma) {
          // this thread's 32 columns live in slab ch/2 at 16-byte chunks (ch&1)*4 .. +3 of row `row` (128B swizzle)
          const uint32_t srow = ostage_addr + (ch >> 1) * kBM * 128 + row * 128;
          const uint32_t sw = row & 7;
          if (has_res) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint4 rv = ld_shared_v4(srow + ((((ch & 1) * 4 + j) ^ sw) << 4));   // residual, then output in place
              const uint32_t w[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                y[j * 8 + 2 * e] += __uint_as_float(w[e] << 16);
                y[j * 8 + 2 * e + 1] += __uint_as_float(w[e] & 0xffff0000u);
              }
            }
          }
#pragma unroll
          for (int c = 0; c < 32; ++c) y[c] = (kEpi == 3) ? gelu_tanh_fast(y[c]) : apply_act(y[c], kEpi - 1);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint4 v;
            v.x = pack_bf16x2(y[j * 8 + 0], y[j * 8 + 1]);
            v.y = pack_bf16x2(y[j * 8 + 2], y[j * 8 + 3]);
            v.z = pack_bf16x2(y[j * 8 + 4], y[j * 8 + 5]);
            v.w = pack_bf16x2(y[j * 8 + 6], y[j * 8 + 7]);
            st_shared_v4(srow + ((((ch & 1) * 4 + j) ^ sw) << 4), v);
          }
        } else {
          // Direct epilogue (split-bf16 planes, fp32 outputs, final layers).  Thread = accumulator row, but a row's 32 columns
          // are only 64 bytes per plane: written straight from the registers, one warp instruction would touch 32 rows x 16 bytes
          // (32 half-used sectors, 32 LSU wavefronts).  Every plane goes through the warp's
          // transpose buffer: rows -> shared memory, then 8 rows x 64 contiguous bytes per instruction to / from global memory.
          const int nvalid = min(32, N - nc);   // multiple of 8 (N % 8 == 0 enforced on the host)
          const uint32_t xw = smem_u32(out_stage) + ewarp * kXposeWarpBytes;
          const uint32_t x_own = xw + lane * kXposePitch;           // this thread's row
          const int m_w0 = m0 + static_cast<int>(quad) * 32;        // first row of this warp
          if (has_res) {
            for (int pl = 0; pl < p.res_planes; ++pl) {
              const __nv_bfloat16* rbase = p.res + pl * p.res_plane_stride + nc;
              __syncwarp();
#pragma unroll
              for (int t = 0; t < 4; ++t) {
                const int piece = t * 32 + static_cast<int>(lane), r = piece >> 2, part = piece & 3;
                if (m_w0 + r < M && part * 8 < nvalid)
                  st_shared_v4(xw + r * kXposePitch + part * 16,
                               *reinterpret_cast<const uint4*>(rbase + static_cast<size_t>(m_w0 + r) * p.ld_res + part * 8));
              }
              __syncwarp();
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                if (j * 8 < nvalid && row_ok) {
                  const uint4 rv = ld_shared_v4(x_own + j * 16);
                  const uint32_t w[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    y[j * 8 + 2 * e] += __uint_as_float(w[e] << 16);
                    y[j * 8 + 2 * e + 1] += __uint_as_float(w[e] & 0xffff0000u);
                  }
                }
              }
            }
          }
          // the activation is a run-time value here: ONE warp-uniform switch per chunk (inside the element loop the compiler
          // kept a compare-and-branch chain per element: 660 instructions per 32-column chunk, a quarter of the warp samples on
          // instruction fetch)
          if (act == 1) {
#pragma unroll
            for (int c = 0; c < 32; ++c) y[c] = fmaxf(y[c], 0.f);
          } else if (act == 2) {
            if (p.fast_gelu) {
#pragma unroll
              for (int c = 0; c < 32; ++c) y[c] = gelu_tanh_fast(y[c]);
            } else {
#pragma unroll
              for (int c = 0; c < 32; ++c) y[c] = gelu_erf_fast(y[c]);
            }
          } else if (act == 3) {
#pragma unroll
            for (int c = 0; c < 32; ++c) y[c] = apply_act(y[c], 3);
          }
          if (p.out_f32 && row_ok) {
            float* op = p.out_f32 + static_cast<size_t>(m) * p.ld_out_f32 + nc;
#pragma unroll
            for (int c = 0; c < 32; c += 4)
              if (c < nvalid) *reinterpret_cast<float4*>(op + c) = make_float4(y[c], y[c + 1], y[c + 2], y[c + 3]);
          }
          if (p.out) {
            for (int pl = 0; pl < p.out_planes; ++pl) {
              __nv_bfloat16* obase = p.out + pl * p.out_plane_stride + p.out_col_off + nc;
              __syncwarp();
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                uint4 v;
                v.x = pack_bf16x2(y[j * 8 + 0], y[j * 8 + 1]);
                v.y = pack_bf16x2(y[j * 8 + 2], y[j * 8 + 3]);
                v.z = pack_bf16x2(y[j * 8 + 4], y[j * 8 + 5]);
                v.w = pack_bf16x2(y[j * 8 + 6], y[j * 8 + 7]);
                st_shared_v4(x_own + j * 16, v);
              }
              __syncwarp();
#pragma unroll
              for (int t = 0; t < 4; ++t) {
                const int piece = t * 32 + static_cast<int>(lane), r = piece >> 2, part = piece & 3;
                if (m_w0 + r < M && part * 8 < nvalid)
                  *reinterpret_cast<uint4*>(obase + static_cast<size_t>(m_w0 + r) * p.ld_out + part * 8) =
                      ld_shared_v4(xw + r * kXposePitch + part * 16);
              }
              if (pl + 1 < p.out_planes) {
                // next plane holds the rounding residual of this one
#pragma unroll
                for (int c = 0; c < 32; ++c) y[c] -= __bfloat162float(__float2bfloat16_rn(y[c]));
              }
            }
          }
        }
      }
      if constexpr (kTma) {
        fence_proxy_async();   // generic-proxy writes -> visible to the TMA (async proxy)
        named_bar_sync(bar_end, 128);
        if (gtid == 0) {
          for (int sl = 0; sl < BN / 64; ++sl)
            if (n0 + sl * 64 < N && m0 < M) tma_store_2d(&maps.out, smem_u32(ostage + sl * kBM * 128), p.out_col_off + n0 + sl * 64, m0);
          tma_store_commit();
        }
      }
    }
  }

  if (kTma && (warp == 0 || warp == 4) && lane == 0) tma_store_wait_all();   // gtid 0 of each warpgroup issued stores
}

// A-resident mode: plain (non-im2col) single-term GEMMs with several column blocks and K <= 256 -- the wide 1x1
// expansions: the A rows of an m-tile are loaded once instead of once per column block (per-SM-unique data is what
// the L2 -> shared-memory path is short of; the W tiles are shared by all SMs and cheap)
// (the resident rows are single buffered: the next m-tile's rows wait for the last MMA on the current ones, a bubble
// that only pays off when the epilogue is heavy (residual) or the m-tile has >= 4 column blocks)
bool wants_a_resident(const GemmParams& p, int BN, bool im2col, size_t max_smem) {
  const int k_iters_h = p.n_terms * p.taps * p.cblocks;
  if (!(!im2col && p.tma_epi && p.n_terms == 1 && p.num_n_tiles >= 2 && (p.res != nullptr || p.num_n_tiles >= 4) &&
        k_iters_h * kAStage <= 64 * 1024 && p.num_n_tiles * BN <= 4096))
    return false;
  // the resident rows, the all-blocks affine table and the staging tiles must leave at least three W stages; otherwise
  // the layer runs with the default schedule
  const size_t staging = static_cast<size_t>(BN / 64) * kBM * 128;   // one per warpgroup
  const size_t need = 1024 + static_cast<size_t>(2) * p.num_n_tiles * BN * 4 + static_cast<size_t>(k_iters_h) * kAStage + 256 +
                      2 * staging + kAccXposeBytes + 3 * static_cast<size_t>(BN) * kBK * 2;
  return need <= max_smem;
}

template <int BN, bool kIm2col, int kEpi>
int launch_gemm(const GemmMaps& maps, GemmParams& p, int num_sms, size_t max_smem, cudaStream_t stream) {
  constexpr int kStageBytes = kAStage + BN * kBK * 2;
  constexpr size_t kStagingBytes = static_cast<size_t>(BN / 64) * kBM * 128;
  const int k_iters_h = p.n_terms * p.taps * p.cblocks;
  p.a_resident = (kEpi != 0 && wants_a_resident(p, BN, kIm2col, max_smem)) ? 1 : 0;
  const size_t sb_bytes = p.a_resident ? static_cast<size_t>(2) * p.num_n_tiles * BN * 4 : static_cast<size_t>(8) * BN * 4;
  const size_t ares_bytes = p.a_resident ? static_cast<size_t>(k_iters_h) * kAStage : 0;
  // one output staging tile per warpgroup (TMA-store epilogue) or the per-warp transpose buffers (direct epilogue)
  const size_t fixed = 1024 + sb_bytes + ares_bytes + 256 + (p.tma_epi ? 2 * kStagingBytes : kXposeBytes) + kAccXposeBytes;
  const size_t stage_bytes = p.a_resident ? static_cast<size_t>(BN) * kBK * 2 : static_cast<size_t>(kStageBytes);
  DCR_REQUIRE(max_smem > fixed + 3 * stage_bytes, "gemm: not enough shared memory");   // kPend + 1 stages at least
  int stages = static_cast<int>((max_smem - fixed) / stage_bytes);
  stages = std::min(stages, 8);
  p.stages = stages;
  const size_t smem = fixed + static_cast<size_t>(stages) * stage_bytes;
  const int grid = std::min(p.num_m_tiles * p.num_n_tiles, num_sms);
  return launch(gemm_bf16_kernel<BN, kIm2col, kEpi>, grid, kThreads, smem, stream, "conv_gemm", maps, p);
}

}  // namespace

int conv_gemm(const ConvGemmDesc& d, cudaStream_t stream) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  if (int rc = require_sm90a(di, "conv_gemm")) return rc;
  DCR_REQUIRE(d.n_terms >= 1 && d.n_terms <= kMaxGemmTerms, "conv_gemm: bad n_terms %d", d.n_terms);
  DCR_REQUIRE(d.C % 8 == 0 && d.N % 8 == 0, "conv_gemm: C (%d) and N (%d) must be multiples of 8", d.C, d.N);
  DCR_REQUIRE(d.kh >= 1 && d.kw >= 1 && d.stride >= 1, "conv_gemm: bad filter geometry");
  DCR_REQUIRE(d.act >= 0 && d.act <= 3, "conv_gemm: unknown activation %d", d.act);
  if (d.exact) return conv_exact(d, stream);
  if (conv3x3_halo_eligible(d)) return conv3x3_halo(d, stream);
  const bool windowed = d.in_stride_w != 0;
  const bool im2col = windowed || !(d.kh == 1 && d.kw == 1 && d.stride == 1 && d.pad_h == 0 && d.pad_w == 0);
  const int P = (d.H + 2 * d.pad_h - d.kh) / d.stride + 1;
  const int Q = (d.W + 2 * d.pad_w - d.kw) / d.stride + 1;
  const long long M = static_cast<long long>(d.B) * P * Q;
  DCR_REQUIRE(M > 0 && M < (1ll << 31), "conv_gemm: M out of range");
  const int cblocks = (d.C + kBK - 1) / kBK;
  const int ktot = d.kh * d.kw * cblocks * kBK;   // padded K of the prepared weights

  GemmMaps maps;
  memset(&maps, 0, sizeof(maps));
  int a_planes = 0, w_planes = 0;
  for (int t = 0; t < d.n_terms; ++t) {
    a_planes = std::max(a_planes, d.term_a[t] + 1);
    w_planes = std::max(w_planes, d.term_w[t] + 1);
  }
  DCR_REQUIRE(a_planes <= 3 && w_planes <= 3, "conv_gemm: at most 3 planes");
  // at most 128 columns: a warpgroup holds a whole 128 x 128 tile (128 accumulator registers per thread).  Two 128-wide
  // ping-pong tiles beat one 128 x 256 tile split over both warpgroups on every 256-wide shape of SSCD ResNet-50 and DINO
  // ViT-S (ResNet layer3/4 3x3 and reduces, ViT qkv / fc1; DESIGN.md section 2): the epilogue no longer stalls the tensor
  // core, which outweighs reading A twice as often
  int BN = d.N <= 64 ? 64 : 128;
  // QuickGELU divides by 1 + exp(-1.702 y) in IEEE single precision, whose rare-operand path is a subroutine call: with
  // a 128-column accumulator live across 32 such calls per chunk ptxas spills, so QuickGELU layers (CLIP) take 64-column
  // tiles
  if (d.act == 3) BN = 64;
  // few output tiles and a long K (the SSCD head: 384 x 512 x 2048 is twelve 128 x 128 tiles, each CTA streaming its K
  // through one SM's L2 port): narrower tiles put more CTAs -- more L2 ports -- on the same K stream
  {
    const long long m_tiles = (M + kBM - 1) / kBM;
    while (BN > 64 && ktot >= 1024 && m_tiles * ((d.N + BN - 1) / BN) * 4 <= di->num_sms) BN /= 2;
  }
  for (int pl = 0; pl < 3; ++pl) {
    const int pa = std::min(pl, a_planes - 1), pw = std::min(pl, w_planes - 1);
    const __nv_bfloat16* abase = d.in + pa * d.in_plane_stride;
    if (im2col) {
      DCR_REQUIRE(windowed || d.ld_in == d.C, "conv_gemm: im2col input must be dense NHWC (ld_in == C)");
      if (int rc = make_tmap_im2col_bf16(&maps.a[pl], abase, d.B, d.H, d.W, d.C, d.pad_h, d.pad_w, d.kh, d.kw, d.stride,
                                         kBK, kBM, d.in_stride_w, d.in_stride_h, d.in_stride_n))
        return rc;
    } else {
      if (int rc = make_tmap_2d_bf16(&maps.a[pl], abase, M, d.C, d.ld_in, kBM, kBK)) return rc;
    }
    if (int rc = make_tmap_2d_bf16(&maps.w[pl], d.weight + pw * d.w_plane_stride, d.N, ktot, ktot, BN, kBK)) return rc;
  }

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = static_cast<int>(M);
  p.N = d.N;
  p.taps = d.kh * d.kw;
  p.kw = d.kw;
  p.cblocks = cblocks;
  p.n_terms = d.n_terms;
  for (int t = 0; t < d.n_terms; ++t) {
    p.term_a[t] = d.term_a[t];
    p.term_w[t] = d.term_w[t];
  }
  p.P = P;
  p.Q = Q;
  p.stride = d.stride;
  p.pad_h = d.pad_h;
  p.pad_w = d.pad_w;
  p.num_m_tiles = static_cast<int>((M + kBM - 1) / kBM);
  p.num_n_tiles = (d.N + BN - 1) / BN;
  p.scale = d.scale;
  p.bias = d.bias;
  p.res = d.res;
  p.ld_res = d.ld_res;
  p.res_planes = d.res ? std::max(1, d.res_planes) : 0;
  p.res_plane_stride = d.res_plane_stride;
  p.out = d.out;
  p.ld_out = d.ld_out;
  p.out_col_off = d.out_col_off;
  p.out_planes = d.out ? std::max(1, d.out_planes) : 0;
  p.out_plane_stride = d.out_plane_stride;
  p.out_f32 = d.out_f32;
  p.ld_out_f32 = d.ld_out_f32;
  p.act = d.act;
  p.fast_gelu = (d.n_terms == 1 && p.out_planes <= 1) ? 1 : 0;
  // tile order: with several column blocks and an A matrix larger than what L2 keeps between the passes, m-fastest order
  // streams A from HBM once per column block
  const double a_bytes = 2.0 * a_planes * (im2col ? static_cast<double>(d.B) * d.H * d.W * d.C : static_cast<double>(M) * d.C);
  const int order = tuning_int("DCR_GEMM_TILE_ORDER", -1);   // tuning / tests: 0 = m-fastest, 1 = n-fastest, default by size
  p.n_fastest = (order >= 0) ? (order == 1 && p.num_n_tiles >= 2) : (p.num_n_tiles >= 2 && a_bytes > 48e6);
  p.tma_epi = (p.out != nullptr && p.out_planes == 1 && p.out_f32 == nullptr && (p.res == nullptr || p.res_planes == 1) &&
               (d.act != 2 || p.fast_gelu) &&   // the TMA-store epilogue's compile-time GELU is the tanh form
               !tuning_flag("DCR_GEMM_DIRECT_EPILOGUE"))
                  ? 1
                  : 0;
  if (p.tma_epi) {
    // dim0 = col_off + N so that a partial last slab is clipped at this op's own columns (concat neighbours intact)
    if (int rc = make_tmap_2d_bf16(&maps.out, p.out, M, p.out_col_off + d.N, p.ld_out, kBM, 64)) return rc;
    if (p.res) {
      if (int rc = make_tmap_2d_bf16(&maps.res, p.res, M, d.N, p.ld_res, kBM, 64)) return rc;
    } else {
      maps.res = maps.out;
    }
  } else {
    maps.out = maps.w[0];
    maps.res = maps.w[0];
  }
  DCR_REQUIRE(p.out == nullptr || (p.ld_out % 8 == 0 && p.out_col_off % 8 == 0), "conv_gemm: output leading dim / offset must be multiples of 8");
  DCR_REQUIRE(p.res == nullptr || p.ld_res % 8 == 0, "conv_gemm: residual leading dim must be a multiple of 8");
  DCR_REQUIRE(p.out_f32 == nullptr || p.ld_out_f32 % 4 == 0, "conv_gemm: fp32 output leading dim must be a multiple of 4");

  const int epi = p.tma_epi ? 1 + p.act : 0;   // compile-time activation on the TMA-store path

#define DCR_LAUNCH_E(BNv, E)                                                                      \
  (im2col ? launch_gemm<BNv, true, E>(maps, p, di->num_sms, di->max_smem_optin, stream)         \
          : launch_gemm<BNv, false, E>(maps, p, di->num_sms, di->max_smem_optin, stream))
#define DCR_LAUNCH(BNv)                                                                          \
  (epi == 0 ? DCR_LAUNCH_E(BNv, 0)                                                                \
            : (epi == 1 ? DCR_LAUNCH_E(BNv, 1) : (epi == 2 ? DCR_LAUNCH_E(BNv, 2) : (epi == 3 ? DCR_LAUNCH_E(BNv, 3) : DCR_LAUNCH_E(64, 4)))))
  switch (BN) {
    case 64: return DCR_LAUNCH(64);
    case 128: return DCR_LAUNCH(128);
    default: return set_error(-1, "conv_gemm: unsupported BN %d", BN);
  }
#undef DCR_LAUNCH_E
#undef DCR_LAUNCH
}

}  // namespace dcr
