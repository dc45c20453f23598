// ResNet stem (7x7 / stride 2 / pad 3 convolution + BatchNorm + ReLU) as a wgmma implicit GEMM whose A operand is an
// OVERLAPPING-WINDOW (Toeplitz) view of the input in shared memory -- every input pixel travels L2 -> shared memory ~1.7
// times instead of 16 times (conv_gemm.cu's space-to-depth path re-reads each stored pixel once per window position and
// filter row, which makes that path ingest bound).
//
// Reference call site: `model(samples)` (utils_ret.py:751) -> torchvision ResNet conv1 / bn1 / relu of the SSCD trunk.
//
// Input layout (stem_rows_kernel in image_in.cu, fused with Resize/CenterCrop/ToTensor/Normalize of diff_retrieval.py:325-330):
// with ip the zero-padded (3 pixels) normalised crop, the image is stored as two "column-parity planes" of 16-byte units
//     plane_e[P * PW + u] = { ip[2P + i][2u + e][c] : i in {0,1}, c in {0,1,2} } + 2 zero channels      (8 bf16)
// so that   out[y][x] = sum_{a<4, e<2, b<4, ch<8} W[a][e][b][ch] * plane_e[(y + a) * PW + (x + b)][ch]
// (filter row 2a+i, filter column 2b+e; the 8th row / column of the 8x8 footprint carries zero weights).  With output
// position m = y * PW + x the A operand of K-chunk (a, e, b) is the SAME linear array shifted by (a * PW + b) units: in a
// K-major SWIZZLE_NONE shared-memory descriptor rows are 16 bytes apart (stride-dimension offset 128 B per 8 rows) and
// the second 16-byte K chunk of an instruction sits leading-dimension-offset = 16 bytes further -- i.e. row m+1 and
// K-chunk b+1 address the same bytes.
// Positions with x >= OW (PW - OW per row) are junk and dropped by the epilogue.
//
// Roles (288 threads, persistent over tiles of 512 positions = 4 MMA row blocks):
//   warps 0-7 two consumer warpgroups, warpgroup h owns output channels [32h, 32h+32): per row block 16 x two
//            m64 x 32 x 16 wgmma (weights 64 x 256, 32 KB, 128B swizzle, resident) -> BN affine + ReLU -> bf16 -> staging
//            -> coalesced NHWC stores of the valid positions
//   warp 8   producer: two cp.async.bulk copies per tile (the even / odd plane windows, 512 + 3*PW + 3 units each)
#include <cuda_bf16.h>

#include <algorithm>
#include <cstring>

#include "dcr_internal.cuh"
#include "host_util.cuh"
#include "ptx.cuh"

namespace dcr {

namespace {

constexpr int kSN = 64;                   // output channels
constexpr int kSTile = 512;               // positions per tile
constexpr int kSBlocks = kSTile / 128;    // MMA row blocks per tile
constexpr int kSThreads = 288;             // warps 0-7 MMA + epilogue, warp 8 producer
constexpr int kWBytes = kSN * 256 * 2;    // resident weights: 4 k-blocks of [64 rows x 128 B]

struct StemParams {
  const __nv_bfloat16* planes;   // [B][2][alloc_units][8]
  long long img_stride;          // elements between images (2 * alloc_units * 8)
  long long plane_stride;        // elements between the two planes (alloc_units * 8)
  int B, OH, OW, PW;
  // work units: a unit is `tiles_per_unit` consecutive 512-position tiles of one image, starting at position
  // unit_begin(part).  Without pooling: unit = one tile.  With pooling: unit = 1/parts of an image (one extra conv row on top).
  int units_per_img, tiles_per_unit, num_units;
  int part_rows;                 // pooling: conv rows owned per part (2 * pooled rows per part)
  int OHp, OWp, prow_per_part;   // pooling: pooled output size, pooled rows per part
  int win_units;                 // units copied per plane and tile: 512 + 3 * PW + 3, rounded up to 8
  int win_stages;
  int ring_rows;                 // pooling: conv rows in the shared-memory ring (a power of two, see stem_ring_rows)
  const float* scale;
  const float* bias;
  __nv_bfloat16* out;            // NHWC [B][OH][OW][64]
};

DCR_DEVICE uint64_t desc_nosw(uint32_t addr) {
  // K-major, no swizzle: 8-row x 16-byte core matrices; LBO (next K chunk) = 16 B, SBO (next used 8-row group) = 256 B:
  // each m64 half of a WgAcc takes every other 8-row group (the odd groups start 128 B later)
  uint64_t d = 0;
  d |= static_cast<uint64_t>((addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(16 >> 4) << 16;
  d |= static_cast<uint64_t>(256 >> 4) << 32;
  return d;
}

DCR_DEVICE void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// first position of a unit
DCR_DEVICE int unit_begin(const StemParams& p, int part, bool pool) {
  if (!pool) return part * kSTile;
  const int row_lo = max(0, part * p.part_rows - 1);     // one conv row above the part's first pooled window
  return row_lo * p.PW;
}

// kPool: the 3x3 / stride 2 / pad 1 max pool that follows the stem (torchvision ResNet.maxpool) is taken in the epilogue:
// conv outputs (post BN + ReLU, bf16) go into a ring of conv rows in shared memory and a pooled row is emitted as soon
// as its three conv rows are complete -- the 112 x 112 x 64 stem activation (411 MB at batch 256) never reaches HBM.
template <bool kPool>
__global__ void __launch_bounds__(kSThreads, 1) stem_conv_kernel(const __grid_constant__ CUtensorMap tmap_w, const StemParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  const int win_bytes = p.win_units * 16;                       // per plane
  const int stage_bytes = (2 * win_bytes + 1023) & ~1023;
  uint8_t* s_w = smem;                                          // 32 KB, 4 k-blocks
  uint8_t* s_win = s_w + kWBytes;                               // win_stages x [even | odd]
  uint8_t* s_out = s_win + p.win_stages * stage_bytes;          // 2 x [128 positions x 128 B] | kPool: ring of conv rows
  const int ring_row_bytes = p.OW * 128;
  const int ring_mask = p.ring_rows - 1;
  uint8_t* acc_xpose = s_out + (kPool ? ((p.ring_rows * ring_row_bytes + 1023) & ~1023) : 2 * 16384);   // [8 warps]
  float* sb = reinterpret_cast<float*>(acc_xpose + 8 * kAccXposeWarpBytes);   // scale[64] | bias[64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sb + 128);
  uint64_t* w_full = bars;
  uint64_t* win_full = bars + 1;      // [4]
  uint64_t* win_empty = bars + 5;     // [4]

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) tma_prefetch_desc(&tmap_w);
  if (warp == 0 && lane == 0) {
    mbar_init(w_full, 1);
    for (int s = 0; s < 4; ++s) {
      mbar_init(&win_full[s], 1);
      mbar_init(&win_empty[s], 8);   // one arrive per consumer warp and tile
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================================== producer =====================================
    if (elect_one()) {
      mbar_arrive_expect_tx(w_full, kWBytes);
      for (int kb = 0; kb < 4; ++kb) tma_load_2d(s_w + kb * 8192, &tmap_w, w_full, kb * 64, 0, kEvictLast);
    }
    __syncwarp();
    PipeState ws(p.win_stages);
    for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
      const int b = unit / p.units_per_img;
      const int mu = unit_begin(p, unit - b * p.units_per_img, kPool);
      for (int t = 0; t < p.tiles_per_unit; ++t, ws.next()) {
        const int m0 = mu + t * kSTile;
        mbar_wait(&win_empty[ws.s], ws.ph ^ 1);
        if (elect_one()) {
          mbar_arrive_expect_tx(&win_full[ws.s], 2 * win_bytes);
          const __nv_bfloat16* src = p.planes + static_cast<size_t>(b) * p.img_stride + static_cast<size_t>(m0) * 8;
          bulk_load(s_win + ws.s * stage_bytes, src, win_bytes, &win_full[ws.s]);
          bulk_load(s_win + ws.s * stage_bytes + win_bytes, src + p.plane_stride, win_bytes, &win_full[ws.s]);
        }
        __syncwarp();
      }
    }
  } else {
    // ===================================== consumer warpgroups =====================================
    const uint32_t ewarp = warp;
    const uint32_t quad = warp & 3;
    const uint32_t half = ewarp >> 2;                 // 32-column half of the 64 channels (= warpgroup)
    const uint32_t row = quad * 32 + lane;            // position inside the row block
    const uint32_t etid = ewarp * 32 + lane;
    const uint32_t xacc = smem_u32(acc_xpose) + warp * kAccXposeWarpBytes;
    const uint32_t win0 = smem_u32(s_win);
    const uint32_t PW = static_cast<uint32_t>(p.PW);
    const uint64_t dw0 = wgmma_desc_sw128(smem_u32(s_w) + half * 32 * 128);
    PipeState ws(p.win_stages);
    const uint32_t sb_addr = smem_u32(sb), so_addr = smem_u32(s_out);
    for (int c = etid; c < kSN; c += 256) {
      st_shared_f32(sb_addr + c * 4, p.scale ? p.scale[c] : 1.f);
      st_shared_f32(sb_addr + (kSN + c) * 4, p.bias ? p.bias[c] : 0.f);
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    float sc[32], bi[32];
#pragma unroll
    for (int c = 0; c < 32; c += 4) {
      const float4 s4 = ld_shared_f4(sb_addr + (half * 32 + c) * 4);
      const float4 b4 = ld_shared_f4(sb_addr + (kSN + half * 32 + c) * 4);
      sc[c] = s4.x; sc[c + 1] = s4.y; sc[c + 2] = s4.z; sc[c + 3] = s4.w;
      bi[c] = b4.x; bi[c + 1] = b4.y; bi[c + 2] = b4.z; bi[c + 3] = b4.w;
    }
    const int positions = p.OH * p.PW;
    mbar_wait(w_full, 0);
    uint32_t tc = 0, blk = 0;
    for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
      const int b = unit / p.units_per_img;
      const int part = unit - b * p.units_per_img;
      const int mu = unit_begin(p, part, kPool);
      // pooling state of this unit: conv rows [row_lo, row_hi) are produced here, pooled rows [next_yp, yp_end) emitted
      const int row_lo = kPool ? max(0, part * p.part_rows - 1) : 0;
      const int row_hi = kPool ? min(p.OH, (part + 1) * p.part_rows) : p.OH;
      int next_yp = part * p.prow_per_part;
      const int yp_end = min(p.OHp, next_yp + p.prow_per_part);
      if constexpr (kPool) asm volatile("bar.sync 2, 256;" ::: "memory");   // nobody still pools the previous unit's rows
      for (int t = 0; t < p.tiles_per_unit; ++t, ++tc, ws.next()) {
        const int m0 = mu + t * kSTile;
        mbar_wait(&win_full[ws.s], ws.ph);
        const uint32_t wbase = win0 + ws.s * stage_bytes;
#pragma unroll 1
        for (int mb = 0; mb < kSBlocks; ++mb, ++blk) {
          WgAcc<32> acc;
          wgmma_fence();
#pragma unroll
          for (int a = 0; a < 4; ++a) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
#pragma unroll
              for (int bp = 0; bp < 2; ++bp) {
                // A: positions mb*128.., shifted by filter row pair a and column pair 2*bp (units of 16 B)
                const uint32_t a_addr = wbase + e * win_bytes + (mb * 128 + a * PW + 2 * bp) * 16;
                const int kc = (a * 2 + e) * 2 + bp;                 // K = 16 chunk of the weights
                const uint64_t db = dw0 + static_cast<uint64_t>((kc >> 2) * (8192 >> 4) + (kc & 3) * 2);
                acc.mma2(desc_nosw(a_addr), desc_nosw(a_addr + 128), db, kc != 0);
              }
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          acc.fence_regs();
          if (mb == kSBlocks - 1 && lane == 0) mbar_arrive(&win_empty[ws.s]);
          uint32_t r[32];
          acc.rows32(0, r, xacc, lane);
          uint4 v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            v[q].x = pack_bf16x2(fmaxf(fmaf(__uint_as_float(r[q * 8 + 0]), sc[q * 8 + 0], bi[q * 8 + 0]), 0.f),
                                 fmaxf(fmaf(__uint_as_float(r[q * 8 + 1]), sc[q * 8 + 1], bi[q * 8 + 1]), 0.f));
            v[q].y = pack_bf16x2(fmaxf(fmaf(__uint_as_float(r[q * 8 + 2]), sc[q * 8 + 2], bi[q * 8 + 2]), 0.f),
                                 fmaxf(fmaf(__uint_as_float(r[q * 8 + 3]), sc[q * 8 + 3], bi[q * 8 + 3]), 0.f));
            v[q].z = pack_bf16x2(fmaxf(fmaf(__uint_as_float(r[q * 8 + 4]), sc[q * 8 + 4], bi[q * 8 + 4]), 0.f),
                                 fmaxf(fmaf(__uint_as_float(r[q * 8 + 5]), sc[q * 8 + 5], bi[q * 8 + 5]), 0.f));
            v[q].w = pack_bf16x2(fmaxf(fmaf(__uint_as_float(r[q * 8 + 6]), sc[q * 8 + 6], bi[q * 8 + 6]), 0.f),
                                 fmaxf(fmaf(__uint_as_float(r[q * 8 + 7]), sc[q * 8 + 7], bi[q * 8 + 7]), 0.f));
          }
          const int mblk = m0 + mb * 128;
          if constexpr (!kPool) {
            // staging row = position inside the block, 128 B per position, 16-byte chunks XOR-swizzled by the row
            const uint32_t stage = so_addr + (blk & 1) * 16384;
            const uint32_t srow = stage + row * 128;
            const uint32_t sw = row & 7;
#pragma unroll
            for (int q = 0; q < 4; ++q) st_shared_v4(srow + (((half * 4 + q) ^ sw) << 4), v[q]);
            asm volatile("bar.sync 2, 256;" ::: "memory");
            // coalesced copy-out: 8 threads per position (16 B each), 32 positions per pass; junk positions are skipped
#pragma unroll
            for (int it = 0; it < 4; ++it) {
              const int pos = it * 32 + static_cast<int>(etid >> 3);
              const int ch16 = static_cast<int>(etid & 7);
              const int m = mblk + pos;
              const int y = m / p.PW, x = m - y * p.PW;
              if (m < positions && x < p.OW) {
                const uint4 o = ld_shared_v4(stage + pos * 128 + ((ch16 ^ (pos & 7)) << 4));
                __nv_bfloat16* dst = p.out + ((static_cast<size_t>(b) * p.OH + y) * p.OW + x) * kSN + ch16 * 8;
                *reinterpret_cast<uint4*>(dst) = o;
              }
            }
            // the staging buffer (blk & 1) is rewritten two blocks later: the barrier of the next block orders that
          } else {
            // conv row ring: ring[y mod ring_rows][x][64 ch], 16-byte chunks XOR-swizzled by x
            const int m = mblk + static_cast<int>(row);
            const int y = m / p.PW, x = m - y * p.PW;
            if (x < p.OW && y >= row_lo && y < row_hi) {
              const uint32_t rrow = so_addr + (y & ring_mask) * ring_row_bytes + x * 128;
#pragma unroll
              for (int q = 0; q < 4; ++q) st_shared_v4(rrow + (((half * 4 + q) ^ (x & 7)) << 4), v[q]);
            }
            asm volatile("bar.sync 2, 256;" ::: "memory");
            // rows <= yc are complete; emit every pooled row whose last conv row is in (the ring depth keeps the rows a
            // slower thread is still pooling, and the rows of the pending pooled row, apart from the rows the next block
            // writes: stem_ring_rows)
            const int yc = min((mblk + 128) / p.PW - 1, row_hi - 1);
            while (next_yp < yp_end && min(2 * next_yp + 1, p.OH - 1) <= yc) {
              // taps outside the image are replaced by the nearest tap INSIDE the window (the maximum is idempotent), so
              // there is no branching and the nine 16-byte loads of an item are independent and all in flight together
              const int y1 = 2 * next_yp;
              const uint32_t r0 = so_addr + (max(y1 - 1, 0) & ring_mask) * ring_row_bytes;
              const uint32_t r1 = so_addr + (y1 & ring_mask) * ring_row_bytes;
              const uint32_t r2 = so_addr + (min(y1 + 1, p.OH - 1) & ring_mask) * ring_row_bytes;
              for (int idx = etid; idx < p.OWp * 8; idx += 256) {
                const int xp = idx >> 3, c = idx & 7;
                const int x1 = 2 * xp, x0 = max(x1 - 1, 0), x2 = min(x1 + 1, p.OW - 1);
                const uint32_t o0 = x0 * 128 + ((c ^ (x0 & 7)) << 4), o1 = x1 * 128 + ((c ^ (x1 & 7)) << 4),
                               o2 = x2 * 128 + ((c ^ (x2 & 7)) << 4);
                uint4 w[9];
                w[0] = ld_shared_v4(r0 + o0); w[1] = ld_shared_v4(r0 + o1); w[2] = ld_shared_v4(r0 + o2);
                w[3] = ld_shared_v4(r1 + o0); w[4] = ld_shared_v4(r1 + o1); w[5] = ld_shared_v4(r1 + o2);
                w[6] = ld_shared_v4(r2 + o0); w[7] = ld_shared_v4(r2 + o1); w[8] = ld_shared_v4(r2 + o2);
                uint4 o;
                {
                  auto mx = [](uint32_t a, uint32_t b) {
                    __nv_bfloat162 r = __hmax2(*reinterpret_cast<const __nv_bfloat162*>(&a), *reinterpret_cast<const __nv_bfloat162*>(&b));
                    return *reinterpret_cast<uint32_t*>(&r);
                  };
                  auto mx9 = [&](auto get) {
                    const uint32_t a = mx(mx(get(w[0]), get(w[1])), mx(get(w[2]), get(w[3])));
                    const uint32_t b = mx(mx(get(w[4]), get(w[5])), mx(get(w[6]), get(w[7])));
                    return mx(mx(a, b), get(w[8]));
                  };
                  o.x = mx9([](const uint4& v) { return v.x; });
                  o.y = mx9([](const uint4& v) { return v.y; });
                  o.z = mx9([](const uint4& v) { return v.z; });
                  o.w = mx9([](const uint4& v) { return v.w; });
                }
                __nv_bfloat16* dst = p.out + ((static_cast<size_t>(b) * p.OHp + next_yp) * p.OWp + xp) * kSN + c * 8;
                *reinterpret_cast<uint4*>(dst) = o;
              }
              ++next_yp;
            }
          }
        }
      }
    }
  }

}

// Conv rows the pooling ring must hold.  While some threads still pool the rows of block k, others already write block
// k+1 (there is no barrier between the pooling loop and the next block's ring stores).  The rows block k may still read
// start at yc(k-1) - 1 >= floor(m_k / PW) - 2 (m_k: first position of block k), and block k+1 writes rows up to
// floor((m_k + 255) / PW) <= floor(m_k / PW) + floor(255 / PW) + 1.  Those rows must fall in distinct ring slots:
// depth >= floor(255 / PW) + 4.  8 rows suffice from PW >= 52 (stem output width 48, a 96-pixel network input); a
// narrower image takes 16, 32 or 64.
int stem_ring_rows(int PW) {
  int r = 8;
  while (r < 255 / PW + 4) r *= 2;
  return r;
}

}  // namespace

// geometry shared by the host graph builder (through dcr_stem_plane_units), stem_rows (image_in.cu) and stem_conv
int stem_fused_pitch(int out_w) { return out_w + 4; }
long long stem_fused_plane_units(int out_h, int out_w) {
  const int PW = stem_fused_pitch(out_w);
  const long long tiles = (static_cast<long long>(out_h) * PW + kSTile - 1) / kSTile;
  return tiles * kSTile + 3ll * PW + 16 + 2 * kSTile;   // read slack: tiles of the pooled schedule may start past a tile boundary
}

int stem_conv(const __nv_bfloat16* planes, int B, int OH, int OW, const __nv_bfloat16* weight, const float* scale, const float* bias,
              __nv_bfloat16* out, cudaStream_t stream, int pool) {
  const DeviceInfo* di = device_info();
  if (!di) return -2;
  if (int rc = require_sm90a(di, "stem_conv")) return rc;
  if (B == 0) return 0;
  StemParams p;
  memset(&p, 0, sizeof(p));
  p.planes = planes; p.B = B; p.OH = OH; p.OW = OW;
  p.PW = stem_fused_pitch(OW);
  p.plane_stride = stem_fused_plane_units(OH, OW) * 8;
  p.img_stride = 2 * p.plane_stride;
  const int tiles_per_img = static_cast<int>((static_cast<long long>(OH) * p.PW + kSTile - 1) / kSTile);
  p.win_units = (kSTile + 3 * p.PW + 3 + 7) & ~7;
  p.scale = scale; p.bias = bias; p.out = out;
  p.OHp = (OH - 1) / 2 + 1;
  p.OWp = (OW - 1) / 2 + 1;
  p.ring_rows = stem_ring_rows(p.PW);
  if (pool) {
    const int parts = (p.OHp % 4 == 0) ? 4 : ((p.OHp % 2 == 0) ? 2 : 1);
    p.units_per_img = parts;
    p.prow_per_part = p.OHp / parts;
    p.part_rows = 2 * p.prow_per_part;
    p.tiles_per_unit = static_cast<int>((static_cast<long long>(p.part_rows + 1) * p.PW + kSTile - 1) / kSTile);
    // the last part's tiles may run past the image's last conv row: the planes carry zero slack for those reads
    const long long last_unit = static_cast<long long>(std::max(0, (parts - 1) * p.part_rows - 1)) * p.PW;
    DCR_REQUIRE(last_unit + static_cast<long long>(p.tiles_per_unit) * kSTile + 3ll * p.PW + 8 <= stem_fused_plane_units(OH, OW),
                "stem_conv: plane slack too small for the pooled schedule (%d x %d)", OH, OW);
  } else {
    p.units_per_img = tiles_per_img;
    p.tiles_per_unit = 1;
    p.prow_per_part = 0;
    p.part_rows = 0;
  }
  p.num_units = B * p.units_per_img;
  CUtensorMap tw;
  if (int rc = make_tmap_2d_bf16(&tw, weight, kSN, 256, 256, kSN, 64)) return rc;
  const size_t stage = (static_cast<size_t>(2) * p.win_units * 16 + 1023) & ~size_t(1023);
  const size_t out_bytes = pool ? ((static_cast<size_t>(p.ring_rows) * OW * 128 + 1023) & ~size_t(1023)) : 2 * 16384;
  const size_t fixed = 1024 + kWBytes + out_bytes + 8 * kAccXposeWarpBytes + 512 + 256;
  // with the pooling ring of a 224-pixel image only one window stage fits: the next tile's window is loaded once the
  // current tile's MMAs have completed
  DCR_REQUIRE(fixed + stage <= di->max_smem_optin, "stem_conv: image too wide for the window buffers (OW = %d)", OW);
  p.win_stages = static_cast<int>(std::min<size_t>(4, (di->max_smem_optin - fixed) / stage));
  const size_t smem = fixed + p.win_stages * stage;
  const int grid = std::min(p.num_units, di->num_sms);
  return launch(pool ? stem_conv_kernel<true> : stem_conv_kernel<false>, grid, kSThreads, smem, stream, "stem_conv", tw, p);
}

}  // namespace dcr
