// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (tiled + im2col loads, tiled stores), wgmma, the ping-pong
// hand-off between two consumer warpgroups.  Everything here is device-only and header-only.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace dcr {

#define DCR_DEVICE __device__ __forceinline__

DCR_DEVICE uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// Dynamic shared memory rounded up to 1024 bytes: the 128-byte swizzle of TMA and wgmma repeats every 1024 bytes, so
// tile bases carved from here line up with it.  Launches reserve 1024 bytes of slack for this.
DCR_DEVICE uint8_t* smem_align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

// two floats -> round-to-nearest bf16 pair, `lo` in the lower half (the lower address once stored)
DCR_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&p);
}

DCR_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
DCR_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
DCR_DEVICE void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
DCR_DEVICE void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

DCR_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
DCR_DEVICE void mbar_arrive_cnt(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
DCR_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
DCR_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// The producer role is a single thread whose instruction stream is on the critical path of the whole pipeline, so the
// wait is one tight asm loop (no predicate -> register -> branch round trip per poll) ...
DCR_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%0], %1;\n\t"
      "@P bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// ... and ring positions advance with a compare instead of `it % stages` / `it / stages` (runtime divisions).
struct PipeState {
  uint32_t s, ph, n;
  DCR_DEVICE explicit PipeState(uint32_t stages) : s(0), ph(0), n(stages) {}
  DCR_DEVICE void next() {
    if (++s == n) {
      s = 0;
      ph ^= 1;
    }
  }
  // past the k ring positions another consumer takes (ping-pong schedules: the other warpgroup's tile)
  DCR_DEVICE void skip(int k) {
    for (int i = 0; i < k; ++i) next();
  }
};

// Register reallocation between warpgroups (executed by all warps of a warpgroup): the producer warpgroup gives registers
// back so that the consumer warpgroups can hold a 128 x 128 fp32 accumulator and its epilogue without spilling.
template <int kRegs>
DCR_DEVICE void wg_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
DCR_DEVICE void wg_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// named barrier among `threads` threads (a warpgroup: 128, both consumer warpgroups: 256)
DCR_DEVICE void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Ping-pong hand-off of two consumer warpgroups that take a CTA's tiles alternately, warpgroup 0 first: a warpgroup
// starts the k-loop of its tile once the other one has issued its last k-block, so each epilogue runs under the other
// warpgroup's k-loop.  turn[g] (count 4: the other warpgroup's warps) completes a phase per hand-over to warpgroup g.
// Warpgroup 1's tile tc waits for phase tc of turn[1] (warpgroup 0's tile tc), warpgroup 0's tile tc > 0 for phase
// tc - 1 of turn[0] (warpgroup 1's tile tc - 1).  A barrier never runs a phase ahead of its waiter, because the next
// hand-over to a warpgroup needs that warpgroup's own hand-over first, so the parity of the phase is enough.
struct PingPong {
  uint64_t* turn;   // [2]
  // tc: tiles this warpgroup has run so far
  DCR_DEVICE void wait(uint32_t wg, uint32_t tc) const {
    if (wg == 1 || tc > 0) mbar_wait(&turn[wg], (wg == 1 ? tc : tc - 1) & 1);
  }
  // one lane of each of the warpgroup's four warps, once the tile's last wgmma has been issued
  DCR_DEVICE void hand_over(uint32_t wg) const { mbar_arrive(&turn[wg ^ 1]); }
};

// ----------------------------------------------------------------------------------------------
// TMA
DCR_DEVICE void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

// tiled loads, complete on this CTA's barrier
DCR_DEVICE void tma_load_2d(void* dst, const void* tmap, uint64_t* bar, int c0, int c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}

// 4-D tiled load / store (coordinates innermost first; loads may start at negative coordinates: zero fill)
DCR_DEVICE void tma_load_4d(void* dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, int c3, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(hint)
      : "memory");
}
DCR_DEVICE void tma_store_4d(const void* tmap, uint32_t src_smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(src_smem), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
DCR_DEVICE void tma_store_2d(const void* tmap, uint32_t src_smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(src_smem), "r"(c0), "r"(c1)
               : "memory");
}
// Tiled stores are issued by one thread and tracked in bulk groups: commit closes the group of the stores issued since
// the last commit; wait_read<N> returns once at most N groups still read their shared-memory source (the older sources
// may be overwritten); wait_all returns once every committed store is complete.
DCR_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
DCR_DEVICE void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
DCR_DEVICE void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// im2col-mode load of an NHWC tensor: coordinates {c, w, h, n} of the first base pixel, filter-tap offsets {w, h}
DCR_DEVICE void tma_load_im2col_4d(void* dst, const void* tmap, uint64_t* bar, int c, int w, int h, int n,
                                   uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w),
      "h"(off_h)
      : "memory");
}

// Explicit shared-state-space vector accesses (32-bit shared addresses): pointers into dynamically carved shared
// memory whose buffer index is a run-time value otherwise compile to GENERIC loads/stores (LD.E / ST.E), which queue
// with the global-memory operations (lg_throttle stalls) and have a longer latency than LDS / STS.
DCR_DEVICE uint4 ld_shared_v4(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr));
  return v;
}
DCR_DEVICE float4 ld_shared_f4(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr));
  return v;
}
DCR_DEVICE void st_shared_v4(uint32_t saddr, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
DCR_DEVICE float2 ld_shared_f2(uint32_t saddr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(saddr));
  return v;
}
DCR_DEVICE uint32_t ld_shared_u32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}
DCR_DEVICE void st_shared_u32(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}
DCR_DEVICE void st_shared_f32(uint32_t saddr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(saddr), "f"(v) : "memory");
}


// ----------------------------------------------------------------------------------------------
// wgmma (Hopper warpgroup MMA): D[regs] (+)= A[smem desc] * B[smem desc], bf16 inputs, fp32 accumulation.
// Executed by all 128 threads of an aligned warpgroup (warps 4i .. 4i+3).
DCR_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
DCR_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
DCR_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }

// m64 x N x k16; kTransB: B is stored MN-major (N contiguous) instead of K-major
template <int N, bool kTransB = false>
DCR_DEVICE void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  static_assert(N == 32 || N == 64 || N == 128, "wgmma_bf16: N must be 32, 64 or 128");
  if constexpr (N == 32) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, %19;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate), "n"(kTransB ? 1 : 0));
  } else if constexpr (N == 64) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, %35;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate), "n"(kTransB ? 1 : 0));
  } else if constexpr (N == 128) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, %67;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate), "n"(kTransB ? 1 : 0));
  }

}

// Shared-memory matrix descriptor (wgmma) for a bf16 tile stored as rows of 128 B with the 128-byte swizzle (8-row x
// 128 B atoms).  start>>4 in [0,14), LBO>>4 in [16,30) (unused for swizzled K-major, 1), SBO>>4 in [32,46) = distance of
// consecutive 8-row groups, layout type 1 (SWIZZLE_128B) in [62,64); base offset 0: the swizzle is a function of the
// absolute shared-memory address, so a start address that is a multiple of 128 B but not of 1024 B (conv3x3_halo.cu)
// needs no correction.  K advances inside the atom by +32 B per k16.
DCR_DEVICE uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t sbo = 1024) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(sbo >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// A 128-row x N-column fp32 accumulator tile held by one warpgroup as two m64 wgmma accumulators.  The A descriptors take
// the tile's 8-row groups two apart (SBO = 2048 B; the second accumulator starts one group, 1024 B, later), so warp w of
// the warpgroup holds exactly rows 32w .. 32w+31 of the tile: the row block its epilogue owns.
template <int N, bool kTransB = false>
struct WgAcc {
  float d[2][N / 2];

  // one k16 step.  a_addr: smem address of row 0 of the 128-row K-major A tile (1024-aligned, plus the k offset);
  // db: descriptor of B for the same k step
  DCR_DEVICE void mma(uint32_t a_addr, uint64_t db, uint32_t accumulate) {
    mma2(wgmma_desc_sw128(a_addr, 2048), wgmma_desc_sw128(a_addr + 1024, 2048), db, accumulate);
  }
  // the same with explicit A descriptors of the two 64-row halves (even / odd 8-row groups)
  DCR_DEVICE void mma2(uint64_t da0, uint64_t da1, uint64_t db, uint32_t accumulate) {
    wgmma_bf16<N, kTransB>(d[0], da0, db, accumulate);
    wgmma_bf16<N, kTransB>(d[1], da1, db, accumulate);
  }
  // keep the compiler from moving accumulator accesses across wgmma_fence / wgmma_wait
  DCR_DEVICE void fence_regs() {
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int i = 0; i < N / 2; ++i) asm volatile("" : "+f"(d[s][i])::"memory");
  }
  // every pair of horizontally adjacent accumulator elements this thread holds: f(row, col, d[row][col], d[row][col + 1])
  // with row in [0, 32) of this warp's row block and col even, in [0, N).  For epilogues that write straight from the
  // accumulator layout (no transpose buffer).
  template <class F>
  DCR_DEVICE void for_each_pair(uint32_t lane, F&& f) const {
    const uint32_t r0 = lane >> 2, c0 = 2 * (lane & 3);
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int i = 0; i < N / 2; i += 2) f(r0 + 8 * s + 16 * ((i >> 1) & 1), 8 * (i >> 2) + c0, d[s][i], d[s][i + 1]);
  }
  // columns [32c, 32c+32) of row `lane` of this warp's 32-row block -> r[0..31], through the warp's 32 x 33 float
  // transpose buffer at shared address xbuf.  c must be a compile-time constant after unrolling (d stays in registers).
  DCR_DEVICE void rows32(int c, uint32_t (&r)[32], uint32_t xbuf, uint32_t lane) const {
    const uint32_t r0 = lane >> 2, c0 = 2 * (lane & 3);
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const uint32_t row = r0 + 8 * s + 16 * ((i >> 1) & 1);
        const uint32_t col = 8 * (i >> 2) + c0 + (i & 1);
        st_shared_f32(xbuf + (row * 33 + col) * 4, d[s][16 * c + i]);
      }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 32; ++j) asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r[j]) : "r"(xbuf + (lane * 33 + j) * 4));
    __syncwarp();
  }
};
constexpr int kAccXposeWarpBytes = 32 * 33 * 4;   // per-warp transpose buffer of WgAcc::rows32

}  // namespace dcr
