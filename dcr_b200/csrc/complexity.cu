// Match-complexity statistics of uint8 HWC images (diff_retrieval.py:497-524): grey-level entropy and the two L1
// total-variation sums (image_stats), and the size / bytes of the baseline JPEG that cv2.imencode writes (jpeg_*).
//
// JPEG pipeline per chunk of n images (DESIGN.md, "Match complexity"):
//   1. jpeg_block_kernel   one thread per 8x8 block: colour conversion, h2v2 downsampling, islow DCT, quantisation;
//                          stores the quantised DC and the bit count of the AC codes.
//   2. jpeg_scan_kernel    one CTA per image: adds the DC code lengths (the DC difference needs the previous block of
//                          the component in MCU order) and turns the counts into bit offsets, a fixed-association scan.
//   3. jpeg_emit_kernel    one thread per block again: recomputes its coefficients and ORs its codes into the image's
//                          big-endian bit buffer at its offset.  OR commutes, so the bits do not depend on the schedule.
//   4. jpeg_finish_kernel  one CTA per image: counts the 0xFF bytes (each is followed by a stuffed 0x00), pads the last
//                          byte with 1-bits, writes the size and, when asked, header + stuffed scan + EOI.
// No coefficient array is kept: the workspace holds per-block DC and offsets and the bit buffers, sized per chunk.
#include <cstring>
#include <vector>

#include "dcr_internal.cuh"
#include "host_util.cuh"

namespace dcr {

namespace {

constexpr int kJpegHeaderBytes = 623;
// Largest code of one block: DC category 11 with the 11-bit chroma code (22 bits), then 63 AC codes of at most 16 bits
// with at most 10 magnitude bits (26 bits each).  An EOB is only sent after a zero (62 codes + EOB < 63 codes) and a
// ZRL (at most 16 bits) stands for 16 zeros that send nothing, so 22 + 63 * 26 bounds every block.
constexpr int kMaxBlockBits = 22 + 63 * 26;

// Annex K.3 tables (bits per code length 1..16, then the symbols)
constexpr unsigned char kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr unsigned char kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
constexpr unsigned char kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr unsigned char kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
constexpr unsigned char kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
    0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
constexpr unsigned char kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
constexpr unsigned char kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
    0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
    0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
    0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
    0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
    0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
    0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
constexpr unsigned char kStdLumaQt[64] = {
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr unsigned char kStdChromaQt[64] = {
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
    99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
// zig-zag position -> natural index, and its inverse
constexpr unsigned char kZigzag[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63};
__constant__ unsigned char c_unzig[64] = {
    0, 1, 5, 6, 14, 15, 27, 28, 2, 4, 7, 13, 16, 26, 29, 42, 3, 8, 12, 17, 25, 30, 41, 43, 9, 11, 18, 24, 31, 40, 44,
    53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48,
    49, 57, 58, 62, 63};

// Everything a kernel needs that depends on the quality: passed by value (kernel parameter space)
struct JpegTables {
  unsigned short qdiv[2][64];        // 8 * quantval (the islow DCT output is scaled by 8), natural order
  unsigned short dc_code[2][12];
  unsigned char dc_size[2][12];
  unsigned short ac_code[2][256];
  unsigned char ac_size[2][256];
};

void make_huff(const unsigned char* bits, const unsigned char* vals, unsigned short* code, unsigned char* size) {
  // jchuff.c jpeg_make_c_derived_tbl: canonical codes in order of length
  unsigned c = 0;
  int p = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < bits[len - 1]; ++i, ++p) {
      code[vals[p]] = static_cast<unsigned short>(c++);
      size[vals[p]] = static_cast<unsigned char>(len);
    }
    c <<= 1;
  }
}

int quality_scale(int quality) { return quality < 50 ? 5000 / quality : 200 - 2 * quality; }

int quant_value(int base, int scale) {   // jcparam.c jpeg_add_quant_table with force_baseline
  int v = (base * scale + 50) / 100;
  return v < 1 ? 1 : (v > 255 ? 255 : v);
}

JpegTables make_tables(int quality) {
  JpegTables t;
  std::memset(&t, 0, sizeof(t));
  const int s = quality_scale(quality);
  for (int i = 0; i < 64; ++i) {
    t.qdiv[0][i] = static_cast<unsigned short>(8 * quant_value(kStdLumaQt[i], s));
    t.qdiv[1][i] = static_cast<unsigned short>(8 * quant_value(kStdChromaQt[i], s));
  }
  make_huff(kDcLumaBits, kDcVals, t.dc_code[0], t.dc_size[0]);
  make_huff(kDcChromaBits, kDcVals, t.dc_code[1], t.dc_size[1]);
  make_huff(kAcLumaBits, kAcLumaVals, t.ac_code[0], t.ac_size[0]);
  make_huff(kAcChromaBits, kAcChromaVals, t.ac_code[1], t.ac_size[1]);
  return t;
}

std::vector<unsigned char> make_header(int h, int w, int quality) {
  std::vector<unsigned char> o = {0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00, 0x01, 0x01, 0x00,
                                  0x00, 0x01, 0x00, 0x01, 0x00, 0x00};
  const int s = quality_scale(quality);
  for (int tid = 0; tid < 2; ++tid) {
    const unsigned char* base = tid == 0 ? kStdLumaQt : kStdChromaQt;
    o.insert(o.end(), {0xFF, 0xDB, 0x00, 0x43, static_cast<unsigned char>(tid)});
    for (int k = 0; k < 64; ++k) o.push_back(static_cast<unsigned char>(quant_value(base[kZigzag[k]], s)));
  }
  o.insert(o.end(), {0xFF, 0xC0, 0x00, 0x11, 8, static_cast<unsigned char>(h >> 8), static_cast<unsigned char>(h & 255),
                     static_cast<unsigned char>(w >> 8), static_cast<unsigned char>(w & 255), 3, 1, 0x22, 0, 2, 0x11, 1,
                     3, 0x11, 1});
  const unsigned char* bits[4] = {kDcLumaBits, kAcLumaBits, kDcChromaBits, kAcChromaBits};
  const unsigned char* vals[4] = {kDcVals, kAcLumaVals, kDcVals, kAcChromaVals};
  const unsigned char cls[4] = {0x00, 0x10, 0x01, 0x11};
  for (int t = 0; t < 4; ++t) {
    int nv = 0;
    for (int i = 0; i < 16; ++i) nv += bits[t][i];
    const int len = 2 + 1 + 16 + nv;
    o.insert(o.end(), {0xFF, 0xC4, static_cast<unsigned char>(len >> 8), static_cast<unsigned char>(len & 255), cls[t]});
    o.insert(o.end(), bits[t], bits[t] + 16);
    o.insert(o.end(), vals[t], vals[t] + nv);
  }
  o.insert(o.end(), {0xFF, 0xDA, 0x00, 0x0C, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
  return o;
}

// ---- block stage -------------------------------------------------------------------------------------------------

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// jfdctint.c jpeg_fdct_islow, one 8-point pass over d[0], d[s], ..., d[7s]; `final` selects the column pass.
template <int S, bool kFinal>
__device__ __forceinline__ void fdct_pass(int* d) {
  constexpr int cb = 13, pb = 2, sh = kFinal ? cb + pb : cb - pb;
  const int t0 = d[0] + d[7 * S], t7 = d[0] - d[7 * S], t1 = d[S] + d[6 * S], t6 = d[S] - d[6 * S];
  const int t2 = d[2 * S] + d[5 * S], t5 = d[2 * S] - d[5 * S], t3 = d[3 * S] + d[4 * S], t4 = d[3 * S] - d[4 * S];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (kFinal) {
    d[0] = descale(t10 + t11, pb);
    d[4 * S] = descale(t10 - t11, pb);
  } else {
    d[0] = (t10 + t11) << pb;
    d[4 * S] = (t10 - t11) << pb;
  }
  int z1 = (t12 + t13) * 4433;
  d[2 * S] = descale(z1 + t13 * 6270, sh);
  d[6 * S] = descale(z1 - t12 * 15137, sh);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  d[7 * S] = descale(t4 * 2446 + z1 + z3, sh);
  d[5 * S] = descale(t5 * 16819 + z2 + z4, sh);
  d[3 * S] = descale(t6 * 25172 + z2 + z3, sh);
  d[S] = descale(t7 * 12299 + z1 + z4, sh);
}

// Which block a thread of the block / emit kernels owns.  Threads [0, n * 4 * mcus) take the Y blocks, the rest the
// chroma blocks (Cb and Cr of one MCU on adjacent threads), so that a warp runs one kind of colour conversion.
struct BlockRef {
  int img, mcu, j;   // j: 0..3 Y (row-major in the MCU), 4 Cb, 5 Cr
};
__device__ __forceinline__ BlockRef block_ref(long long g, int n, int mcus) {
  const long long ny = static_cast<long long>(n) * 4 * mcus;
  BlockRef r;
  if (g < ny) {
    r.img = static_cast<int>(g / (4 * mcus));
    const int rem = static_cast<int>(g - static_cast<long long>(r.img) * 4 * mcus);
    r.mcu = rem >> 2;
    r.j = rem & 3;
  } else {
    const long long c = g - ny;
    r.img = static_cast<int>(c / (2 * mcus));
    const int rem = static_cast<int>(c - static_cast<long long>(r.img) * 2 * mcus);
    r.mcu = rem >> 1;
    r.j = 4 + (rem & 1);
  }
  return r;
}

// Quantised coefficients of one block, written to zz[0..63] in zig-zag order; returns the mask of non-zero positions.
// Colour conversion: jccolor.c rgb_ycc_convert with cv2's channel order (the array is read as BGR).
__device__ __forceinline__ unsigned long long block_coefs(const unsigned char* __restrict__ img, int w, int mcus_x,
                                                          const BlockRef& b, const JpegTables& t, short* zz) {
  const int my = b.mcu / mcus_x, mx = b.mcu - my * mcus_x;
  int d[64];
  if (b.j < 4) {
    const int y0 = my * 16 + (b.j >> 1) * 8, x0 = mx * 16 + (b.j & 1) * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const unsigned char* p = img + (static_cast<size_t>(y0 + r) * w + x0) * 3;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int B = __ldg(p + 3 * c), G = __ldg(p + 3 * c + 1), R = __ldg(p + 3 * c + 2);
        d[r * 8 + c] = ((19595 * R + 38470 * G + 7471 * B + 32768) >> 16) - 128;
      }
    }
  } else {
    const bool cb = b.j == 4;
    const int kr = cb ? -11059 : 32768, kg = cb ? -21709 : -27439, kb = cb ? 32768 : -5329;
    const int off = (128 << 16) + 32767;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const unsigned char* p0 = img + (static_cast<size_t>(my * 16 + 2 * r) * w + mx * 16) * 3;
      const unsigned char* p1 = p0 + static_cast<size_t>(w) * 3;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        int s = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const unsigned char* p = ((q >> 1) ? p1 : p0) + 3 * (2 * c + (q & 1));
          s += (kr * __ldg(p + 2) + kg * __ldg(p + 1) + kb * __ldg(p) + off) >> 16;
        }
        d[r * 8 + c] = ((s + 1 + (c & 1)) >> 2) - 128;   // jcsample.c h2v2_downsample: bias 1, 2, 1, 2, ...
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) fdct_pass<1, false>(d + 8 * r);
#pragma unroll
  for (int c = 0; c < 8; ++c) fdct_pass<8, true>(d + c);
  const int tbl = b.j < 4 ? 0 : 1;
  unsigned long long mask = 0;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int q = t.qdiv[tbl][i];
    const int a = d[i] < 0 ? -d[i] : d[i];
    int v = (a + (q >> 1)) / q;                         // jcdctmgr.c quantize: round half up, sign restored
    v = d[i] < 0 ? -v : v;
    const int k = c_unzig[i];
    zz[k] = static_cast<short>(v);
    mask |= static_cast<unsigned long long>(v != 0) << k;
  }
  return mask;
}

__device__ __forceinline__ int nbits(int v) {
  const int a = v < 0 ? -v : v;
  return a ? 32 - __clz(a) : 0;
}
__device__ __forceinline__ unsigned magnitude(int v, int nb) {
  return static_cast<unsigned>(v < 0 ? v - 1 : v) & ((1u << nb) - 1u);
}

struct BitCounter {
  unsigned bits = 0;
  __device__ void put(unsigned, int len) { bits += len; }
};

// Writes MSB-first codes into a zeroed big-endian bit buffer (bit p is bit 31 - p % 32 of word p / 32).  Words are
// OR-ed in, so the first and last word of a block may be shared with its neighbours.
struct BitWriter {
  unsigned* buf;
  unsigned word;
  int fill;                  // bits of the current word already taken
  unsigned long long acc;    // pending bits, left-aligned
  __device__ BitWriter(unsigned* b, unsigned pos) : buf(b), word(pos >> 5), fill(pos & 31), acc(0) {}
  __device__ void put(unsigned code, int len) {   // len <= 32
    acc |= static_cast<unsigned long long>(code) << (64 - fill - len);
    fill += len;
    if (fill >= 32) {
      atomicOr(buf + word, static_cast<unsigned>(acc >> 32));
      acc <<= 32;
      fill -= 32;
      ++word;
    }
  }
  __device__ void flush() {
    if (fill > 0) atomicOr(buf + word, static_cast<unsigned>(acc >> 32));
  }
};

// jchuff.c encode_one_block after the DC: run lengths, ZRL, EOB.  Codes and magnitudes go out together (<= 26 bits).
template <class Sink>
__device__ __forceinline__ void encode_ac(const short* zz, unsigned long long mask, int tbl, const JpegTables& t,
                                          Sink& s) {
  mask &= ~1ull;
  int last = 0;
  while (mask) {
    const int k = __ffsll(static_cast<long long>(mask)) - 1;
    mask &= mask - 1;
    int run = k - last - 1;
    while (run > 15) {
      s.put(t.ac_code[tbl][0xF0], t.ac_size[tbl][0xF0]);
      run -= 16;
    }
    const int v = zz[k], nb = nbits(v), sym = (run << 4) + nb;
    s.put((static_cast<unsigned>(t.ac_code[tbl][sym]) << nb) | magnitude(v, nb), t.ac_size[tbl][sym] + nb);
    last = k;
  }
  if (last < 63) s.put(t.ac_code[tbl][0], t.ac_size[tbl][0]);
}

// index (within the image, MCU order) of the block whose DC predicts block b, or -1 for the first of its component
__device__ __forceinline__ int dc_predecessor(int b) {
  const int m = b / 6, j = b - m * 6;
  if (j < 4) return j > 0 ? b - 1 : (m > 0 ? b - 3 : -1);
  return m > 0 ? b - 6 : -1;
}

constexpr int kBlockThreads = 128;

__global__ void __launch_bounds__(kBlockThreads)
    jpeg_block_kernel(const unsigned char* __restrict__ images, int n, int h, int w, const __grid_constant__ JpegTables t,
                      short* __restrict__ dc, unsigned* __restrict__ ac_bits) {
  __shared__ short zz_s[kBlockThreads][66];   // 33-word rows: no bank conflicts on a common zig-zag position
  const int mcus_x = w >> 4, mcus = mcus_x * (h >> 4), nb = 6 * mcus;
  const long long g = static_cast<long long>(blockIdx.x) * kBlockThreads + threadIdx.x;
  if (g >= static_cast<long long>(n) * nb) return;
  const BlockRef b = block_ref(g, n, mcus);
  short* zz = zz_s[threadIdx.x];
  const unsigned long long mask = block_coefs(images + static_cast<size_t>(b.img) * h * w * 3, w, mcus_x, b, t, zz);
  BitCounter cnt;
  encode_ac(zz, mask, b.j < 4 ? 0 : 1, t, cnt);
  const size_t slot = static_cast<size_t>(b.img) * nb + b.mcu * 6 + b.j;
  dc[slot] = zz[0];
  ac_bits[slot] = cnt.bits;
}

// ---- per-image scan ----------------------------------------------------------------------------------------------

// Exclusive scan of one value per thread over the CTA (fixed association: warp shuffles, then the warp totals in
// order).  Returns the prefix; *total receives the CTA sum.  Every thread must call it.
template <int kThreads>
__device__ unsigned block_exclusive_scan(unsigned v, unsigned* total) {
  __shared__ unsigned warp_sum[kThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[wid] = x;
  __syncthreads();
  unsigned before = 0, all = 0;
#pragma unroll 1
  for (int i = 0; i < kThreads / 32; ++i) {
    if (i < wid) before += warp_sum[i];
    all += warp_sum[i];
  }
  __syncthreads();   // warp_sum may be reused by the next call
  *total = all;
  return before + x - v;
}

constexpr int kScanThreads = 1024;

__global__ void __launch_bounds__(kScanThreads)
    jpeg_scan_kernel(int nb, const __grid_constant__ JpegTables t, const short* __restrict__ dc,
                     unsigned* __restrict__ bits, unsigned* __restrict__ total_bits) {
  const size_t base = static_cast<size_t>(blockIdx.x) * nb;
  const short* d = dc + base;
  unsigned* bb = bits + base;
  const int per = (nb + kScanThreads - 1) / kScanThreads;
  const int lo = min(nb, static_cast<int>(threadIdx.x) * per), hi = min(nb, lo + per);
  auto block_bits = [&](int b) {
    const int p = dc_predecessor(b);
    const int diff = d[b] - (p >= 0 ? d[p] : 0), nbt = nbits(diff), tbl = (b % 6) < 4 ? 0 : 1;
    return bb[b] + t.dc_size[tbl][nbt] + nbt;
  };
  unsigned s = 0;
  for (int b = lo; b < hi; ++b) s += block_bits(b);
  unsigned total;
  unsigned off = block_exclusive_scan<kScanThreads>(s, &total);
  for (int b = lo; b < hi; ++b) {
    const unsigned v = block_bits(b);   // read before bb[b] is overwritten with the offset
    bb[b] = off;
    off += v;
  }
  if (threadIdx.x == 0) total_bits[blockIdx.x] = total;
}

// ---- emit and finish ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlockThreads)
    jpeg_emit_kernel(const unsigned char* __restrict__ images, int n, int h, int w, const __grid_constant__ JpegTables t,
                     const short* __restrict__ dc, const unsigned* __restrict__ offsets, unsigned* __restrict__ bitbuf,
                     size_t words_per_image) {
  __shared__ short zz_s[kBlockThreads][66];
  const int mcus_x = w >> 4, mcus = mcus_x * (h >> 4), nb = 6 * mcus;
  const long long g = static_cast<long long>(blockIdx.x) * kBlockThreads + threadIdx.x;
  if (g >= static_cast<long long>(n) * nb) return;
  const BlockRef b = block_ref(g, n, mcus);
  short* zz = zz_s[threadIdx.x];
  const unsigned long long mask = block_coefs(images + static_cast<size_t>(b.img) * h * w * 3, w, mcus_x, b, t, zz);
  const int bi = b.mcu * 6 + b.j, p = dc_predecessor(bi), tbl = b.j < 4 ? 0 : 1;
  const size_t ibase = static_cast<size_t>(b.img) * nb;
  const int diff = zz[0] - (p >= 0 ? dc[ibase + p] : 0), nbt = nbits(diff);
  BitWriter wr(bitbuf + static_cast<size_t>(b.img) * words_per_image, offsets[ibase + bi]);
  wr.put((static_cast<unsigned>(t.dc_code[tbl][nbt]) << nbt) | magnitude(diff, nbt), t.dc_size[tbl][nbt] + nbt);
  encode_ac(zz, mask, tbl, t, wr);
  wr.flush();
}

constexpr int kFinishThreads = 512;

__device__ __forceinline__ unsigned scan_byte(const unsigned* buf, unsigned k, unsigned nbytes, unsigned pad_bits) {
  unsigned v = (buf[k >> 2] >> (24 - 8 * (k & 3))) & 0xFFu;
  if (k == nbytes - 1) v |= (1u << pad_bits) - 1u;   // the last byte is padded with 1-bits
  return v;
}

__global__ void __launch_bounds__(kFinishThreads)
    jpeg_finish_kernel(const unsigned* __restrict__ bitbuf, size_t words_per_image, const unsigned* __restrict__ total_bits,
                       const unsigned char* __restrict__ header, long long* __restrict__ sizes,
                       unsigned char* __restrict__ out, long long out_stride) {
  const unsigned* buf = bitbuf + static_cast<size_t>(blockIdx.x) * words_per_image;
  const unsigned tb = total_bits[blockIdx.x], nbytes = (tb + 7) >> 3, pad = (8 - (tb & 7)) & 7;
  const unsigned per = (nbytes + kFinishThreads - 1) / kFinishThreads;
  const unsigned lo = min(nbytes, threadIdx.x * per), hi = min(nbytes, lo + per);
  unsigned ff = 0;
  for (unsigned k = lo; k < hi; ++k) ff += scan_byte(buf, k, nbytes, pad) == 0xFFu;
  unsigned total_ff;
  unsigned before = block_exclusive_scan<kFinishThreads>(ff, &total_ff);
  const long long size = kJpegHeaderBytes + static_cast<long long>(nbytes) + total_ff + 2;
  if (threadIdx.x == 0) sizes[blockIdx.x] = size;
  if (out == nullptr) return;
  unsigned char* o = out + static_cast<size_t>(blockIdx.x) * out_stride;
  for (int i = threadIdx.x; i < kJpegHeaderBytes; i += kFinishThreads) o[i] = header[i];
  for (unsigned k = lo; k < hi; ++k) {
    const unsigned v = scan_byte(buf, k, nbytes, pad);
    const size_t at = kJpegHeaderBytes + static_cast<size_t>(k) + before;
    o[at] = static_cast<unsigned char>(v);
    if (v == 0xFFu) {
      o[at + 1] = 0;
      ++before;
    }
  }
  if (threadIdx.x == 0) {
    o[size - 2] = 0xFF;
    o[size - 1] = 0xD9;
  }
}

// ---- entropy and total variation -----------------------------------------------------------------------------------

constexpr int kStatsThreads = 256;

// One CTA per image.  Grey value: skimage's rgb2gray + img_as_ubyte in fp64 with every product and sum rounded on its
// own (no contraction), in the order x = c/255; g = (x0*0.2125 + x1*0.7154) + x2*0.0721; u = rint(g*255).
__global__ void __launch_bounds__(kStatsThreads)
    image_stats_kernel(const unsigned char* __restrict__ images, int h, int w, double* __restrict__ out_entropy,
                       long long* __restrict__ out_tv) {
  __shared__ unsigned hist[256];
  __shared__ double term[256];
  __shared__ unsigned long long red[2][kStatsThreads / 32];
  const unsigned char* img = images + static_cast<size_t>(blockIdx.x) * h * w * 3;
  hist[threadIdx.x] = 0;
  __syncthreads();
  unsigned long long th = 0, tw = 0;
  const int npx = h * w, row = 3 * w;
  for (int p = threadIdx.x; p < npx; p += kStatsThreads) {
    const int y = p / w, x = p - y * w;
    const unsigned char* px = img + static_cast<size_t>(p) * 3;
    const int c0 = __ldg(px), c1 = __ldg(px + 1), c2 = __ldg(px + 2);
    const double inv = 1.0 / 255;
    const double g = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(c0, inv), 0.2125), __dmul_rn(__dmul_rn(c1, inv), 0.7154)),
                               __dmul_rn(__dmul_rn(c2, inv), 0.0721));
    const double u = fmin(fmax(rint(__dmul_rn(g, 255.0)), 0.0), 255.0);
    atomicAdd(&hist[static_cast<int>(u)], 1u);
    if (x + 1 < w) tw += abs(__ldg(px + 3) - c0) + abs(__ldg(px + 4) - c1) + abs(__ldg(px + 5) - c2);
    if (y + 1 < h) th += abs(__ldg(px + row) - c0) + abs(__ldg(px + row + 1) - c1) + abs(__ldg(px + row + 2) - c2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    th += __shfl_down_sync(0xffffffffu, th, o);
    tw += __shfl_down_sync(0xffffffffu, tw, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = th;
    red[1][threadIdx.x >> 5] = tw;
  }
  __syncthreads();
  // sklearn.metrics.cluster.entropy: -sum (p/N)(log p - log N) over the non-empty bins, 0 when one bin is used
  const unsigned cnt = hist[threadIdx.x];
  const double nn = static_cast<double>(npx);
  term[threadIdx.x] = cnt ? __dmul_rn(static_cast<double>(cnt) / nn, log(static_cast<double>(cnt)) - log(nn)) : 0.0;
  const int used = __syncthreads_count(cnt != 0);
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < 256; ++i) s = __dadd_rn(s, term[i]);
    out_entropy[blockIdx.x] = used <= 1 ? 0.0 : -s;
    unsigned long long a = 0, b = 0;
    for (int i = 0; i < kStatsThreads / 32; ++i) {
      a += red[0][i];
      b += red[1][i];
    }
    out_tv[2 * blockIdx.x] = static_cast<long long>(a);
    out_tv[2 * blockIdx.x + 1] = static_cast<long long>(b);
  }
}

int check_jpeg_size(const char* what, int h, int w) {
  DCR_REQUIRE(h >= 16 && w >= 16 && h <= 4096 && w <= 4096 && h % 16 == 0 && w % 16 == 0,
              "%s: %d x %d images: height and width must be multiples of 16 in 16..4096 (the edge replication libjpeg "
              "applies to other sizes is not implemented)", what, h, w);
  return 0;
}

// The workspace.  With a null base only nb, words_per_image and bytes are meaningful.
struct JpegLayout {
  int nb;                    // blocks per image
  size_t words_per_image;    // bit-buffer words per image
  short* dc;
  unsigned *bits, *total, *buf;
  unsigned char* header;
  size_t bytes;
};

JpegLayout jpeg_layout(int n, int h, int w, void* base = nullptr) {
  JpegLayout l;
  l.nb = 6 * (h / 16) * (w / 16);
  l.words_per_image = (static_cast<size_t>(l.nb) * kMaxBlockBits + 31) / 32;
  Carve c{static_cast<uint8_t*>(base)};
  l.dc = c.take<short>(static_cast<size_t>(n) * l.nb);
  l.bits = c.take<unsigned>(static_cast<size_t>(n) * l.nb);
  l.total = c.take<unsigned>(n);
  l.header = c.take<unsigned char>(kJpegHeaderBytes);
  // the bit buffer comes last and is not rounded up: take(0) only places it
  l.buf = c.take<unsigned>(0);
  l.bytes = c.bytes + sizeof(unsigned) * l.words_per_image * static_cast<size_t>(n);
  return l;
}

}  // namespace

int image_stats(const unsigned char* images, int n, int h, int w, double* out_entropy, long long* out_tv,
                cudaStream_t stream) {
  DCR_REQUIRE(n >= 0, "dcr_image_stats: bad n %d", n);
  DCR_REQUIRE(h >= 1 && w >= 1 && static_cast<long long>(h) * w <= (1ll << 26),
              "dcr_image_stats: bad image size %d x %d (1 .. 2^26 pixels)", h, w);
  if (n == 0) return 0;
  DCR_REQUIRE(images && out_entropy && out_tv, "dcr_image_stats: null pointer argument");
  if (!device_info()) return -2;
  return launch(image_stats_kernel, n, kStatsThreads, 0, stream, "dcr_image_stats", images, h, w, out_entropy, out_tv);
}

size_t jpeg_workspace_size(int n, int h, int w) {
  if (n < 0) {
    set_error(-1, "dcr_jpeg_workspace_size: bad n %d", n);
    return 0;
  }
  if (check_jpeg_size("dcr_jpeg_workspace_size", h, w) != 0) return 0;
  return jpeg_layout(n, h, w).bytes;
}

long long jpeg_max_bytes(int h, int w) {
  if (check_jpeg_size("dcr_jpeg_max_bytes", h, w) != 0) return -1;
  // header, every scan byte stuffed, EOI; rounded up to 16 bytes so that consecutive files stay aligned
  const long long scan = (static_cast<long long>(jpeg_layout(1, h, w).nb) * kMaxBlockBits + 7) / 8;
  return (kJpegHeaderBytes + 2 * scan + 2 + 15) / 16 * 16;
}

int jpeg_encode(const unsigned char* images, int n, int h, int w, int quality, long long* out_sizes,
                unsigned char* out_bytes, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  DCR_REQUIRE(n >= 0, "dcr_jpeg_encode: bad n %d", n);
  if (check_jpeg_size("dcr_jpeg_encode", h, w) != 0) return -1;
  DCR_REQUIRE(quality >= 1 && quality <= 100, "dcr_jpeg_encode: quality %d outside 1..100", quality);
  if (n == 0) return 0;
  DCR_REQUIRE(images && out_sizes && workspace, "dcr_jpeg_encode: null pointer argument");
  const JpegLayout l = jpeg_layout(n, h, w, workspace);
  DCR_REQUIRE(workspace_bytes >= l.bytes, "dcr_jpeg_encode: workspace too small (%zu < %zu)", workspace_bytes, l.bytes);
  DCR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "dcr_jpeg_encode: workspace must be 256-byte aligned");
  if (!device_info()) return -2;
  const JpegTables t = make_tables(quality);
  const std::vector<unsigned char> header = make_header(h, w, quality);
  DCR_REQUIRE(header.size() == kJpegHeaderBytes, "dcr_jpeg_encode: internal header size %zu", header.size());
  // pageable source: staged before the call returns, so `header` may go out of scope
  DCR_CUDA_CHECK(cudaMemcpyAsync(l.header, header.data(), kJpegHeaderBytes, cudaMemcpyHostToDevice, stream));
  DCR_CUDA_CHECK(cudaMemsetAsync(l.buf, 0, sizeof(unsigned) * l.words_per_image * static_cast<size_t>(n), stream));
  const long long blocks = static_cast<long long>(n) * l.nb;
  const unsigned grid = static_cast<unsigned>((blocks + kBlockThreads - 1) / kBlockThreads);
  if (int rc = launch(jpeg_block_kernel, grid, kBlockThreads, 0, stream, "dcr_jpeg_encode", images, n, h, w, t, l.dc, l.bits))
    return rc;
  if (int rc = launch(jpeg_scan_kernel, n, kScanThreads, 0, stream, "dcr_jpeg_encode", l.nb, t, l.dc, l.bits, l.total))
    return rc;
  if (int rc = launch(jpeg_emit_kernel, grid, kBlockThreads, 0, stream, "dcr_jpeg_encode", images, n, h, w, t, l.dc, l.bits,
                      l.buf, l.words_per_image))
    return rc;
  return launch(jpeg_finish_kernel, n, kFinishThreads, 0, stream, "dcr_jpeg_encode", l.buf, l.words_per_image, l.total,
                l.header, out_sizes, out_bytes, out_bytes ? jpeg_max_bytes(h, w) : 0);
}

}  // namespace dcr
