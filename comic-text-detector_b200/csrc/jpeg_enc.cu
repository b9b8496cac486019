// GPU JPEG encode (C ABI `ctd_jpeg_encoder_*`, `ctd_jpeg_encode`, include/ctd_b200.h): every image of a call at once,
// byte for byte the baseline file cv2.imencode('.jpg', img, params) writes with its libjpeg-turbo 3.1 (JCS_EXT_BGR or
// JCS_GRAYSCALE input, JDCT_ISLOW, force_baseline quality tables).  oracle/jpeg_enc_ref.py restates every rule;
// tests/test_cpu_jpeg_encode.py pins it to cv2.
//
// The blocks of all images are numbered in scan order (MCU by MCU, components in order inside an MCU; a grey image is
// one non-interleaved component, one block per MCU).  Stages:
//   1. jpeg_block_kernel, 64 threads per block: colour conversion (jccolor.c tables), edge replication and
//      downsampling (jcprepct.c / jcsample.c) of the block's samples read straight from the strided source,
//      jpeg_fdct_islow, the reciprocal quantiser; int16 coefficients in zig-zag order.  A dummy block (an interleaved
//      MCU past the component's width or height) is its reference block's DC with zero AC (jccoefct.c).
//   2. jpeg_symbol_kernel<kCount>, one thread per block of an OPTIMIZE image: warp-aggregated symbol histograms.
//   3. jpeg_table_kernel, one warp per table: jpeg_gen_optimal_table on the counts, or Annex K.3; the codes.
//   4. jpeg_header_kernel, one thread per image: SOI, APP0, DQT, SOF0, DHT, DRI, SOS into the file buffer.
//   5. jpeg_symbol_kernel<kLength>: each block's bit length; a 64-bit scan of them; a scan of the intervals' byte
//      lengths (every restart interval is padded to a byte).
//   6. jpeg_symbol_kernel<kEmit>: each block ORs its codes, MSB first, into the zeroed word buffer; the last block of
//      an interval adds the 1-bit padding.
//   7. a scan of the 0xFF bytes per word, then jpeg_stuff_kernel writes every byte at its place in the file (a 00
//      after each FF), the RSTn markers and EOI; jpeg_copy_kernel moves the files, 16 bytes a thread, into mapped
//      pinned host memory.  The call synchronises once, at the end.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/ctd_b200.h"
#include "scan.cuh"

int ctd_fail(ctd_handle* h, int code, const char* fmt, ...);

namespace ctd {
namespace jenc {
namespace {

constexpr int kMaxSlots = 6;            // blocks per MCU: 4 luma + 2 chroma at 4:2:0 and 4:1:1
constexpr int64_t kBlockBitsMax = 1665; // 16 + 11 DC bits, 63 AC coefficients of 16 + 10 bits
constexpr int kHdrMax = 2048;           // SOI .. SOS: at most 20 + 2 * 69 + 19 + 4 * 277 + 6 + 14 bytes
constexpr int kMaxSide = 65500;         // JPEG_MAX_DIMENSION

struct JImg {
  const uint8_t* src;
  int64_t sh, sw, sc;
  int32_t h, w, nc, optimize, rst;      // rst: MCUs per restart interval (0: the scan is one interval)
  int32_t maxh, maxv, mcux, mcuy, bpm, nint;
  int32_t hs[3], vs[3], wib[3], hib[3];
  int32_t rows[3];                      // downsampled rows before the last one is repeated to whole iMCU rows
  int32_t first[3], last[3];            // first / last slot of each component in an MCU
  int8_t scomp[kMaxSlots], sdx[kMaxSlots], sdy[kMaxSlots];
  int64_t blk0, nblk, int0, out_off;
  uint32_t recip[2][64], corr[2][64], shift[2][64];   // natural order
  uint8_t qz[2][64];                    // the tables in zig-zag order, for DQT
};

struct HTab {                           // one Huffman table: its DHT payload and per-symbol codes
  uint8_t bits[16];
  uint8_t vals[256];
  int32_t nvals;
  uint32_t code[256];                   // code | size << 16
};

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_std_bits[4][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                          {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125},
                                          {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0},
                                          {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119}};
__constant__ uint8_t c_std_ac_luma[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
    0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
__constant__ uint8_t c_std_ac_chroma[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
    0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
    0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
    0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
    0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
    0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
    0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// last i in [0, n) with a[i] <= v (a non-decreasing, a[0] <= v)
__device__ __forceinline__ int64_t last_le(const int64_t* a, int64_t n, int64_t v) {
  int64_t lo = 0, hi = n - 1;
  while (lo < hi) {
    int64_t mid = (lo + hi + 1) >> 1;
    if (a[mid] <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct BlkPos {
  int img, c, slot, rx, ry;             // (rx, ry): the block whose samples are transformed
  int64_t mcu;
  bool dummy;
};

__device__ __forceinline__ BlkPos locate(const JImg* imgs, const int64_t* blk0, int n, int64_t g) {
  BlkPos P;
  P.img = (int)last_le(blk0, n, g);
  const JImg& im = imgs[P.img];
  int64_t local = g - im.blk0;
  P.mcu = local / im.bpm;
  P.slot = (int)(local - P.mcu * im.bpm);
  int c = P.c = im.scomp[P.slot];
  int mx = (int)(P.mcu % im.mcux), my = (int)(P.mcu / im.mcux);
  int bx = mx * im.hs[c] + im.sdx[P.slot], by = my * im.vs[c] + im.sdy[P.slot];
  bool real_y = by < im.hib[c];
  P.dummy = !real_y || bx >= im.wib[c];
  // a right-edge dummy repeats the row's last real block; a bottom dummy row the MCU's last block of the row above
  P.rx = real_y ? min(bx, im.wib[c] - 1) : min(mx * im.hs[c] + im.hs[c] - 1, im.wib[c] - 1);
  P.ry = min(by, im.hib[c] - 1);
  return P;
}

// ---- 1. block transform ----------------------------------------------------------------------------------------------
__device__ __forceinline__ int comp_value(const JImg& im, int c, int y, int x) {
  const uint8_t* p = im.src + y * im.sh + x * im.sw;
  if (im.nc == 1) return p[0];
  int b = p[0], g = p[im.sc], r = p[2 * im.sc];
  if (c == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (c == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__device__ __forceinline__ int64_t descale(int64_t x, int n) { return (x + ((int64_t)1 << (n - 1))) >> n; }

// one row (stride 1, pass 1) or column (stride 8, pass 2) of jpeg_fdct_islow
template <bool kPass1>
__device__ void fdct_line(int32_t* d, int s) {
  int64_t t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s], t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
  int64_t t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s], t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
  int64_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  constexpr int sh = kPass1 ? 13 - 2 : 13 + 2;
  d[0] = (int32_t)(kPass1 ? (t10 + t11) * 4 : descale(t10 + t11, 2));
  d[4 * s] = (int32_t)(kPass1 ? (t10 - t11) * 4 : descale(t10 - t11, 2));
  int64_t z1 = (t12 + t13) * 4433;
  d[2 * s] = (int32_t)descale(z1 + t13 * 6270, sh);
  d[6 * s] = (int32_t)descale(z1 - t12 * 15137, sh);
  z1 = t4 + t7;
  int64_t z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  int64_t z5 = (z3 + z4) * 9633;
  t4 *= 2446;
  t5 *= 16819;
  t6 *= 25172;
  t7 *= 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  d[7 * s] = (int32_t)descale(t4 + z1 + z3, sh);
  d[5 * s] = (int32_t)descale(t5 + z2 + z4, sh);
  d[3 * s] = (int32_t)descale(t6 + z2 + z3, sh);
  d[s] = (int32_t)descale(t7 + z1 + z4, sh);
}

constexpr int kBlocksPerCta = 4;

__global__ void __launch_bounds__(64 * kBlocksPerCta) jpeg_block_kernel(const JImg* imgs, const int64_t* blk0, int n,
                                                                         int64_t NB, int16_t* coef) {
  __shared__ int32_t s[kBlocksPerCta][64];
  __shared__ uint8_t zz_of[64];
  int lb = threadIdx.x >> 6, t = threadIdx.x & 63;
  if (threadIdx.x < 64) zz_of[c_zigzag[threadIdx.x]] = (uint8_t)threadIdx.x;
  int64_t g = (int64_t)blockIdx.x * kBlocksPerCta + lb;
  bool live = g < NB;
  BlkPos P{};
  if (live) {
    P = locate(imgs, blk0, n, g);
    const JImg& im = imgs[P.img];
    int c = P.c, he = im.maxh / im.hs[c], ve = im.maxv / im.vs[c];
    int sx = P.rx * 8 + (t & 7), sy = P.ry * 8 + (t >> 3);
    int r = min(sy, im.rows[c] - 1);
    int sum = 0;
    for (int j = 0; j < ve; ++j) {
      int y = min(r * ve + j, im.h - 1);
      for (int i = 0; i < he; ++i) sum += comp_value(im, c, y, min(sx * he + i, im.w - 1));
    }
    int v;
    if (he == 1 && ve == 1) v = sum;
    else if (he == 2 && ve == 1) v = (sum + (sx & 1)) >> 1;          // h2v1: bias 0, 1, 0, 1, ...
    else if (he == 2 && ve == 2) v = (sum + 1 + (sx & 1)) >> 2;      // h2v2: bias 1, 2, 1, 2, ...
    else v = (sum + he * ve / 2) / (he * ve);                         // int_downsample
    s[lb][t] = v - 128;
  }
  __syncthreads();
  if (live && t < 8) fdct_line<true>(&s[lb][8 * t], 1);
  __syncthreads();
  if (live && t < 8) fdct_line<false>(&s[lb][t], 8);
  __syncthreads();
  if (!live) return;
  const JImg& im = imgs[P.img];
  int tq = min(P.c, 1), zz = zz_of[t];
  int x = s[lb][t];
  int q = 0;
  if (!P.dummy || zz == 0) {
    uint64_t a = (uint64_t)abs(x);
    q = (int)(((a + im.corr[tq][t]) * im.recip[tq][t]) >> im.shift[tq][t]);
    if (x < 0) q = -q;
  }
  coef[g * 64 + zz] = (int16_t)q;
}

// ---- 2, 5, 6. symbols ---------------------------------------------------------------------------------------------------
enum SymMode { kCount, kLength, kEmit };

__device__ __forceinline__ int nbits_of(int a) { return a ? 32 - __clz(a) : 0; }

// v (nb <= 32 bits) at bit p of the MSB-first stream in 32-bit words
__device__ __forceinline__ void put_bits(uint32_t* w, uint64_t p, uint32_t v, int nb) {
  if (nb == 0) return;
  uint64_t k = p >> 5;
  int sh = 32 - (int)(p & 31) - nb;
  if (sh >= 0) {
    atomicOr(&w[k], v << sh);
  } else {
    atomicOr(&w[k], v >> -sh);
    atomicOr(&w[k + 1], v << (32 + sh));
  }
}

struct SymArgs {
  const JImg* imgs;
  const int64_t* blk0;
  const int64_t* int0;
  int n;
  int64_t NB;
  const int16_t* coef;
  uint32_t* hist;                       // [4 n][256] counts (kCount)
  const HTab* tabs;                     // [4 n] (kLength, kEmit)
  uint32_t* blen;                       // block bit lengths (kLength)
  const uint64_t* boff;                 // block bit offsets, exclusive, [NB + 1] (kEmit)
  const uint32_t* ioff;                 // interval byte offsets, exclusive, [NI + 1] (kEmit)
  uint32_t* words;                      // the stream (kEmit)
};

// one thread per block, in warp-uniform steps so that kCount can aggregate equal symbols across the warp
template <int kMode>
__global__ void __launch_bounds__(256) jpeg_symbol_kernel(SymArgs a) {
  int lane = threadIdx.x & 31;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g - lane < a.NB;
       g += (int64_t)gridDim.x * blockDim.x) {
    bool live = g < a.NB;
    int dct = 0, act = 0;
    int diff = 0;
    const int16_t* cb = a.coef + (live ? g : 0) * 64;
    const JImg* im = nullptr;
    BlkPos P{};
    if (live) {
      P = locate(a.imgs, a.blk0, a.n, g);
      im = &a.imgs[P.img];
      if (kMode == kCount && !im->optimize) live = false;
      int tq = min(P.c, 1);
      dct = 4 * P.img + 2 * tq;
      act = dct + 1;
      // the DC predictor: the component's previous block in the interval
      int64_t pred = -1;
      if (P.slot != im->first[P.c]) pred = g - 1;
      else if (P.mcu != 0 && (im->rst == 0 || P.mcu % im->rst != 0)) pred = g - P.slot - im->bpm + im->last[P.c];
      diff = cb[0] - (pred >= 0 ? a.coef[pred * 64] : 0);
    }
    uint64_t pos = 0;
    uint32_t bits = 0;
    if (kMode == kEmit && live) {
      int64_t q = (P.mcu / (im->rst ? im->rst : (int64_t)1 << 62)) + im->int0;
      int64_t qfirst = im->blk0 + (q - im->int0) * (int64_t)(im->rst ? im->rst * im->bpm : 0);
      pos = (uint64_t)a.ioff[q] * 8 + (a.boff[g] - a.boff[qfirst]);
    }
    auto symbol = [&](int tab, int sym, uint32_t extra, int nb) {
      if (kMode == kCount) {
        uint32_t key = live ? (uint32_t)(tab * 256 + sym) : 0xffffffffu;
        unsigned peers = __match_any_sync(0xffffffffu, key);
        if (live && (__ffs(peers) - 1) == lane) atomicAdd(&a.hist[key], __popc(peers));
        return;
      }
      if (!live) return;
      uint32_t c = a.tabs[tab].code[sym];
      int cs = c >> 16;
      if (kMode == kLength) {
        bits += cs + nb;
      } else {
        put_bits(a.words, pos, ((c & 0xffff) << nb) | (extra & ((1u << nb) - 1)), cs + nb);
        pos += cs + nb;
      }
    };
    {
      int m = abs(diff), nb = nbits_of(m);
      symbol(dct, nb, (uint32_t)(diff < 0 ? diff - 1 : diff), nb);
    }
    int r = 0;
    for (int k = 1; k < 64; ++k) {
      int v = live ? cb[k] : 0;
      bool emit = v != 0;
      if (!emit) r++;
      if (kMode == kCount) {
        // runs of 16 zeros before a coefficient (ZRL) are rare: counted directly
        if (emit && live && r > 15) atomicAdd(&a.hist[act * 256 + 0xF0], r >> 4);
        int nb = nbits_of(abs(v));
        uint32_t key = emit && live ? (uint32_t)(act * 256 + ((r & 15) << 4) + nb) : 0xffffffffu;
        unsigned peers = __match_any_sync(0xffffffffu, key);
        if (key != 0xffffffffu && (__ffs(peers) - 1) == lane) atomicAdd(&a.hist[key], __popc(peers));
        if (emit) r = 0;
        continue;
      }
      if (!emit || !live) continue;
      while (r > 15) {
        symbol(act, 0xF0, 0, 0);
        r -= 16;
      }
      int nb = nbits_of(abs(v));
      symbol(act, (r << 4) + nb, (uint32_t)(v < 0 ? v - 1 : v), nb);
      r = 0;
    }
    if (kMode == kCount) {
      uint32_t key = live && r > 0 ? (uint32_t)(act * 256) : 0xffffffffu;
      unsigned peers = __match_any_sync(0xffffffffu, key);
      if (key != 0xffffffffu && (__ffs(peers) - 1) == lane) atomicAdd(&a.hist[key], __popc(peers));
      continue;
    }
    if (live && r > 0) symbol(act, 0, 0, 0);   // EOB
    if (!live) continue;
    if (kMode == kLength) {
      a.blen[g] = bits;
    } else {
      // the interval's last block pads it to a byte with 1-bits
      int64_t local_next = g + 1 - im->blk0;
      bool last = local_next == im->nblk || (im->rst && (local_next % ((int64_t)im->rst * im->bpm)) == 0);
      int pad = (int)((8 - (pos & 7)) & 7);
      if (last && pad) put_bits(a.words, pos, (1u << pad) - 1, pad);
    }
  }
}

// ---- 3. Huffman tables ---------------------------------------------------------------------------------------------
constexpr int kTableWarps = 4;

__device__ __forceinline__ uint64_t warp_min64(uint64_t v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    uint64_t u = __shfl_xor_sync(0xffffffffu, v, o);
    v = u < v ? u : v;
  }
  return v;
}

// jchuff.c jpeg_gen_optimal_table, one warp per table: the two smallest nonzero counts (ties to the larger symbol) by
// warp reductions, the merges and code-size chains by lane 0.  Counts stay below the reference's 10^9 sentinel: a call
// holds fewer than 2^31 / 418 blocks, so a table fewer than 64 * 5.2e6 symbols.
__global__ void __launch_bounds__(32 * kTableWarps) jpeg_table_kernel(const JImg* imgs, int n, const uint32_t* hist,
                                                                      HTab* tabs) {
  __shared__ uint32_t freq_s[kTableWarps][257];
  __shared__ int16_t others_s[kTableWarps][257];
  __shared__ uint8_t size_s[kTableWarps][257];
  int wl = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int w = blockIdx.x * kTableWarps + wl;
  if (w >= 4 * n) return;
  const JImg& im = imgs[w >> 2];
  int k = w & 3;
  if (im.nc == 1 && k >= 2) return;
  HTab& T = tabs[w];
  if (!im.optimize) {
    if (lane < 16) T.bits[lane] = c_std_bits[k][lane];
    int nv = (k & 1) ? 162 : 12;
    for (int s = lane; s < nv; s += 32) T.vals[s] = (k & 1) ? (k == 1 ? c_std_ac_luma[s] : c_std_ac_chroma[s]) : s;
    if (lane == 0) T.nvals = nv;
  } else {
    uint32_t* freq = freq_s[wl];
    int16_t* others = others_s[wl];
    uint8_t* codesize = size_s[wl];
    for (int s = lane; s < 257; s += 32) {
      freq[s] = s < 256 ? hist[w * 256 + s] : 1;   // the pseudo-symbol 256 keeps every code from being all ones
      others[s] = -1;
      codesize[s] = 0;
    }
    __syncwarp();
    for (;;) {
      uint64_t b1 = ~0ull;
      for (int s = lane; s < 257; s += 32)
        if (freq[s]) b1 = min(b1, (uint64_t)freq[s] << 9 | (uint64_t)(511 - s));
      b1 = warp_min64(b1);
      int c1 = 511 - (int)(b1 & 511);
      uint64_t b2 = ~0ull;
      for (int s = lane; s < 257; s += 32)
        if (freq[s] && s != c1) b2 = min(b2, (uint64_t)freq[s] << 9 | (uint64_t)(511 - s));
      b2 = warp_min64(b2);
      if (b2 == ~0ull) break;
      int c2 = 511 - (int)(b2 & 511);
      if (lane == 0) {
        freq[c1] += freq[c2];
        freq[c2] = 0;
        codesize[c1]++;
        while (others[c1] >= 0) {
          c1 = others[c1];
          codesize[c1]++;
        }
        others[c1] = (int16_t)c2;
        codesize[c2]++;
        while (others[c2] >= 0) {
          c2 = others[c2];
          codesize[c2]++;
        }
      }
      __syncwarp();
    }
    if (lane == 0) {
      int bits[33] = {0};
      for (int s = 0; s < 257; ++s)
        if (codesize[s]) bits[codesize[s]]++;
      for (int i = 32; i > 16; --i) {
        while (bits[i] > 0) {
          int j = i - 2;
          while (bits[j] == 0) j--;
          bits[i] -= 2;
          bits[i - 1]++;
          bits[j + 1] += 2;
          bits[j]--;
        }
      }
      int i = 16;
      while (bits[i] == 0) i--;
      bits[i]--;
      for (int l = 1; l <= 16; ++l) T.bits[l - 1] = (uint8_t)bits[l];
      // the symbols by code size (the sizes before the 16-bit limit), then by value
      int start[33], p = 0;
      for (int l = 1; l <= 32; ++l) {
        start[l] = p;
        for (int s = 0; s < 256; ++s) p += codesize[s] == l;
      }
      for (int s = 0; s < 256; ++s)
        if (codesize[s]) T.vals[start[codesize[s]]++] = (uint8_t)s;
      T.nvals = p;
    }
  }
  __syncwarp();
  // jpeg_make_c_derived_tbl
  for (int s = lane; s < 256; s += 32) T.code[s] = 0;
  __syncwarp();
  if (lane == 0) {
    uint32_t code = 0;
    int p = 0;
    for (int l = 1; l <= 16; ++l) {
      for (int j = 0; j < T.bits[l - 1]; ++j) T.code[T.vals[p++]] = code++ | (uint32_t)l << 16;
      code <<= 1;
    }
  }
}

// ---- 4. headers ----------------------------------------------------------------------------------------------------------
__global__ void jpeg_header_kernel(const JImg* imgs, int n, const HTab* tabs, uint8_t* file, int32_t* hdr_len) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const JImg& im = imgs[i];
  uint8_t* o = file + im.out_off;
  int p = 0;
  auto b = [&](int v) { o[p++] = (uint8_t)v; };
  auto marker = [&](int m, int len) { b(0xFF); b(m); b(len >> 8); b(len & 255); };
  b(0xFF);
  b(0xD8);
  marker(0xE0, 16);
  const uint8_t jfif[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  for (int k = 0; k < 14; ++k) b(jfif[k]);
  int ntq = im.nc == 1 ? 1 : 2;
  for (int t = 0; t < ntq; ++t) {
    marker(0xDB, 67);
    b(t);
    for (int k = 0; k < 64; ++k) b(im.qz[t][k]);
  }
  marker(0xC0, 8 + 3 * im.nc);
  b(8);
  b(im.h >> 8);
  b(im.h & 255);
  b(im.w >> 8);
  b(im.w & 255);
  b(im.nc);
  for (int c = 0; c < im.nc; ++c) {
    b(c + 1);
    b(im.hs[c] << 4 | im.vs[c]);
    b(min(c, 1));
  }
  for (int k = 0; k < 2 * ntq; ++k) {
    const HTab& T = tabs[4 * i + k];
    marker(0xC4, 2 + 1 + 16 + T.nvals);
    b((k & 1) << 4 | (k >> 1));
    for (int l = 0; l < 16; ++l) b(T.bits[l]);
    for (int s = 0; s < T.nvals; ++s) b(T.vals[s]);
  }
  if (im.rst) {
    marker(0xDD, 4);
    b(im.rst >> 8);
    b(im.rst & 255);
  }
  marker(0xDA, 6 + 2 * im.nc);
  b(im.nc);
  for (int c = 0; c < im.nc; ++c) {
    b(c + 1);
    b(c ? 0x11 : 0x00);
  }
  b(0);
  b(63);
  b(0);
  hdr_len[i] = p;
}

// ---- 5. interval lengths -------------------------------------------------------------------------------------------
struct BlkLenItem {
  const uint32_t* blen;
  __device__ uint64_t operator()(int64_t g) const { return blen[g]; }
};
struct OffOut {                        // exclusive offsets and, after the last item, the total
  uint64_t* off;
  int64_t n;
  __device__ void operator()(int64_t j, uint64_t e, uint64_t v) const {
    off[j] = e;
    if (j == n - 1) off[n] = e + v;
  }
};
struct IntBytesItem {
  const JImg* imgs;
  const int64_t* int0;
  int n;
  const uint64_t* boff;
  __device__ uint32_t operator()(int64_t q) const {
    const JImg& im = imgs[last_le(int0, n, q)];
    int64_t span = im.rst ? (int64_t)im.rst * im.bpm : im.nblk;
    int64_t b0 = im.blk0 + (q - im.int0) * span, b1 = min(b0 + span, im.blk0 + im.nblk);
    return (uint32_t)((boff[b1] - boff[b0] + 7) >> 3);
  }
};
struct Off32Out {
  uint32_t* off;
  int64_t n;
  __device__ void operator()(int64_t j, uint32_t e, uint32_t v) const {
    off[j] = e;
    if (j == n - 1) off[n] = e + v;
  }
};

// ---- 7. stuffing, markers, files -----------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t stream_byte(const uint32_t* w, int64_t j) {
  return (uint8_t)(w[j >> 2] >> (24 - 8 * (j & 3)));
}
__device__ __forceinline__ uint32_t ff_in_word(uint32_t x) {
  uint32_t c = 0;
  for (int k = 0; k < 4; ++k) c += ((x >> (8 * k)) & 0xff) == 0xff;
  return c;
}
struct FFItem {
  const uint32_t* words;
  const uint32_t* total;                // the stream's bytes: ioff[NI]
  __device__ uint32_t operator()(int64_t k) const { return 4 * k < *total ? ff_in_word(words[k]) : 0; }
};
struct FFOut {
  uint32_t* ffw;
  __device__ void operator()(int64_t k, uint32_t e, uint32_t) const { ffw[k] = e; }
};
// 0xFF bytes of the stream before byte j
__device__ __forceinline__ uint32_t ff_before(const uint32_t* ffw, const uint32_t* w, int64_t j) {
  uint32_t c = ffw[j >> 2];
  for (int64_t k = j & ~(int64_t)3; k < j; ++k) c += stream_byte(w, k) == 0xff;
  return c;
}

__global__ void jpeg_stuff_kernel(const JImg* imgs, const int64_t* int0, int n, int64_t NI, const uint32_t* ioff,
                                  const uint32_t* words, const uint32_t* ffw, const int32_t* hdr_len, uint8_t* file,
                                  int64_t* fsize, int64_t nwords) {
  const uint32_t total = ioff[NI];
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nwords; k += (int64_t)gridDim.x * blockDim.x) {
    if (4 * k >= total) return;
    for (int64_t j = 4 * k; j < 4 * k + 4 && j < total; ++j) {
      // the interval of byte j: the last one starting at or before it (intervals are never empty)
      int64_t lo = 0, hi = NI - 1;
      while (lo < hi) {
        int64_t mid = (lo + hi + 1) >> 1;
        if (ioff[mid] <= j) lo = mid; else hi = mid - 1;
      }
      int64_t q = lo;
      int i = (int)last_le(int0, n, q);
      const JImg& im = imgs[i];
      uint32_t u0 = ioff[im.int0];
      uint8_t v = stream_byte(words, j);
      int64_t p = im.out_off + hdr_len[i] + (j - u0) + (ff_before(ffw, words, j) - ff_before(ffw, words, u0)) +
                  2 * (q - im.int0);
      file[p++] = v;
      if (v == 0xFF) file[p++] = 0;
      if (j + 1 == (int64_t)ioff[q + 1]) {
        file[p] = 0xFF;
        if (q + 1 < im.int0 + im.nint) {
          file[p + 1] = (uint8_t)(0xD0 + ((q - im.int0) & 7));
        } else {
          file[p + 1] = 0xD9;
          fsize[i] = p + 2 - im.out_off;
        }
      }
    }
  }
}

__global__ void jpeg_copy_kernel(const JImg* imgs, const int64_t* unit0, int n, int64_t nunits, const uint8_t* file,
                                 const int64_t* fsize, uint8_t* out, int64_t* out_sizes) {
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < nunits; u += (int64_t)gridDim.x * blockDim.x) {
    int i = (int)last_le(unit0, n, u);
    int64_t p0 = (u - unit0[i]) * 16;
    if (p0 == 0) out_sizes[i] = fsize[i];
    if (p0 >= fsize[i]) continue;
    int64_t o = imgs[i].out_off + p0;
    *reinterpret_cast<uint4*>(out + o) = *reinterpret_cast<const uint4*>(file + o);
  }
}

}  // namespace
}  // namespace jenc
}  // namespace ctd

using namespace ctd;
using namespace ctd::jenc;

struct ctd_jpeg_encoder {
  int device = 0;
  cudaStream_t stream = nullptr;
  uint8_t* stage = nullptr;    // pinned: descriptors, then host images
  size_t stage_cap = 0;
  uint8_t* dev = nullptr;      // device scratch of one call
  size_t dev_cap = 0;
  uint8_t* out = nullptr;      // mapped pinned: the files and their sizes
  size_t out_cap = 0;
};

#define JCK(expr)                                                                                           \
  do {                                                                                                      \
    cudaError_t _e = (expr);                                                                                \
    if (_e != cudaSuccess)                                                                                  \
      return ctd_fail(nullptr, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

extern "C" CTD_API int ctd_jpeg_encoder_create(int32_t device, ctd_jpeg_encoder** out) {
  if (!out) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_encoder_create: bad argument");
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n)
    return ctd_fail(nullptr, CTD_E_NO_DEVICE, "ctd_jpeg_encoder_create: no CUDA device %d (no CPU fallback)", device);
  cudaDeviceProp prop;
  JCK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return ctd_fail(nullptr, CTD_E_NO_DEVICE, "device %d is sm_%d%d, not sm_90", device, prop.major, prop.minor);
  JCK(cudaSetDevice(device));
  ctd_jpeg_encoder* e = new ctd_jpeg_encoder;
  e->device = device;
  cudaError_t r = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
  if (r != cudaSuccess) {
    ctd_jpeg_encoder_destroy(e);
    return ctd_fail(nullptr, CTD_E_CUDA, "ctd_jpeg_encoder_create: %s", cudaGetErrorString(r));
  }
  *out = e;
  return CTD_OK;
}

extern "C" CTD_API void ctd_jpeg_encoder_destroy(ctd_jpeg_encoder* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  cudaFreeHost(e->stage);
  cudaFreeHost(e->out);
  cudaFree(e->dev);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

namespace {

enum BufKind { kPinned, kDevice, kMapped };
int grow(uint8_t** buf, size_t* cap, size_t need, BufKind kind) {
  if (*cap >= need) return CTD_OK;
  if (kind == kDevice) cudaFree(*buf); else cudaFreeHost(*buf);
  *buf = nullptr;
  *cap = 0;
  size_t n = need + need / 4;
  cudaError_t e = kind == kDevice ? cudaMalloc((void**)buf, n)
                : cudaHostAlloc((void**)buf, n, kind == kMapped ? cudaHostAllocMapped : cudaHostAllocDefault);
  if (e != cudaSuccess) return ctd_fail(nullptr, CTD_E_CUDA, "jpeg encoder: allocating %zu bytes: %s", n, cudaGetErrorString(e));
  *cap = n;
  return CTD_OK;
}

size_t al16(size_t v) { return (v + 15) & ~(size_t)15; }

struct Carve {
  size_t off = 0;
  size_t take(size_t bytes) {
    size_t o = off;
    off = (off + bytes + 255) & ~(size_t)255;
    return o;
  }
};

int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

const int kStdQ[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29,
     51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120,
     101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99}};
const int kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// jpeg_set_quality (force_baseline) and compute_reciprocal of the divisor 8 q (libjpeg-turbo jcdctmgr.c)
void quant_setup(JImg& p, int quality) {
  int q = std::min(std::max(quality, 1), 100);
  int scale = q < 50 ? 5000 / q : 200 - 2 * q;
  for (int t = 0; t < 2; ++t) {
    int tab[64];
    for (int k = 0; k < 64; ++k) tab[k] = std::min(std::max((kStdQ[t][k] * scale + 50) / 100, 1), 255);
    for (int k = 0; k < 64; ++k) p.qz[t][k] = (uint8_t)tab[kZigzag[k]];
    for (int k = 0; k < 64; ++k) {
      uint32_t d = 8u * tab[k];
      int b = 31 - __builtin_clz(d), r = 16 + b;
      uint64_t fq = ((uint64_t)1 << r) / d, fr = ((uint64_t)1 << r) % d;
      uint32_t c = d / 2;
      if (fr == 0) {
        fq >>= 1;
        r--;
      } else if (fr <= d / 2) {
        c++;
      } else {
        fq++;
      }
      p.recip[t][k] = (uint32_t)fq;
      p.corr[t][k] = c;
      p.shift[t][k] = (uint32_t)r;
    }
  }
}

}  // namespace

extern "C" CTD_API int ctd_jpeg_encode(ctd_jpeg_encoder* e, const ctd_png_image* in, const ctd_jpeg_params* prm,
                                       int32_t n, const uint8_t** files, int64_t* sizes) {
  if (!e || n < 0 || (n && (!in || !prm || !files || !sizes)))
    return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_encode: bad argument");
  if (n == 0) return CTD_OK;
  JCK(cudaSetDevice(e->device));
  // validate every image and lay out every buffer before any GPU work
  std::vector<JImg> im(n);
  std::vector<int64_t> blk0(n + 1), int0(n + 1), unit0(n + 1);
  int64_t NB = 0, NI = 0, ubytes = 0, out_bytes = 0, nunits = 0, host_bytes = 0;
  bool any_opt = false;
  for (int i = 0; i < n; ++i) {
    const ctd_png_image& s = in[i];
    const ctd_jpeg_params& P = prm[i];
    if (!s.data || s.height < 1 || s.width < 1 || (s.channels != 1 && s.channels != 3) || s.bit_depth != 8)
      return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_encode: image %d: need u8 [h][w] or [h][w][3] with h, w >= 1 "
                      "(got %dx%dx%d, %d bits)", i, s.height, s.width, s.channels, s.bit_depth);
    if (s.height > kMaxSide || s.width > kMaxSide)
      return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_encode: image %d: side above %d", i, kMaxSide);
    int hv = 0;
    switch (P.sampling) {
      case 0x411111: hv = 0x41; break;
      case 0x221111: hv = 0x22; break;
      case 0x211111: hv = 0x21; break;
      case 0x121111: hv = 0x12; break;
      case 0x111111: hv = 0x11; break;
      default: break;
    }
    if (P.quality < 0 || P.quality > 100 || !hv || P.restart_interval < 0 || P.restart_interval > 65535)
      return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_encode: image %d: quality %d, sampling 0x%x or restart interval "
                      "%d out of range", i, P.quality, P.sampling, P.restart_interval);
    if (s.on_device) {
      if (s.stride_h < 0 || s.stride_w < 0 || s.stride_c < 0)
        return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_encode: image %d: negative stride", i);
      cudaPointerAttributes a;
      if (cudaPointerGetAttributes(&a, s.data) != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != e->device) {
        cudaGetLastError();
        return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_encode: image %d is not device memory of GPU %d", i, e->device);
      }
    }
    JImg& p = im[i];
    memset(&p, 0, sizeof(JImg));
    p.h = s.height;
    p.w = s.width;
    p.nc = s.channels;
    p.optimize = P.optimize != 0;
    p.rst = P.restart_interval;
    any_opt |= p.optimize;
    // a grey image is one component at 1x1, whatever the sampling parameter
    int H = p.nc == 3 ? hv >> 4 : 1, V = p.nc == 3 ? hv & 15 : 1;
    for (int c = 0; c < p.nc; ++c) {
      p.hs[c] = c ? 1 : H;
      p.vs[c] = c ? 1 : V;
    }
    p.maxh = H;
    p.maxv = V;
    int64_t groups = cdiv(p.h, p.maxv);
    for (int c = 0; c < p.nc; ++c) {
      p.wib[c] = (int32_t)cdiv((int64_t)p.w * p.hs[c], p.maxh * 8);
      p.hib[c] = (int32_t)cdiv((int64_t)p.h * p.vs[c], p.maxv * 8);
      p.rows[c] = (int32_t)(groups * p.vs[c]);
    }
    if (p.nc == 1) {
      p.mcux = p.wib[0];
      p.mcuy = p.hib[0];
    } else {
      p.mcux = (int32_t)cdiv(p.w, p.maxh * 8);
      p.mcuy = (int32_t)cdiv(p.h, p.maxv * 8);
    }
    int slot = 0;
    for (int c = 0; c < p.nc; ++c) {
      p.first[c] = slot;
      for (int dy = 0; dy < p.vs[c]; ++dy)
        for (int dx = 0; dx < p.hs[c]; ++dx) {
          p.scomp[slot] = (int8_t)c;
          p.sdx[slot] = (int8_t)dx;
          p.sdy[slot] = (int8_t)dy;
          slot++;
        }
      p.last[c] = slot - 1;
    }
    p.bpm = slot;
    int64_t nmcu = (int64_t)p.mcux * p.mcuy;
    p.nblk = nmcu * p.bpm;
    p.nint = (int32_t)(p.rst ? cdiv(nmcu, p.rst) : 1);
    quant_setup(p, P.quality);
    p.blk0 = blk0[i] = NB;
    p.int0 = int0[i] = NI;
    NB += p.nblk;
    NI += p.nint;
    int64_t ub = cdiv(p.nblk * kBlockBitsMax, 8) + p.nint;      // the stream before stuffing, intervals padded
    ubytes += ub;
    int64_t fmax = (int64_t)al16(kHdrMax + 2 * ub + 2 * p.nint + 2);
    p.out_off = out_bytes;
    out_bytes += fmax;
    unit0[i] = nunits;
    nunits += fmax / 16;
    if (!s.on_device) host_bytes += al16((size_t)p.h * p.w * p.nc);
  }
  blk0[n] = NB;
  int0[n] = NI;
  unit0[n] = nunits;
  if (out_bytes >= (int64_t)1 << 31)
    return ctd_fail(nullptr, CTD_E_CAPACITY, "ctd_jpeg_encode: the files' bound is %lld bytes in one call (%lld blocks); "
                    "encode fewer (< 2^31 bytes, 418 per block)", (long long)out_bytes, (long long)NB);
  const int64_t nwords = ubytes / 4 + 2;
  // device scratch
  Carve c;
  size_t o_coef = c.take(128 * NB), o_blen = c.take(4 * NB), o_boff = c.take(8 * (NB + 1));
  size_t o_ioff = c.take(4 * (NI + 1)), o_words = c.take(4 * nwords), o_ffw = c.take(4 * nwords);
  size_t o_tiles = c.take(8 * (std::max(std::max(NB, NI), nwords) / kScanTile + 2));
  size_t o_hist = c.take(4 * 256 * 4 * (size_t)n), o_tabs = c.take(sizeof(HTab) * 4 * n);
  size_t o_hdr = c.take(4 * n), o_fsize = c.take(8 * n), o_file = c.take(out_bytes);
  size_t o_imgs = c.take(sizeof(JImg) * n), o_blk0 = c.take(8 * (n + 1)), o_int0 = c.take(8 * (n + 1));
  size_t o_unit0 = c.take(8 * (n + 1)), o_host = c.take(host_bytes);
  size_t meta = c.off - o_imgs;   // descriptors and host pixels: staged, then one copy
  int rc;
  if ((rc = grow(&e->dev, &e->dev_cap, c.off, kDevice))) return rc;
  if ((rc = grow(&e->stage, &e->stage_cap, meta, kPinned))) return rc;
  if ((rc = grow(&e->out, &e->out_cap, out_bytes + 8 * n + 16, kMapped))) return rc;
  uint8_t* D = e->dev;
  uint8_t* S = e->stage;
  int64_t hoff = 0;
  for (int i = 0; i < n; ++i) {
    const ctd_png_image& s = in[i];
    JImg& p = im[i];
    if (s.on_device) {
      p.src = s.data;
      p.sh = s.stride_h;
      p.sw = s.stride_w;
      p.sc = s.stride_c;
    } else {
      size_t bytes = (size_t)p.h * p.w * p.nc;
      memcpy(S + (o_host - o_imgs) + hoff, s.data, bytes);
      p.src = D + o_host + hoff;
      p.sh = (int64_t)p.w * p.nc;
      p.sw = p.nc;
      p.sc = 1;
      hoff += al16(bytes);
    }
  }
  memcpy(S, im.data(), sizeof(JImg) * n);
  memcpy(S + (o_blk0 - o_imgs), blk0.data(), 8 * (n + 1));
  memcpy(S + (o_int0 - o_imgs), int0.data(), 8 * (n + 1));
  memcpy(S + (o_unit0 - o_imgs), unit0.data(), 8 * (n + 1));
  cudaStream_t st = e->stream;
  for (int i = 0; i < n; ++i)
    if (in[i].on_device && in[i].event) JCK(cudaStreamWaitEvent(st, (cudaEvent_t)in[i].event, 0));
  JCK(cudaMemcpyAsync(D + o_imgs, S, meta, cudaMemcpyHostToDevice, st));
  if (any_opt) JCK(cudaMemsetAsync(D + o_hist, 0, 4 * 256 * 4 * (size_t)n, st));
  JCK(cudaMemsetAsync(D + o_words, 0, 4 * nwords, st));

  const JImg* dimgs = (const JImg*)(D + o_imgs);
  const int64_t* dblk0 = (const int64_t*)(D + o_blk0);
  const int64_t* dint0 = (const int64_t*)(D + o_int0);
  int16_t* coef = (int16_t*)(D + o_coef);
  uint32_t* blen = (uint32_t*)(D + o_blen);
  uint64_t* boff = (uint64_t*)(D + o_boff);
  uint32_t* ioff = (uint32_t*)(D + o_ioff);
  uint32_t* words = (uint32_t*)(D + o_words);
  uint32_t* ffw = (uint32_t*)(D + o_ffw);
  uint32_t* hist = (uint32_t*)(D + o_hist);
  HTab* tabs = (HTab*)(D + o_tabs);
  int32_t* hdr_len = (int32_t*)(D + o_hdr);
  int64_t* fsize = (int64_t*)(D + o_fsize);
  uint8_t* file = D + o_file;
  uint8_t* dout = nullptr;                 // the mapped output as the kernels address it
  JCK(cudaHostGetDevicePointer((void**)&dout, e->out, 0));
  int64_t* dsizes = (int64_t*)(dout + al16(out_bytes));
  const int64_t* hsizes = (const int64_t*)(e->out + al16(out_bytes));
  const int kT = 256;
  auto grid = [](int64_t items, int threads) { return (unsigned)std::min<int64_t>(cdiv(items, threads), 132 * 16); };

  SymArgs a{dimgs, dblk0, dint0, n, NB, coef, hist, tabs, blen, boff, ioff, words};
  jpeg_block_kernel<<<(unsigned)cdiv(NB, kBlocksPerCta), 64 * kBlocksPerCta, 0, st>>>(dimgs, dblk0, n, NB, coef);
  if (any_opt) jpeg_symbol_kernel<kCount><<<grid(NB, kT), kT, 0, st>>>(a);
  jpeg_table_kernel<<<(unsigned)cdiv(4 * n, kTableWarps), 32 * kTableWarps, 0, st>>>(dimgs, n, hist, tabs);
  jpeg_header_kernel<<<(unsigned)cdiv(n, 64), 64, 0, st>>>(dimgs, n, tabs, file, hdr_len);
  jpeg_symbol_kernel<kLength><<<grid(NB, kT), kT, 0, st>>>(a);
  run_scan<uint64_t>(NB, BlkLenItem{blen}, OffOut{boff, NB}, (uint64_t*)(D + o_tiles), st);
  run_scan<uint32_t>(NI, IntBytesItem{dimgs, dint0, n, boff}, Off32Out{ioff, NI}, (uint32_t*)(D + o_tiles), st);
  jpeg_symbol_kernel<kEmit><<<grid(NB, kT), kT, 0, st>>>(a);
  run_scan<uint32_t>(nwords, FFItem{words, ioff + NI}, FFOut{ffw}, (uint32_t*)(D + o_tiles), st);
  jpeg_stuff_kernel<<<grid(nwords, kT), kT, 0, st>>>(dimgs, dint0, n, NI, ioff, words, ffw, hdr_len, file, fsize,
                                                     nwords);
  jpeg_copy_kernel<<<grid(nunits, kT), kT, 0, st>>>(dimgs, (const int64_t*)(D + o_unit0), n, nunits, file, fsize, dout,
                                                    dsizes);
  JCK(cudaGetLastError());
  JCK(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    files[i] = e->out + im[i].out_off;
    sizes[i] = hsizes[i];
  }
  return CTD_OK;
}
