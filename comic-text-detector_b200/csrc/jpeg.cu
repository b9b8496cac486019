// GPU JPEG decode (C ABI `ctd_jpeg_decoder_*`, `ctd_jpeg_decode`, include/ctd_b200.h): every page of a call at once,
// byte for byte the u8 BGR page cv2.imdecode(buf, IMREAD_COLOR) returns with its libjpeg-turbo.
//
// Stages, each one launch over all pages:
//   1. jpeg_sync_kernel, in rounds: Huffman decode by self-synchronisation.  Each restart interval's bits are cut into
//      subsequences of `sub_bits` bits.  A decoder state is (bit offset of the next codeword, block index in the MCU,
//      zig-zag index k).  The first subsequence of an interval starts from the exact state (0, 0, 0), every other one
//      from a guess (its first bit, 0, 0).  A round decodes every subsequence from its start state up to the first
//      codeword that starts past its end and stores that end state as the next subsequence's start.  Rounds repeat
//      until no start state changes; then every start state is exact, by induction from the interval's start (the
//      worst case is serial, one subsequence per round, and still ends).  A round also counts the blocks each
//      subsequence completes, sums its DC differences per component and notes whether it met an invalid code or a run
//      past coefficient 63.  Such an error ends the block and decoding goes on (an error state that stopped the
//      decode would keep a wrongly guessed subsequence from ever falling into step): the error only counts at the
//      fixpoint, where every start is exact.  Rounds run in bounded groups per
//      host check of a device "changed" flag: no cooperative launch.
//   2. jpeg_scan_kernel (one CTA per page): exclusive scan of the block counts (each subsequence's first block) and a
//      per-component prefix sum of the DC differences that restarts at every interval (each subsequence's DC
//      predictors).  It checks that every interval decodes to exactly its MCUs, ends on an MCU boundary with fewer
//      than 8 bits left, and that no subsequence met an error; otherwise the page is CTD_JPEG_ENTROPY.
//   3. jpeg_write_kernel: each subsequence decoded once more from its exact state, coefficients written de-zig-zagged
//      into a zeroed int16 [block][64] buffer in MCU order, DC as absolute values (32-bit sums stored as int16, as
//      libjpeg's JCOEF).
//   4. jpeg_idct_kernel: dequantisation and jidctint.c's jpeg_idct_islow (13-bit constants, PASS1_BITS 2) into
//      per-component u8 planes, through the post-IDCT range-limit table.  libjpeg-turbo's SIMD IDCT (what cv2 runs)
//      works in 16-bit lanes and saturates where the C table wraps; they agree while dequantised coefficients and
//      pass-1 values stay within +-16383 and outputs within [-512, 511].  A block outside that marks its page
//      CTD_JPEG_RANGE, and the page goes to cv2.  Real encoders stay far inside.
//   5. jpeg_color_kernel: jdsample.c's fancy h2v1 / h2v2 upsampling (box filter for chroma at most 2 samples wide, as
//      jinit_upsampler chooses), jdcolor.c's YCbCr->RGB tables, stored as BGR at the pixel's EXIF-oriented position in
//      the caller's page.
// oracle/jpeg_ref.py restates every rule in numpy; tests/test_cpu_jpeg.py pins it to cv2.imdecode.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "jpeg.h"

int ctd_fail(ctd_handle* h, int code, const char* fmt, ...);

namespace ctd {
namespace jpeg {
namespace {

constexpr int kDefaultSubBits = 1024;   // the fastest of 1024..16384 on an H100 (DESIGN §7.9)
constexpr int kRoundsPerCheck = 8;

struct DPage {
  int32_t w, h, ncomp, mcux, bpm, orient, out_w, out_h, hmax, vmax;
  int32_t nmcu, restart;                 // restart: MCUs per interval (nmcu without DRI)
  int32_t blk_comp[6], blk_dx[6], blk_dy[6];
  int32_t tab_dc[3], tab_ac[3], quant[3], ch[3], cv[3], plane_w[3];
  int32_t first_iv, n_iv, first_sub, n_sub;
  int64_t coef_blk, nblocks;             // first block in the coefficient buffer, block count
  int64_t plane_off[3];
  uint8_t* dst;
};

struct DInterval {
  int64_t byte;                          // first byte in the staged bits
  int32_t bits, first_sub, n_sub, page, first_mcu;
};

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

__device__ __forceinline__ uint64_t pack(uint32_t pos, int blk, int k) {
  return pos | ((uint64_t)blk << 32) | ((uint64_t)k << 40);
}

// 32 bits of the stream from bit `pos` (the staging buffer has slack past its last byte)
__device__ __forceinline__ uint32_t peek32(const uint8_t* b, uint32_t pos) {
  const uint8_t* p = b + (pos >> 3);
  uint32_t w = ((uint32_t)__ldg(p) << 24) | ((uint32_t)__ldg(p + 1) << 16) | ((uint32_t)__ldg(p + 2) << 8) | __ldg(p + 3);
  int s = pos & 7;
  return s ? (w << s) | (__ldg(p + 4) >> (8 - s)) : w;
}

// one Huffman symbol from the window x: its code length (0: invalid) and value
__device__ __forceinline__ int huff(const HuffTable* __restrict__ t, uint32_t x, int* sym) {
  uint32_t e = t->lut[x >> (32 - kLutBits)];
  if (e) {
    *sym = e & 0xff;
    return e >> 8;
  }
  for (int L = kLutBits + 1; L <= 16; ++L) {
    int code = (int)(x >> (32 - L));
    if (code <= t->maxcode[L]) {
      *sym = t->vals[(code + t->valoff[L]) & 0xff];
      return L;
    }
  }
  return 0;
}

// Decodes from state st until the next codeword starts at or past `stop` (or does not fit in the interval's `nbits`).
// Counts completed blocks and sums DC differences per component; with WRITE, also stores coefficients of the blocks
// from `blk_index` on, DC as the running predictor dc[].  An invalid code (1 bit consumed) or a run past coefficient 63
// sets *err and ends the block: decoding goes on, so that a subsequence started from a wrong guess can still fall into
// step with the true codeword boundaries; from an exact start, *err means the data is not clean.
template <bool WRITE>
__device__ uint64_t run(const DPage& pg, const HuffTable* __restrict__ tabs, const uint8_t* bits, uint32_t nbits,
                        uint32_t stop, uint64_t st, int* count, int* err, int dc[3], int16_t* coef,
                        int64_t blk_index) {
  uint32_t pos = (uint32_t)st;
  int blk = (int)((st >> 32) & 0xff), k = (int)((st >> 40) & 0xff);
  int cnt = 0, bad = 0;
  while (pos < stop) {
    uint32_t x = peek32(bits, pos);
    int c = pg.blk_comp[blk];
    int sym;
    int len = huff(tabs + (k == 0 ? pg.tab_dc[c] : pg.tab_ac[c]), x, &sym);
    if (!len) {
      if (pos + 16 > nbits) break;   // the lookup read past the interval: its end, not an error
      bad = 1;
      pos += 1;
      k = 64;
      sym = 0;
    }
    int s = !len ? 0 : k == 0 ? sym : (sym & 15);
    if (pos + len + s > nbits) break;
    int v = 0;
    if (s) {
      uint32_t r = (x << len) >> (32 - s);
      v = r < (1u << (s - 1)) ? (int)r - (1 << s) + 1 : (int)r;
    }
    pos += len + s;
    if (!len) {
      // an invalid code: the block ends here
    } else if (k == 0) {
      dc[c] = (int)((uint32_t)dc[c] + (uint32_t)v);
      if (WRITE) coef[blk_index * 64] = (int16_t)dc[c];
      k = 1;
    } else {
      int r = sym >> 4;
      if (s) {
        k += r;
        if (k > 63) {
          bad = 1;
          k = 64;
        } else {
          if (WRITE) coef[blk_index * 64 + c_zigzag[k]] = (int16_t)v;
          ++k;
        }
      } else if (r == 15) {
        k += 16;
        if (k > 64) {
          bad = 1;
          k = 64;
        }
      } else {
        k = 64;
      }
    }
    if (k == 64) {
      k = 0;
      ++cnt;
      ++blk_index;
      if (++blk == pg.bpm) blk = 0;
    }
  }
  *count = cnt;
  *err = bad;
  return pack(pos, blk, k);
}

struct Scratch {
  uint64_t* start;   // [n_sub] start state of each subsequence
  uint64_t* iend;    // [n_iv] end state of each interval's last subsequence
  int32_t* cnt;      // [n_sub] blocks completed
  int32_t* err;      // [n_sub] an invalid code or a run past coefficient 63 met
  int32_t* dcp;      // [n_sub][3] DC difference sums
  int32_t* blk0;     // [n_sub] first block (within the page)
  int32_t* dc0;      // [n_sub][3] DC predictors at the start
};

__global__ void jpeg_sync_kernel(const DPage* __restrict__ pages, const DInterval* __restrict__ ivs,
                                 const int32_t* __restrict__ sub_iv, const HuffTable* __restrict__ tabs,
                                 const uint8_t* __restrict__ bits, Scratch sc, int n_sub, int sub_bits,
                                 int* __restrict__ changed) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_sub) return;
  const DInterval I = ivs[sub_iv[j]];
  const DPage& pg = pages[I.page];
  int local = j - I.first_sub;
  bool last = local + 1 == I.n_sub;
  uint32_t stop = last ? (uint32_t)I.bits : (uint32_t)(local + 1) * (uint32_t)sub_bits;
  uint64_t st = local ? *(volatile uint64_t*)&sc.start[j] : 0ull;
  int dc[3] = {0, 0, 0}, cnt = 0, err = 0;
  uint64_t end = run<false>(pg, tabs, bits + I.byte, (uint32_t)I.bits, stop, st, &cnt, &err, dc, nullptr, 0);
  sc.cnt[j] = cnt;
  sc.err[j] = err;
  for (int c = 0; c < 3; ++c) sc.dcp[j * 3 + c] = dc[c];
  if (last) {
    sc.iend[sub_iv[j]] = end;
  } else if (*(volatile uint64_t*)&sc.start[j + 1] != end) {
    *(volatile uint64_t*)&sc.start[j + 1] = end;
    *changed = 1;
  }
}

// one CTA of 1024 threads per page
__global__ void __launch_bounds__(1024) jpeg_scan_kernel(const DPage* __restrict__ pages,
                                                         const DInterval* __restrict__ ivs, Scratch sc,
                                                         int32_t* __restrict__ status) {
  const DPage& pg = pages[blockIdx.x];
  __shared__ int s_cnt[1024], s_dc[3][1024], s_flag[1024];
  __shared__ int carry_cnt, carry_dc[3], bad;
  int t = threadIdx.x;
  if (t == 0) {
    carry_cnt = 0;
    carry_dc[0] = carry_dc[1] = carry_dc[2] = 0;
    bad = 0;
  }
  __syncthreads();   // the end checks below may set `bad` from any thread
  // per-interval end checks
  for (int i = t; i < pg.n_iv; i += blockDim.x) {
    const DInterval& I = ivs[pg.first_iv + i];
    uint64_t e = sc.iend[pg.first_iv + i];
    uint32_t pos = (uint32_t)e;
    if ((e >> 32) != 0 || pos > (uint32_t)I.bits || (uint32_t)I.bits - pos >= 8) bad = 1;
  }
  __syncthreads();
  for (int base = 0; base < pg.n_sub; base += blockDim.x) {
    int j = pg.first_sub + base + t;
    bool in = base + t < pg.n_sub;
    int cnt = in ? sc.cnt[j] : 0;
    if (in && sc.err[j]) bad = 1;
    int dc[3];
    for (int c = 0; c < 3; ++c) dc[c] = in ? sc.dcp[j * 3 + c] : 0;
    // a subsequence that starts an interval resets the DC predictors
    int first = 0, iv_first_mcu = 0;
    if (in) {
      // the interval of subsequence j: found through the page's intervals (binary search on first_sub)
      int lo = pg.first_iv, hi = pg.first_iv + pg.n_iv - 1;
      while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (ivs[mid].first_sub <= j) lo = mid; else hi = mid - 1;
      }
      first = ivs[lo].first_sub == j;
      iv_first_mcu = ivs[lo].first_mcu;
    }
    s_cnt[t] = cnt;
    s_flag[t] = first;
    for (int c = 0; c < 3; ++c) s_dc[c][t] = dc[c];
    __syncthreads();
    // inclusive Hillis-Steele scans: plain for the counts, segmented at interval starts for the DC sums
    for (int off = 1; off < blockDim.x; off <<= 1) {
      int a = 0, f = 0, d[3] = {0, 0, 0};
      if (t >= off) {
        a = s_cnt[t - off];
        f = s_flag[t - off];
        for (int c = 0; c < 3; ++c) d[c] = s_dc[c][t - off];
      }
      __syncthreads();
      if (t >= off) {
        s_cnt[t] += a;
        if (!s_flag[t]) {
          for (int c = 0; c < 3; ++c) s_dc[c][t] = (int)((uint32_t)s_dc[c][t] + (uint32_t)d[c]);
          s_flag[t] = f;
        }
      }
      __syncthreads();
    }
    if (in) {
      int ex_cnt = carry_cnt + s_cnt[t] - cnt;
      sc.blk0[j] = ex_cnt;
      if (first && (int64_t)ex_cnt != (int64_t)iv_first_mcu * pg.bpm) atomicExch(&bad, 1);
      // exclusive DC predictors: 0 at an interval's first subsequence; the chunk's carry only where no interval
      // starts between the chunk's first subsequence and this one
      for (int c = 0; c < 3; ++c) {
        int ex = (int)((uint32_t)s_dc[c][t] - (uint32_t)dc[c]);
        if (first) ex = 0;
        else if (!s_flag[t]) ex = (int)((uint32_t)ex + (uint32_t)carry_dc[c]);
        sc.dc0[j * 3 + c] = ex;
      }
    }
    __syncthreads();
    if (t == blockDim.x - 1) {
      carry_cnt += s_cnt[t];
      for (int c = 0; c < 3; ++c)
        carry_dc[c] = s_flag[t] ? s_dc[c][t] : (int)((uint32_t)carry_dc[c] + (uint32_t)s_dc[c][t]);
    }
    __syncthreads();
  }
  if (t == 0 && ((int64_t)carry_cnt != pg.nblocks || bad)) status[blockIdx.x] = CTD_JPEG_ENTROPY;
}

__global__ void jpeg_write_kernel(const DPage* __restrict__ pages, const DInterval* __restrict__ ivs,
                                  const int32_t* __restrict__ sub_iv, const HuffTable* __restrict__ tabs,
                                  const uint8_t* __restrict__ bits, Scratch sc, int n_sub, int sub_bits,
                                  const int32_t* __restrict__ status, int16_t* __restrict__ coef) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_sub) return;
  const DInterval I = ivs[sub_iv[j]];
  if (status[I.page]) return;
  const DPage& pg = pages[I.page];
  int local = j - I.first_sub;
  uint32_t stop = local + 1 == I.n_sub ? (uint32_t)I.bits : (uint32_t)(local + 1) * (uint32_t)sub_bits;
  uint64_t st = local ? sc.start[j] : 0ull;
  int dc[3] = {sc.dc0[j * 3], sc.dc0[j * 3 + 1], sc.dc0[j * 3 + 2]}, cnt, err;
  run<true>(pg, tabs, bits + I.byte, (uint32_t)I.bits, stop, st, &cnt, &err, dc, coef, pg.coef_blk + sc.blk0[j]);
}

__device__ __forceinline__ int descale(int64_t x, int n) { return (int)((x + (1ll << (n - 1))) >> n); }

// one jpeg_idct_islow pass over 8 values (64-bit products: overflow-free for any int16 x 16-bit quantiser input)
__device__ __forceinline__ void idct8(const int64_t* v, int shift, int* o) {
  int64_t z2 = v[2], z3 = v[6];
  int64_t z1 = (z2 + z3) * 4433;
  int64_t tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
  int64_t tmp0 = (v[0] + v[4]) * 8192, tmp1 = (v[0] - v[4]) * 8192;
  int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int64_t a0 = v[7], a1 = v[5], a2 = v[3], a3 = v[1];
  int64_t y1 = a0 + a3, y2 = a1 + a2, y3 = a0 + a2, y4 = a1 + a3;
  int64_t z5 = (y3 + y4) * 9633;
  a0 *= 2446;
  a1 *= 16819;
  a2 *= 25172;
  a3 *= 12299;
  y1 *= -7373;
  y2 *= -20995;
  y3 = y3 * -16069 + z5;
  y4 = y4 * -3196 + z5;
  a0 += y1 + y3;
  a1 += y2 + y4;
  a2 += y2 + y3;
  a3 += y1 + y4;
  o[0] = descale(t10 + a3, shift);
  o[7] = descale(t10 - a3, shift);
  o[1] = descale(t11 + a2, shift);
  o[6] = descale(t11 - a2, shift);
  o[2] = descale(t12 + a1, shift);
  o[5] = descale(t12 - a1, shift);
  o[3] = descale(t13 + a0, shift);
  o[4] = descale(t13 - a0, shift);
}

// the post-IDCT range limit of jdmaster.c prepare_range_limit_table, indexed with x & 1023
__device__ __forceinline__ uint32_t range_limit(int x) {
  int i = x & 1023;
  return i < 128 ? i + 128 : i < 512 ? 255 : i < 896 ? 0 : i - 896;
}

constexpr int kIdctBlocks = 32;   // blocks per CTA, 8 threads per block

// grid (ceil(max blocks / kIdctBlocks), pages)
__global__ void __launch_bounds__(256) jpeg_idct_kernel(const DPage* __restrict__ pages,
                                                        const int32_t* __restrict__ quant,
                                                        const int16_t* __restrict__ coef, uint8_t* __restrict__ planes,
                                                        int32_t* __restrict__ status) {
  const DPage& pg = pages[blockIdx.y];
  __shared__ int s_in[kIdctBlocks][8][9];
  __shared__ int s_ws[kIdctBlocks][8][9];
  int lb = threadIdx.x >> 3, t = threadIdx.x & 7;
  int64_t b = (int64_t)blockIdx.x * kIdctBlocks + lb;
  bool live = b < pg.nblocks && status[blockIdx.y] == 0;
  int m = 0, r = 0, c = 0;
  bool ok = true;
  if (live) {
    m = (int)(b / pg.bpm);
    r = (int)(b - (int64_t)m * pg.bpm);
    c = pg.blk_comp[r];
    const int32_t* q = quant + pg.quant[c] * 64 + t * 8;
    int4 raw = *reinterpret_cast<const int4*>(coef + (pg.coef_blk + b) * 64 + t * 8);
    const int16_t* v = reinterpret_cast<const int16_t*>(&raw);
    for (int u = 0; u < 8; ++u) {
      int d = v[u] * q[u];
      ok &= d >= -16383 && d <= 16383;
      s_in[lb][t][u] = d;
    }
  }
  __syncthreads();
  if (live) {   // column t
    int64_t col[8];
    int o[8];
    for (int y = 0; y < 8; ++y) col[y] = s_in[lb][y][t];
    idct8(col, 11, o);
    for (int y = 0; y < 8; ++y) {
      ok &= o[y] >= -16383 && o[y] <= 16383;
      s_ws[lb][y][t] = o[y];
    }
  }
  __syncthreads();
  if (!live) return;
  int64_t row[8];
  int o[8];
  for (int x = 0; x < 8; ++x) row[x] = s_ws[lb][t][x];
  idct8(row, 18, o);
  uint32_t lo = 0, hi = 0;
  for (int x = 0; x < 8; ++x) {
    ok &= o[x] >= -512 && o[x] <= 511;
    uint32_t px = range_limit(o[x]);
    if (x < 4) lo |= px << (8 * x); else hi |= px << (8 * (x - 4));
  }
  if (!ok) atomicCAS(&status[blockIdx.y], 0, CTD_JPEG_RANGE);
  int mx = m % pg.mcux, my = m / pg.mcux;
  int px = (mx * pg.ch[c] + pg.blk_dx[r]) * 8, py = (my * pg.cv[c] + pg.blk_dy[r]) * 8 + t;
  *reinterpret_cast<uint2*>(planes + pg.plane_off[c] + (int64_t)py * pg.plane_w[c] + px) = make_uint2(lo, hi);
}

// jdcolor.c build_ycc_rgb_table
__device__ __forceinline__ void ycc_bgr(int y, int cb, int cr, uint8_t* o) {
  int x = cr - 128, z = cb - 128;
  int r = y + (int)((91881ll * x + 32768) >> 16);
  int g = y + (int)((-46802ll * x + -22554ll * z + 32768) >> 16);
  int b = y + (int)((116130ll * z + 32768) >> 16);
  o[0] = (uint8_t)min(max(b, 0), 255);
  o[1] = (uint8_t)min(max(g, 0), 255);
  o[2] = (uint8_t)min(max(r, 0), 255);
}

// jdsample.c: one chroma sample of output pixel (x, y); C: the plane, cw x chh real samples, row stride pw (64-bit: a
// 65535-row plane is past 2^31 bytes)
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ C, int64_t pw, int cw, int chh, int hf, int vf, int x,
                                      int y) {
  if (hf == 1) return C[y * pw + x];   // 4:4:4
  int i = x >> 1;
  if (cw <= 2) return C[(vf == 2 ? y >> 1 : y) * pw + i];   // box filter (jinit_upsampler)
  bool odd = x & 1;
  int in = odd ? min(i + 1, cw - 1) : max(i - 1, 0);
  if (vf == 1) {
    const uint8_t* row = C + y * pw;
    return (3 * row[i] + row[in] + (odd ? 2 : 1)) >> 2;
  }
  int j = y >> 1;
  int jn = (y & 1) ? min(j + 1, chh - 1) : max(j - 1, 0);
  const uint8_t* r0 = C + j * pw;
  const uint8_t* r1 = C + jn * pw;
  int cs = 3 * r0[i] + r1[i], cn = 3 * r0[in] + r1[in];
  return (3 * cs + cn + (odd ? 7 : 8)) >> 4;
}

// grid (ceil(max pixels / 256), pages): one thread per frame pixel
__global__ void __launch_bounds__(256) jpeg_color_kernel(const DPage* __restrict__ pages,
                                                         const uint8_t* __restrict__ planes,
                                                         const int32_t* __restrict__ status) {
  const DPage& pg = pages[blockIdx.y];
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)pg.w * pg.h || status[blockIdx.y]) return;
  int y = (int)(i / pg.w), x = (int)(i - (int64_t)y * pg.w);
  int Y = planes[pg.plane_off[0] + (int64_t)y * pg.plane_w[0] + x];
  uint8_t o[3];
  if (pg.ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
  } else {
    int cw = (pg.w + pg.hmax - 1) / pg.hmax, chh = (pg.h + pg.vmax - 1) / pg.vmax;
    int cb = chroma(planes + pg.plane_off[1], pg.plane_w[1], cw, chh, pg.hmax, pg.vmax, x, y);
    int cr = chroma(planes + pg.plane_off[2], pg.plane_w[2], cw, chh, pg.hmax, pg.vmax, x, y);
    ycc_bgr(Y, cb, cr, o);
  }
  // OpenCV ExifTransform: transpose for 5..8, then flip (1: columns, 0: rows, -1: both)
  int orow = y, ocol = x;
  int ot = pg.orient;
  if (ot >= 5) {
    orow = x;
    ocol = y;
  }
  bool fc = ot == 2 || ot == 3 || ot == 6 || ot == 7, fr = ot == 3 || ot == 4 || ot == 7 || ot == 8;
  if (fc) ocol = pg.out_w - 1 - ocol;
  if (fr) orow = pg.out_h - 1 - orow;
  uint8_t* d = pg.dst + ((int64_t)orow * pg.out_w + ocol) * 3;
  d[0] = o[0];
  d[1] = o[1];
  d[2] = o[2];
}

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace
}  // namespace jpeg
}  // namespace ctd

using namespace ctd::jpeg;

struct ctd_jpeg_decoder {
  int device = 0, sub_bits = kDefaultSubBits;
  cudaStream_t stream = nullptr;
  uint8_t* host = nullptr;   // pinned staging: descriptors, tables and bits of one call
  size_t host_cap = 0;
  uint8_t* dev = nullptr;    // its device mirror
  size_t dev_cap = 0;
  uint8_t* work = nullptr;   // scratch, coefficients and planes
  size_t work_cap = 0;
  int* flags = nullptr;      // pinned copy of the rounds' changed flags
};

#define JCK(expr)                                                                                           \
  do {                                                                                                      \
    cudaError_t _e = (expr);                                                                                \
    if (_e != cudaSuccess)                                                                                  \
      return ctd_fail(nullptr, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

extern "C" CTD_API int ctd_jpeg_decoder_create(int32_t device, int32_t subsequence_bits, ctd_jpeg_decoder** out) {
  if (!out || subsequence_bits < 0) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_decoder_create: bad argument");
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n)
    return ctd_fail(nullptr, CTD_E_NO_DEVICE, "ctd_jpeg_decoder_create: no CUDA device %d (no CPU fallback)", device);
  cudaDeviceProp prop;
  JCK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return ctd_fail(nullptr, CTD_E_NO_DEVICE, "device %d is sm_%d%d, not sm_90", device, prop.major, prop.minor);
  JCK(cudaSetDevice(device));
  ctd_jpeg_decoder* d = new ctd_jpeg_decoder;
  d->device = device;
  if (subsequence_bits) d->sub_bits = subsequence_bits;
  cudaError_t e = cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&d->flags, kRoundsPerCheck * sizeof(int));
  if (e != cudaSuccess) {
    ctd_jpeg_decoder_destroy(d);
    return ctd_fail(nullptr, CTD_E_CUDA, "ctd_jpeg_decoder_create: %s", cudaGetErrorString(e));
  }
  *out = d;
  return CTD_OK;
}

extern "C" CTD_API void ctd_jpeg_decoder_destroy(ctd_jpeg_decoder* d) {
  if (!d) return;
  cudaSetDevice(d->device);
  if (d->stream) cudaStreamSynchronize(d->stream);
  cudaFreeHost(d->host);
  cudaFreeHost(d->flags);
  cudaFree(d->dev);
  cudaFree(d->work);
  if (d->stream) cudaStreamDestroy(d->stream);
  delete d;
}

namespace {

// grows a pinned or device buffer to at least `need` bytes (by a quarter more, as the engine's pinned buffers grow)
int grow(uint8_t** buf, size_t* cap, size_t need, bool pinned) {
  if (*cap >= need) return CTD_OK;
  if (pinned) cudaFreeHost(*buf); else cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  size_t n = need + need / 4;
  cudaError_t e = pinned ? cudaMallocHost((void**)buf, n) : cudaMalloc((void**)buf, n);
  if (e != cudaSuccess) return ctd_fail(nullptr, CTD_E_CUDA, "jpeg decoder: allocating %zu bytes: %s", n, cudaGetErrorString(e));
  *cap = n;
  return CTD_OK;
}

}  // namespace

extern "C" CTD_API int ctd_jpeg_decode(ctd_jpeg_decoder* d, const uint8_t* const* data, const size_t* len, int32_t n,
                                       uint8_t* const* dst, int32_t* status) {
  if (!d || n < 0 || (n && (!data || !len || !dst || !status)))
    return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_decode: bad argument");
  JCK(cudaSetDevice(d->device));
  // 1. host: parse every file, lay out the call
  std::vector<Frame> frames(n);
  std::vector<int> live;   // indices of the files the GPU decodes
  for (int i = 0; i < n; ++i) {
    status[i] = data[i] ? parse(data[i], len[i], &frames[i]) : CTD_JPEG_NOT_JPEG;
    if (status[i] == CTD_JPEG_OK) {
      if (!dst[i]) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_jpeg_decode: file %d decodes but dst[%d] is NULL", i, i);
      live.push_back(i);
    }
  }
  if (live.empty()) return CTD_OK;
  const int S = d->sub_bits;
  int np = (int)live.size();
  int64_t n_iv = 0, n_sub = 0, n_tab = 0, bits_bytes = 0;
  int64_t max_blocks = 0, max_px = 0;
  for (int i : live) {
    const Frame& f = frames[i];
    n_iv += f.n_intervals;
    n_tab += (int64_t)f.tables.size();
    int64_t ecs = (int64_t)(f.scan_end - f.scan_begin);
    bits_bytes += align_up(ecs, 16);
    // subsequences per interval are not known before staging; bound them by the scan's bits
    n_sub += f.n_intervals + ecs * 8 / S;
    int64_t bpm = 0;
    for (int c = 0; c < f.ncomp; ++c) bpm += f.ch[c] * f.cv[c];
    int64_t nb = bpm * f.mcux * f.mcuy;
    max_blocks = std::max(max_blocks, nb);
    max_px = std::max(max_px, (int64_t)f.w * f.h);
  }
  // subsequences are indexed with int32 (and launched one thread each)
  if (n_sub > INT32_MAX / 2)
    return ctd_fail(nullptr, CTD_E_CAPACITY, "ctd_jpeg_decode: %lld subsequences of %d bits in one call; decode fewer "
                    "files per call or use longer subsequences", (long long)n_sub, S);
  size_t o_pages = 0;
  size_t o_ivs = align_up(o_pages + np * sizeof(DPage), 256);
  size_t o_subiv = align_up(o_ivs + n_iv * sizeof(DInterval), 256);
  size_t o_start = align_up(o_subiv + n_sub * sizeof(int32_t), 256);
  size_t o_tabs = align_up(o_start + n_sub * sizeof(uint64_t), 256);
  size_t o_quant = align_up(o_tabs + n_tab * sizeof(HuffTable), 256);
  size_t o_status = align_up(o_quant + (size_t)np * 3 * 64 * sizeof(int32_t), 256);
  size_t o_bits = align_up(o_status + np * sizeof(int32_t), 256);
  size_t host_bytes = align_up(o_bits + bits_bytes + 16, 256);
  int rc = grow(&d->host, &d->host_cap, host_bytes, true);
  if (rc) return rc;
  uint8_t* H = d->host;
  DPage* pages = (DPage*)(H + o_pages);
  DInterval* ivs = (DInterval*)(H + o_ivs);
  int32_t* sub_iv = (int32_t*)(H + o_subiv);
  uint64_t* start = (uint64_t*)(H + o_start);
  HuffTable* tabs = (HuffTable*)(H + o_tabs);
  int32_t* quant = (int32_t*)(H + o_quant);
  int32_t* dstatus = (int32_t*)(H + o_status);
  uint8_t* bits = H + o_bits;
  // 2. host: stage every scan, fill the descriptors
  std::vector<int64_t> ib;
  std::vector<int32_t> ibits;
  int64_t iv = 0, sub = 0, tab = 0, blk = 0, plane = 0, boff = 0;
  for (int p = 0; p < np; ++p) {
    const Frame& f = frames[live[p]];
    DPage& g = pages[p];
    memset(&g, 0, sizeof(g));
    g.w = f.w;
    g.h = f.h;
    g.ncomp = f.ncomp;
    g.hmax = f.hmax;
    g.vmax = f.vmax;
    g.orient = f.orient;
    g.out_w = f.orient >= 5 ? f.h : f.w;
    g.out_h = f.orient >= 5 ? f.w : f.h;
    g.mcux = f.mcux;
    int mcuy = f.mcuy;
    g.nmcu = g.mcux * mcuy;
    g.restart = f.restart ? f.restart : g.nmcu;
    int r = 0;
    for (int c = 0; c < f.ncomp; ++c) {
      g.ch[c] = f.ch[c];
      g.cv[c] = f.cv[c];
      for (int by = 0; by < f.cv[c]; ++by)
        for (int bx = 0; bx < f.ch[c]; ++bx, ++r) {
          g.blk_comp[r] = c;
          g.blk_dx[r] = bx;
          g.blk_dy[r] = by;
        }
      g.tab_dc[c] = (int32_t)(tab + f.dc[c]);
      g.tab_ac[c] = (int32_t)(tab + f.ac[c]);
      g.quant[c] = p * 3 + c;
      memcpy(quant + (p * 3 + c) * 64, f.quant[f.q[c]], 64 * sizeof(int32_t));
      g.plane_w[c] = g.mcux * f.ch[c] * 8;
      g.plane_off[c] = plane;
      plane += align_up((int64_t)g.plane_w[c] * mcuy * f.cv[c] * 8, 256);
    }
    g.bpm = r;
    g.nblocks = (int64_t)g.bpm * g.nmcu;
    g.coef_blk = blk;
    blk += g.nblocks;
    g.dst = dst[live[p]];
    for (size_t t = 0; t < f.tables.size(); ++t) tabs[tab + t] = f.tables[t];
    tab += (int64_t)f.tables.size();
    ib.assign(f.n_intervals + 1, 0);
    ibits.assign(f.n_intervals, 0);
    size_t nbytes = stage(data[live[p]], f, bits + boff, ib.data(), ibits.data());
    g.first_iv = (int32_t)iv;
    g.n_iv = f.n_intervals;
    g.first_sub = (int32_t)sub;
    for (int k = 0; k < f.n_intervals; ++k) {
      DInterval& I = ivs[iv + k];
      I.byte = boff + ib[k];
      I.bits = ibits[k];
      I.page = p;
      I.first_mcu = k * g.restart;
      I.first_sub = (int32_t)sub;
      I.n_sub = (int32_t)std::max<int64_t>(1, ((int64_t)ibits[k] + S - 1) / S);
      for (int s = 0; s < I.n_sub; ++s) {
        sub_iv[sub + s] = (int32_t)(iv + k);
        start[sub + s] = (uint64_t)s * S;   // the guess: a codeword starts at the subsequence's first bit, block 0, k 0
      }
      sub += I.n_sub;
    }
    g.n_sub = (int32_t)(sub - g.first_sub);
    iv += f.n_intervals;
    dstatus[p] = 0;
    boff += align_up(nbytes, 16);
  }
  memset(bits + boff, 0, 16);   // slack for the last lookahead
  // 3. device buffers
  size_t w_iend = 0;   // scratch arrays, changed flags, coefficients, planes
  size_t w_cnt = align_up(w_iend + n_iv * sizeof(uint64_t), 256);
  size_t w_err = align_up(w_cnt + sub * sizeof(int32_t), 256);
  size_t w_dcp = align_up(w_err + sub * sizeof(int32_t), 256);
  size_t w_blk0 = align_up(w_dcp + sub * 3 * sizeof(int32_t), 256);
  size_t w_dc0 = align_up(w_blk0 + sub * sizeof(int32_t), 256);
  size_t w_flags = align_up(w_dc0 + sub * 3 * sizeof(int32_t), 256);
  size_t w_coef = align_up(w_flags + kRoundsPerCheck * sizeof(int), 256);
  size_t w_planes = align_up(w_coef + (size_t)blk * 128, 256);
  size_t work_bytes = w_planes + plane;
  if ((rc = grow(&d->dev, &d->dev_cap, host_bytes, false))) return rc;
  if ((rc = grow(&d->work, &d->work_cap, work_bytes, false))) return rc;
  uint8_t* D = d->dev;
  uint8_t* W = d->work;
  cudaStream_t st = d->stream;
  JCK(cudaMemcpyAsync(D, H, o_bits + boff + 16, cudaMemcpyHostToDevice, st));
  JCK(cudaMemsetAsync(W + w_coef, 0, (size_t)blk * 128, st));
  const DPage* gp = (const DPage*)(D + o_pages);
  const DInterval* giv = (const DInterval*)(D + o_ivs);
  const int32_t* gsub = (const int32_t*)(D + o_subiv);
  const HuffTable* gtab = (const HuffTable*)(D + o_tabs);
  const int32_t* gq = (const int32_t*)(D + o_quant);
  int32_t* gstatus = (int32_t*)(D + o_status);
  const uint8_t* gbits = D + o_bits;
  int16_t* coef = (int16_t*)(W + w_coef);
  uint8_t* planes = W + w_planes;
  int* changed = (int*)(W + w_flags);
  Scratch sc{(uint64_t*)(D + o_start), (uint64_t*)(W + w_iend), (int32_t*)(W + w_cnt), (int32_t*)(W + w_err),
             (int32_t*)(W + w_dcp),
             (int32_t*)(W + w_blk0), (int32_t*)(W + w_dc0)};
  // 4. self-synchronising rounds, kRoundsPerCheck per look at the flags
  int ns = (int)sub;
  dim3 sg((ns + 127) / 128);
  for (;;) {
    JCK(cudaMemsetAsync(changed, 0, kRoundsPerCheck * sizeof(int), st));
    for (int r = 0; r < kRoundsPerCheck; ++r)
      jpeg_sync_kernel<<<sg, 128, 0, st>>>(gp, giv, gsub, gtab, gbits, sc, ns, S, changed + r);
    JCK(cudaGetLastError());
    JCK(cudaMemcpyAsync(d->flags, changed, kRoundsPerCheck * sizeof(int), cudaMemcpyDeviceToHost, st));
    JCK(cudaStreamSynchronize(st));
    if (!d->flags[kRoundsPerCheck - 1]) break;
  }
  // 5. offsets, coefficients, IDCT, colour
  jpeg_scan_kernel<<<np, 1024, 0, st>>>(gp, giv, sc, gstatus);
  jpeg_write_kernel<<<sg, 128, 0, st>>>(gp, giv, gsub, gtab, gbits, sc, ns, S, gstatus, coef);
  jpeg_idct_kernel<<<dim3((unsigned)((max_blocks + kIdctBlocks - 1) / kIdctBlocks), np), 256, 0, st>>>(gp, gq, coef,
                                                                                                       planes, gstatus);
  jpeg_color_kernel<<<dim3((unsigned)((max_px + 255) / 256), np), 256, 0, st>>>(gp, planes, gstatus);
  JCK(cudaGetLastError());
  JCK(cudaMemcpyAsync(dstatus, gstatus, np * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  JCK(cudaStreamSynchronize(st));
  for (int p = 0; p < np; ++p) status[live[p]] = dstatus[p];
  return CTD_OK;
}
