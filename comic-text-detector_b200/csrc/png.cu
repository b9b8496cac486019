// GPU PNG encode (C ABI `ctd_png_encoder_*`, `ctd_png_encode`, include/ctd_b200.h): every image of a call at once,
// byte for byte the file cv2.imencode('.png', img) writes with its libpng 1.6 and zlib 1.2.11 (compression level 1,
// strategy Z_RLE, filter SUB, memLevel 8).  oracle/png_ref.py restates every rule; tests/test_cpu_png.py pins it to cv2.
//
// Stages, each one launch (or one scan) over the concatenated filtered streams of all images:
//   1. png_filter_kernel: the SUB-filtered stream (filter byte, row bytes minus the bytes one pixel left, BGR stored
//      as RGB) read straight from the strided source.
//   2. scan of run starts (a byte != its predecessor, or an image's first byte): the start of every maximal run.
//   3. scan of tokens per run, in deflate_rle's closed form: a run of R bytes is one literal, (R-1)/258 matches of 258
//      and, with r = (R-1) % 258, a match of r if r >= 3, else r literals (every match has distance 1).
//   4. png_token_kernel: each token from its run (binary search), its stream position, and the histograms of its
//      deflate block (block b of an image holds its tokens [16383 b, 16383 (b+1)); the rest, maybe none, is the
//      final block).
//   5. png_tree_kernel, one thread per block: trees.c's build_tree / gen_bitlen / gen_codes / build_bl_tree and
//      _tr_flush_block's choice of a stored, static or dynamic block, the dynamic header's bits.
//   6. png_offset_kernel, one thread per image: each block's bit offset (a stored block aligns to a byte), the deflate
//      length, Adler-32 from per-segment partial sums, the file size.
//   7. scan of token bit costs, then png_emit_kernel / png_block_kernel OR every code into the zeroed bit buffer.
//   8. png_crc_kernel (one thread per IDAT chunk) and png_assemble_kernel (16 bytes a thread) write the files into
//      mapped pinned host memory.  The call synchronises once, at the end.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/ctd_b200.h"
#include "scan.cuh"

int ctd_fail(ctd_handle* h, int code, const char* fmt, ...);

namespace ctd {
namespace png {
namespace {

constexpr int kMaxMatch = 258, kMinMatch = 3;
constexpr int kBlockTokens = 16383;          // lit_bufsize - 1 at memLevel 8
constexpr int kLCodes = 286, kDCodes = 30, kBLCodes = 19, kMaxBits = 15, kMaxBLBits = 7, kEndBlock = 256;
constexpr int kHeapSize = 2 * kLCodes + 1;
constexpr int kIdat = 8192;                  // libpng's zbuffer: IDAT chunk payload
constexpr int kHdrWords = 40;                // dynamic header bits: <= 74 + 316 * 7 < 40 * 64
constexpr int kAdlerSeg = 16384;
constexpr int64_t kStoredSpan = 32506;       // oracle/png_ref.py stored_ok

struct PImg {
  const uint8_t* src;
  int64_t sh, sw, sc;
  int32_t h, w, c, ftype;
  int64_t pos0, N, rowlen;
  int64_t seg0, word0, out_off, chunk0;
};

struct PBlk {
  int64_t start, len;        // stream bytes of the block, relative to its image
  int64_t tok_first;         // first token (global index)
  int64_t bits;              // the block's bits after its 3-bit type, EOB included (not for stored)
  uint64_t bitpos;           // offset of the block in its image's deflate bits
  int32_t img, ntok, form, last;
  int32_t hdr_bits;          // 3 + the dynamic header
  uint32_t eob;              // code | len << 16
};

struct State {               // device-side results of the scans
  uint32_t nruns;
  uint32_t ntok;
};

__constant__ uint8_t c_extra_lbits[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint8_t c_extra_dbits[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_extra_blbits[19] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};
__constant__ uint8_t c_bl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// tr_static_init's length code of (match length - 3) and its base
__device__ __forceinline__ int length_code(int lc) {
  if (lc == 255) return 28;
  if (lc < 8) return lc;
  int e = 31 - __clz(lc) - 2;                 // extra bits of codes 8..27: lc in [2^(e+2), 2^(e+3))
  return 4 * e + 4 + ((lc >> e) & 3);
}
__device__ __forceinline__ int base_length(int code) {
  if (code < 8) return code;
  if (code == 28) return 0;
  int e = (code - 4) >> 2;
  return (4 + (code & 3)) << e;
}
__host__ __device__ __forceinline__ int64_t imin64(int64_t a, int64_t b) { return a < b ? a : b; }
__device__ __forceinline__ uint32_t bi_reverse(uint32_t c, int n) { return __brev(c) >> (32 - n); }

// static trees (trees.c tr_static_init): literal/length lengths 8 / 9 / 7 / 8, distance codes 5 bits
__device__ __forceinline__ int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }
__device__ __forceinline__ uint32_t static_lcode(int n) {
  uint32_t c = n < 144 ? 0x30 + n : n < 256 ? 0x190 + (n - 144) : n < 280 ? n - 256 : 0xC0 + (n - 280);
  return bi_reverse(c, static_llen(n));
}

__device__ __forceinline__ int find_img(const int64_t* pos, int n, int64_t g) {   // last i with pos[i] <= g
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (pos[mid] <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- stage items -------------------------------------------------------------------------------------------------
struct RunStartItem {
  const uint8_t* f;
  const int64_t* pos;
  int n;
  __device__ uint32_t operator()(int64_t j) const {
    if (j == 0 || f[j] != f[j - 1]) return 1;
    int i = find_img(pos, n, j);
    return pos[i] == j;
  }
};
struct RunStartOut {
  const int64_t* pos;
  int n;
  int64_t N;
  uint32_t* runs;
  uint32_t* first_run;
  State* st;
  __device__ void operator()(int64_t j, uint32_t e, uint32_t v) const {
    if (v) {
      runs[e] = (uint32_t)j;
      int i = find_img(pos, n, j);
      if (pos[i] == j) first_run[i] = e;
    }
    if (j == N - 1) {
      runs[e + v] = (uint32_t)N;
      st->nruns = e + v;
    }
  }
};

__device__ __forceinline__ uint32_t run_tokens(uint32_t R) {
  uint32_t q = (R - 1) / kMaxMatch, r = (R - 1) % kMaxMatch;
  return 1 + q + (r >= kMinMatch ? 1 : r);
}
struct RunTokItem {
  const uint32_t* runs;
  const State* st;
  __device__ uint32_t operator()(int64_t k) const {
    if (k >= st->nruns) return 0;
    return run_tokens(runs[k + 1] - runs[k]);
  }
};
struct RunTokOut {
  uint32_t* tok_off;
  State* st;
  __device__ void operator()(int64_t k, uint32_t e, uint32_t v) const {
    uint32_t nr = st->nruns;
    if (k < nr) tok_off[k] = e;
    if (k == nr - 1) {
      tok_off[nr] = e + v;
      st->ntok = e + v;
    }
  }
};

// ---- 1. filter -----------------------------------------------------------------------------------------------------
__global__ void png_filter_kernel(const PImg* imgs, const int64_t* pos, int n, int64_t N, uint8_t* f) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < N; g += (int64_t)gridDim.x * blockDim.x) {
    const PImg& im = imgs[find_img(pos, n, g)];
    int64_t q = g - im.pos0;
    int64_t y = q / im.rowlen, col = q - y * im.rowlen;
    if (col == 0) {
      f[g] = (uint8_t)im.ftype;
      continue;
    }
    int64_t b = col - 1;
    int64_t x = b / im.c;
    int ch = (int)(b - x * im.c);
    int sc = im.c == 3 ? 2 - ch : 0;       // BGR -> RGB
    const uint8_t* row = im.src + y * im.sh;
    uint8_t v = row[x * im.sw + sc * im.sc];
    if (im.ftype == 1 && x > 0) v = (uint8_t)(v - row[(x - 1) * im.sw + sc * im.sc]);
    f[g] = v;
  }
}

// ---- 4. tokens ----------------------------------------------------------------------------------------------------
// per image: first token, token count, first block, block count (after the run and token scans)
__global__ void png_imginfo_kernel(const PImg* imgs, int n, const uint32_t* first_run, const uint32_t* tok_off,
                                   const State* st, int64_t* tok0, int64_t* blk0, PBlk* blks) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int64_t b = 0;
  for (int i = 0; i < n; ++i) {
    int64_t t0 = tok_off[first_run[i]];
    int64_t t1 = i + 1 < n ? (int64_t)tok_off[first_run[i + 1]] : (int64_t)st->ntok;
    tok0[i] = t0;
    blk0[i] = b;
    int64_t T = t1 - t0, nb = T / kBlockTokens + 1;
    for (int64_t k = 0; k < nb; ++k) {
      PBlk& B = blks[b + k];
      B.img = i;
      B.tok_first = t0 + k * kBlockTokens;
      B.ntok = (int32_t)imin64(kBlockTokens, T - k * kBlockTokens);
      B.last = k == nb - 1;
      if (B.ntok == 0) B.start = imgs[i].N;     // the empty final block after 16383 k tokens
    }
    b += nb;
  }
  tok0[n] = st->ntok;
  blk0[n] = b;
}

__global__ void png_token_kernel(const uint8_t* f, const uint32_t* runs, const uint32_t* tok_off, const State* st,
                                 const int64_t* pos, const int64_t* tok0, const int64_t* blk0, int n,
                                 uint16_t* tok, PBlk* blks, uint32_t* hist) {
  int64_t T = st->ntok;
  uint32_t nr = st->nruns;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t - threadIdx.x < T;
       t += (int64_t)gridDim.x * blockDim.x) {
    bool live = t < T;
    uint32_t key = 0xffffffffu;
    if (live) {
      uint32_t lo = 0, hi = nr - 1;                // last run k with tok_off[k] <= t
      while (lo < hi) {
        uint32_t mid = (lo + hi + 1) >> 1;
        if (tok_off[mid] <= t) lo = mid; else hi = mid - 1;
      }
      uint32_t k = lo, s0 = runs[k], R = runs[k + 1] - s0;
      uint32_t i = (uint32_t)(t - tok_off[k]);
      uint32_t q = (R - 1) / kMaxMatch, r = (R - 1) % kMaxMatch;
      uint8_t lit = f[s0];
      uint16_t v;
      uint32_t p;                                  // the token's stream position
      if (i == 0) { v = lit; p = s0; }
      else if (i <= q) { v = 256 + kMaxMatch; p = s0 + 1 + (i - 1) * kMaxMatch; }
      else if (r >= kMinMatch) { v = 256 + r; p = s0 + 1 + q * kMaxMatch; }
      else { v = lit; p = s0 + 1 + q * kMaxMatch + (i - 1 - q); }
      tok[t] = v;
      int im = 0;
      {
        int a = 0, b = n - 1;
        while (a < b) {
          int mid = (a + b + 1) >> 1;
          if (tok0[mid] <= t) a = mid; else b = mid - 1;
        }
        im = a;
      }
      int64_t li = t - tok0[im];
      int64_t blk = blk0[im] + li / kBlockTokens;
      if (li % kBlockTokens == 0) blks[blk].start = (int64_t)p - pos[im];
      int sym = v < 256 ? v : 257 + length_code(v - 256 - kMinMatch);
      key = (uint32_t)(blk * kLCodes + sym);
    }
    // warp-aggregated histogram: runs of one byte give long streams of one symbol
    unsigned peers = __match_any_sync(0xffffffffu, key);
    if (live && (__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(&hist[key], __popc(peers));
  }
}

// ---- 5. trees (trees.c, zlib 1.2.11) ------------------------------------------------------------------------------
struct TreeWork {
  uint32_t freq[kHeapSize];
  uint16_t len[kHeapSize];
  uint16_t dad[kHeapSize];
  int heap[kHeapSize];
  uint8_t depth[kHeapSize];
  uint16_t bl_count[kMaxBits + 1];
  int heap_len, heap_max;
  int64_t opt_len, static_len;
};

struct TreeDesc {
  int elems, base, max_length, max_code;
  const uint8_t* extra;
  bool has_static;
  bool lit;                  // literal/length static tree (else distance)
};

__device__ __forceinline__ bool smaller(const TreeWork& s, int n, int m) {
  return s.freq[n] < s.freq[m] || (s.freq[n] == s.freq[m] && s.depth[n] <= s.depth[m]);
}

__device__ void pqdownheap(TreeWork& s, int k) {
  int v = s.heap[k];
  int j = k << 1;
  while (j <= s.heap_len) {
    if (j < s.heap_len && smaller(s, s.heap[j + 1], s.heap[j])) j++;
    if (smaller(s, v, s.heap[j])) break;
    s.heap[k] = s.heap[j];
    k = j;
    j <<= 1;
  }
  s.heap[k] = v;
}

__device__ __forceinline__ int stree_len(const TreeDesc& d, int n) { return d.lit ? static_llen(n) : 5; }

__device__ void gen_bitlen(TreeWork& s, const TreeDesc& d) {
  for (int b = 0; b <= kMaxBits; ++b) s.bl_count[b] = 0;
  s.len[s.heap[s.heap_max]] = 0;
  int overflow = 0, h;
  for (h = s.heap_max + 1; h < kHeapSize; ++h) {
    int n = s.heap[h];
    int bits = s.len[s.dad[n]] + 1;
    if (bits > d.max_length) bits = d.max_length, overflow++;
    s.len[n] = (uint16_t)bits;
    if (n > d.max_code) continue;
    s.bl_count[bits]++;
    int xbits = n >= d.base ? d.extra[n - d.base] : 0;
    int64_t f = s.freq[n];
    s.opt_len += f * (bits + xbits);
    if (d.has_static) s.static_len += f * (stree_len(d, n) + xbits);
  }
  if (overflow == 0) return;
  do {
    int bits = d.max_length - 1;
    while (s.bl_count[bits] == 0) bits--;
    s.bl_count[bits]--;
    s.bl_count[bits + 1] += 2;
    s.bl_count[d.max_length]--;
    overflow -= 2;
  } while (overflow > 0);
  for (int bits = d.max_length; bits != 0; bits--) {
    int n = s.bl_count[bits];
    while (n != 0) {
      int m = s.heap[--h];
      if (m > d.max_code) continue;
      if (s.len[m] != bits) {
        s.opt_len += ((int64_t)bits - s.len[m]) * (int64_t)s.freq[m];
        s.len[m] = (uint16_t)bits;
      }
      n--;
    }
  }
}

// build_tree over s.freq[0, elems); codes out (code | len << 16) for [0, elems)
__device__ void build_tree(TreeWork& s, TreeDesc& d, uint32_t* codes) {
  s.heap_len = 0;
  s.heap_max = kHeapSize;
  int max_code = -1;
  for (int n = 0; n < d.elems; ++n) {
    if (s.freq[n] != 0) {
      s.heap[++s.heap_len] = max_code = n;
      s.depth[n] = 0;
    } else {
      s.len[n] = 0;
    }
  }
  while (s.heap_len < 2) {
    int node = s.heap[++s.heap_len] = max_code < 2 ? ++max_code : 0;
    s.freq[node] = 1;
    s.depth[node] = 0;
    s.opt_len--;
    if (d.has_static) s.static_len -= stree_len(d, node);
  }
  d.max_code = max_code;
  for (int n = s.heap_len / 2; n >= 1; n--) pqdownheap(s, n);
  int node = d.elems;
  do {
    int n = s.heap[1];
    s.heap[1] = s.heap[s.heap_len--];
    pqdownheap(s, 1);
    int m = s.heap[1];
    s.heap[--s.heap_max] = n;
    s.heap[--s.heap_max] = m;
    s.freq[node] = s.freq[n] + s.freq[m];
    s.depth[node] = (uint8_t)((s.depth[n] >= s.depth[m] ? s.depth[n] : s.depth[m]) + 1);
    s.dad[n] = s.dad[m] = (uint16_t)node;
    s.heap[1] = node++;
    pqdownheap(s, 1);
  } while (s.heap_len >= 2);
  s.heap[--s.heap_max] = s.heap[1];
  gen_bitlen(s, d);
  uint32_t next_code[kMaxBits + 1];
  uint32_t code = 0;
  for (int bits = 1; bits <= kMaxBits; ++bits) {
    code = (code + s.bl_count[bits - 1]) << 1;
    next_code[bits] = code;
  }
  for (int n = 0; n < d.elems; ++n) {
    int l = n <= max_code ? s.len[n] : 0;
    codes[n] = l ? (bi_reverse(next_code[l]++, l) | (uint32_t)l << 16) : 0;
  }
}

struct BitSink {             // the dynamic header's bits, LSB first
  uint64_t* w;
  int n;
  __device__ void put(uint32_t v, int nb) {
    if (nb == 0) return;
    int k = n >> 6, sh = n & 63;
    w[k] |= (uint64_t)v << sh;
    if (sh + nb > 64) w[k + 1] |= (uint64_t)v >> (64 - sh);
    n += nb;
  }
};

// scan_tree (send == nullptr) / send_tree over lens[0, max_code], with the guard at max_code + 1
__device__ void walk_tree(uint16_t* lens, int max_code, uint32_t* blfreq, const uint32_t* blcodes, BitSink* send) {
  int prevlen = -1, nextlen = lens[0], count = 0, max_count = 7, min_count = 4;
  if (nextlen == 0) max_count = 138, min_count = 3;
  lens[max_code + 1] = 0xffff;
  auto code = [&](int c) { send->put(blcodes[c] & 0xffff, blcodes[c] >> 16); };
  for (int n = 0; n <= max_code; ++n) {
    int curlen = nextlen;
    nextlen = lens[n + 1];
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      if (send) { do code(curlen); while (--count != 0); }
      else blfreq[curlen] += count;
    } else if (curlen != 0) {
      if (curlen != prevlen) {
        if (send) { code(curlen); count--; }
        else blfreq[curlen]++;
      }
      if (send) { code(16); send->put(count - 3, 2); }
      else blfreq[16]++;
    } else if (count <= 10) {
      if (send) { code(17); send->put(count - 3, 3); }
      else blfreq[17]++;
    } else {
      if (send) { code(18); send->put(count - 11, 7); }
      else blfreq[18]++;
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) max_count = 138, min_count = 3;
    else if (curlen == nextlen) max_count = 6, min_count = 3;
    else max_count = 7, min_count = 4;
  }
}

__global__ void __launch_bounds__(64) png_tree_kernel(PBlk* blks, const int64_t* blk0, int n, const uint32_t* hist,
                                                      const int64_t* img_N, uint32_t* lcodes, uint32_t* dcodes,
                                                      uint64_t* hdr, TreeWork* work) {
  int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= blk0[n]) return;
  PBlk& B = blks[b];
  // the block's bytes: up to the next block's start (or the image's end)
  int64_t end = B.last ? img_N[B.img] : blks[b + 1].start;
  B.len = end - B.start;
  TreeWork& s = work[b];
  s.opt_len = s.static_len = 0;
  uint32_t matches = 0;
  for (int k = 0; k < kLCodes; ++k) {
    s.freq[k] = hist[b * kLCodes + k];
    if (k > kEndBlock) matches += s.freq[k];
  }
  s.freq[kEndBlock] = 1;
  uint32_t* lc = lcodes + b * kLCodes;
  TreeDesc ld{kLCodes, 257, kMaxBits, -1, c_extra_lbits, true, true};
  build_tree(s, ld, lc);
  uint16_t llens[kLCodes + 1];
  for (int k = 0; k < kLCodes; ++k) llens[k] = k <= ld.max_code ? s.len[k] : 0;
  // distance tree: only code 0 (distance 1) can have a frequency
  for (int k = 0; k < kDCodes; ++k) s.freq[k] = 0;
  s.freq[0] = matches;
  uint32_t dc[kDCodes];
  TreeDesc dd{kDCodes, 0, kMaxBits, -1, c_extra_dbits, true, false};
  build_tree(s, dd, dc);
  uint16_t dlens[kDCodes + 1];
  for (int k = 0; k < kDCodes; ++k) dlens[k] = k <= dd.max_code ? s.len[k] : 0;
  dcodes[b] = dc[0];
  // build_bl_tree
  for (int k = 0; k < kBLCodes; ++k) s.freq[k] = 0;
  walk_tree(llens, ld.max_code, s.freq, nullptr, nullptr);
  walk_tree(dlens, dd.max_code, s.freq, nullptr, nullptr);
  uint32_t blc[kBLCodes];
  TreeDesc bd{kBLCodes, 0, kMaxBLBits, -1, c_extra_blbits, false, false};
  build_tree(s, bd, blc);
  int max_blindex;
  for (max_blindex = kBLCodes - 1; max_blindex >= 3; max_blindex--)
    if ((blc[c_bl_order[max_blindex]] >> 16) != 0) break;
  s.opt_len += 3 * ((int64_t)max_blindex + 1) + 5 + 5 + 4;
  // _tr_flush_block
  int64_t opt_lenb = (s.opt_len + 3 + 7) >> 3, static_lenb = (s.static_len + 3 + 7) >> 3;
  if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
  uint64_t* hw = hdr + b * kHdrWords;
  for (int k = 0; k < kHdrWords; ++k) hw[k] = 0;
  BitSink sink{hw, 0};
  if (B.len + 4 <= opt_lenb && B.len <= kStoredSpan) {
    B.form = 0;
    sink.put(0 + B.last, 3);
    B.bits = 0;
  } else if (static_lenb == opt_lenb) {
    B.form = 1;
    sink.put((1 << 1) + B.last, 3);
    B.bits = s.static_len;
    for (int k = 0; k < kLCodes; ++k) lc[k] = static_lcode(k) | (uint32_t)static_llen(k) << 16;
    dcodes[b] = 0 | 5u << 16;
    B.eob = static_lcode(kEndBlock) | 7u << 16;
  } else {
    B.form = 2;
    sink.put((2 << 1) + B.last, 3);
    int lcodes_n = ld.max_code + 1, dcodes_n = dd.max_code + 1;
    sink.put(lcodes_n - 257, 5);
    sink.put(dcodes_n - 1, 5);
    sink.put(max_blindex + 1 - 4, 4);
    for (int r = 0; r <= max_blindex; ++r) sink.put(blc[c_bl_order[r]] >> 16, 3);
    walk_tree(llens, ld.max_code, nullptr, blc, &sink);
    walk_tree(dlens, dd.max_code, nullptr, blc, &sink);
    B.bits = s.opt_len - (sink.n - 3);           // the tokens and EOB
    B.eob = lc[kEndBlock];
  }
  B.hdr_bits = sink.n;
}

// ---- 6. offsets, Adler-32, sizes ------------------------------------------------------------------------------------
__global__ void png_adler_kernel(const uint8_t* f, const PImg* imgs, const int64_t* seg_img, int64_t nseg,
                                 uint32_t* seg_ab) {
  int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nseg) return;
  const PImg& im = imgs[seg_img[g]];
  int64_t s0 = (g - im.seg0) * kAdlerSeg, L = imin64(kAdlerSeg, im.N - s0);
  const uint8_t* p = f + im.pos0 + s0;
  uint64_t a = 0, b = 0;
  for (int64_t k = 0; k < L; ++k) {
    a += p[k];
    b += a;
  }
  seg_ab[2 * g] = (uint32_t)(a % 65521);
  seg_ab[2 * g + 1] = (uint32_t)(b % 65521);
}

__device__ uint32_t crc_update(uint32_t c, const uint8_t* p, int n, const uint32_t* tab) {
  for (int k = 0; k < n; ++k) c = tab[(c ^ p[k]) & 0xff] ^ (c >> 8);
  return c;
}
__device__ void make_crc_table(uint32_t* tab) {
  for (int k = threadIdx.x; k < 256; k += blockDim.x) {
    uint32_t c = k;
    for (int j = 0; j < 8; ++j) c = c & 1 ? 0xedb88320u ^ (c >> 1) : c >> 1;
    tab[k] = c;
  }
  __syncthreads();
}

struct ImgOut {
  int64_t D;                 // deflate bytes
  int64_t Z;                 // zlib stream bytes
  int64_t size;              // file bytes
  uint32_t adler, ihdr_crc;
  uint8_t zhdr[2];
};

__global__ void png_offset_kernel(const PImg* imgs, int n, const int64_t* blk0, PBlk* blks, const uint32_t* seg_ab,
                                  ImgOut* io, int64_t* sizes) {
  __shared__ uint32_t tab[256];
  make_crc_table(tab);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PImg& im = imgs[i];
  uint64_t cur = 0;
  for (int64_t b = blk0[i]; b < blk0[i + 1]; ++b) {
    PBlk& B = blks[b];
    B.bitpos = cur;
    if (B.form == 0) cur = ((cur + 3 + 7) & ~(uint64_t)7) + 32 + 8 * (uint64_t)B.len;
    else cur += B.hdr_bits + B.bits;
  }
  ImgOut& o = io[i];
  o.D = (int64_t)((cur + 7) >> 3);
  uint64_t A = 1, Bs = 0;
  int64_t nseg = (im.N + kAdlerSeg - 1) / kAdlerSeg;
  for (int64_t g = 0; g < nseg; ++g) {
    int64_t L = imin64(kAdlerSeg, im.N - g * kAdlerSeg);
    Bs = (Bs + (uint64_t)(L % 65521) * A + seg_ab[2 * (im.seg0 + g) + 1]) % 65521;
    A = (A + seg_ab[2 * (im.seg0 + g)]) % 65521;
  }
  o.adler = (uint32_t)(Bs << 16 | A);
  // zlib header: level 1 (FLEVEL 0); CINFO as libpng leaves it (png_deflate_claim's windowBits, optimize_cmf)
  int64_t ds = im.N;
  int wbits = 15;
  if (ds <= 16384) {
    uint32_t half = 1u << (wbits - 1);
    while (ds + 262 <= half) half >>= 1, wbits--;
  }
  if (wbits == 8) wbits = 9;
  int cinfo = wbits - 8;
  if (ds <= 16384) {
    uint32_t half = 1u << (cinfo + 7);
    if (ds <= half) {
      do half >>= 1, cinfo--;
      while (cinfo > 0 && ds <= half);
    }
  }
  uint32_t cmf = 0x08 | cinfo << 4;
  o.zhdr[0] = (uint8_t)cmf;
  o.zhdr[1] = (uint8_t)(31 - ((cmf << 8) % 31));
  o.Z = 2 + o.D + 4;
  int64_t chunks = (o.Z + kIdat - 1) / kIdat;
  o.size = 8 + 25 + o.Z + 12 * chunks + 12;
  uint8_t ih[17] = {'I', 'H', 'D', 'R', (uint8_t)(im.w >> 24), (uint8_t)(im.w >> 16), (uint8_t)(im.w >> 8),
                    (uint8_t)im.w, (uint8_t)(im.h >> 24), (uint8_t)(im.h >> 16), (uint8_t)(im.h >> 8), (uint8_t)im.h,
                    8, (uint8_t)(im.c == 3 ? 2 : 0), 0, 0, 0};
  o.ihdr_crc = crc_update(0xffffffffu, ih, 17, tab) ^ 0xffffffffu;
  sizes[i] = o.size;
}

// ---- 7. bits ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void or_bits(uint64_t* w, uint64_t p, uint64_t v, int nb) {
  if (nb == 0) return;
  uint64_t k = p >> 6;
  int sh = (int)(p & 63);
  atomicOr((unsigned long long*)&w[k], (unsigned long long)(v << sh));
  if (sh + nb > 64) atomicOr((unsigned long long*)&w[k + 1], (unsigned long long)(v >> (64 - sh)));
}

// (value, bits) of token t with its block's codes
__device__ __forceinline__ uint64_t token_code(uint16_t v, const uint32_t* lc, uint32_t dc, int* nb) {
  if (v < 256) {
    *nb = lc[v] >> 16;
    return lc[v] & 0xffff;
  }
  int l = v - 256 - kMinMatch, code = length_code(l);
  uint32_t c = lc[257 + code];
  int n = c >> 16;
  uint64_t val = c & 0xffff;
  int xb = c_extra_lbits[code];
  if (xb) {
    val |= (uint64_t)(l - base_length(code)) << n;
    n += xb;
  }
  val |= (uint64_t)(dc & 0xffff) << n;
  n += dc >> 16;
  *nb = n;
  return val;
}

__device__ __forceinline__ int64_t block_of(const int64_t* tok0, const int64_t* blk0, int n, int64_t t) {
  int a = 0, b = n - 1;
  while (a < b) {
    int mid = (a + b + 1) >> 1;
    if (tok0[mid] <= t) a = mid; else b = mid - 1;
  }
  return blk0[a] + (t - tok0[a]) / kBlockTokens;
}

struct CostItem {
  const uint16_t* tok;
  const int64_t *tok0, *blk0;
  int n;
  const PBlk* blks;
  const uint32_t *lcodes, *dcodes;
  const State* st;
  __device__ uint64_t operator()(int64_t t) const {
    if (t >= st->ntok) return 0;
    int64_t b = block_of(tok0, blk0, n, t);
    if (blks[b].form == 0) return 0;
    int nb;
    token_code(tok[t], lcodes + b * kLCodes, dcodes[b], &nb);
    return nb;
  }
};
struct CostOut {
  uint64_t* off;
  __device__ void operator()(int64_t t, uint64_t e, uint64_t) const { off[t] = e; }
};

__global__ void png_emit_kernel(const uint16_t* tok, const uint64_t* off, const int64_t* tok0, const int64_t* blk0,
                                int n, const PBlk* blks, const uint32_t* lcodes, const uint32_t* dcodes,
                                const PImg* imgs, const State* st, uint64_t* words) {
  int64_t T = st->ntok;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t b = block_of(tok0, blk0, n, t);
    const PBlk& B = blks[b];
    if (B.form == 0) continue;
    int nb;
    uint64_t v = token_code(tok[t], lcodes + b * kLCodes, dcodes[b], &nb);
    uint64_t p = B.bitpos + B.hdr_bits + (off[t] - off[B.tok_first]);
    or_bits(words + imgs[B.img].word0, p, v, nb);
  }
}

// one warp per block: its header (type bits, dynamic trees) and EOB, or a stored block's length and bytes
__global__ void png_block_kernel(const PBlk* blks, const int64_t* blk0, int n, const uint64_t* hdr, const uint8_t* f,
                                 const PImg* imgs, uint64_t* words) {
  int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (b >= blk0[n]) return;
  const PBlk& B = blks[b];
  const PImg& im = imgs[B.img];
  uint64_t* w = words + im.word0;
  const uint64_t* h = hdr + b * kHdrWords;
  if (B.form != 0) {
    for (int k = lane; k * 64 < B.hdr_bits; k += 32) or_bits(w, B.bitpos + 64 * k, h[k], min(64, B.hdr_bits - 64 * k));
    if (lane == 0) or_bits(w, B.bitpos + B.hdr_bits + B.bits - (B.eob >> 16), B.eob & 0xffff, B.eob >> 16);
    return;
  }
  if (lane == 0) or_bits(w, B.bitpos, h[0], 3);
  uint64_t q = (B.bitpos + 3 + 7) & ~(uint64_t)7;
  if (lane == 0) or_bits(w, q, (uint64_t)(B.len & 0xffff) | (uint64_t)(~B.len & 0xffff) << 16, 32);
  uint64_t byte0 = (q >> 3) + 4;
  const uint8_t* src = f + im.pos0 + B.start;
  for (int64_t j = lane; j < B.len; j += 32) or_bits(w, (byte0 + j) * 8, src[j], 8);
}

// ---- 8. container -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t zbyte(const ImgOut& o, const uint64_t* w, int64_t z) {
  if (z < 2) return o.zhdr[z];
  z -= 2;
  if (z < o.D) return (uint8_t)(w[z >> 3] >> (8 * (z & 7)));
  z -= o.D;
  return (uint8_t)(o.adler >> (8 * (3 - z)));
}

__global__ void png_crc_kernel(const PImg* imgs, const int64_t* chunk_img, int64_t nchunks, const ImgOut* io,
                               const uint64_t* words, uint32_t* crcs) {
  __shared__ uint32_t tab[256];
  make_crc_table(tab);
  int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nchunks) return;
  int i = (int)chunk_img[g];
  const PImg& im = imgs[i];
  const ImgOut& o = io[i];
  int64_t c = g - im.chunk0, z0 = c * kIdat;
  if (z0 >= o.Z) return;
  int64_t z1 = imin64(z0 + kIdat, o.Z);
  const uint8_t idat[4] = {'I', 'D', 'A', 'T'};
  uint32_t crc = crc_update(0xffffffffu, idat, 4, tab);
  const uint64_t* w = words + im.word0;
  for (int64_t z = z0; z < z1; ++z) crc = tab[(crc ^ zbyte(o, w, z)) & 0xff] ^ (crc >> 8);
  crcs[g] = crc ^ 0xffffffffu;
}

__device__ __forceinline__ uint8_t be32(uint32_t v, int k) { return (uint8_t)(v >> (8 * (3 - k))); }

__global__ void png_assemble_kernel(const PImg* imgs, const int64_t* unit0, int n, int64_t nunits, const ImgOut* io,
                                    const uint64_t* words, const uint32_t* crcs, uint8_t* out) {
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < nunits; u += (int64_t)gridDim.x * blockDim.x) {
    int i = find_img(unit0, n, u);
    const PImg& im = imgs[i];
    const ImgOut& o = io[i];
    int64_t p0 = (u - unit0[i]) * 16;
    if (p0 >= o.size) continue;
    const uint64_t* w = words + im.word0;
    int64_t chunks = (o.Z + kIdat - 1) / kIdat, idat_end = 33 + o.Z + 12 * chunks;
    alignas(16) uint8_t v[16];
    for (int k = 0; k < 16; ++k) {
      int64_t p = p0 + k;
      uint8_t x = 0;
      if (p < 8) {
        const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
        x = sig[p];
      } else if (p < 33) {
        int q = (int)(p - 8);
        const uint8_t head[8] = {0, 0, 0, 13, 'I', 'H', 'D', 'R'};
        if (q < 8) x = head[q];
        else if (q < 12) x = be32(im.w, q - 8);
        else if (q < 16) x = be32(im.h, q - 12);
        else if (q == 16) x = 8;
        else if (q == 17) x = im.c == 3 ? 2 : 0;
        else if (q < 21) x = 0;
        else x = be32(o.ihdr_crc, q - 21);
      } else if (p < idat_end) {
        int64_t q = p - 33, c = q / (kIdat + 12), r = q - c * (kIdat + 12);
        int64_t clen = imin64(kIdat, o.Z - c * kIdat);
        if (r < 4) x = be32((uint32_t)clen, (int)r);
        else if (r < 8) x = "IDAT"[r - 4];
        else if (r < 8 + clen) x = zbyte(o, w, c * kIdat + r - 8);
        else x = be32(crcs[im.chunk0 + c], (int)(r - 8 - clen));
      } else if (p < o.size) {
        const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
        x = iend[p - idat_end];
      }
      v[k] = x;
    }
    *reinterpret_cast<uint4*>(out + im.out_off + p0) = *reinterpret_cast<const uint4*>(v);
  }
}

}  // namespace
}  // namespace png
}  // namespace ctd

using namespace ctd;
using namespace ctd::png;

struct ctd_png_encoder {
  int device = 0;
  cudaStream_t stream = nullptr;
  uint8_t* stage = nullptr;    // pinned: host images, then descriptors
  size_t stage_cap = 0;
  uint8_t* dev = nullptr;      // device scratch of one call
  size_t dev_cap = 0;
  uint8_t* out = nullptr;      // mapped pinned: the files and their sizes
  size_t out_cap = 0;
  std::vector<const uint8_t*> files;
};

#define PCK(expr)                                                                                           \
  do {                                                                                                      \
    cudaError_t _e = (expr);                                                                                \
    if (_e != cudaSuccess)                                                                                  \
      return ctd_fail(nullptr, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

extern "C" CTD_API int ctd_png_encoder_create(int32_t device, ctd_png_encoder** out) {
  if (!out) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_encoder_create: bad argument");
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n)
    return ctd_fail(nullptr, CTD_E_NO_DEVICE, "ctd_png_encoder_create: no CUDA device %d (no CPU fallback)", device);
  cudaDeviceProp prop;
  PCK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return ctd_fail(nullptr, CTD_E_NO_DEVICE, "device %d is sm_%d%d, not sm_90", device, prop.major, prop.minor);
  PCK(cudaSetDevice(device));
  ctd_png_encoder* e = new ctd_png_encoder;
  e->device = device;
  cudaError_t r = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
  if (r != cudaSuccess) {
    ctd_png_encoder_destroy(e);
    return ctd_fail(nullptr, CTD_E_CUDA, "ctd_png_encoder_create: %s", cudaGetErrorString(r));
  }
  *out = e;
  return CTD_OK;
}

extern "C" CTD_API void ctd_png_encoder_destroy(ctd_png_encoder* e) {
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
int grow_buf(uint8_t** buf, size_t* cap, size_t need, BufKind kind) {
  if (*cap >= need) return CTD_OK;
  if (kind == kDevice) cudaFree(*buf); else cudaFreeHost(*buf);
  *buf = nullptr;
  *cap = 0;
  size_t n = need + need / 4;
  cudaError_t e = kind == kDevice ? cudaMalloc((void**)buf, n)
                : cudaHostAlloc((void**)buf, n, kind == kMapped ? cudaHostAllocMapped : cudaHostAllocDefault);
  if (e != cudaSuccess) return ctd_fail(nullptr, CTD_E_CUDA, "png encoder: allocating %zu bytes: %s", n, cudaGetErrorString(e));
  *cap = n;
  return CTD_OK;
}

size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

// carves consecutive 256-byte aligned pieces out of one allocation
struct Carve {
  size_t off = 0;
  size_t take(size_t bytes) {
    size_t o = off;
    off = (off + bytes + 255) & ~(size_t)255;
    return o;
  }
};

int64_t blocks_for(int64_t n, int threads) { return (n + threads - 1) / threads; }

}  // namespace

extern "C" CTD_API int ctd_png_encode(ctd_png_encoder* e, const ctd_png_image* in, int32_t n, const uint8_t** files,
                                      int64_t* sizes) {
  if (!e || n < 0 || (n && (!in || !files || !sizes))) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_encode: bad argument");
  if (n == 0) return CTD_OK;
  PCK(cudaSetDevice(e->device));
  // validate every image before any GPU work
  std::vector<PImg> im(n);
  int64_t N = 0, host_bytes = 0, nseg = 0, words = 0, out_bytes = 0, nchunks = 0, nblk_max = 0, nunits = 0;
  std::vector<int64_t> pos(n + 1), unit0(n + 1), img_N(n);
  for (int i = 0; i < n; ++i) {
    const ctd_png_image& s = in[i];
    if (!s.data || s.height < 1 || s.width < 1 || (s.channels != 1 && s.channels != 3) || s.bit_depth != 8)
      return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_encode: image %d: need u8 [h][w] or [h][w][3] with h, w >= 1 "
                      "(got %dx%dx%d, %d bits)", i, s.height, s.width, s.channels, s.bit_depth);
    if (s.height >= (1 << 30) || s.width >= (1 << 30))
      return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_encode: image %d: side of 2^30 or more", i);
    if (s.on_device) {
      if (s.stride_h < 0 || s.stride_w < 0 || s.stride_c < 0)
        return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_encode: image %d: negative stride", i);
      cudaPointerAttributes a;
      if (cudaPointerGetAttributes(&a, s.data) != cudaSuccess || a.type != cudaMemoryTypeDevice || a.device != e->device) {
        cudaGetLastError();
        return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_encode: image %d is not device memory of GPU %d", i, e->device);
      }
    }
    PImg& p = im[i];
    p.h = s.height;
    p.w = s.width;
    p.c = s.channels;
    p.ftype = s.width == 1 ? 0 : 1;     // png_write_start_row drops SUB for one-pixel-wide images
    p.rowlen = 1 + (int64_t)s.width * s.channels;
    p.N = p.rowlen * s.height;
    p.pos0 = N;
    pos[i] = N;
    img_N[i] = p.N;
    N += p.N;
    p.seg0 = nseg;
    nseg += (p.N + kAdlerSeg - 1) / kAdlerSeg;
    int64_t nb = p.N / kBlockTokens + 1;
    nblk_max += nb;
    int64_t Dmax = p.N + 6 * nb + 8, Zmax = Dmax + 6;
    p.word0 = words;
    words += Dmax / 8 + 2;
    p.chunk0 = nchunks;
    nchunks += (Zmax + kIdat - 1) / kIdat;
    int64_t fmax = align16(8 + 25 + Zmax + 12 * ((Zmax + kIdat - 1) / kIdat) + 12);
    p.out_off = out_bytes;
    out_bytes += fmax;
    unit0[i] = nunits;
    nunits += fmax / 16;
    if (!s.on_device) host_bytes += align16((size_t)p.h * p.w * p.c);
  }
  pos[n] = N;
  unit0[n] = nunits;
  if (N >= (int64_t)1 << 31)
    return ctd_fail(nullptr, CTD_E_CAPACITY, "ctd_png_encode: %lld filtered bytes in one call; encode fewer (< 2^31)",
                    (long long)N);
  // device scratch
  Carve c;
  size_t o_f = c.take(N + 8), o_runs = c.take(4 * (N + 1)), o_tok_off = c.take(4 * (N + 1)), o_tok = c.take(2 * N);
  size_t o_off = c.take(8 * N), o_tiles = c.take(8 * (N / kScanTile + 2));
  size_t o_first = c.take(4 * n), o_tok0 = c.take(8 * (n + 1)), o_blk0 = c.take(8 * (n + 1)), o_state = c.take(sizeof(State));
  size_t o_blks = c.take(sizeof(PBlk) * nblk_max), o_hist = c.take(4 * kLCodes * nblk_max);
  size_t o_lc = c.take(4 * kLCodes * nblk_max), o_dc = c.take(4 * nblk_max), o_hdr = c.take(8 * kHdrWords * nblk_max);
  size_t o_work = c.take(sizeof(TreeWork) * nblk_max);
  size_t o_seg = c.take(8 * nseg), o_io = c.take(sizeof(ImgOut) * n);
  size_t o_words = c.take(8 * words), o_crc = c.take(4 * nchunks);
  size_t o_imgs = c.take(sizeof(PImg) * n), o_pos = c.take(8 * (n + 1)), o_unit0 = c.take(8 * (n + 1));
  size_t o_imgN = c.take(8 * n), o_segimg = c.take(8 * nseg), o_chimg = c.take(8 * nchunks), o_host = c.take(host_bytes);
  size_t meta = c.off - o_imgs;   // descriptors and host pixels: staged, then one copy
  int rc;
  if ((rc = grow_buf(&e->dev, &e->dev_cap, c.off, kDevice))) return rc;
  if ((rc = grow_buf(&e->stage, &e->stage_cap, meta, kPinned))) return rc;
  if ((rc = grow_buf(&e->out, &e->out_cap, out_bytes + 8 * n + 16, kMapped))) return rc;
  uint8_t* D = e->dev;
  uint8_t* S = e->stage;
  // stage host pixels and descriptors
  int64_t hoff = 0;
  for (int i = 0; i < n; ++i) {
    const ctd_png_image& s = in[i];
    PImg& p = im[i];
    if (s.on_device) {
      p.src = s.data;
      p.sh = s.stride_h;
      p.sw = s.stride_w;
      p.sc = s.stride_c;
    } else {
      size_t bytes = (size_t)p.h * p.w * p.c;
      memcpy(S + (o_host - o_imgs) + hoff, s.data, bytes);
      p.src = D + o_host + hoff;
      p.sh = (int64_t)p.w * p.c;
      p.sw = p.c;
      p.sc = 1;
      hoff += align16(bytes);
    }
  }
  int64_t* seg_img = (int64_t*)(S + (o_segimg - o_imgs));
  int64_t* chunk_img = (int64_t*)(S + (o_chimg - o_imgs));
  for (int i = 0; i < n; ++i) {
    int64_t s1 = i + 1 < n ? im[i + 1].seg0 : nseg, c1 = i + 1 < n ? im[i + 1].chunk0 : nchunks;
    for (int64_t g = im[i].seg0; g < s1; ++g) seg_img[g] = i;
    for (int64_t g = im[i].chunk0; g < c1; ++g) chunk_img[g] = i;
  }
  memcpy(S + (o_imgs - o_imgs), im.data(), sizeof(PImg) * n);
  memcpy(S + (o_pos - o_imgs), pos.data(), 8 * (n + 1));
  memcpy(S + (o_unit0 - o_imgs), unit0.data(), 8 * (n + 1));
  memcpy(S + (o_imgN - o_imgs), img_N.data(), 8 * n);
  cudaStream_t st = e->stream;
  for (int i = 0; i < n; ++i)
    if (in[i].on_device && in[i].event) PCK(cudaStreamWaitEvent(st, (cudaEvent_t)in[i].event, 0));
  PCK(cudaMemcpyAsync(D + o_imgs, S, meta, cudaMemcpyHostToDevice, st));
  PCK(cudaMemsetAsync(D + o_hist, 0, 4 * kLCodes * nblk_max, st));
  PCK(cudaMemsetAsync(D + o_words, 0, 8 * words, st));

  const PImg* dimgs = (const PImg*)(D + o_imgs);
  const int64_t* dpos = (const int64_t*)(D + o_pos);
  uint8_t* f = D + o_f;
  uint32_t* runs = (uint32_t*)(D + o_runs);
  uint32_t* tok_off = (uint32_t*)(D + o_tok_off);
  uint16_t* tok = (uint16_t*)(D + o_tok);
  uint64_t* off = (uint64_t*)(D + o_off);
  uint32_t* first_run = (uint32_t*)(D + o_first);
  int64_t* tok0 = (int64_t*)(D + o_tok0);
  int64_t* blk0 = (int64_t*)(D + o_blk0);
  State* state = (State*)(D + o_state);
  PBlk* blks = (PBlk*)(D + o_blks);
  uint32_t* hist = (uint32_t*)(D + o_hist);
  uint32_t* lcodes = (uint32_t*)(D + o_lc);
  uint32_t* dcodes = (uint32_t*)(D + o_dc);
  uint64_t* hdr = (uint64_t*)(D + o_hdr);
  TreeWork* work = (TreeWork*)(D + o_work);
  uint32_t* seg_ab = (uint32_t*)(D + o_seg);
  ImgOut* io = (ImgOut*)(D + o_io);
  uint64_t* wbuf = (uint64_t*)(D + o_words);
  uint32_t* crcs = (uint32_t*)(D + o_crc);
  uint8_t* dout = nullptr;                 // the mapped output as the kernels address it
  PCK(cudaHostGetDevicePointer((void**)&dout, e->out, 0));
  int64_t* dsizes = (int64_t*)(dout + align16(out_bytes));
  const int64_t* hsizes = (const int64_t*)(e->out + align16(out_bytes));
  const int kT = 256;
  unsigned grid = (unsigned)imin64(blocks_for(N, kT), 132 * 16);

  png_filter_kernel<<<grid, kT, 0, st>>>(dimgs, dpos, n, N, f);
  run_scan<uint32_t>(N, RunStartItem{f, dpos, n}, RunStartOut{dpos, n, N, runs, first_run, state}, (uint32_t*)(D + o_tiles), st);
  run_scan<uint32_t>(N, RunTokItem{runs, state}, RunTokOut{tok_off, state}, (uint32_t*)(D + o_tiles), st);
  png_imginfo_kernel<<<1, 1, 0, st>>>(dimgs, n, first_run, tok_off, state, tok0, blk0, blks);
  png_token_kernel<<<grid, kT, 0, st>>>(f, runs, tok_off, state, dpos, tok0, blk0, n, tok, blks, hist);
  png_tree_kernel<<<(unsigned)blocks_for(nblk_max, 64), 64, 0, st>>>(blks, blk0, n, hist, (const int64_t*)(D + o_imgN),
                                                                     lcodes, dcodes, hdr, work);
  png_adler_kernel<<<(unsigned)blocks_for(nseg, kT), kT, 0, st>>>(f, dimgs, (const int64_t*)(D + o_segimg), nseg, seg_ab);
  png_offset_kernel<<<(unsigned)blocks_for(n, 128), 128, 0, st>>>(dimgs, n, blk0, blks, seg_ab, io, dsizes);
  run_scan<uint64_t>(N, CostItem{tok, tok0, blk0, n, blks, lcodes, dcodes, state}, CostOut{off}, (uint64_t*)(D + o_tiles), st);
  png_emit_kernel<<<grid, kT, 0, st>>>(tok, off, tok0, blk0, n, blks, lcodes, dcodes, dimgs, state, wbuf);
  png_block_kernel<<<(unsigned)blocks_for(nblk_max * 32, kT), kT, 0, st>>>(blks, blk0, n, hdr, f, dimgs, wbuf);
  png_crc_kernel<<<(unsigned)blocks_for(nchunks, 128), 128, 0, st>>>(dimgs, (const int64_t*)(D + o_chimg), nchunks, io,
                                                                     wbuf, crcs);
  png_assemble_kernel<<<(unsigned)imin64(blocks_for(nunits, kT), 132 * 16), kT, 0, st>>>(
      dimgs, (const int64_t*)(D + o_unit0), n, nunits, io, wbuf, crcs, dout);
  PCK(cudaGetLastError());
  PCK(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    files[i] = e->out + im[i].out_off;
    sizes[i] = hsizes[i];
  }
  return CTD_OK;
}
