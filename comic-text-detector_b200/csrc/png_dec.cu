// GPU PNG decode (C ABI `ctd_png_decoder_*`, `ctd_png_decode`, include/ctd_b200.h): every file of a call at once,
// byte for byte the page cv2.imdecode(buf, IMREAD_COLOR) returns with its libpng 1.6 and zlib 1.2.11.
// oracle/png_decode_ref.py restates every rule; tests/test_cpu_png_decode.py pins it to cv2.
//
// Host: png_plan.cpp's chunk walk (with every chunk's CRC-32), then one pinned staging buffer holding a descriptor
// per file and the zlib streams (IDAT payloads, chunk headers removed), uploaded in one copy.  Device, one launch each:
//   1. png_inflate_kernel, one CTA per file, looping over the file's deflate blocks on the device: thread 0 parses each
//      header and builds the tables; a Huffman block is decoded in chunks of self-synchronised subsequences (pass 1
//      rounds to the fixpoint, a scan, pass 2 from the exact starts), and the match bytes pass 2 could not copy are
//      resolved by pointer jumping.  Every read is bounded by the staged stream, every distance is checked against the
//      output so far and the window before any copy, and the output must end exactly at h * (1 + rowbytes) with the
//      final block's stream ending 4 bytes (the Adler-32) before the zlib stream does.  Any failure marks the file
//      CTD_PNG_DATA.
//   2. png_adler_kernel: Adler-32 of each inflated stream from per-CTA partial sums.
//   3. png_unfilter_kernel, one CTA per file, in place: checks the Adler-32 and the filter types, then reconstructs
//      rows as a wavefront.  Thread t of a group of kUnfilterThreads rows handles row t's bytes [32 s', 32 s' + 32) at
//      step s = s' + t, so a row's bytes run one 32-byte piece behind the row above (every filter reads the row above
//      at the same or lower offsets, and its own row at lower ones).
//   4. png_convert_kernel, one thread per pixel: bit-depth expansion, palette lookup, high byte of 16-bit samples,
//      grey / RGB to BGR, alpha dropped, stored at the pixel's eXIf-oriented position in the caller's page.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "png_dec.h"

int ctd_fail(ctd_handle* h, int code, const char* fmt, ...);

namespace ctd {
namespace png {
namespace {

constexpr int kLutBits = 10;
constexpr int kInflateThreads = 256;    // subsequences per chunk of a Huffman block
constexpr int kDefaultSubBits = 512;
constexpr int kUnfilterThreads = 256;
constexpr int kPiece = 32;              // bytes of a row one unfilter thread handles per step
constexpr int kAdlerBytes = 16384;      // bytes per CTA of png_adler_kernel
constexpr uint32_t kAdlerMod = 65521;

struct DFile {
  int64_t in_off, out_off;
  uint8_t* dst;
  int32_t in_len, out_len;
  int32_t w, h, rowbytes, bpp, depth, ctype, orient, out_w, out_h, window;
  uint32_t adler;
  uint8_t plte[256 * 3];
};

__constant__ uint16_t c_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                        31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                         193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// One canonical Huffman code: 10-bit lookup ((length << 9) | symbol, 0 for a longer or unused code) and puff.c's
// count / sorted-symbol form for the longer codes.
struct Code {
  uint16_t lut[1 << kLutBits];
  uint16_t count[16];
  uint16_t sym[288];
};

// inflate_table's checks and the tables, by one thread.  single_ok: a lone one-bit code is allowed (litlen and
// distance sets, as zlib allows them).  False for a set zlib refuses.
__device__ bool build_code(const uint8_t* lens, int n, bool single_ok, Code* c) {
  for (int l = 0; l < 16; ++l) c->count[l] = 0;
  for (int s = 0; s < n; ++s) c->count[lens[s]]++;
  int left = 1, maxlen = 0;
  for (int l = 1; l < 16; ++l) {
    left = (left << 1) - c->count[l];
    if (left < 0) return false;   // over-subscribed
    if (c->count[l]) maxlen = l;
  }
  if (maxlen == 0) return false;
  if (left > 0 && !(single_ok && maxlen == 1)) return false;   // incomplete
  uint16_t offs[16], next[16];
  c->count[0] = 0;   // unused symbols
  offs[1] = 0;
  for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + c->count[l];
  for (int s = 0; s < n; ++s)
    if (lens[s]) c->sym[offs[lens[s]]++] = (uint16_t)s;
  for (int i = 0; i < (1 << kLutBits); ++i) c->lut[i] = 0;
  int code = 0;
  for (int l = 1; l < 16; ++l) {
    next[l] = (uint16_t)code;
    code = (code + c->count[l]) << 1;
  }
  for (int s = 0; s < n; ++s) {
    int L = lens[s];
    if (!L || L > kLutBits) {
      if (L) next[L]++;
      continue;
    }
    int cd = next[L]++, r = 0;
    for (int b = 0; b < L; ++b) r |= ((cd >> b) & 1) << (L - 1 - b);
    for (int j = r; j < (1 << kLutBits); j += 1 << L) c->lut[j] = (uint16_t)((L << 9) | s);
  }
  return true;
}

// The bit reader of one thread: LSB-first, 64-bit buffer, reads past the staged stream return zero bits and are caught
// by the consumed-bits check.
struct Bits {
  const uint8_t* in;
  uint32_t n, pos;   // staged bytes, next byte to load
  uint64_t buf;
  int cnt;
  __device__ void refill() {
    while (cnt <= 56) {
      buf |= (uint64_t)(pos < n ? in[pos] : 0) << cnt;
      ++pos;
      cnt += 8;
    }
  }
  __device__ uint32_t take(int k) {
    uint32_t v = (uint32_t)(buf & ((1ull << k) - 1));
    buf >>= k;
    cnt -= k;
    return v;
  }
  __device__ int64_t consumed() const { return (int64_t)pos * 8 - cnt; }
};

// one symbol (the buffer holds at least 15 bits); -1 for an invalid code
__device__ __forceinline__ int decode_sym(Bits& b, const Code* c) {
  uint32_t e = c->lut[b.buf & ((1 << kLutBits) - 1)];
  if (e) {
    b.take(e >> 9);
    return e & 511;
  }
  int code = 0, first = 0, index = 0;   // puff.c decode()
  for (int len = 1; len < 16; ++len) {
    code |= (int)((b.buf >> (len - 1)) & 1);
    int count = c->count[len];
    if (code - count < first) {
      b.take(len);
      return c->sym[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// Decodes whole steps (a literal, or a length with its distance) from bit `start` until the reader reaches bit `stop`
// or decodes EOB.  Pass 1 (out == nullptr) only counts: the end bit, the bytes produced, EOB seen.  An invalid code
// consumes one bit and sets `bad`, and the decode goes on, so a subsequence started at a wrong guess still reaches
// its end.  Pass 2 (from an exact start, output position o) writes every literal and every match byte whose source
// is already final (before the chunk, or earlier in this thread's own output and itself final); any other match
// byte gets its source in src[] and its bit in unres[].  Distances are checked before any byte is written.
struct Step {
  int64_t end;
  uint32_t n;
  bool eob, bad;
};

__device__ Step run(const uint8_t* in, uint32_t nbytes, int64_t start, int64_t stop, const Code* lit, const Code* dist,
                    uint8_t* out, uint32_t* src, uint32_t* unres, uint32_t o, uint32_t o_chunk, uint32_t out_len,
                    uint32_t window) {
  Step r{start, 0, false, false};
  const int64_t nbits = (int64_t)nbytes * 8;
  if (start >= nbits) return r;   // a guessed start past the stream: nothing to decode
  stop = min(stop, nbits);
  Bits b{in, nbytes, (uint32_t)(start >> 3), 0, 0};
  b.refill();
  b.take((int)(start & 7));
  const uint32_t o0 = o;
  while (b.consumed() < stop) {
    if (o - o0 > out_len) { r.bad = true; break; }
    b.refill();
    int sym = decode_sym(b, lit);
    if (sym < 0) {
      r.bad = true;
      b.take(1);
      continue;
    }
    if (sym < 256) {
      if (out) {
        if (o >= out_len) { r.bad = true; break; }
        out[o] = (uint8_t)sym;
      }
      ++o;
      continue;
    }
    if (sym == 256) {
      r.eob = true;
      break;
    }
    sym -= 257;
    if (sym >= 29) {
      r.bad = true;
      continue;
    }
    uint32_t len = c_len_base[sym] + b.take(c_len_extra[sym]);
    int ds = decode_sym(b, dist);
    if (ds < 0 || ds >= 30) {
      r.bad = true;
      continue;
    }
    uint32_t d = c_dist_base[ds] + b.take(c_dist_extra[ds]);
    if (out) {
      if (d > o || d > window || o + len > out_len) { r.bad = true; break; }
      for (uint32_t i = 0; i < len; ++i) {
        uint32_t q = o - d + i % d, p = o + i;
        bool final_q = q < o_chunk || (q >= o0 && !((unres[q >> 5] >> (q & 31)) & 1));
        if (final_q) {
          out[p] = out[q];
        } else {
          src[p] = q;
          atomicOr(&unres[p >> 5], 1u << (p & 31));
        }
      }
    }
    o += len;
  }
  r.end = b.consumed();
  r.n = o - o0;
  return r;
}

enum { kCmdHuff = 0, kCmdStored = 1, kCmdDone = 2, kCmdError = 3 };

// One CTA of kInflateThreads per file, looping over the file's deflate blocks on the device.  Thread 0 parses each
// block header and builds the block's tables in shared memory.  A Huffman block is decoded in chunks of
// kInflateThreads subsequences of sub_bits bits: rounds of pass 1 from guessed starts until no start changes (the
// fixpoint of jpeg_sync_kernel), a scan of the bytes each subsequence produces, pass 2 from the exact starts, then
// the match bytes pass 2 could not copy are resolved by pointer jumping over src[] and gathered.
__global__ void __launch_bounds__(kInflateThreads) png_inflate_kernel(const DFile* __restrict__ files,
                                                                      const uint8_t* __restrict__ bytes, uint8_t* work,
                                                                      uint32_t* src_all, uint32_t* unres_all,
                                                                      int64_t sub_bits, int32_t* __restrict__ status,
                                                                      int32_t* __restrict__ stats) {
  __shared__ Code s_lit, s_dist;
  __shared__ uint8_t s_lens[19 + 286 + 30];
  __shared__ int64_t s_start[kInflateThreads + 1], s_end[kInflateThreads];
  __shared__ uint32_t s_off[kInflateThreads + 1];
  __shared__ int64_t s_bit;   // next block header, or the current chunk's first bit
  __shared__ uint32_t s_o;    // bytes written so far
  __shared__ int s_cmd, s_last, s_stop, s_changed, s_bad, s_unres;
  __shared__ uint32_t s_stored_len;
  const DFile& f = files[blockIdx.x];
  const int t = threadIdx.x;
  const uint8_t* in = bytes + f.in_off;
  const uint32_t nbytes = (uint32_t)f.in_len, out_len = (uint32_t)f.out_len;
  const int64_t nbits = (int64_t)nbytes * 8;
  uint8_t* out = work + f.out_off;
  uint32_t* src = src_all + f.out_off;
  uint32_t* unres = unres_all + f.out_off / 32;
  int blocks = 0, rounds = 0;
  bool failed = false;
  if (t == 0) {
    s_bad = 0;
    s_bit = 16;   // after the zlib header
    s_o = 0;
    s_last = 0;
  }
  __syncthreads();
  for (;;) {
    // 1. the block header, by thread 0
    if (t == 0) {
      int cmd = kCmdHuff;
      if (s_last) {
        int64_t end = (s_bit + 7) / 8;
        cmd = (end + 4 == (int64_t)nbytes && s_o == out_len) ? kCmdDone : kCmdError;
      } else {
        Bits b{in, nbytes, (uint32_t)(s_bit >> 3), 0, 0};
        b.refill();
        b.take((int)(s_bit & 7));
        s_last = b.take(1);
        int type = b.take(2);
        bool ok = true;
        if (type == 0) {
          b.take(b.cnt & 7);
          uint32_t len = b.take(16), nlen = b.take(16);
          ok = (len ^ 0xffffu) == nlen && s_o + len <= out_len && b.consumed() / 8 + len <= nbytes;
          s_stored_len = len;
          cmd = kCmdStored;
        } else if (type == 3) {
          ok = false;
        } else if (type == 1) {
          for (int s = 0; s < 288; ++s) s_lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
          for (int s = 0; s < 32; ++s) s_lens[288 + s] = 5;   // codes 30 and 31 exist and are invalid
          ok = build_code(s_lens, 288, true, &s_lit) && build_code(s_lens + 288, 32, true, &s_dist);
        } else {
          int nlit = b.take(5) + 257, ndist = b.take(5) + 1, ncl = b.take(4) + 4;
          ok = nlit <= 286 && ndist <= 30;
          for (int i = 0; i < 19; ++i) s_lens[c_clen_order[i]] = 0;
          b.refill();
          for (int i = 0; i < ncl; ++i) s_lens[c_clen_order[i]] = (uint8_t)b.take(3);
          ok = ok && build_code(s_lens, 19, false, &s_lit);   // the code-length code, in the litlen slot
          int k = 0;
          while (ok && k < nlit + ndist) {
            b.refill();
            int sym = decode_sym(b, &s_lit);
            if (sym < 0) { ok = false; break; }
            if (sym < 16) {
              s_lens[19 + k++] = (uint8_t)sym;
              continue;
            }
            int rep, v = 0;
            if (sym == 16) {
              if (k == 0) { ok = false; break; }
              v = s_lens[19 + k - 1];
              rep = 3 + b.take(2);
            } else if (sym == 17) {
              rep = 3 + b.take(3);
            } else {
              rep = 11 + b.take(7);
            }
            if (k + rep > nlit + ndist) { ok = false; break; }
            while (rep--) s_lens[19 + k++] = (uint8_t)v;
          }
          if (ok) {
            for (int i = 0; i < nlit + ndist; ++i) s_lens[i] = s_lens[19 + i];
            ok = s_lens[256] != 0 && build_code(s_lens, nlit, true, &s_lit) &&
                 build_code(s_lens + nlit, ndist, true, &s_dist);
          }
        }
        if (!ok || b.consumed() > nbits) cmd = kCmdError;
        s_bit = b.consumed();
      }
      s_cmd = cmd;
    }
    __syncthreads();
    const int cmd = s_cmd;
    if (cmd == kCmdError || cmd == kCmdDone) break;
    ++blocks;
    if (cmd == kCmdStored) {
      const uint32_t len = s_stored_len, o = s_o;
      const int64_t at = s_bit / 8;
      for (uint32_t i = t; i < len; i += kInflateThreads) out[o + i] = in[at + i];
      __syncthreads();
      if (t == 0) {
        s_bit = (at + len) * 8;
        s_o = o + len;
      }
      __syncthreads();
      continue;
    }
    // 2. the Huffman block, chunk by chunk
    for (;;) {
      const int64_t b0 = s_bit;
      const uint32_t o_chunk = s_o;
      int64_t stop = b0 + (int64_t)(t + 1) * sub_bits;
      s_start[t] = b0 + (int64_t)t * sub_bits;
      Step r;
      for (;;) {   // pass 1 rounds
        if (t == 0) {
          s_stop = kInflateThreads;
          s_changed = 0;
        }
        __syncthreads();
        r = run(in, nbytes, s_start[t], stop, &s_lit, &s_dist, nullptr, nullptr, nullptr, 0, 0, out_len, f.window);
        s_end[t] = r.end;
        if (r.eob) atomicMin(&s_stop, t);
        __syncthreads();
        ++rounds;
        if (t < s_stop && t + 1 < kInflateThreads && s_start[t + 1] != r.end) {
          s_start[t + 1] = r.end;
          s_changed = 1;
        }
        __syncthreads();
        const bool again = s_changed;
        __syncthreads();   // every thread has read the flag before thread 0 clears it for the next round
        if (!again) break;
      }
      const int last = s_stop;   // the subsequence holding EOB, or kInflateThreads
      s_off[t + 1] = t <= last ? r.n : 0;
      __syncthreads();
      if (t == 0) {
        uint64_t acc = o_chunk;
        s_off[0] = o_chunk;
        for (int i = 1; i <= kInflateThreads; ++i) {
          acc += s_off[i];
          s_off[i] = acc > out_len ? out_len + 1 : (uint32_t)acc;
        }
        s_bad = acc > out_len;
        s_unres = 0;
      }
      __syncthreads();
      if (s_bad) {
        failed = true;
        break;
      }
      // pass 2 from the exact starts
      if (t <= last && t < kInflateThreads) {
        Step w = run(in, nbytes, s_start[t], stop, &s_lit, &s_dist, out, src, unres, s_off[t], o_chunk, out_len,
                     f.window);
        if (w.bad || w.n != s_off[t + 1] - s_off[t]) s_bad = 1;
      }
      __syncthreads();
      const uint32_t o_end = s_off[kInflateThreads];
      const int64_t chunk_end = s_end[last < kInflateThreads ? last : kInflateThreads - 1];
      if (s_bad || chunk_end > nbits) {
        failed = true;
        break;
      }
      // LZ77 resolution: pointer jumping over the bytes pass 2 left, then one gather
      const uint32_t w0 = o_chunk >> 5, w1 = (o_end + 31) >> 5;
      for (uint32_t wd = w0 + t; wd < w1; wd += kInflateThreads)
        if (unres[wd]) s_unres = 1;
      __syncthreads();
      if (s_unres) {
        for (;;) {
          if (t == 0) s_changed = 0;
          __syncthreads();
          for (uint32_t wd = w0 + t; wd < w1; wd += kInflateThreads) {
            uint32_t m = unres[wd];
            while (m) {
              uint32_t p = (wd << 5) + __ffs(m) - 1;
              m &= m - 1;
              uint32_t q = src[p];
              if (q >= o_chunk && ((unres[q >> 5] >> (q & 31)) & 1)) {
                src[p] = src[q];
                s_changed = 1;
              }
            }
          }
          __syncthreads();
          const bool again = s_changed;
          __syncthreads();
          if (!again) break;
        }
        for (uint32_t wd = w0 + t; wd < w1; wd += kInflateThreads) {
          uint32_t m = unres[wd];
          while (m) {
            uint32_t p = (wd << 5) + __ffs(m) - 1;
            m &= m - 1;
            out[p] = out[src[p]];
          }
        }
        __syncthreads();
        for (uint32_t wd = w0 + t; wd < w1; wd += kInflateThreads) unres[wd] = 0;
      }
      __syncthreads();
      if (t == 0) {
        s_o = o_end;
        s_bit = chunk_end;
      }
      __syncthreads();
      if (last < kInflateThreads) break;   // EOB: the next block header follows
    }
    if (failed) break;
  }
  if (t == 0) {
    if (failed || s_cmd != kCmdDone) status[blockIdx.x] = CTD_PNG_DATA;
    stats[2 * blockIdx.x] = blocks;
    stats[2 * blockIdx.x + 1] = rounds;
  }
}

// grid (ceil(max filtered / kAdlerBytes), files): sums[2 f] += sum of bytes, sums[2 f + 1] += sum of (len - i) * byte,
// each mod 65521
__global__ void __launch_bounds__(256) png_adler_kernel(const DFile* __restrict__ files, const uint8_t* __restrict__ work,
                                                        const int32_t* __restrict__ status,
                                                        unsigned long long* __restrict__ sums) {
  const DFile& f = files[blockIdx.y];
  int64_t i0 = (int64_t)blockIdx.x * kAdlerBytes;
  if (i0 >= f.out_len || status[blockIdx.y]) return;
  int64_t i1 = min((int64_t)f.out_len, i0 + kAdlerBytes);
  const uint8_t* p = work + f.out_off;
  uint64_t a = 0, w = 0;
  for (int64_t i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
    uint32_t v = p[i];
    a += v;
    w += (uint64_t)((f.out_len - i) % kAdlerMod) * v;
  }
  __shared__ uint64_t s_a[256], s_w[256];
  s_a[threadIdx.x] = a % kAdlerMod;
  s_w[threadIdx.x] = w % kAdlerMod;
  __syncthreads();
  for (int s = 128; s; s >>= 1) {
    if (threadIdx.x < s) {
      s_a[threadIdx.x] += s_a[threadIdx.x + s];
      s_w[threadIdx.x] += s_w[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    atomicAdd(&sums[2 * blockIdx.y], (unsigned long long)(s_a[0] % kAdlerMod));
    atomicAdd(&sums[2 * blockIdx.y + 1], (unsigned long long)(s_w[0] % kAdlerMod));
  }
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
  int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// one CTA per file, in place on the inflated stream
__global__ void __launch_bounds__(kUnfilterThreads) png_unfilter_kernel(const DFile* __restrict__ files, uint8_t* work,
                                                                        const unsigned long long* __restrict__ sums,
                                                                        int32_t* __restrict__ status) {
  const DFile& f = files[blockIdx.x];
  __shared__ int s_bad;
  if (status[blockIdx.x]) return;
  const int t = threadIdx.x;
  const int64_t stride = 1 + (int64_t)f.rowbytes;
  uint8_t* img = work + f.out_off;
  if (t == 0) {
    uint32_t a = (uint32_t)((1 + sums[2 * blockIdx.x]) % kAdlerMod);
    uint32_t bsum = (uint32_t)(((uint64_t)f.out_len + sums[2 * blockIdx.x + 1]) % kAdlerMod);
    s_bad = ((bsum << 16) | a) != f.adler;
  }
  __syncthreads();
  for (int y = t; y < f.h; y += kUnfilterThreads)
    if (img[y * stride] > 4) s_bad = 1;
  __syncthreads();
  if (s_bad) {
    if (t == 0) status[blockIdx.x] = CTD_PNG_DATA;
    return;
  }
  const int rb = f.rowbytes, bpp = f.bpp;
  const int pieces = (rb + kPiece - 1) / kPiece;
  for (int y0 = 0; y0 < f.h; y0 += kUnfilterThreads) {
    const int y = y0 + t;
    const bool live = y < f.h;
    uint8_t* row = img + (int64_t)y * stride + 1;
    const uint8_t* up = row - stride;
    const int ft = live ? row[-1] : 0;
    for (int s = 0; s < pieces + kUnfilterThreads - 1; ++s) {
      int pc = s - t;
      if (live && pc >= 0 && pc < pieces && ft) {
        int x1 = min(rb, (pc + 1) * kPiece);
        for (int x = pc * kPiece; x < x1; ++x) {
          int a = x >= bpp ? row[x - bpp] : 0;
          int b = y > 0 ? up[x] : 0;
          int c = (x >= bpp && y > 0) ? up[x - bpp] : 0;
          int pr = ft == 1 ? a : ft == 2 ? b : ft == 3 ? (a + b) >> 1 : paeth(a, b, c);
          row[x] = (uint8_t)(row[x] + pr);
        }
      }
      __syncthreads();
    }
  }
}

// grid (ceil(max pixels / 256), files): one thread per image pixel
__global__ void __launch_bounds__(256) png_convert_kernel(const DFile* __restrict__ files, const uint8_t* __restrict__ work,
                                                          const int32_t* __restrict__ status) {
  const DFile& f = files[blockIdx.y];
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)f.w * f.h || status[blockIdx.y]) return;
  int y = (int)(i / f.w), x = (int)(i - (int64_t)y * f.w);
  const uint8_t* row = work + f.out_off + (int64_t)y * (1 + (int64_t)f.rowbytes) + 1;
  const int d = f.depth;
  uint8_t B, G, R;
  if (d < 8) {   // grey or palette of 1, 2 or 4 bits, most significant bits first
    int bit = x * d;
    int v = (row[bit >> 3] >> (8 - d - (bit & 7))) & ((1 << d) - 1);
    if (f.ctype == 3) {
      R = f.plte[3 * v], G = f.plte[3 * v + 1], B = f.plte[3 * v + 2];
    } else {
      B = G = R = (uint8_t)(v * (d == 1 ? 255 : d == 2 ? 85 : 17));
    }
  } else {
    const int sb = d >> 3;   // bytes per sample; a 16-bit sample keeps its first (high) byte
    switch (f.ctype) {
      case 0: case 4:
        B = G = R = row[(int64_t)x * sb * (f.ctype == 4 ? 2 : 1)];
        break;
      case 3: {
        int v = row[x];
        R = f.plte[3 * v], G = f.plte[3 * v + 1], B = f.plte[3 * v + 2];
        break;
      }
      default: {   // RGB, RGBA
        const uint8_t* px = row + (int64_t)x * sb * (f.ctype == 6 ? 4 : 3);
        R = px[0], G = px[sb], B = px[2 * sb];
      }
    }
  }
  // OpenCV ExifTransform: transpose for 5..8, then flip (columns for 2, 3, 6, 7; rows for 3, 4, 7, 8)
  int orow = y, ocol = x, ot = f.orient;
  if (ot >= 5) {
    orow = x;
    ocol = y;
  }
  if (ot == 2 || ot == 3 || ot == 6 || ot == 7) ocol = f.out_w - 1 - ocol;
  if (ot == 3 || ot == 4 || ot == 7 || ot == 8) orow = f.out_h - 1 - orow;
  uint8_t* o = f.dst + ((int64_t)orow * f.out_w + ocol) * 3;
  o[0] = B;
  o[1] = G;
  o[2] = R;
}

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// grows a pinned or device buffer to at least `need` bytes (by a quarter more, as the JPEG decoder's buffers grow)
int grow(uint8_t** buf, size_t* cap, size_t need, bool pinned) {
  if (*cap >= need) return CTD_OK;
  if (pinned) cudaFreeHost(*buf); else cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  size_t n = need + need / 4;
  cudaError_t e = pinned ? cudaMallocHost((void**)buf, n) : cudaMalloc((void**)buf, n);
  if (e != cudaSuccess) return ctd_fail(nullptr, CTD_E_CUDA, "png decoder: allocating %zu bytes: %s", n, cudaGetErrorString(e));
  *cap = n;
  return CTD_OK;
}

}  // namespace
}  // namespace png
}  // namespace ctd

using namespace ctd::png;

struct ctd_png_decoder {
  int device = 0;
  int64_t sub_bits = kDefaultSubBits;
  int64_t blocks = 0, rounds = 0;   // of the last call's GPU-decoded files
  cudaStream_t stream = nullptr;
  uint8_t* host = nullptr;   // pinned staging: descriptors, statuses and zlib streams of one call
  size_t host_cap = 0;
  uint8_t* dev = nullptr;    // its device mirror
  size_t dev_cap = 0;
  uint8_t* work = nullptr;   // Adler sums and the inflated streams
  size_t work_cap = 0;
};

#define PCK(expr)                                                                                           \
  do {                                                                                                      \
    cudaError_t _e = (expr);                                                                                \
    if (_e != cudaSuccess)                                                                                  \
      return ctd_fail(nullptr, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

extern "C" CTD_API int ctd_png_decoder_create(int32_t device, int32_t subsequence_bits, ctd_png_decoder** out) {
  if (!out || subsequence_bits < 0) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_decoder_create: bad argument");
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n)
    return ctd_fail(nullptr, CTD_E_NO_DEVICE, "ctd_png_decoder_create: no CUDA device %d (no CPU fallback)", device);
  cudaDeviceProp prop;
  PCK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return ctd_fail(nullptr, CTD_E_NO_DEVICE, "device %d is sm_%d%d, not sm_90", device, prop.major, prop.minor);
  PCK(cudaSetDevice(device));
  ctd_png_decoder* d = new ctd_png_decoder;
  d->device = device;
  if (subsequence_bits) d->sub_bits = subsequence_bits;
  cudaError_t e = cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    ctd_png_decoder_destroy(d);
    return ctd_fail(nullptr, CTD_E_CUDA, "ctd_png_decoder_create: %s", cudaGetErrorString(e));
  }
  *out = d;
  return CTD_OK;
}

extern "C" CTD_API void ctd_png_decoder_destroy(ctd_png_decoder* d) {
  if (!d) return;
  cudaSetDevice(d->device);
  if (d->stream) cudaStreamSynchronize(d->stream);
  cudaFreeHost(d->host);
  cudaFree(d->dev);
  cudaFree(d->work);
  if (d->stream) cudaStreamDestroy(d->stream);
  delete d;
}

extern "C" CTD_API int ctd_png_decode(ctd_png_decoder* d, const uint8_t* const* data, const size_t* len, int32_t n,
                                      uint8_t* const* dst, int32_t* status) {
  if (!d || n < 0 || (n && (!data || !len || !dst || !status)))
    return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_decode: bad argument");
  PCK(cudaSetDevice(d->device));
  // 1. host: walk every file (CRCs included), lay out the call
  std::vector<File> files(n);
  std::vector<int> live;
  for (int i = 0; i < n; ++i) {
    status[i] = data[i] ? parse(data[i], len[i], &files[i], true) : CTD_PNG_NOT_PNG;
    if (status[i] == CTD_PNG_OK) {
      if (!dst[i]) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_decode: file %d decodes but dst[%d] is NULL", i, i);
      live.push_back(i);
    }
  }
  d->blocks = d->rounds = 0;
  if (live.empty()) return CTD_OK;
  const int np = (int)live.size();
  // the per-file grids of the Adler-32 and convert kernels put the file in gridDim.y
  if (np > 65535)
    return ctd_fail(nullptr, CTD_E_CAPACITY, "ctd_png_decode: %d decodable files in one call (at most 65535)", np);
  size_t in_bytes = 0, out_bytes = 0;
  int64_t max_out = 0, max_px = 0;
  for (int i : live) {
    in_bytes += align_up(files[i].zlen, 16);
    out_bytes += align_up((size_t)files[i].filtered, 256);
    max_out = std::max(max_out, files[i].filtered);
    max_px = std::max(max_px, (int64_t)files[i].w * files[i].h);
  }
  size_t o_files = 0;
  size_t o_status = align_up(o_files + np * sizeof(DFile), 256);
  size_t o_stats = align_up(o_status + np * sizeof(int32_t), 256);
  size_t o_in = align_up(o_stats + 2 * np * sizeof(int32_t), 256);
  size_t host_bytes = o_in + in_bytes + 16;
  int rc = grow(&d->host, &d->host_cap, host_bytes, true);
  if (rc) return rc;
  uint8_t* H = d->host;
  DFile* df = (DFile*)(H + o_files);
  int32_t* dstatus = (int32_t*)(H + o_status);
  // 2. host: stage every zlib stream, fill the descriptors
  size_t boff = 0, ooff = 0;
  static const int kChannels[7] = {1, 0, 3, 1, 2, 0, 4};
  for (int p = 0; p < np; ++p) {
    const File& f = files[live[p]];
    DFile& g = df[p];
    memset(&g, 0, sizeof(g));
    uint8_t* s = H + o_in + boff;
    size_t k = 0;
    for (size_t c = 0; c < f.idat_off.size(); ++c) {
      memcpy(s + k, data[live[p]] + f.idat_off[c], f.idat_len[c]);
      k += f.idat_len[c];
    }
    g.in_off = (int64_t)boff;
    g.in_len = (int32_t)f.zlen;
    g.out_off = (int64_t)ooff;
    g.out_len = (int32_t)f.filtered;
    g.dst = dst[live[p]];
    g.w = f.w;
    g.h = f.h;
    g.rowbytes = (int32_t)f.rowbytes;
    g.bpp = std::max(1, kChannels[f.ctype] * f.depth / 8);
    g.depth = f.depth;
    g.ctype = f.ctype;
    g.orient = f.orient;
    g.out_w = f.orient >= 5 ? f.h : f.w;
    g.out_h = f.orient >= 5 ? f.w : f.h;
    g.window = f.window;
    const uint8_t* a = s + f.zlen - 4;
    g.adler = ((uint32_t)a[0] << 24) | ((uint32_t)a[1] << 16) | ((uint32_t)a[2] << 8) | a[3];
    memcpy(g.plte, f.plte, sizeof(g.plte));
    dstatus[p] = 0;
    boff += align_up(f.zlen, 16);
    ooff += align_up((size_t)f.filtered, 256);
  }
  memset(H + o_in + boff, 0, 16);
  // 3. device buffers
  // Adler sums, the inflated streams, each output byte's LZ77 source and a bit per byte left for pointer jumping
  size_t w_sums = 0, w_out = align_up(w_sums + 2 * np * sizeof(unsigned long long), 256);
  size_t w_src = align_up(w_out + out_bytes, 256), w_unres = align_up(w_src + 4 * out_bytes, 256);
  if ((rc = grow(&d->dev, &d->dev_cap, host_bytes, false))) return rc;
  if ((rc = grow(&d->work, &d->work_cap, w_unres + out_bytes / 8, false))) return rc;
  uint8_t* D = d->dev;
  uint8_t* W = d->work;
  cudaStream_t st = d->stream;
  const DFile* gf = (const DFile*)(D + o_files);
  int32_t* gstatus = (int32_t*)(D + o_status);
  unsigned long long* sums = (unsigned long long*)(W + w_sums);
  uint8_t* out = W + w_out;
  PCK(cudaMemcpyAsync(D, H, host_bytes, cudaMemcpyHostToDevice, st));
  PCK(cudaMemsetAsync(sums, 0, 2 * np * sizeof(unsigned long long), st));
  PCK(cudaMemsetAsync(W + w_unres, 0, out_bytes / 8, st));
  int32_t* gstats = (int32_t*)(D + o_stats);
  // 4. inflate, Adler-32, unfilter, convert
  png_inflate_kernel<<<np, kInflateThreads, 0, st>>>(gf, D + o_in, out, (uint32_t*)(W + w_src),
                                                     (uint32_t*)(W + w_unres), d->sub_bits, gstatus, gstats);
  png_adler_kernel<<<dim3((unsigned)((max_out + kAdlerBytes - 1) / kAdlerBytes), np), 256, 0, st>>>(gf, out, gstatus, sums);
  png_unfilter_kernel<<<np, kUnfilterThreads, 0, st>>>(gf, out, sums, gstatus);
  png_convert_kernel<<<dim3((unsigned)((max_px + 255) / 256), np), 256, 0, st>>>(gf, out, gstatus);
  PCK(cudaGetLastError());
  PCK(cudaMemcpyAsync(dstatus, gstatus, (o_in - o_status), cudaMemcpyDeviceToHost, st));
  PCK(cudaStreamSynchronize(st));
  const int32_t* stats = (const int32_t*)(H + o_stats);
  for (int p = 0; p < np; ++p) {
    status[live[p]] = dstatus[p];
    d->blocks += stats[2 * p];
    d->rounds += stats[2 * p + 1];
  }
  return CTD_OK;
}

extern "C" CTD_API int ctd_png_decoder_stats(const ctd_png_decoder* d, int64_t* blocks, int64_t* rounds) {
  if (!d || !blocks || !rounds) return ctd_fail(nullptr, CTD_E_INVALID, "ctd_png_decoder_stats: bad argument");
  *blocks = d->blocks;
  *rounds = d->rounds;
  return CTD_OK;
}
