// Host side of the GPU JPEG decoder (C ABI `ctd_jpeg_probe`, include/ctd_b200.h): the marker walk that decides
// whether the GPU path takes a file, and the staging step that prepares its scan for upload.
//
// The walk accepts exactly the files whose decode jpeg.cu restates: baseline / extended sequential Huffman, 8-bit,
// one interleaved scan of every component in frame order, one component or YCbCr with luma 1x1 / 2x1 / 2x2 and chroma
// 1x1.  Colour space follows libjpeg-turbo's guess (jdapimin.c default_decompress_parms) only where it is certainly
// YCbCr: an Adobe APP14 transform other than 1, or component ids 'R', 'G', 'B', send the file to cv2.  The Huffman
// tables are checked as jdhuff.c jpeg_make_d_derived_tbl checks them (no all-ones code, DC symbols <= 15).  The scan
// is walked to its EOI: restart markers must come in order and number one less than the intervals; any other marker,
// fill bytes or a missing EOI decline the file.  EXIF orientation is read from IFD0 as OpenCV's ExifReader reads it,
// and the block must parse cleanly (every entry's data inside it, orientation one SHORT in 1..8, and only one
// orientation entry).  A scan of 2^28 bytes or more (bit offsets past int32) is left to cv2 as well.
// Stateless and thread-safe.  oracle/jpeg_ref.py restates the same rules in numpy.
#include <string.h>

#include "jpeg.h"

namespace ctd {
namespace jpeg {
namespace {

const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

inline int u16be(const uint8_t* p) { return (p[0] << 8) | p[1]; }

constexpr size_t kMaxScanBytes = size_t(1) << 28;   // 2^31 bits

// jdhuff.c jpeg_make_d_derived_tbl plus a kLutBits lookahead table; false for a table libjpeg refuses
bool derive(const uint8_t* counts, const uint8_t* vals, int nvals, bool dc, HuffTable* t) {
  memset(t, 0, sizeof(*t));
  memcpy(t->vals, vals, nvals);
  int code = 0, k = 0;
  for (int L = 1; L <= 16; ++L) {
    t->valoff[L] = k - code;
    t->maxcode[L] = counts[L - 1] ? code + counts[L - 1] - 1 : -1;
    for (int i = 0; i < counts[L - 1]; ++i, ++k, ++code) {
      if (code >= (1 << L) - 1) return false;   // the all-ones code of each length stays unused
      if (L <= kLutBits) {
        int shift = kLutBits - L;
        for (int j = 0; j < (1 << shift); ++j) t->lut[(code << shift) | j] = (uint16_t)((L << 8) | vals[k]);
      }
    }
    if (code >= (1 << L)) return false;
    code <<= 1;
  }
  t->maxcode[0] = -1;
  t->maxcode[17] = 0x7fffffff;
  if (dc)
    for (int i = 0; i < nvals; ++i)
      if (vals[i] > 15) return false;
  return true;
}

// the scan from its first byte: restart markers in order, then EOI.  Sets scan_end and n_intervals.
int walk_scan(const uint8_t* d, size_t n, Frame* f) {
  size_t q = f->scan_begin;
  int rst = 0;
  for (;;) {
    const void* ff = q < n ? memchr(d + q, 0xFF, n - q) : nullptr;
    if (!ff) return CTD_JPEG_TRUNCATED;
    q = (const uint8_t*)ff - d;
    if (q + 1 >= n) return CTD_JPEG_TRUNCATED;
    uint8_t m = d[q + 1];
    if (m == 0x00) {
      q += 2;
    } else if (m >= 0xD0 && m <= 0xD7) {
      if (!f->restart || m != 0xD0 + (rst & 7)) return CTD_JPEG_ENTROPY;
      ++rst;
      q += 2;
    } else if (m == 0xD9) {
      f->scan_end = q;
      break;
    } else {
      return (m == 0xDA || m == 0xDC) ? CTD_JPEG_SCANS : CTD_JPEG_ENTROPY;
    }
  }
  // the decoder keeps an interval's bit offsets in 32 bits
  if (f->scan_end - f->scan_begin >= kMaxScanBytes) return CTD_JPEG_SIZE;
  int64_t nmcu = (int64_t)f->mcux * f->mcuy;
  int64_t nint = f->restart ? (nmcu + f->restart - 1) / f->restart : 1;
  if (rst + 1 != nint) return CTD_JPEG_ENTROPY;
  f->n_intervals = (int)nint;
  return CTD_JPEG_OK;
}

}  // namespace

struct Tiff {
  const uint8_t* p;
  size_t n;
  bool le;
  uint32_t u16(size_t o) const { return le ? p[o] | (p[o + 1] << 8) : (p[o] << 8) | p[o + 1]; }
  uint32_t u32(size_t o) const {
    return le ? p[o] | (p[o + 1] << 8) | (p[o + 2] << 16) | ((uint32_t)p[o + 3] << 24)
              : ((uint32_t)p[o] << 24) | (p[o + 1] << 16) | (p[o + 2] << 8) | p[o + 3];
  }
};

int exif_orientation(const uint8_t* p, size_t n) {
  if (n < 8 || !((p[0] == 'I' && p[1] == 'I') || (p[0] == 'M' && p[1] == 'M'))) return 0;
  Tiff t{p, n, p[0] == 'I'};
  if (t.u16(2) != 42) return 0;
  uint64_t ifd = t.u32(4);
  if (ifd < 8 || ifd + 2 > n) return 0;
  uint64_t cnt = t.u16(ifd);
  if (ifd + 2 + 12 * cnt > n) return 0;
  static const int kSize[13] = {0, 1, 1, 2, 4, 8, 1, 1, 2, 4, 8, 4, 8};
  int orient = 1;
  bool seen = false;
  for (uint64_t i = 0; i < cnt; ++i) {
    size_t o = ifd + 2 + 12 * i;
    uint32_t tag = t.u16(o), typ = t.u16(o + 2), c = t.u32(o + 4);
    if (typ < 1 || typ > 12) return 0;
    uint64_t nb = (uint64_t)kSize[typ] * c;
    if (nb > 4 && (uint64_t)t.u32(o + 8) + nb > n) return 0;
    if (tag == 0x0112) {
      // a second orientation entry: OpenCV takes the first, other readers the last; left to cv2
      if (seen) return 0;
      seen = true;
      if (typ != 3 || c != 1) return 0;
      orient = (int)t.u16(o + 8);
      if (orient < 1 || orient > 8) return 0;
    }
  }
  return orient;
}

int parse(const uint8_t* d, size_t n, Frame* f) {
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return CTD_JPEG_NOT_JPEG;
  struct Ht { bool set = false; uint8_t counts[16]; uint8_t vals[256]; int nvals = 0; } ht[2][4];
  bool qset[4] = {false, false, false, false};
  bool frame = false, exif = false;
  int adobe = -1;
  int cid[3] = {0, 0, 0};
  size_t p = 2;
  for (;;) {
    if (p >= n) return CTD_JPEG_TRUNCATED;
    if (d[p] != 0xFF) return CTD_JPEG_NOT_JPEG;
    while (p < n && d[p] == 0xFF) ++p;   // fill bytes before a marker
    if (p >= n) return CTD_JPEG_TRUNCATED;
    uint8_t m = d[p++];
    if (m == 0xD9) return CTD_JPEG_TRUNCATED;   // EOI before any scan
    if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
    if (p + 2 > n) return CTD_JPEG_TRUNCATED;
    size_t L = u16be(d + p);
    if (L < 2 || p + L > n) return CTD_JPEG_TRUNCATED;
    const uint8_t* s = d + p + 2;
    size_t sl = L - 2;
    p += L;
    if (m == 0xC0 || m == 0xC1) {
      if (frame) return CTD_JPEG_SCANS;
      if (sl < 6) return CTD_JPEG_TRUNCATED;
      if (s[0] != 8) return CTD_JPEG_PRECISION;
      f->h = u16be(s + 1);
      f->w = u16be(s + 3);
      f->ncomp = s[5];
      if (f->h == 0) return CTD_JPEG_SCANS;   // height defined by DNL
      if (f->w == 0) return CTD_JPEG_TRUNCATED;
      if (sl != 6 + 3 * (size_t)f->ncomp) return CTD_JPEG_TRUNCATED;
      if (f->ncomp != 1 && f->ncomp != 3) return CTD_JPEG_COLOR;
      for (int c = 0; c < f->ncomp; ++c) {
        cid[c] = s[6 + 3 * c];
        f->ch[c] = s[7 + 3 * c] >> 4;
        f->cv[c] = s[7 + 3 * c] & 15;
        f->q[c] = s[8 + 3 * c];
        if (f->q[c] > 3) return CTD_JPEG_TABLES;
      }
      frame = true;
    } else if (m == 0xC2 || m == 0xC6) {
      return CTD_JPEG_PROGRESSIVE;
    } else if (m >= 0xC9 && m <= 0xCF) {
      return m == 0xCA || m == 0xCE ? CTD_JPEG_PROGRESSIVE : CTD_JPEG_ARITHMETIC;
    } else if (m == 0xC3 || m == 0xC5 || m == 0xC7) {
      return CTD_JPEG_LOSSLESS;
    } else if (m == 0xC4) {
      size_t q = 0;
      while (q < sl) {
        if (q + 17 > sl) return CTD_JPEG_TABLES;
        int tc = s[q] >> 4, th = s[q] & 15, tot = 0;
        for (int i = 0; i < 16; ++i) tot += s[q + 1 + i];
        if (tc > 1 || th > 3 || tot > 256 || q + 17 + tot > sl) return CTD_JPEG_TABLES;
        Ht& h = ht[tc][th];
        h.set = true;
        memcpy(h.counts, s + q + 1, 16);
        memcpy(h.vals, s + q + 17, tot);
        h.nvals = tot;
        q += 17 + tot;
      }
    } else if (m == 0xDB) {
      size_t q = 0;
      while (q < sl) {
        int pq = s[q] >> 4, tq = s[q] & 15;
        size_t sz = pq ? 128 : 64;
        if (pq > 1 || tq > 3 || q + 1 + sz > sl) return CTD_JPEG_TABLES;
        for (int i = 0; i < 64; ++i) {
          int v = pq ? u16be(s + q + 1 + 2 * i) : s[q + 1 + i];
          if (v > 32767) return CTD_JPEG_TABLES;   // libjpeg-turbo's SIMD IDCT multiplies in 16 bits
          f->quant[tq][kZigzag[i]] = v;
        }
        qset[tq] = true;
        q += 1 + sz;
      }
    } else if (m == 0xDD) {
      if (sl != 2) return CTD_JPEG_TRUNCATED;
      f->restart = u16be(s);
    } else if (m == 0xE1 && sl >= 6 && memcmp(s, "Exif\0\0", 6) == 0) {
      if (exif) return CTD_JPEG_EXIF;
      exif = true;
      f->orient = exif_orientation(s + 6, sl - 6);
      if (!f->orient) return CTD_JPEG_EXIF;
    } else if (m == 0xEE && sl >= 12 && memcmp(s, "Adobe", 5) == 0) {
      adobe = s[11];
    } else if (m == 0xDA) {
      if (!frame) return CTD_JPEG_TRUNCATED;
      int ns = sl ? s[0] : 0;
      if (sl != 4 + 2 * (size_t)ns || ns != f->ncomp) return CTD_JPEG_SCANS;
      int tdc[3], tac[3];
      for (int c = 0; c < ns; ++c) {
        if (s[1 + 2 * c] != cid[c]) return CTD_JPEG_SCANS;
        tdc[c] = s[2 + 2 * c] >> 4;
        tac[c] = s[2 + 2 * c] & 15;
        if (tdc[c] > 3 || tac[c] > 3) return CTD_JPEG_TABLES;
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return CTD_JPEG_PROGRESSIVE;
      if (f->ncomp == 3) {
        if ((cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B') || (adobe >= 0 && adobe != 1)) return CTD_JPEG_COLOR;
        bool luma_ok = (f->ch[0] == 1 && f->cv[0] == 1) || (f->ch[0] == 2 && f->cv[0] == 1) ||
                       (f->ch[0] == 2 && f->cv[0] == 2);
        if (!luma_ok || f->ch[1] != 1 || f->cv[1] != 1 || f->ch[2] != 1 || f->cv[2] != 1) return CTD_JPEG_SAMPLING;
        f->hmax = f->ch[0];
        f->vmax = f->cv[0];
      } else {
        f->ch[0] = f->cv[0] = 1;
        f->hmax = f->vmax = 1;
      }
      f->tables.clear();
      for (int c = 0; c < ns; ++c) {
        if (!qset[f->q[c]]) return CTD_JPEG_TABLES;
        for (int k = 0; k < 2; ++k) {
          const Ht& h = ht[k][k ? tac[c] : tdc[c]];
          HuffTable t;
          if (!h.set || !derive(h.counts, h.vals, h.nvals, k == 0, &t)) return CTD_JPEG_TABLES;
          (k ? f->ac : f->dc)[c] = (int)f->tables.size();
          f->tables.push_back(t);
        }
      }
      f->mcux = (f->w + 8 * f->hmax - 1) / (8 * f->hmax);
      f->mcuy = (f->h + 8 * f->vmax - 1) / (8 * f->vmax);
      f->scan_begin = p;
      return walk_scan(d, n, f);
    } else if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) {
      // other APPn and COM: skipped, as libjpeg skips them
    } else {
      return m == 0x00 ? CTD_JPEG_NOT_JPEG : CTD_JPEG_SCANS;
    }
  }
}

size_t stage(const uint8_t* d, const Frame& f, uint8_t* out, int64_t* interval_byte, int32_t* interval_bits) {
  size_t q = f.scan_begin, o = 0;
  int iv = 0;
  interval_byte[0] = 0;
  while (q < f.scan_end) {
    const void* ff = memchr(d + q, 0xFF, f.scan_end - q);
    size_t e = ff ? (size_t)((const uint8_t*)ff - d) : f.scan_end;
    memcpy(out + o, d + q, e - q);
    o += e - q;
    q = e;
    if (q >= f.scan_end) break;
    if (d[q + 1] == 0x00) {
      out[o++] = 0xFF;
    } else {   // RSTn: parse() has checked the order
      interval_bits[iv] = (int32_t)((o - interval_byte[iv]) * 8);
      interval_byte[++iv] = (int64_t)o;
    }
    q += 2;
  }
  interval_bits[iv] = (int32_t)((o - interval_byte[iv]) * 8);
  return o;
}

}  // namespace jpeg
}  // namespace ctd

extern "C" CTD_API int ctd_jpeg_probe(const uint8_t* data, size_t len, ctd_jpeg_info* info) {
  if (!data || !info) return CTD_E_INVALID;
  memset(info, 0, sizeof(*info));
  ctd::jpeg::Frame f;
  info->status = ctd::jpeg::parse(data, len, &f);
  if (info->status != CTD_JPEG_OK) return CTD_OK;
  bool t = f.orient >= 5;
  info->height = t ? f.w : f.h;
  info->width = t ? f.h : f.w;
  info->frame_height = f.h;
  info->frame_width = f.w;
  info->components = f.ncomp;
  info->h_samp = f.hmax;
  info->v_samp = f.vmax;
  info->orientation = f.orient;
  info->restart_interval = f.restart;
  info->ecs_bytes = (int64_t)(f.scan_end - f.scan_begin);
  return CTD_OK;
}
