// Host side of the GPU PNG decoder (C ABI `ctd_png_probe`, include/ctd_b200.h): the chunk walk that decides whether
// the GPU path takes a file.
//
// The walk accepts exactly the files whose decode png_dec.cu restates: a valid IHDR first, non-interlaced, one of the
// colour type / bit depth pairs of the header's list, PLTE (once, before IDAT, 1..256 whole entries) for palette
// images and no PLTE otherwise, IDAT chunks in one run, no APNG chunk, at most one eXIf that parses as OpenCV's
// ExifReader parses a JPEG's Exif block, only known critical chunks, and an empty IEND.  The zlib header must be a
// deflate stream without a preset dictionary.  Anything libpng would treat as an error or a warning that can change
// the pixels is declined here, so cv2 decides it.  Stateless and thread-safe.  oracle/png_decode_ref.py restates the
// same rules in numpy.
#include <string.h>

#include <algorithm>

#include "jpeg.h"
#include "png_dec.h"

namespace ctd {
namespace png {
namespace {

const uint8_t kSig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};

inline uint32_t u32be(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}

// CRC-32 (ISO 3309, as PNG and zlib use it), eight bytes a step
struct CrcTables {
  uint32_t t[8][256];
  CrcTables() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = c & 1 ? 0xedb88320u ^ (c >> 1) : c >> 1;
      t[0][i] = c;
    }
    for (int k = 1; k < 8; ++k)
      for (int i = 0; i < 256; ++i) t[k][i] = t[0][t[k - 1][i] & 0xff] ^ (t[k - 1][i] >> 8);
  }
};

uint32_t crc32(const uint8_t* p, size_t n) {
  static const CrcTables T;
  uint32_t c = 0xffffffffu;
  for (; n >= 8; p += 8, n -= 8) {
    uint32_t a = c ^ (p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24));
    uint32_t b = p[4] | (p[5] << 8) | (p[6] << 16) | ((uint32_t)p[7] << 24);
    c = T.t[7][a & 0xff] ^ T.t[6][(a >> 8) & 0xff] ^ T.t[5][(a >> 16) & 0xff] ^ T.t[4][a >> 24] ^ T.t[3][b & 0xff] ^
        T.t[2][(b >> 8) & 0xff] ^ T.t[1][(b >> 16) & 0xff] ^ T.t[0][b >> 24];
  }
  while (n--) c = T.t[0][(c ^ *p++) & 0xff] ^ (c >> 8);
  return c ^ 0xffffffffu;
}

bool depth_ok(int ctype, int depth) {
  switch (ctype) {
    case 0: return depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16;
    case 3: return depth == 1 || depth == 2 || depth == 4 || depth == 8;
    case 2: case 4: case 6: return depth == 8 || depth == 16;
    default: return false;
  }
}

bool is_letter(uint8_t c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); }

}  // namespace

int parse(const uint8_t* d, size_t n, File* f, bool check_crc) {
  if (n < 8 || memcmp(d, kSig, 8) != 0) return CTD_PNG_NOT_PNG;
  if (n < 8 + 8 || u32be(d + 8) != 13 || memcmp(d + 12, "IHDR", 4) != 0) return CTD_PNG_NOT_PNG;
  if (n < 8 + 25) return CTD_PNG_TRUNCATED;
  const uint8_t* ih = d + 16;
  uint32_t w = u32be(ih), h = u32be(ih + 4);
  int depth = ih[8], ctype = ih[9];
  if (w == 0 || h == 0 || w > 0x7fffffffu || h > 0x7fffffffu || ih[10] != 0 || ih[11] != 0 || !depth_ok(ctype, depth))
    return CTD_PNG_HEADER;
  if (ih[12] == 1) return CTD_PNG_INTERLACED;
  if (ih[12] != 0) return CTD_PNG_HEADER;
  static const int kChannels[7] = {1, 0, 3, 1, 2, 0, 4};
  int64_t bits = (int64_t)kChannels[ctype] * depth;
  f->w = (int)std::min<uint32_t>(w, 0x7fffffff);
  f->h = (int)std::min<uint32_t>(h, 0x7fffffff);
  f->depth = depth;
  f->ctype = ctype;
  f->rowbytes = ((int64_t)w * bits + 7) / 8;
  f->filtered = (int64_t)h * (1 + f->rowbytes);
  // libpng's default user limits and OpenCV's pixel limit; the decoder keeps output offsets in 32 bits
  bool size_ok = w <= 1000000 && h <= 1000000 && (int64_t)w * h <= (int64_t(1) << 30) && f->filtered < (int64_t(1) << 31);
  bool ihdr_crc_ok = !check_crc || crc32(d + 12, 17) == u32be(d + 29);
  bool plte = false, exif = false, idat_done = false;
  size_t p = 33;
  for (;;) {
    if (p + 12 > n) return CTD_PNG_TRUNCATED;
    uint32_t L = u32be(d + p);
    const uint8_t* t = d + p + 4;
    if (L > 0x7fffffffu || p + 12 + (size_t)L > n) return CTD_PNG_TRUNCATED;
    if (!is_letter(t[0]) || !is_letter(t[1]) || !is_letter(t[2]) || !is_letter(t[3])) return CTD_PNG_CHUNKS;
    const uint8_t* s = t + 4;
    if (check_crc && crc32(t, 4 + (size_t)L) != u32be(s + L)) return CTD_PNG_CRC;
    bool is_idat = memcmp(t, "IDAT", 4) == 0;
    if (!is_idat && !f->idat_off.empty()) idat_done = true;
    if (is_idat) {
      if (idat_done) return CTD_PNG_CHUNKS;
      if (ctype == 3 && !plte) return CTD_PNG_CHUNKS;
      f->idat_off.push_back((size_t)(s - d));
      f->idat_len.push_back(L);
      f->zlen += L;
    } else if (memcmp(t, "IEND", 4) == 0) {
      if (L != 0) return CTD_PNG_CHUNKS;
      break;
    } else if (memcmp(t, "PLTE", 4) == 0) {
      if (ctype != 3 || plte || !f->idat_off.empty() || L == 0 || L % 3 || L > 768) return CTD_PNG_CHUNKS;
      plte = true;
      f->plte_n = (int)(L / 3);
      memcpy(f->plte, s, L);
    } else if (memcmp(t, "acTL", 4) == 0 || memcmp(t, "fcTL", 4) == 0 || memcmp(t, "fdAT", 4) == 0) {
      return CTD_PNG_APNG;
    } else if (memcmp(t, "eXIf", 4) == 0) {
      if (exif) return CTD_PNG_EXIF;
      exif = true;
      f->orient = jpeg::exif_orientation(s, L);
      if (!f->orient) return CTD_PNG_EXIF;
    } else if (!(t[0] & 0x20)) {
      return CTD_PNG_CHUNKS;   // IHDR again or an unknown critical chunk
    }
    p += 12 + (size_t)L;
  }
  if (f->idat_off.empty()) return CTD_PNG_TRUNCATED;
  if (!ihdr_crc_ok) return CTD_PNG_CRC;
  if (!size_ok || f->zlen >= (size_t(1) << 30)) return CTD_PNG_SIZE;
  // the zlib header: its first two bytes, wherever the IDAT chunks split them
  uint8_t hdr[2];
  size_t k = 0;
  for (size_t c = 0; c < f->idat_off.size() && k < 2; ++c)
    for (size_t j = 0; j < f->idat_len[c] && k < 2; ++j) hdr[k++] = d[f->idat_off[c] + j];
  if (k < 2 || f->zlen < 6) return CTD_PNG_ZLIB;
  if ((hdr[0] & 15) != 8 || (hdr[0] >> 4) > 7 || ((hdr[0] << 8) | hdr[1]) % 31 != 0 || (hdr[1] & 0x20))
    return CTD_PNG_ZLIB;
  f->window = 1 << ((hdr[0] >> 4) + 8);
  return CTD_PNG_OK;
}

}  // namespace png
}  // namespace ctd

extern "C" CTD_API int ctd_png_probe(const uint8_t* data, size_t len, ctd_png_info* info) {
  if (!data || !info) return CTD_E_INVALID;
  memset(info, 0, sizeof(*info));
  ctd::png::File f;
  info->status = ctd::png::parse(data, len, &f, false);
  if (info->status != CTD_PNG_OK) return CTD_OK;
  bool t = f.orient >= 5;
  info->height = t ? f.w : f.h;
  info->width = t ? f.h : f.w;
  info->image_height = f.h;
  info->image_width = f.w;
  info->bit_depth = f.depth;
  info->color_type = f.ctype;
  info->orientation = f.orient;
  info->palette_entries = f.plte_n;
  info->zlib_bytes = (int64_t)f.zlen;
  return CTD_OK;
}
