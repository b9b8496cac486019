// Internal interface between the JPEG host parser (jpeg_plan.cpp) and the GPU decoder (jpeg.cu).
#pragma once
#include <stdint.h>

#include <vector>

#include "../../include/ctd_b200.h"

namespace ctd {
namespace jpeg {

constexpr int kLutBits = 9;   // Huffman codes up to this length are decoded by one table lookup

// One Huffman table as the GPU reads it (jdhuff.c's derived table plus a lookahead table).
struct HuffTable {
  uint16_t lut[1 << kLutBits];   // (length << 8) | symbol for codes of <= kLutBits bits, 0 for longer codes
  int32_t maxcode[18];           // largest code of each length, -1 if none; maxcode[17] = INT32_MAX sentinel
  int32_t valoff[17];            // index into vals of a code of length L: code + valoff[L]
  uint8_t vals[256];
};

// The parsed headers of one file the GPU path takes.
struct Frame {
  int h = 0, w = 0, ncomp = 0, hmax = 1, vmax = 1, mcux = 0, mcuy = 0, restart = 0, orient = 1;
  int ch[3] = {1, 1, 1}, cv[3] = {1, 1, 1};  // sampling factors (forced to 1x1 for one component)
  int dc[3] = {0, 0, 0}, ac[3] = {0, 0, 0};  // Huffman table slot of each component in `tables`
  int q[3] = {0, 0, 0};                      // quantisation table of each component in `quant`
  std::vector<HuffTable> tables;             // the tables the scan uses
  int32_t quant[4][64] = {};                 // natural order
  size_t scan_begin = 0, scan_end = 0;       // entropy-coded bytes [begin, end): up to the EOI marker
  int n_intervals = 0;
};

// The marker walk and the scan's structure check: CTD_JPEG_OK and the frame, or the reason code.
int parse(const uint8_t* data, size_t len, Frame* f);

// IFD0 orientation of an Exif payload (a TIFF header and its IFDs: after "Exif\0\0" in a JPEG, the whole eXIf chunk
// of a PNG) as OpenCV's ExifReader reads it: 1..8, or 0 when the block does not parse cleanly
int exif_orientation(const uint8_t* p, size_t n);

// Unstuffs the scan of a parsed file into out (at most scan_end - scan_begin bytes): FF00 -> FF, RSTn dropped.
// Writes each restart interval's first byte offset (relative to out) and bit length.  Returns the bytes written.
size_t stage(const uint8_t* data, const Frame& f, uint8_t* out, int64_t* interval_byte, int32_t* interval_bits);

}  // namespace jpeg
}  // namespace ctd
