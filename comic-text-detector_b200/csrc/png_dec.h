// Internal interface between the PNG host parser (png_plan.cpp) and the GPU decoder (png_dec.cu).
#pragma once
#include <stdint.h>

#include <vector>

#include "../../include/ctd_b200.h"

namespace ctd {
namespace png {

// The parsed chunks of one file the GPU path takes.
struct File {
  int w = 0, h = 0, depth = 0, ctype = 0, orient = 1, plte_n = 0;
  uint8_t plte[256 * 3] = {};            // RGB entries, zero past plte_n
  std::vector<size_t> idat_off, idat_len;  // payload of each IDAT chunk in the file
  size_t zlen = 0;                       // bytes of the zlib stream (all IDAT payloads)
  int window = 0;                        // LZ77 window the zlib header declares
  int64_t rowbytes = 0, filtered = 0;    // bytes of one row, h * (1 + rowbytes)
};

// The chunk walk: CTD_PNG_OK and the file, or the reason code.  check_crc: also check every chunk's CRC-32
// (CTD_PNG_CRC).
int parse(const uint8_t* data, size_t len, File* f, bool check_crc);

}  // namespace png
}  // namespace ctd
