// Text-line crops (C ABI `ctd_transform_regions`, include/ctd_b200.h): `cv2.warpPerspective(img, M, (w, h))` with
// INTER_LINEAR / BORDER_CONSTANT 0, followed for vertical lines by `cv2.rotate(.., ROTATE_90_COUNTERCLOCKWISE)`, for
// every line of a page in ONE launch (reference utils/textblock.py:162-194; the matrices come from ctd_region_plan,
// csrc/region_plan.cpp).  The same kernel crops every line of every page of a ctd_submit_pages batch with a textheight
// in one launch (pipeline.cu): each crop record carries its page's byte offset and size, so the pages are read in
// place.
//
// Work split: the host (RegionJob) cuts every crop into tiles of kRegionTilePx consecutive output pixels (row-major in
// the RETURNED array, i.e. after the rotation) and uploads a tile table {region, first pixel}; one CTA per tile, one
// thread per output pixel, all three channels, the rotation folded into the index map.  A crop of 48 x 4000 px is
// spread over 750 CTAs, a 48 x 60 one takes 12, so the grid is balanced whatever the mix of line lengths.
//
// Sampling, bit-exact with OpenCV's fixed-point warp (imgwarp.cpp's perspective invoker + remap's bilinear path):
//   X0 = (M0*xb + M1*y) + M2,  W = (M6*xb + M7*y) + M8 + M6*x1,  W = W ? 32/W : 0,  X = rint((X0 + M0*x1) * W)
// (same for Y), where M is the inverse matrix and xb + x1 = x with xb the start of OpenCV's pixel block: the invoker
// walks the output in blocks of bw0 = min(1024 / min(16, h), w) columns and forms the row terms per block, so the
// grouping of the sums depends on the block start and the kernel reproduces it.  The integer part X >> 5 picks the
// tap, the fraction X & 31 the weight of OpenCV's 32 x 32 table of 15-bit coefficients ((32-fx)(32-fy)*32 ...); each of
// the four taps reads 0 outside the page (BORDER_CONSTANT, per tap) and the result is (sum + 2^14) >> 15.
// The double-precision steps use __dmul_rn / __dadd_rn / __ddiv_rn so that nvcc cannot contract them into FMAs
// (an FMA changes which way rint() resolves the exact .5 ties integer line quads produce).
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "engine.h"

#define CK(expr)                                                                                      \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) return ctd_fail(h, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

namespace {

using ctd::kRegionTilePx;
using ctd::RegionDev;
using ctd::RegionTile;

__global__ void __launch_bounds__(kRegionTilePx) k_warp_regions(const uint8_t* __restrict__ pages,
                                                               const RegionDev* __restrict__ regs,
                                                               const RegionTile* __restrict__ tiles,
                                                               uint8_t* __restrict__ out) {
  const RegionTile t = tiles[blockIdx.x];
  const RegionDev& r = regs[t.region];
  const uint8_t* page = pages + r.page_off;
  const int ih = r.ih, iw = r.iw;
  const int p = t.first + int(threadIdx.x);
  const int ow = r.out_w;
  if (p >= r.out_h * ow) return;
  const int oy = p / ow, ox = p - oy * ow;
  int x, y;   // pixel of the warped image: out[i][j] = warp[j][w-1-i] for the counter-clockwise rotation
  if (r.rotate) {
    x = r.warp_w - 1 - oy;
    y = ox;
  } else {
    x = ox;
    y = oy;
  }
  const int xb = (x / r.bw0) * r.bw0, x1 = x - xb;
  const double dxb = double(xb), dy = double(y), dx1 = double(x1);
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(r.m[0], dxb), __dmul_rn(r.m[1], dy)), r.m[2]);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(r.m[3], dxb), __dmul_rn(r.m[4], dy)), r.m[5]);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(r.m[6], dxb), __dmul_rn(r.m[7], dy)), r.m[8]);
  double W = __dadd_rn(W0, __dmul_rn(r.m[6], dx1));
  W = W != 0.0 ? __ddiv_rn(32.0, W) : 0.0;
  double fX = __dmul_rn(__dadd_rn(X0, __dmul_rn(r.m[0], dx1)), W);
  double fY = __dmul_rn(__dadd_rn(Y0, __dmul_rn(r.m[3], dx1)), W);
  // std::max(INT_MIN, std::min(INT_MAX, v)) with its NaN behaviour (a NaN becomes INT_MAX)
  fX = fX < double(INT_MAX) ? fX : double(INT_MAX);
  fX = double(INT_MIN) < fX ? fX : double(INT_MIN);
  fY = fY < double(INT_MAX) ? fY : double(INT_MAX);
  fY = double(INT_MIN) < fY ? fY : double(INT_MIN);
  const int X = __double2int_rn(fX), Y = __double2int_rn(fY);
  const int sx = max(-32768, min(32767, X >> 5)), sy = max(-32768, min(32767, Y >> 5));   // saturate_cast<short>
  const int fx = X & 31, fy = Y & 31;
  const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
  const bool in_x0 = unsigned(sx) < unsigned(iw), in_x1 = unsigned(sx + 1) < unsigned(iw);
  const bool in_y0 = unsigned(sy) < unsigned(ih), in_y1 = unsigned(sy + 1) < unsigned(ih);
  const long long t00 = ((long long)sy * iw + sx) * 3;   // only dereferenced for taps inside the page
  const uint8_t* row0 = page + t00;
  const uint8_t* row1 = page + t00 + (long long)iw * 3;
  uint8_t* dst = out + r.offset + size_t(p) * 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int v00 = in_y0 && in_x0 ? __ldg(row0 + k) : 0;
    const int v01 = in_y0 && in_x1 ? __ldg(row0 + 3 + k) : 0;
    const int v10 = in_y1 && in_x0 ? __ldg(row1 + k) : 0;
    const int v11 = in_y1 && in_x1 ? __ldg(row1 + 3 + k) : 0;
    const int s = v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11;
    dst[k] = uint8_t(min(255, max(0, (s + (1 << 14)) >> 15)));
  }
}

}  // namespace

cudaError_t ctd::warp_regions_launch(const uint8_t* d_pages, const RegionDev* d_regs, const RegionTile* d_tiles,
                                     int n_tiles, uint8_t* d_out, cudaStream_t s) {
  if (n_tiles <= 0) return cudaSuccess;
  k_warp_regions<<<unsigned(n_tiles), kRegionTilePx, 0, s>>>(d_pages, d_regs, d_tiles, d_out);
  return cudaGetLastError();
}

int RegionJob::add(const ctd_region* plan, int n, long long page_off, int ih, int iw, long long out_base) {
  for (int i = 0; i < n; ++i) {
    const ctd_region& r = plan[i];
    if (r.status != 0) continue;
    if (r.out_h < 1 || r.out_w < 1 || r.offset < 0 || (r.rotate != 0 && r.rotate != 1) ||
        (long long)r.out_h * r.out_w > INT_MAX / 4)
      return i;
    const size_t px = size_t(r.out_h) * r.out_w;
    out_bytes = std::max(out_bytes, size_t(out_base + r.offset) + px * 3);
    RegionDev d{};
    d.offset = out_base + r.offset;
    d.page_off = page_off;
    d.out_h = r.out_h;
    d.out_w = r.out_w;
    d.rotate = r.rotate;
    d.ih = ih;
    d.iw = iw;
    const int ww = r.rotate ? r.out_h : r.out_w, wh = r.rotate ? r.out_w : r.out_h;
    d.warp_w = ww;
    const int bh0 = std::min(16, wh);   // OpenCV's block shape for a ww x wh destination
    d.bw0 = std::min(1024 / bh0, ww);
    memcpy(d.m, r.inverse, sizeof(d.m));
    const int ri = int(regs.size());
    regs.push_back(d);
    for (size_t f = 0; f < px; f += kRegionTilePx) tiles.push_back(RegionTile{ri, int(f)});
  }
  return -1;
}

static size_t al256(size_t v) { return (v + 255) / 256 * 256; }
size_t RegionJob::table_bytes() const {
  return al256(regs.size() * sizeof(RegionDev)) + al256(tiles.size() * sizeof(RegionTile));
}
void RegionJob::write_tables(char* dst) const {
  memcpy(dst, regs.data(), regs.size() * sizeof(RegionDev));
  memcpy(dst + al256(regs.size() * sizeof(RegionDev)), tiles.data(), tiles.size() * sizeof(RegionTile));
}

extern "C" int ctd_transform_regions(ctd_handle* h, const uint8_t* page, int32_t ih, int32_t iw, int32_t page_on_device,
                                     const ctd_region* plan, int32_t n, uint8_t* pixels_out, size_t pixels_bytes) {
  if (!h || !page || n < 0 || (n > 0 && !plan)) return CTD_E_INVALID;
  if (ih < 1 || iw < 1) return ctd_fail(h, CTD_E_SHAPE, "bad page size %dx%d", ih, iw);
  RegionJob job;
  if (int bad = job.add(plan, n, 0, ih, iw, 0); bad >= 0) {
    const ctd_region& r = plan[bad];
    return ctd_fail(h, CTD_E_INVALID, "malformed plan entry %d (%dx%d at offset %lld)", bad, r.out_h, r.out_w,
                    (long long)r.offset);
  }
  const size_t total = job.out_bytes;
  if (total > 0 && !pixels_out) return CTD_E_INVALID;
  if (pixels_bytes < total)
    return ctd_fail(h, CTD_E_CAPACITY, "the crops need %zu bytes, the output holds %zu", total, pixels_bytes);
  if (job.tiles.empty()) return CTD_OK;
  if (job.tiles.size() > size_t(INT_MAX)) return ctd_fail(h, CTD_E_INVALID, "too many crop pixels");
  CK(cudaSetDevice(h->cfg.device));
  const size_t tb = job.table_bytes();
  const size_t rb = al256(job.regs.size() * sizeof(RegionDev));
  const size_t pb = page_on_device ? 0 : al256(size_t(ih) * iw * 3);
  if (int rc = h->io_scratch.grow(h, tb + pb + total, h->stream)) return rc;
  char* base = reinterpret_cast<char*>(h->io_scratch.p);
  std::vector<char> stage(tb);
  job.write_tables(stage.data());
  CK(cudaMemcpyAsync(base, stage.data(), tb, cudaMemcpyHostToDevice, h->stream));
  const uint8_t* d_page = page;
  if (!page_on_device) {
    CK(cudaMemcpyAsync(base + tb, page, size_t(ih) * iw * 3, cudaMemcpyHostToDevice, h->stream));
    d_page = reinterpret_cast<const uint8_t*>(base + tb);
  }
  uint8_t* d_out = reinterpret_cast<uint8_t*>(base + tb + pb);
  CK(ctd::warp_regions_launch(d_page, reinterpret_cast<const RegionDev*>(base),
                              reinterpret_cast<const RegionTile*>(base + rb), int(job.tiles.size()), d_out, h->stream));
  CK(cudaMemcpyAsync(pixels_out, d_out, total, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}
