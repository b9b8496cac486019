// cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR) for uint8 images on the GPU, bit-exact with OpenCV 4.x
// (modules/imgproc/src/resize.cpp), as used by the reference's letterbox (utils/imgproc_utils.py:86-117 via
// preprocess_img, inference.py:72-83) and by the mask back-projection (inference.py:164-168).
//   * source coordinate f = (float)((d + 0.5) * scale - 0.5), scale = (double)src / dst; s = floor(f); f -= s
//   * COLUMNS: s < 0 -> (pixel 0, weight 1); s >= W-1 -> (last pixel, weight 1)
//     ROWS: fractional weights are kept, only the two row indices are clipped to [0, H-1]
//   * weights: cvRound(w * 2048) as int16 (round half to even)
//   * horizontal: S = a0*p[x0] + a1*p[x1] (int32); vertical: (((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2
//   * dst*2 == src in both axes: computed as INTER_AREA, (p00+p01+p10+p11+2)>>2
// Oracle: oracle/resize_ref.py (pinned against the installed cv2, tests/test_cpu_resize.py).
// The output may be a window of a larger zero-padded canvas (letterbox: bottom/right padding).
// letterbox_tensor_kernel writes the same letterbox as the network tensor of preprocess_img (inference.py:72-83):
// f32 or f16 NCHW planes of v / 255, or u8 NHWC, in either channel order.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace ctd {

struct AxisTap { int i0, i1, w0, w1; };

__device__ __forceinline__ AxisTap axis_tap(int d, int ssize, int dsize, bool clamp_weights) {
  const double scale = (double)ssize / (double)dsize;
  // (d + 0.5) * scale - 0.5 with separately rounded product and difference (no FMA contraction), then float
  float f = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_weights) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= ssize - 1) { f = 0.f; s = ssize - 1; }
  }
  AxisTap t;
  t.w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), 2048.0f));
  t.w1 = __float2int_rn(__fmul_rn(f, 2048.0f));
  t.i0 = min(max(s, 0), ssize - 1);
  t.i1 = min(max(s + 1, 0), ssize - 1);
  return t;
}

// One output pixel (all C channels) of the dh x dw resize of src, written at `o`; pixels outside the dh x dw image are
// zero (letterbox padding).  Every kernel of this file computes its pixels here, so the single-image and the batched
// paths cannot drift apart.
template <int C>
__device__ __forceinline__ void resize_pixel(const uint8_t* __restrict__ src, int sh, int sw, size_t src_pitch,
                                             uint8_t* __restrict__ o, int x, int y, int dh, int dw) {
  if (x >= dw || y >= dh) {
#pragma unroll
    for (int c = 0; c < C; ++c) o[c] = 0;
    return;
  }
  if (dw * 2 == sw && dh * 2 == sh) {   // INTER_LINEAR -> INTER_AREA for the exact 2x2 decimation
    const uint8_t* p0 = src + size_t(2 * y) * src_pitch + size_t(2 * x) * C;
    const uint8_t* p1 = p0 + src_pitch;
#pragma unroll
    for (int c = 0; c < C; ++c) o[c] = uint8_t((int(p0[c]) + int(p0[C + c]) + int(p1[c]) + int(p1[C + c]) + 2) >> 2);
    return;
  }
  const AxisTap tx = axis_tap(x, sw, dw, true), ty = axis_tap(y, sh, dh, false);
  const uint8_t* r0 = src + size_t(ty.i0) * src_pitch;
  const uint8_t* r1 = src + size_t(ty.i1) * src_pitch;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const int s0 = tx.w0 * int(r0[size_t(tx.i0) * C + c]) + tx.w1 * int(r0[size_t(tx.i1) * C + c]);
    const int s1 = tx.w0 * int(r1[size_t(tx.i0) * C + c]) + tx.w1 * int(r1[size_t(tx.i1) * C + c]);
    o[c] = uint8_t((((ty.w0 * (s0 >> 4)) >> 16) + ((ty.w1 * (s1 >> 4)) >> 16) + 2) >> 2);
  }
}

// One thread per canvas pixel.
template <int C>
__global__ void resize_linear_u8_kernel(const uint8_t* __restrict__ src, int sh, int sw, size_t src_pitch,
                                        uint8_t* __restrict__ dst, int dh, int dw, int canvas_h, int canvas_w) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= canvas_w || y >= canvas_h) return;
  resize_pixel<C>(src, sh, sw, src_pitch, dst + (size_t(y) * canvas_w + x) * C, x, y, dh, dw);
}

// Letterbox of every page of a batch: blockIdx.z = page, one thread per pixel of its net_h x net_w canvas.
__global__ void letterbox_batch_kernel(const uint8_t* __restrict__ src, const PageGeom* __restrict__ tab,
                                       uint8_t* __restrict__ dst, int net_h, int net_w) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= net_w) return;
  const PageGeom g = tab[blockIdx.z];
  uint8_t* o = dst + ((size_t(blockIdx.z) * net_h + y) * net_w + x) * 3;
  resize_pixel<3>(src + g.src_off, g.ih, g.iw, size_t(g.iw) * 3, o, x, y, g.unpad_h, g.unpad_w);
}

// v / 255 as numpy's `astype(float32) / 255` computes it: a correctly rounded float32 division (__fdiv_rn(v, 255.f)),
// which is not v * RN(1/255) (the two differ on 126 of the 256 u8 values).  The product by RN(1/255) corrected once by
// its fma residual equals the division on all 256 values (checked in exact arithmetic, tests/test_cpu_preprocess.py),
// and needs no call to __fdiv_rn's slow path, whose register saves would spill.
__device__ __forceinline__ float unit_f32(uint8_t v) {
  const float r = 0x1.010102p-8f;   // RN(1 / 255)
  const float x = float(v);
  const float q0 = __fmul_rn(x, r);
  return __fmaf_rn(__fmaf_rn(-q0, 255.0f, x), r, q0);
}

// The letterbox of every page of a batch written as the tensor `preprocess_img` makes (ctd_preprocess_pages):
// blockIdx.z = page, blockIdx.y = row, each thread kPx consecutive pixels of the row, each computed by resize_pixel<3>
// and packed into the thread's output words as soon as it is computed (so few values are live across the double
// divisions of axis_tap).  NCHW: one 16-byte store per plane (4 f32 or 8 f16 values); NHWC u8: 16 pixels = three
// 16-byte stores.  Reverse: output channel k is channel 2 - k of the page.
template <int Fmt, bool Reverse>
__global__ void __launch_bounds__(128) letterbox_tensor_kernel(const uint8_t* __restrict__ src,
                                                               const PageGeom* __restrict__ tab, void* __restrict__ dst,
                                                               int net_h, int net_w) {
  constexpr int kPx = Fmt == PRE_F32_NCHW ? 4 : Fmt == PRE_F16_NCHW ? 8 : 16;
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * kPx;
  const int y = blockIdx.y;
  if (x0 >= net_w) return;
  const PageGeom g = tab[blockIdx.z];
  // f32: w[k][i] = the bits of pixel i of plane k; f16: w[k][i / 2] holds pixels i, i + 1 of plane k (low half first);
  // u8: w[0..11] are the 48 bytes of the 16 pixels, little-endian
  uint32_t w[3][4] = {};
#pragma unroll
  for (int i = 0; i < kPx; ++i) {
    uint8_t p[3];
    resize_pixel<3>(src + g.src_off, g.ih, g.iw, size_t(g.iw) * 3, p, x0 + i, y, g.unpad_h, g.unpad_w);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const uint8_t v = p[Reverse ? 2 - k : k];
      if constexpr (Fmt == PRE_F32_NCHW) {
        w[k][i] = __float_as_uint(unit_f32(v));
      } else if constexpr (Fmt == PRE_F16_NCHW) {
        w[k][i / 2] |= uint32_t(__half_as_ushort(__float2half_rn(unit_f32(v)))) << (16 * (i % 2));
      } else {
        const int j = 3 * i + k;
        w[j / 16][(j / 4) % 4] |= uint32_t(v) << (8 * (j % 4));
      }
    }
  }
  if constexpr (Fmt == PRE_U8_NHWC) {
    uint4* o = reinterpret_cast<uint4*>(static_cast<uint8_t*>(dst) +
                                        ((size_t(blockIdx.z) * net_h + y) * net_w + x0) * 3);
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = make_uint4(w[k][0], w[k][1], w[k][2], w[k][3]);
  } else {
    constexpr int kElem = Fmt == PRE_F32_NCHW ? 4 : 2;
    const size_t plane = size_t(net_h) * net_w;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const size_t at = (size_t(blockIdx.z) * 3 + k) * plane + size_t(y) * net_w + x0;
      *reinterpret_cast<uint4*>(static_cast<uint8_t*>(dst) + at * kElem) = make_uint4(w[k][0], w[k][1], w[k][2], w[k][3]);
    }
  }
}

// Mask back-projection of every page of a batch: one CTA per output row over the pages' stacked rows (page p owns rows
// [row0, row0 + ih)), so no CTA is launched for a row that does not exist; the threads stride over the row's columns.
__global__ void backproject_batch_kernel(const uint8_t* __restrict__ mask, int net_h, int net_w,
                                         const PageGeom* __restrict__ tab, int n, uint8_t* __restrict__ dst) {
  const int r = blockIdx.x;
  int lo = 0, hi = n - 1;   // last page with row0 <= r
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab[mid].row0 <= r) lo = mid; else hi = mid - 1;
  }
  const PageGeom g = tab[lo];
  const int y = r - g.row0;
  const uint8_t* src = mask + size_t(lo) * net_h * net_w;
  uint8_t* orow = dst + g.dst_off + size_t(y) * g.iw;
  for (int x = threadIdx.x; x < g.iw; x += blockDim.x)
    resize_pixel<1>(src, g.unpad_h, g.unpad_w, size_t(net_w), orow + x, x, y, g.ih, g.iw);
}

cudaError_t resize_linear_u8_launch(const uint8_t* src, int sh, int sw, size_t src_pitch, int channels, uint8_t* dst,
                                    int dh, int dw, int canvas_h, int canvas_w, cudaStream_t s) {
  if (sh < 1 || sw < 1 || dh < 1 || dw < 1 || canvas_h < dh || canvas_w < dw) return cudaErrorInvalidValue;
  const dim3 grid(unsigned((canvas_w + 127) / 128), unsigned(canvas_h));
  if (channels == 3) resize_linear_u8_kernel<3><<<grid, 128, 0, s>>>(src, sh, sw, src_pitch, dst, dh, dw, canvas_h, canvas_w);
  else if (channels == 1) resize_linear_u8_kernel<1><<<grid, 128, 0, s>>>(src, sh, sw, src_pitch, dst, dh, dw, canvas_h, canvas_w);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t letterbox_batch_launch(const uint8_t* src, const PageGeom* d_tab, int n, uint8_t* dst, int net_h, int net_w,
                                   cudaStream_t s) {
  if (n < 1 || net_h < 1 || net_w < 1) return cudaErrorInvalidValue;
  letterbox_batch_kernel<<<dim3(unsigned((net_w + 127) / 128), unsigned(net_h), unsigned(n)), 128, 0, s>>>(src, d_tab, dst,
                                                                                                        net_h, net_w);
  return cudaGetLastError();
}

template <int Fmt, bool Reverse>
static void letterbox_tensor_launch_t(const uint8_t* src, const PageGeom* d_tab, int n, void* dst, int net_h, int net_w,
                                      cudaStream_t s) {
  constexpr int kPx = Fmt == PRE_F32_NCHW ? 4 : Fmt == PRE_F16_NCHW ? 8 : 16;
  const dim3 grid(unsigned((net_w / kPx + 127) / 128), unsigned(net_h), unsigned(n));
  letterbox_tensor_kernel<Fmt, Reverse><<<grid, 128, 0, s>>>(src, d_tab, dst, net_h, net_w);
}

cudaError_t letterbox_tensor_launch(const uint8_t* src, const PageGeom* d_tab, int n, void* dst, int net_h, int net_w,
                                    int format, bool reverse, cudaStream_t s) {
  if (n < 1 || net_h < 1 || net_w < 16 || net_w % 16 || (uintptr_t(dst) & 15)) return cudaErrorInvalidValue;
  switch (format * 2 + (reverse ? 1 : 0)) {
    case PRE_F32_NCHW * 2: letterbox_tensor_launch_t<PRE_F32_NCHW, false>(src, d_tab, n, dst, net_h, net_w, s); break;
    case PRE_F32_NCHW * 2 + 1: letterbox_tensor_launch_t<PRE_F32_NCHW, true>(src, d_tab, n, dst, net_h, net_w, s); break;
    case PRE_F16_NCHW * 2: letterbox_tensor_launch_t<PRE_F16_NCHW, false>(src, d_tab, n, dst, net_h, net_w, s); break;
    case PRE_F16_NCHW * 2 + 1: letterbox_tensor_launch_t<PRE_F16_NCHW, true>(src, d_tab, n, dst, net_h, net_w, s); break;
    case PRE_U8_NHWC * 2: letterbox_tensor_launch_t<PRE_U8_NHWC, false>(src, d_tab, n, dst, net_h, net_w, s); break;
    case PRE_U8_NHWC * 2 + 1: letterbox_tensor_launch_t<PRE_U8_NHWC, true>(src, d_tab, n, dst, net_h, net_w, s); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t backproject_batch_launch(const uint8_t* mask, int net_h, int net_w, const PageGeom* d_tab, int n,
                                     int total_rows, uint8_t* dst, cudaStream_t s) {
  if (n < 1 || total_rows < 1) return cudaErrorInvalidValue;
  backproject_batch_kernel<<<unsigned(total_rows), 256, 0, s>>>(mask, net_h, net_w, d_tab, n, dst);
  return cudaGetLastError();
}

}  // namespace ctd
