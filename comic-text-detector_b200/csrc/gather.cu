// Batched strided page gather (ctd_submit_pages, ctd_submit_refine): every page of a batch that is already in device
// memory, laid out with any strides (a sub-window of a larger image, a permuted channels-first image), copied in one
// launch into the packed page buffer of the batch (u8 BGR [ih][iw][3] at the page's page_off), where the letterbox,
// refine_mask and the crop kernels read it; in the same launch, the batch's masks in device memory (u8 [ih][iw], any
// strides: a channel of a page) into its packed mask plane.  One CTA per row over the stacked rows of the gathered
// images, as backproject_batch_kernel.
// gather_outputs_kernel is the ingest of ctd_submit_outputs: a caller's network outputs (float32 or float16, any
// strides) staged into the engine's post-processing workspace in one launch, with postprocess_mask's u8 cast and the DB
// threshold fused.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <type_traits>

#include "kernels.h"

namespace ctd {

namespace {

// bytes [0, nb) of s to d when s and d agree modulo sizeof(W): a byte head up to d's W boundary, W-wide copies, a
// byte tail
template <typename W>
__device__ __forceinline__ void copy_same_phase(const uint8_t* __restrict__ s, uint8_t* __restrict__ d, int nb) {
  constexpr int kW = int(sizeof(W));
  const int head = min(nb, int((kW - int(uintptr_t(d) & (kW - 1))) & (kW - 1)));
  const int nw = (nb - head) / kW;
  for (int i = threadIdx.x; i < head; i += blockDim.x) d[i] = s[i];
  const W* sw = reinterpret_cast<const W*>(s + head);
  W* dw = reinterpret_cast<W*>(d + head);
  for (int j = threadIdx.x; j < nw; j += blockDim.x) dw[j] = sw[j];
  for (int i = head + nw * kW + threadIdx.x; i < nb; i += blockDim.x) d[i] = s[i];
}

// the same when s and d disagree modulo 4: aligned 4-byte stores, each assembled from the two aligned source words it
// straddles.  The second word holds at least one byte of the run, so it lies inside the source allocation.
__device__ __forceinline__ void copy_shifted(const uint8_t* __restrict__ s, uint8_t* __restrict__ d, int nb) {
  const int head = min(nb, int((4 - int(uintptr_t(d) & 3)) & 3));
  const int nw = (nb - head) >> 2;
  for (int i = threadIdx.x; i < head; i += blockDim.x) d[i] = s[i];
  const uint8_t* sp = s + head;
  const int k = int(uintptr_t(sp) & 3);   // 1..3 here
  const uint32_t* sa = reinterpret_cast<const uint32_t*>(sp - k);
  uint32_t* dw = reinterpret_cast<uint32_t*>(d + head);
  for (int j = threadIdx.x; j < nw; j += blockDim.x) dw[j] = __funnelshift_r(sa[j], sa[j + 1], 8 * k);
  for (int i = head + nw * 4 + threadIdx.x; i < nb; i += blockDim.x) d[i] = s[i];
}

__global__ void __launch_bounds__(256) gather_pages_kernel(const GatherPage* __restrict__ tab, int n) {
  const int r = blockIdx.x;
  int lo = 0, hi = n - 1;   // last page with row0 <= r
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab[mid].row0 <= r) lo = mid; else hi = mid - 1;
  }
  const GatherPage g = tab[lo];
  const int y = r - g.row0;
  const int nb = g.iw * g.ch;
  const uint8_t* s = g.src + y * g.sh;
  uint8_t* d = g.dst + size_t(y) * nb;
  if (g.fast) {
    const uintptr_t phase = uintptr_t(s) ^ uintptr_t(d);
    if ((phase & 15) == 0) copy_same_phase<uint4>(s, d, nb);
    else if ((phase & 3) == 0) copy_same_phase<uint32_t>(s, d, nb);
    else copy_shifted(s, d, nb);
    return;
  }
  if (g.ch == 1) {
    for (int i = threadIdx.x; i < nb; i += blockDim.x) d[i] = s[i * g.sw];
    return;
  }
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    const int x = i / 3, c = i - 3 * x;
    d[i] = s[x * g.sw + c * g.sc];
  }
}

constexpr int kOutThreads = 256;
constexpr int kBlkPerThread = 8;   // blks elements per thread of a blks CTA

__device__ __forceinline__ bool finite_f(float v) { return (__float_as_uint(v) & 0x7f800000u) != 0x7f800000u; }

__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(__half v) { return __half2float(v); }
__device__ __forceinline__ float round_half(float v) { return __half2float(__float2half_rn(v)); }

// postprocess_mask's `(p * 255).astype(np.uint8)`: the product rounded to float32 (T = float) or, on a float16 map, to
// float16 (numpy's half arithmetic: the float product of two halves is exact, so rounding it once is RN_half of the
// exact product), truncated to int32 (0x80000000 where it does not fit, as cvttss2si gives it; numpy casts a half
// through float), and the low byte of that
template <typename T>
__device__ __forceinline__ uint32_t mask_byte(float p) {
  float v = __fmul_rn(p, 255.f);
  if constexpr (sizeof(T) == 2) v = round_half(v);
  return (v >= -2147483648.f && v < 2147483648.f) ? uint32_t(__float2int_rz(v)) & 0xffu : 0u;
}

// 4 consecutive elements of a row, one aligned load: 16 bytes of float, 8 of __half
template <typename T>
using Vec4 = typename std::conditional<sizeof(T) == 4, uint4, uint2>::type;

// row y of one page's mask and lines channel 0 of element T into the staging planes: 4 elements per thread and load
// (16 bytes of f32, 8 of f16, so every thread of a 1024-wide row has work at either size) when both rows are
// contiguous and aligned to a load, else one strided element per thread.  thresh is the DB threshold in the page's
// precision.  Returns the non-finite bits (2: mask, 4: lines).
template <typename T>
__device__ __forceinline__ uint32_t gather_row(const OutputGather& g, int y, int w, float thresh, uint8_t* __restrict__ mo,
                                               uint8_t* __restrict__ bo, float* __restrict__ lo) {
  using V = Vec4<T>;
  const T* ms = static_cast<const T*>(g.mask) + y * g.msh;
  const T* ls = static_cast<const T*>(g.lines) + y * g.lsh;
  uint32_t bad = 0;
  const bool vec = g.msw == 1 && g.lsw == 1 && (w & 3) == 0 && ((uintptr_t(ms) | uintptr_t(ls)) & (sizeof(V) - 1)) == 0;
  if (vec) {
    for (int x4 = threadIdx.x; x4 < (w >> 2); x4 += kOutThreads) {
      const V mr = __ldg(reinterpret_cast<const V*>(ms) + x4);
      const V lr = __ldg(reinterpret_cast<const V*>(ls) + x4);
      T mv[4], lv[4];
      memcpy(mv, &mr, sizeof(V));
      memcpy(lv, &lr, sizeof(V));
      uint32_t mb = 0, bb = 0;
      float lf[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float m = widen(mv[k]);
        lf[k] = widen(lv[k]);
        if (finite_f(m)) mb |= mask_byte<T>(m) << (8 * k);
        else bad |= 2;
        if (!finite_f(lf[k])) { bad |= 4; lf[k] = 0.f; }
        bb |= uint32_t(lf[k] > thresh) << (8 * k);
      }
      reinterpret_cast<uint32_t*>(mo)[x4] = mb;
      reinterpret_cast<uint32_t*>(bo)[x4] = bb;
      reinterpret_cast<float4*>(lo)[x4] = make_float4(lf[0], lf[1], lf[2], lf[3]);
    }
  } else {
    for (int x = threadIdx.x; x < w; x += kOutThreads) {
      const float m = widen(ms[x * g.msw]);
      float l = widen(ls[x * g.lsw]);
      if (!finite_f(m)) bad |= 2;
      if (!finite_f(l)) { bad |= 4; l = 0.f; }
      mo[x] = finite_f(m) ? uint8_t(mask_byte<T>(m)) : 0;
      bo[x] = l > thresh ? 1 : 0;
      lo[x] = l;
    }
  }
  return bad;
}

// grid (h + blks CTAs per page, n).  CTA x < h: row x of the page's mask and lines channel 0 (gather_row, in the
// page's dtype); the others: kBlkPerThread * 256 blks elements each, in row-major order of the workspace rows
__global__ void __launch_bounds__(kOutThreads) gather_outputs_kernel(const OutputGather* __restrict__ tab, int h, int w,
                                                                     int no, int ws_rows, float thresh,
                                                                     uint8_t* __restrict__ mask_u8,
                                                                     float* __restrict__ lines,
                                                                     uint8_t* __restrict__ bitmap,
                                                                     float* __restrict__ blks,
                                                                     int32_t* __restrict__ flags) {
  const int page = blockIdx.y;
  const OutputGather g = tab[page];
  uint32_t bad = 0;
  if (int(blockIdx.x) < h) {
    const int y = blockIdx.x;
    const size_t o = (size_t(page) * h + y) * w;
    float* lo = lines + size_t(page) * 2 * h * w + size_t(y) * w;
    bad = g.half ? gather_row<__half>(g, y, w, round_half(thresh), mask_u8 + o, bitmap + o, lo)
                 : gather_row<float>(g, y, w, thresh, mask_u8 + o, bitmap + o, lo);
  } else {
    const size_t total = size_t(ws_rows) * no;
    const size_t e0 = size_t(blockIdx.x - h) * kOutThreads * kBlkPerThread;
    float* out = blks + size_t(page) * total;
#pragma unroll
    for (int k = 0; k < kBlkPerThread; ++k) {
      const size_t e = e0 + size_t(k) * kOutThreads + threadIdx.x;
      if (e >= total) break;
      const int r = int(e / no), c = int(e - size_t(r) * no);
      float v;
      if (r < g.rows) {
        const long long i = r * g.bsr + c * g.bsc;
        v = g.half ? __half2float(static_cast<const __half*>(g.blks)[i]) : static_cast<const float*>(g.blks)[i];
        if (!finite_f(v)) { bad |= 1; v = 0.f; }
      } else {
        v = c == 4 ? __int_as_float(0x7fc00000) : 0.f;   // NaN objectness: `obj > conf_thres` is false
      }
      out[e] = v;
    }
  }
  if (bad) atomicOr(flags + page, int(bad));
}

}  // namespace

cudaError_t gather_outputs_launch(const OutputGather* d_tab, int n, int h, int w, int no, int ws_rows, float thresh,
                                  uint8_t* mask_u8, float* lines, uint8_t* bitmap, float* blks, int32_t* flags,
                                  cudaStream_t s) {
  if (n < 1 || h < 1 || w < 1 || no < 1 || ws_rows < 0) return cudaErrorInvalidValue;
  const size_t per_cta = size_t(kOutThreads) * kBlkPerThread;
  const unsigned blk_ctas = unsigned((size_t(ws_rows) * no + per_cta - 1) / per_cta);
  gather_outputs_kernel<<<dim3(unsigned(h) + blk_ctas, unsigned(n)), kOutThreads, 0, s>>>(
      d_tab, h, w, no, ws_rows, thresh, mask_u8, lines, bitmap, blks, flags);
  return cudaGetLastError();
}

cudaError_t gather_pages_launch(const GatherPage* d_tab, int n, int total_rows, cudaStream_t s) {
  if (n < 1 || total_rows < 1) return cudaErrorInvalidValue;
  gather_pages_kernel<<<unsigned(total_rows), 256, 0, s>>>(d_tab, n);
  return cudaGetLastError();
}

namespace {
struct ParamWords {
  uint4 w[240];   // 3840 bytes: with the other arguments, inside the 4 KB kernel parameter space
};
__global__ void param_words_kernel(const __grid_constant__ ParamWords p, int n, uint4* __restrict__ dst) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = p.w[i];
}
}  // namespace

cudaError_t upload_table_launch(const void* host, size_t bytes, void* dst, cudaStream_t s) {
  if (bytes % 16 || (uintptr_t(dst) & 15)) return cudaErrorInvalidValue;
  const size_t chunk = sizeof(ParamWords);
  for (size_t off = 0; off < bytes; off += chunk) {
    ParamWords p;
    const size_t b = bytes - off < chunk ? bytes - off : chunk;
    memcpy(p.w, static_cast<const char*>(host) + off, b);
    param_words_kernel<<<1, 256, 0, s>>>(p, int(b / 16), reinterpret_cast<uint4*>(static_cast<char*>(dst) + off));
  }
  return cudaGetLastError();
}

}  // namespace ctd
