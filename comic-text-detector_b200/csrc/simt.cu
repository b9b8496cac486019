// CUDA-core kernels: the fp32-accurate / bisecting convolution path (same op descriptors and
// weight packing as the tensor-core path) and the thin layers that are HBM-bound by nature
// (stem from u8, pools, nearest upsample, the seg/DB tails).  T = float or __half storage,
// arithmetic always fp32.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "kernels.h"

namespace ctd {

__device__ __forceinline__ float ldf(const float* p) { return *p; }
__device__ __forceinline__ float ldf(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ void stf(float* p, float v) { *p = v; }
__device__ __forceinline__ void stf(__half* p, float v) { *p = __float2half_rn(v); }

__device__ __forceinline__ float act_f(float v, int act) {
  switch (act) {
    case CTD_ACT_SILU: return v / (1.0f + expf(-v));
    case CTD_ACT_LEAKY: return v > 0.f ? v : 0.1f * v;
    case CTD_ACT_RELU: return fmaxf(v, 0.f);
    case CTD_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
    default: return v;
  }
}

void fill_conv_geom_taps(ConvGeom& g, int kind, int ksize, int stride) {
  memset(g.tap_dy, 0, sizeof(g.tap_dy));
  memset(g.tap_dx, 0, sizeof(g.tap_dx));
  if (kind == CTD_OP_DECONV4) {
    // out = 2*in - 1 + k  (k=4, s=2, p=1).  Output phase py: taps (ky, dy): py=0 -> (1,0),(3,-1); py=1 -> (0,+1),(2,0)
    g.n_phase = 4;
    g.taps = 4;
    g.out_mul = 2;
    g.in_stride = 1;
    const int d[2][2] = {{0, -1}, {1, 0}};
    for (int ph = 0; ph < 4; ++ph)
      for (int t = 0; t < 4; ++t) {
        g.tap_dy[ph][t] = int8_t(d[ph >> 1][t >> 1]);
        g.tap_dx[ph][t] = int8_t(d[ph & 1][t & 1]);
      }
  } else {
    g.n_phase = 1;
    g.taps = ksize * ksize;
    g.out_mul = 1;
    g.in_stride = stride;
    const int pad = ksize / 2;
    for (int t = 0; t < g.taps; ++t) {
      g.tap_dy[0][t] = int8_t(t / ksize - pad);
      g.tap_dx[0][t] = int8_t(t % ksize - pad);
    }
  }
}

// ---------------------------------------------------------------------------------------
// generic implicit-GEMM convolution on CUDA cores: CTA = 64 grid pixels x 64 couts, K chunks of 16
template <typename T>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvSimtParams p) {
  const ConvGeom& g = p.g;
  __shared__ float As[16][64 + 4];
  __shared__ float Ws[16][64 + 4];
  const int tid = threadIdx.x;
  const int phase = blockIdx.z;
  const long long npix = (long long)g.n_img * g.gh * g.gw;
  const long long pix0 = (long long)blockIdx.x * 64;
  const int co0 = blockIdx.y * 64;
  const int tx = tid & 15, ty = tid >> 4;  // tx -> couts (4 each), ty -> pixels (4 each)

  // loader roles
  const int lp = tid >> 2;        // pixel within tile loaded by this thread (0..63)
  const int lk = (tid & 3) * 4;   // first of 4 consecutive channels in the 16-chunk
  const long long lpix = pix0 + lp;
  int ln = 0, ly = 0, lx = 0;
  const bool lvalid = lpix < npix;
  if (lvalid) {
    ln = int(lpix / (g.gh * g.gw));
    const int r = int(lpix - (long long)ln * g.gh * g.gw);
    ly = r / g.gw;
    lx = r - ly * g.gw;
  }
  const int wco = tid >> 2;       // cout within tile whose weights this thread loads

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const T* wbase = static_cast<const T*>(p.w) + (size_t(phase) * g.cout_pad) * g.k_total;
  for (int tap = 0; tap < g.taps; ++tap) {
    const int sy = ly * g.in_stride + g.tap_dy[phase][tap];
    const int sx = lx * g.in_stride + g.tap_dx[phase][tap];
    const bool inb = lvalid && sy >= 0 && sy < g.src_h && sx >= 0 && sx < g.src_w;
    int kglob = tap * g.cin_total;
    for (int s = 0; s < g.n_src; ++s) {
      const T* sp = static_cast<const T*>(p.src[s]);
      const size_t poff = (size_t(ln) * g.src_h * g.src_w + size_t(sy) * g.src_w + sx) * g.src_cstride[s];
      for (int c0 = 0; c0 < g.src_c[s]; c0 += 16) {
#pragma unroll
        for (int e = 0; e < 4; ++e) As[lk + e][lp] = inb ? ldf(sp + poff + c0 + lk + e) : 0.f;
        const int co = co0 + wco;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          Ws[lk + e][wco] = co < g.cout_pad ? ldf(wbase + size_t(co) * g.k_total + kglob + c0 + lk + e) : 0.f;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          float a[4], w[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
          for (int j = 0; j < 4; ++j) w[j] = Ws[k][tx * 4 + j];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
        __syncthreads();
      }
      kglob += g.src_c[s];
    }
  }
  // epilogue
  const int ph_y = phase >> 1, ph_x = phase & 1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long pix = pix0 + ty * 4 + i;
    if (pix >= npix) continue;
    const int n = int(pix / (g.gh * g.gw));
    const int r = int(pix - (long long)n * g.gh * g.gw);
    const int gy = r / g.gw, gx = r - gy * g.gw;
    const int oy = gy * g.out_mul + ph_y, ox = gx * g.out_mul + ph_x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = co0 + tx * 4 + j;
      if (co >= g.cout) continue;
      float v = acc[i][j] + p.bias[co];
      if (p.dst != nullptr) {
        T* o = static_cast<T*>(p.dst) + (size_t(n) * g.dst_h * g.dst_w + size_t(oy) * g.dst_w + ox) * g.dst_cstride +
               g.dst_coff + co;
        v = act_f(v, g.act);
        if (g.residual) v += ldf(o);
        stf(o, v);
      } else {
        const int no = 5 + p.nc;
        const int a = co / no, oo = co - a * no;
        const float s = 1.0f / (1.0f + expf(-v));
        float rr;
        if (oo == 0) rr = (s * 2.0f - 0.5f + float(gx)) * p.det_stride;
        else if (oo == 1) rr = (s * 2.0f - 0.5f + float(gy)) * p.det_stride;
        else if (oo == 2) rr = (s * 2.0f) * (s * 2.0f) * p.anchor_wh[2 * a];
        else if (oo == 3) rr = (s * 2.0f) * (s * 2.0f) * p.anchor_wh[2 * a + 1];
        else rr = s;
        float* rows = p.blks + (size_t(n) * p.blks_rows_per_img + p.level_row0) * no;
        rows[(size_t(a) * g.gh * g.gw + size_t(gy) * g.gw + gx) * no + oo] = rr;
      }
    }
  }
}

template <typename T>
cudaError_t conv_simt_launch(const ConvSimtParams& p, cudaStream_t s) {
  const long long npix = (long long)p.g.n_img * p.g.gh * p.g.gw;
  dim3 grid(unsigned((npix + 63) / 64), unsigned((p.g.cout_pad + 63) / 64), unsigned(p.g.n_phase));
  conv_simt_kernel<T><<<grid, 256, 0, s>>>(p);
  return cudaGetLastError();
}
template cudaError_t conv_simt_launch<float>(const ConvSimtParams&, cudaStream_t);
template cudaError_t conv_simt_launch<__half>(const ConvSimtParams&, cudaStream_t);

// ---------------------------------------------------------------------------------------
// stem: Conv 6x6 s2 p2, 3 -> cout(32), reads the BGR HWC page: u8 with the /255 fused (inference.py:78), or the f32
// staging page of a float input as it is
__device__ __forceinline__ float page_value(const uint8_t* p) { return float(*p) / 255.0f; }
__device__ __forceinline__ float page_value(const float* p) { return *p; }

template <typename T, typename P>
__global__ void __launch_bounds__(256) stem_kernel(const P* __restrict__ pages, int n, int h, int w,
                                                   const float* __restrict__ wgt, const float* __restrict__ bias,
                                                   T* __restrict__ dst, int dst_cstride, int dst_coff, int cout,
                                                   int act) {
  // CTA: 8x32 output pixels; input patch (2*8+4) x (2*32+4) x 3
  constexpr int TH = 8, TW = 32;
  constexpr int PH = 2 * TH + 4, PW = 2 * TW + 4;
  __shared__ float patch[PH][PW * 3];
  __shared__ float ws[108 * 32];
  __shared__ float bs[32];
  const int oh = h / 2, ow = w / 2;
  const int tiles_x = (ow + TW - 1) / TW, tiles_y = (oh + TH - 1) / TH;
  const int img = blockIdx.x / (tiles_x * tiles_y);
  const int tr = blockIdx.x % (tiles_x * tiles_y);
  const int oy0 = (tr / tiles_x) * TH, ox0 = (tr % tiles_x) * TW;
  const int iy0 = oy0 * 2 - 2, ix0 = ox0 * 2 - 2;
  for (int i = threadIdx.x; i < 108 * 32; i += 256) {
    // ws[k][co] <- wgt[co][k]
    const int co = i & 31, k = i >> 5;
    ws[i] = co < cout ? wgt[co * 108 + k] : 0.f;
  }
  if (threadIdx.x < 32) bs[threadIdx.x] = threadIdx.x < cout ? bias[threadIdx.x] : 0.f;
  const P* page = pages + size_t(img) * h * w * 3;
  for (int i = threadIdx.x; i < PH * PW * 3; i += 256) {
    const int py = i / (PW * 3), rem = i - py * (PW * 3);
    const int px = rem / 3, c = rem - px * 3;
    const int iy = iy0 + py, ix = ix0 + px;
    float v = 0.f;
    if (iy >= 0 && iy < h && ix >= 0 && ix < w) v = page_value(page + (size_t(iy) * w + ix) * 3 + c);
    patch[py][rem] = v;
  }
  __syncthreads();
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  float acc[32];
#pragma unroll
  for (int co = 0; co < 32; ++co) acc[co] = bs[co];
  for (int ky = 0; ky < 6; ++ky)
#pragma unroll
    for (int kc = 0; kc < 18; ++kc) {  // kc = kx*3 + c
      const float a = patch[ty * 2 + ky][tx * 6 + kc];
      const float* wr = &ws[(ky * 18 + kc) * 32];
#pragma unroll
      for (int co = 0; co < 32; ++co) acc[co] = fmaf(a, wr[co], acc[co]);
    }
  const int oy = oy0 + ty, ox = ox0 + tx;
  if (oy < oh && ox < ow) {
    T* o = dst + (size_t(img) * oh * ow + size_t(oy) * ow + ox) * dst_cstride + dst_coff;
    for (int co = 0; co < cout; ++co) stf(o + co, act_f(acc[co], act));
  }
}

template <typename T, typename P>
cudaError_t stem_launch(const P* pages, int n, int h, int w, const float* wgt, const float* bias, T* dst,
                        int dst_cstride, int dst_coff, int cout, int act, cudaStream_t s) {
  if (cout > 32) return cudaErrorInvalidValue;
  const int oh = h / 2, ow = w / 2;
  const int tiles = ((ow + 31) / 32) * ((oh + 7) / 8);
  stem_kernel<T, P><<<n * tiles, 256, 0, s>>>(pages, n, h, w, wgt, bias, dst, dst_cstride, dst_coff, cout, act);
  return cudaGetLastError();
}
template cudaError_t stem_launch<float, uint8_t>(const uint8_t*, int, int, int, const float*, const float*, float*, int,
                                                 int, int, int, cudaStream_t);
template cudaError_t stem_launch<__half, uint8_t>(const uint8_t*, int, int, int, const float*, const float*, __half*,
                                                  int, int, int, int, cudaStream_t);
template cudaError_t stem_launch<float, float>(const float*, int, int, int, const float*, const float*, float*, int,
                                               int, int, int, cudaStream_t);
template cudaError_t stem_launch<__half, float>(const float*, int, int, int, const float*, const float*, __half*, int,
                                                int, int, int, cudaStream_t);

// ---------------------------------------------------------------------------------------
// input pre-pass: f32 or f16 NCHW -> HWC staging page.  One thread per 4 pixels (h * w is a multiple of 4096): three
// 4-pixel plane loads (16 bytes of f32, 8 of f16), then the 12 values of the 4 pixels as three 16-byte (f32) or 8-byte
// (fp16) stores.
__device__ __forceinline__ void st_hwc4(float* d, const float (&v)[12]) {
  float4* o = reinterpret_cast<float4*>(d);
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
}
__device__ __forceinline__ void st_hwc4(__half* d, const float (&v)[12]) {
  uint2* o = reinterpret_cast<uint2*>(d);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const __half2 a = __floats2half2_rn(v[4 * k], v[4 * k + 1]), b = __floats2half2_rn(v[4 * k + 2], v[4 * k + 3]);
    uint2 u;
    memcpy(&u.x, &a, 4);
    memcpy(&u.y, &b, 4);
    o[k] = u;
  }
}

// pixels 4q .. 4q + 3 of a plane, widened exactly to float
__device__ __forceinline__ float4 ld_px4(const float* p, size_t q) { return __ldcs(reinterpret_cast<const float4*>(p) + q); }
__device__ __forceinline__ float4 ld_px4(const __half* p, size_t q) {
  const uint2 u = __ldcs(reinterpret_cast<const uint2*>(p) + q);
  __half2 a, b;
  memcpy(&a, &u.x, 4);
  memcpy(&b, &u.y, 4);
  const float2 fa = __half22float2(a), fb = __half22float2(b);
  return make_float4(fa.x, fa.y, fb.x, fb.y);
}

template <typename X, typename S>
__global__ void __launch_bounds__(256) nchw_to_hwc_kernel(const X* __restrict__ x, size_t hw4, size_t total4,
                                                          S* __restrict__ dst) {
  const size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x;
  if (i >= total4) return;
  const size_t img = i / hw4, q = i - img * hw4;
  const X* src = x + img * 3 * hw4 * 4;
  const float4 b = ld_px4(src, q), g = ld_px4(src + hw4 * 4, q), r = ld_px4(src + 2 * hw4 * 4, q);
  const float v[12] = {b.x, g.x, r.x, b.y, g.y, r.y, b.z, g.z, r.z, b.w, g.w, r.w};
  st_hwc4(dst + i * 12, v);
}

template <typename X, typename S>
cudaError_t nchw_to_hwc_launch(const X* x, int n, int h, int w, S* dst, cudaStream_t s) {
  if ((size_t(h) * w) % 4) return cudaErrorInvalidValue;
  const size_t hw4 = size_t(h) * w / 4, total4 = size_t(n) * hw4;
  nchw_to_hwc_kernel<X, S><<<unsigned((total4 + 255) / 256), 256, 0, s>>>(x, hw4, total4, dst);
  return cudaGetLastError();
}
template cudaError_t nchw_to_hwc_launch<float, float>(const float*, int, int, int, float*, cudaStream_t);
template cudaError_t nchw_to_hwc_launch<float, __half>(const float*, int, int, int, __half*, cudaStream_t);
template cudaError_t nchw_to_hwc_launch<__half, float>(const __half*, int, int, int, float*, cudaStream_t);
template cudaError_t nchw_to_hwc_launch<__half, __half>(const __half*, int, int, int, __half*, cudaStream_t);

// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void avgpool2_kernel(const T* __restrict__ src, int n, int h, int w, int c, int scs, T* __restrict__ dst,
                                int dcs) {
  const int oh = h / 2, ow = w / 2;
  const long long total = (long long)n * oh * ow * c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = int(i % c);
    long long r = i / c;
    const int ox = int(r % ow);
    r /= ow;
    const int oy = int(r % oh);
    const int img = int(r / oh);
    const T* s0 = src + ((size_t(img) * h + 2 * oy) * w + 2 * ox) * scs + ch;
    const float v = (ldf(s0) + ldf(s0 + scs) + ldf(s0 + size_t(w) * scs) + ldf(s0 + size_t(w) * scs + scs)) * 0.25f;
    stf(dst + ((size_t(img) * oh + oy) * ow + ox) * dcs + ch, v);
  }
}
template <typename T>
cudaError_t avgpool2_launch(const T* src, int n, int h, int w, int c, int scs, T* dst, int dcs, cudaStream_t s) {
  const long long total = (long long)n * (h / 2) * (w / 2) * c;
  avgpool2_kernel<T><<<unsigned((total + 255) / 256), 256, 0, s>>>(src, n, h, w, c, scs, dst, dcs);
  return cudaGetLastError();
}
template cudaError_t avgpool2_launch<float>(const float*, int, int, int, int, int, float*, int, cudaStream_t);
template cudaError_t avgpool2_launch<__half>(const __half*, int, int, int, int, int, __half*, int, cudaStream_t);

// 8-channel vectors (16 bytes of fp16 / 32 bytes of fp32)
struct Vec8 { float v[8]; };
__device__ __forceinline__ Vec8 ldv8(const __half* p) {
  Vec8 r;
  const uint4 q = *reinterpret_cast<const uint4*>(p);
  const __half2* hh = reinterpret_cast<const __half2*>(&q);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t = __half22float2(hh[e]);
    r.v[2 * e] = t.x;
    r.v[2 * e + 1] = t.y;
  }
  return r;
}
__device__ __forceinline__ Vec8 ldv8(const float* p) {
  Vec8 r;
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
__device__ __forceinline__ void stv8(__half* p, const Vec8& r) {
  uint4 q;
  __half2* hh = reinterpret_cast<__half2*>(&q);
#pragma unroll
  for (int e = 0; e < 4; ++e) hh[e] = __floats2half2_rn(r.v[2 * e], r.v[2 * e + 1]);
  *reinterpret_cast<uint4*>(p) = q;
}
__device__ __forceinline__ void stv8(float* p, const Vec8& r) {
  *reinterpret_cast<float4*>(p) = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(r.v[4], r.v[5], r.v[6], r.v[7]);
}

// SPPF pools: buf[..., 0:c] = x (already written); writes y1=mp5(x), y2=mp5(y1)=mp9(x), y3=mp13(x)
// into channel slots [c,2c), [2c,3c), [3c,4c).  Chained 5x5 s1 p2 max pools equal 9x9 / 13x13 windows
// clipped at the border (-inf padding).  One thread = one pixel x 8 channels.
template <typename T>
__global__ void sppf_pool_kernel(T* __restrict__ buf, int n, int h, int w, int c, int cs) {
  const int c8 = c / 8;
  const long long total = (long long)n * h * w * c8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = int(i % c8) * 8;
  long long r = i / c8;
  const int x = int(r % w);
  r /= w;
  const int y = int(r % h);
  const int img = int(r / h);
  const T* base = buf + size_t(img) * h * w * cs + ch;
  Vec8 m5, m9, m13;
#pragma unroll
  for (int e = 0; e < 8; ++e) m5.v[e] = m9.v[e] = m13.v[e] = -INFINITY;
  for (int dy = -6; dy <= 6; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= h) continue;
    for (int dx = -6; dx <= 6; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= w) continue;
      const Vec8 v = ldv8(base + (size_t(yy) * w + xx) * cs);
      const int ad = max(abs(dy), abs(dx));
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        m13.v[e] = fmaxf(m13.v[e], v.v[e]);
        if (ad <= 4) m9.v[e] = fmaxf(m9.v[e], v.v[e]);
        if (ad <= 2) m5.v[e] = fmaxf(m5.v[e], v.v[e]);
      }
    }
  }
  T* o = buf + ((size_t(img) * h + y) * w + x) * cs + ch;
  stv8(o + c, m5);
  stv8(o + 2 * c, m9);
  stv8(o + 3 * c, m13);
}
// Same result, whole image of one 8-channel group resident in shared memory: the three chained 5x5 pools run as
// separable row / column passes (2 x 5 reads per level instead of one 13x13 window per pixel).
template <typename T>
__global__ void sppf_pool_tile_kernel(T* __restrict__ buf, int h, int w, int c, int cs) {
  extern __shared__ __align__(16) unsigned char sppf_sm[];
  T* a = reinterpret_cast<T*>(sppf_sm);
  T* b = a + size_t(h) * w * 8;
  const int ch = blockIdx.x * 8, img = blockIdx.y, hw = h * w;
  T* base = buf + size_t(img) * hw * cs + ch;
  for (int i = threadIdx.x; i < hw; i += blockDim.x) stv8(a + size_t(i) * 8, ldv8(base + size_t(i) * cs));
  __syncthreads();
  for (int level = 1; level <= 3; ++level) {
    for (int i = threadIdx.x; i < hw; i += blockDim.x) {   // row pass a -> b
      const int y = i / w, x = i - y * w;
      Vec8 m = ldv8(a + size_t(i) * 8);
#pragma unroll
      for (int d = -2; d <= 2; ++d) {
        if (d == 0 || x + d < 0 || x + d >= w) continue;
        const Vec8 v = ldv8(a + size_t(i + d) * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) m.v[e] = fmaxf(m.v[e], v.v[e]);
      }
      stv8(b + size_t(i) * 8, m);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < hw; i += blockDim.x) {   // column pass b -> a (+ output slot `level`)
      const int y = i / w;
      Vec8 m = ldv8(b + size_t(i) * 8);
#pragma unroll
      for (int d = -2; d <= 2; ++d) {
        if (d == 0 || y + d < 0 || y + d >= h) continue;
        const Vec8 v = ldv8(b + size_t(i + d * w) * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) m.v[e] = fmaxf(m.v[e], v.v[e]);
      }
      stv8(a + size_t(i) * 8, m);
      stv8(base + size_t(i) * cs + size_t(level) * c, m);
    }
    __syncthreads();
  }
}

template <typename T>
cudaError_t sppf_pool_launch(T* buf, int n, int h, int w, int c, int cs, cudaStream_t s) {
  if (c % 8 || cs % 8) return cudaErrorInvalidValue;
  const size_t smem = size_t(2) * h * w * 8 * sizeof(T);
  if (smem <= 200 * 1024) {
    // per device, so set on every launch (cheap; a process may own engines on several GPUs)
    cudaFuncSetAttribute(sppf_pool_tile_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    sppf_pool_tile_kernel<T><<<dim3(c / 8, n), 256, smem, s>>>(buf, h, w, c, cs);
    return cudaGetLastError();
  }
  const long long total = (long long)n * h * w * (c / 8);
  sppf_pool_kernel<T><<<unsigned((total + 127) / 128), 128, 0, s>>>(buf, n, h, w, c, cs);
  return cudaGetLastError();
}
template cudaError_t sppf_pool_launch<float>(float*, int, int, int, int, int, cudaStream_t);
template cudaError_t sppf_pool_launch<__half>(__half*, int, int, int, int, int, cudaStream_t);

template <typename T>
__global__ void upsample2_kernel(const T* __restrict__ src, int n, int h, int w, int c, int scs, T* __restrict__ dst,
                                 int dcs) {
  const int oh = 2 * h, ow = 2 * w, c8 = c / 8;
  const long long total = (long long)n * oh * ow * c8;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = int(i % c8) * 8;
  long long r = i / c8;
  const int ox = int(r % ow);
  r /= ow;
  const int oy = int(r % oh);
  const int img = int(r / oh);
  stv8(dst + ((size_t(img) * oh + oy) * ow + ox) * dcs + ch, ldv8(src + ((size_t(img) * h + oy / 2) * w + ox / 2) * scs + ch));
}
template <typename T>
cudaError_t upsample2_launch(const T* src, int n, int h, int w, int c, int scs, T* dst, int dcs, cudaStream_t s) {
  if (c % 8 || scs % 8 || dcs % 8) return cudaErrorInvalidValue;
  const long long total = (long long)n * 4 * h * w * (c / 8);
  upsample2_kernel<T><<<unsigned((total + 255) / 256), 256, 0, s>>>(src, n, h, w, c, scs, dst, dcs);
  return cudaGetLastError();
}
template cudaError_t upsample2_launch<float>(const float*, int, int, int, int, int, float*, int, cudaStream_t);
template cudaError_t upsample2_launch<__half>(const __half*, int, int, int, int, int, __half*, int, cudaStream_t);

// ---------------------------------------------------------------------------------------
// seg tail: ConvTranspose2d(C,1,4,2,1,bias=False) + Sigmoid (basemodel.py:57-60) and
// postprocess_mask's (p*255).astype(uint8) (inference.py:96-99).
// CTA = 16x16 input pixels.  Each thread first forms the 16 per-tap partial dot products
// part[ky][kx] = sum_c x[c] * w[c][ky][kx] of ITS input pixel (one 128-byte vector load), the
// partials go to shared memory, then 14x14 threads each assemble a 2x2 output block from the
// partials of the 3x3 neighbourhood (out = 2*in - 1 + k).  HBM traffic = the input once (+31% halo)
// plus the 5 bytes/pixel of output.
__device__ __forceinline__ void load8(const __half* p, float* f) {
  const uint4 r = *reinterpret_cast<const uint4*>(p);
  const __half2* hh = reinterpret_cast<const __half2*>(&r);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t = __half22float2(hh[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
}
__device__ __forceinline__ void load8(const float* p, float* f) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

template <typename T>
__global__ void __launch_bounds__(256) seg_tail_kernel(const T* __restrict__ src, int n, int h, int w, int c, int cs,
                                                       const float* __restrict__ wgt, float* __restrict__ mask_f32,
                                                       uint8_t* __restrict__ mask_u8) {
  extern __shared__ float sm[];
  float* wsm = sm;                 // [c][16]  (ci major, tap = ky*4+kx)
  float* part = sm + c * 16;       // [256][17]
  for (int i = threadIdx.x; i < 16 * c; i += 256) wsm[i] = wgt[i];
  __syncthreads();
  const int tiles_x = (w + 13) / 14, tiles_y = (h + 13) / 14;
  const int img = blockIdx.x / (tiles_x * tiles_y);
  const int tr = blockIdx.x % (tiles_x * tiles_y);
  const int q0y = (tr / tiles_x) * 14, q0x = (tr % tiles_x) * 14;  // first q block of this CTA
  const int lx = threadIdx.x & 15, ly = threadIdx.x >> 4;
  // phase 1: threads 0..127 each form the partials of TWO input pixels (rows ly and ly+8 of the tile), so
  // every weight vector read from shared memory feeds 8 FMAs instead of 4
  if (threadIdx.x < 128) {
    const int ix = q0x - 1 + lx;
    const int iy0 = q0y - 1 + ly, iy1 = iy0 + 8;
    const bool v0 = iy0 >= 0 && iy0 < h && ix >= 0 && ix < w;
    const bool v1 = iy1 >= 0 && iy1 < h && ix >= 0 && ix < w;
    float a0[16], a1[16];
#pragma unroll
    for (int t = 0; t < 16; ++t) { a0[t] = 0.f; a1[t] = 0.f; }
    const T* sp0 = src + ((size_t(img) * h + (v0 ? iy0 : 0)) * w + (v0 ? ix : 0)) * cs;
    const T* sp1 = src + ((size_t(img) * h + (v1 ? iy1 : 0)) * w + (v1 ? ix : 0)) * cs;
    for (int c0 = 0; c0 < c; c0 += 8) {
      float x0[8], x1[8];
      load8(sp0 + c0, x0);
      load8(sp1 + c0, x1);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float4* wr = reinterpret_cast<const float4*>(wsm + (c0 + e) * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 ww = wr[q];
          a0[4 * q + 0] = fmaf(x0[e], ww.x, a0[4 * q + 0]);
          a0[4 * q + 1] = fmaf(x0[e], ww.y, a0[4 * q + 1]);
          a0[4 * q + 2] = fmaf(x0[e], ww.z, a0[4 * q + 2]);
          a0[4 * q + 3] = fmaf(x0[e], ww.w, a0[4 * q + 3]);
          a1[4 * q + 0] = fmaf(x1[e], ww.x, a1[4 * q + 0]);
          a1[4 * q + 1] = fmaf(x1[e], ww.y, a1[4 * q + 1]);
          a1[4 * q + 2] = fmaf(x1[e], ww.z, a1[4 * q + 2]);
          a1[4 * q + 3] = fmaf(x1[e], ww.w, a1[4 * q + 3]);
        }
      }
    }
#pragma unroll
    for (int t = 0; t < 16; ++t) {
      part[(ly * 16 + lx) * 17 + t] = v0 ? a0[t] : 0.f;
      part[((ly + 8) * 16 + lx) * 17 + t] = v1 ? a1[t] : 0.f;
    }
  }
  __syncthreads();
  if (lx >= 14 || ly >= 14) return;
  const int qy = q0y + ly, qx = q0x + lx;
  if (qy >= h || qx >= w) return;
  // local index of input pixel (qy+dy, qx+dx) is (ly+1+dy, lx+1+dx)
  auto P = [&](int dy, int dx, int ky, int kx) { return part[((ly + 1 + dy) * 16 + (lx + 1 + dx)) * 17 + ky * 4 + kx]; };
  float o[2][2];
#pragma unroll
  for (int py = 0; py < 2; ++py)
#pragma unroll
    for (int px = 0; px < 2; ++px) {
      // oy = 2*qy + py: taps (dy,ky): py=0 -> (0,1),(-1,3); py=1 -> (0,2),(+1,0)
      const int dyA = 0, kyA = py ? 2 : 1, dyB = py ? 1 : -1, kyB = py ? 0 : 3;
      const int dxA = 0, kxA = px ? 2 : 1, dxB = px ? 1 : -1, kxB = px ? 0 : 3;
      o[py][px] = P(dyA, dxA, kyA, kxA) + P(dyA, dxB, kyA, kxB) + P(dyB, dxA, kyB, kxA) + P(dyB, dxB, kyB, kxB);
    }
  const int H = 2 * h, W = 2 * w;
#pragma unroll
  for (int py = 0; py < 2; ++py) {
    const size_t o_idx = (size_t(img) * H + 2 * qy + py) * W + 2 * qx;
    const float s0 = 1.0f / (1.0f + expf(-o[py][0])), s1 = 1.0f / (1.0f + expf(-o[py][1]));
    *reinterpret_cast<float2*>(mask_f32 + o_idx) = make_float2(s0, s1);
    *reinterpret_cast<uchar2*>(mask_u8 + o_idx) = make_uchar2((uint8_t)(s0 * 255.0f), (uint8_t)(s1 * 255.0f));
  }
}
template <typename T>
cudaError_t seg_tail_launch(const T* src, int n, int h, int w, int c, int cs, const float* wgt, float* mask_f32,
                            uint8_t* mask_u8, cudaStream_t s) {
  if (c % 8 != 0 || cs % 8 != 0) return cudaErrorInvalidValue;
  const int tiles = ((w + 13) / 14) * ((h + 13) / 14);
  const size_t smem = (size_t(c) * 16 + 256 * 17) * sizeof(float);
  seg_tail_kernel<T><<<n * tiles, 256, smem, s>>>(src, n, h, w, c, cs, wgt, mask_f32, mask_u8);
  return cudaGetLastError();
}
template cudaError_t seg_tail_launch<float>(const float*, int, int, int, int, int, const float*, float*, uint8_t*,
                                            cudaStream_t);
template cudaError_t seg_tail_launch<__half>(const __half*, int, int, int, int, int, const float*, float*, uint8_t*,
                                             cudaStream_t);

// ---------------------------------------------------------------------------------------
// DB tail (basemodel.py:99-103 binarize[3..6] and 138-142 thresh[3..7]); input = 32 channels at
// 1/4 resolution: [0,16) = ReLU(BN(binarize conv3x3)), [16,32) = ReLU(BN(thresh conv3x3)).
// params (fp32), per branch b in {0: binarize, 1: thresh}, base = b*1105:
//   w3[ci][co][dy][dx] (16*16*4, BN folded), b3[co] (16), w6[co][dy][dx] (16*4), b6 (1)
// One thread per 1/4-res pixel: 16 in -> 2x2x16 -> 4x4 outputs per branch.
// lines[n][0] = sigmoid(binarize) (shrink), lines[n][1] = sigmoid(thresh)  (basemodel.py:114-125)
template <typename T>
__global__ void __launch_bounds__(128) db_tail_kernel(const T* __restrict__ src, int n, int h, int w, int cs,
                                                      const float* __restrict__ params, float* __restrict__ lines,
                                                      uint8_t* __restrict__ bitmap, float db_thresh) {
  // shared layout per branch: w3s[d1][ci][co] (1024), b3 (16), w6s[d2][co] (64), b6 (1) -> float4 reads over co
  __shared__ __align__(16) float prm[2 * 1108];
  for (int i = threadIdx.x; i < 2 * 1105; i += blockDim.x) {
    const int b = i / 1105, r = i - b * 1105;
    float v = params[i];
    int dstp;
    if (r < 1024) {
      const int d1 = r & 3, co = (r >> 2) & 15, ci = r >> 6;
      dstp = d1 * 256 + ci * 16 + co;
    } else if (r < 1040) {
      dstp = r;
    } else if (r < 1104) {
      const int q = r - 1040, d2 = q & 3, co = q >> 2;
      dstp = 1040 + d2 * 16 + co;
    } else {
      dstp = 1104;
    }
    prm[b * 1108 + dstp] = v;
  }
  __syncthreads();
  const long long total = (long long)n * h * w;
  // grid-stride: the 8.8 KB parameter re-layout above is paid once per CTA, not once per 128 pixels
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
  const int x = int(i % w), y = int((i / w) % h), img = int(i / ((long long)w * h));
  const T* sp = src + i * cs;
  const int H = 4 * h, W = 4 * w;
  float xin[32];
  load8(sp, xin);
  load8(sp + 8, xin + 8);
  load8(sp + 16, xin + 16);
  load8(sp + 24, xin + 24);
#pragma unroll 1
  for (int b = 0; b < 2; ++b) {
    const float* w3s = prm + b * 1108;
    const float* b3 = w3s + 1024;
    const float* w6s = b3 + 16;
    const float b6 = w6s[64];
    float res[16];
#pragma unroll
    for (int d1 = 0; d1 < 4; ++d1) {  // first deconv position (dy1,dx1)
      float t[16];
#pragma unroll
      for (int co = 0; co < 16; ++co) t[co] = b3[co];
#pragma unroll
      for (int ci = 0; ci < 16; ++ci) {
        const float xv = xin[b * 16 + ci];
        const float4* wr = reinterpret_cast<const float4*>(w3s + d1 * 256 + ci * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 ww = wr[q];
          t[4 * q + 0] = fmaf(xv, ww.x, t[4 * q + 0]);
          t[4 * q + 1] = fmaf(xv, ww.y, t[4 * q + 1]);
          t[4 * q + 2] = fmaf(xv, ww.z, t[4 * q + 2]);
          t[4 * q + 3] = fmaf(xv, ww.w, t[4 * q + 3]);
        }
      }
#pragma unroll
      for (int co = 0; co < 16; ++co) t[co] = fmaxf(t[co], 0.f);
#pragma unroll
      for (int d2 = 0; d2 < 4; ++d2) {
        float a = b6;
        const float4* wr = reinterpret_cast<const float4*>(w6s + d2 * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 ww = wr[q];
          a = fmaf(t[4 * q + 0], ww.x, a);
          a = fmaf(t[4 * q + 1], ww.y, a);
          a = fmaf(t[4 * q + 2], ww.z, a);
          a = fmaf(t[4 * q + 3], ww.w, a);
        }
        const int oy = (d1 >> 1) * 2 + (d2 >> 1), ox = (d1 & 1) * 2 + (d2 & 1);
        res[oy * 4 + ox] = 1.0f / (1.0f + expf(-a));
      }
    }
    float* outp = lines + ((size_t(img) * 2 + b) * H + 4 * y) * W + 4 * x;
#pragma unroll
    for (int oy = 0; oy < 4; ++oy) {
      *reinterpret_cast<float4*>(outp + size_t(oy) * W) = make_float4(res[oy * 4], res[oy * 4 + 1], res[oy * 4 + 2], res[oy * 4 + 3]);
      if (b == 0) {
        uchar4 bm = make_uchar4(res[oy * 4] > db_thresh, res[oy * 4 + 1] > db_thresh, res[oy * 4 + 2] > db_thresh,
                                res[oy * 4 + 3] > db_thresh);
        *reinterpret_cast<uchar4*>(bitmap + (size_t(img) * H + 4 * y + oy) * W + 4 * x) = bm;
      }
    }
  }
  }
}
template <typename T>
cudaError_t db_tail_launch(const T* src, int n, int h, int w, int cs, const float* params, float* lines,
                           uint8_t* bitmap, float db_thresh, cudaStream_t s) {
  const long long total = (long long)n * h * w;
  const long long blocks = (total + 127) / 128;
  const long long cap = 132LL * 16;   // a few resident CTAs per SM, each looping over its share of the pixels
  db_tail_kernel<T><<<unsigned(blocks < cap ? blocks : cap), 128, 0, s>>>(src, n, h, w, cs, params, lines, bitmap, db_thresh);
  return cudaGetLastError();
}
template cudaError_t db_tail_launch<float>(const float*, int, int, int, int, const float*, float*, uint8_t*, float,
                                           cudaStream_t);
template cudaError_t db_tail_launch<__half>(const __half*, int, int, int, int, const float*, float*, uint8_t*, float,
                                            cudaStream_t);


// ---------------------------------------------------------------------------------------------
// split-fp16 mode: fp32 NHWC channel slice -> hi = fp16(x), lo = fp16((x - hi) * kSplitLoScale) planes (4 channels
// per thread)
__global__ void split_planes_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo,
                                    size_t npix, int c4, int cstride) {
  const size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x;
  if (i >= npix * size_t(c4)) return;
  const size_t pix = i / size_t(c4);
  const int q = int(i - pix * size_t(c4));
  const size_t off = pix * size_t(cstride) + size_t(q) * 4;
  const float4 v = *reinterpret_cast<const float4*>(src + off);
  const __half h0 = __float2half_rn(v.x), h1 = __float2half_rn(v.y), h2 = __float2half_rn(v.z), h3 = __float2half_rn(v.w);
  const __half l0 = __float2half_rn((v.x - __half2float(h0)) * kSplitLoScale);
  const __half l1 = __float2half_rn((v.y - __half2float(h1)) * kSplitLoScale);
  const __half l2 = __float2half_rn((v.z - __half2float(h2)) * kSplitLoScale);
  const __half l3 = __float2half_rn((v.w - __half2float(h3)) * kSplitLoScale);
  __half2 hh[2] = {__halves2half2(h0, h1), __halves2half2(h2, h3)};
  __half2 ll[2] = {__halves2half2(l0, l1), __halves2half2(l2, l3)};
  *reinterpret_cast<uint2*>(hi + off) = *reinterpret_cast<uint2*>(hh);
  *reinterpret_cast<uint2*>(lo + off) = *reinterpret_cast<uint2*>(ll);
}

cudaError_t split_planes_launch(const float* src, __half* hi, __half* lo, size_t npix, int c, int cstride,
                                cudaStream_t s) {
  if (c % 4 || cstride % 4) return cudaErrorInvalidValue;
  const size_t total = npix * size_t(c / 4);
  if (total == 0) return cudaSuccess;
  split_planes_kernel<<<unsigned((total + 255) / 256), 256, 0, s>>>(src, hi, lo, npix, c / 4, cstride);
  return cudaGetLastError();
}

}  // namespace ctd
