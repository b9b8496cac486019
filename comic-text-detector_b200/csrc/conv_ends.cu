// The network's two ends on the tensor cores (sm_90a): the stem and the seg tail.
//
// Both are small GEMMs (N = 32 / 8, K = 192 / 576) over large images, so their time is the bytes they move.  Each
// 16x16-pixel output tile loads its input region ONCE into shared memory with one TMA box, halo included, and TMA's
// out-of-bounds zero fill stands in for the convolution padding.  The consumers build the wgmma A fragments of every
// tap from that one tile with ldmatrix (wgmma with A in registers); B (the weights, 12 / 9 KB) is loaded once per CTA.
//
// Persistent, one CTA per SM, 384 threads: warpgroup 0 = TMA producer (one elected thread, a ring of input stages, so
// the next tiles load under the current one's MMAs and stores), warpgroups 1 and 2 = consumers, each owning 8 pixel
// rows of the tile (two m64 row blocks).
//
//   stem      u8 BGR page rows 2*y0-2 .. 2*y0+33, bytes of pixels 2*x0-2 .. 2*x0+37 (a 144-byte box)  ->  each consumer
//             warpgroup converts its rows to the fp16 space-to-depth tile (s2d pixel (Y, X), channel (dy*2+dx)*3 + c =
//             page(2Y+dy, 2X+dx, c) / 255, channels 12..15 zero) -> 3 filter rows x (4-pixel window x 16 channels) =
//             K 192, the compiler's window weight order -> bias + SiLU -> fp16 NHWC slice through a TMA store.
//             The same kernel also reads an fp16 HWC page (the staging page of a float input, ctd_forward_tensor): the
//             box keeps its 144 elements per row (288 bytes) and the conversion copies the fp16 values as they are.
//   seg tail  fp16 input tile (16+2) x (16+2) pixels x 64 channels, 128-byte swizzle -> 9 taps x 64 channels, the
//             4 output channels being the sub-pixel phases of ConvT 4x4 s2 p1 -> sigmoid -> each warpgroup's 16 x 32
//             mask pixels staged in shared memory and written as whole rows (f32 and truncated u8).
//
// Every accumulator sees the same k16 MMAs, in the same order, on the same fp16 values as the generic form of these
// ops (tap, then 16-channel K step), so the results do not depend on the tiling.
#include <cstring>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "kernels.h"
#include "ptx.cuh"

namespace ctd {

namespace {

constexpr int kThreads = 384;
constexpr int kTile = 16;   // output tile: 16 x 16 pixels; consumer warpgroup wg owns rows 8*wg .. 8*wg + 7

constexpr uint32_t align1k(uint32_t x) { return (x + 1023u) & ~1023u; }

// ---- stem; P = uint8_t (the u8 pages) or __half (the fp16 staging page of a float input)
template <typename P>
struct StemT {
  static constexpr int kBoxRows = 2 * kTile + 4;      // page rows of a tile: s2d rows y0-1 .. y0+16
  // elements per page row: s2d pixels x0-1 .. x0+18 are the 120 elements from 6*x0 - 6; the box starts 10 elements
  // earlier, at 6*x0 - 16, so that its innermost coordinate is 16-byte aligned (144 bytes per row for u8, 288 for fp16)
  static constexpr int kBoxElems = 144;
  static constexpr int kBoxSkip = 10;
  static constexpr int kStageBytes = kBoxRows * kBoxElems * int(sizeof(P));
  static constexpr int kStageStride = (kStageBytes + 127) / 128 * 128;   // TMA destinations are 128-byte aligned
  static constexpr int kStages = 4;
  static constexpr int kS2dRows = kTile / 2 + 2;      // s2d rows of one warpgroup: its 8 rows and one halo row each side
  static constexpr int kS2dCols = kTile + 4;          // s2d pixels x0-1 .. x0+18: the 4-pixel windows of 16 outputs
  static constexpr int kS2dBytes = kS2dRows * kS2dCols * 32;
  static constexpr int kWBytes = 3 * 32 * 128;        // 3 filter rows x 32 output channels x 64 fp16
  static constexpr int kStgBytes = 8 * kTile * 64;    // 128 pixels x 32 fp16 per consumer warpgroup
  static constexpr uint32_t kW = 0;
  static constexpr uint32_t kStg = align1k(kW + kWBytes);
  static constexpr uint32_t kIn = kStg + 2 * kStgBytes;
  static constexpr uint32_t kS2d = kIn + kStages * kStageStride;
  static constexpr uint32_t kBar = kS2d + 2 * kS2dBytes;
  static constexpr uint32_t kLut = kBar + 256;          // u8 pages: fp16(u8 / 255) for the 256 byte values
  static constexpr size_t kSmem = 1024 + kLut + (sizeof(P) == 1 ? 512 : 0);
};
static_assert(StemT<uint8_t>::kSmem <= 227 * 1024 && StemT<__half>::kSmem <= 227 * 1024, "stem: shared memory");

// ---- seg tail
struct Seg {
  static constexpr int kHalo = kTile + 2;
  static constexpr int kInBytes = kHalo * kHalo * 128;   // (16+2)^2 pixels x 64 fp16
  static constexpr int kStageBytes = int(align1k(kInBytes));   // stages stay 1024-aligned for the 128-byte swizzle
  static constexpr int kStages = 3;
  static constexpr int kWBytes = 9 * 8 * 128;            // 9 taps x 8 rows (4 phases + 4 zero) x 64 fp16
  static constexpr int kStgPitch = 48;                   // floats per staged mask row: 32 + 16 (no bank conflicts)
  static constexpr int kStgBytes = 2 * 8 * kStgPitch * 4;   // 16 mask rows per consumer warpgroup
  static constexpr uint32_t kW = 0;
  static constexpr uint32_t kIn = align1k(kW + kWBytes);
  static constexpr uint32_t kStg = kIn + kStages * kStageBytes;
  static constexpr uint32_t kBar = kStg + 2 * kStgBytes;
  static constexpr size_t kSmem = 1024 + kBar + 256;
};
static_assert(Seg::kSmem <= 227 * 1024, "seg tail: shared memory");

int g_sms = 132;

}  // namespace

// Both kernels: barriers at `bar`: full[S] | empty[S] | weights.  Returns the 1024-aligned shared base.
__device__ __forceinline__ uint32_t ends_smem_base(uint8_t* smem) { return (smem_u32(smem) + 1023u) & ~1023u; }

// keeps the compiler from reusing (or moving accesses to) an A register set that an in-flight wgmma may still read
__device__ __forceinline__ void fence_a_set(uint32_t (&set)[2][4][4]) {
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_fence_regs(set[m][k]);
}

__device__ __forceinline__ void ends_decode(const ConvEndsParams& p, int t, int& img, int& y0, int& x0) {
  const int per_img = p.tiles_x * p.tiles_y;
  img = t / per_img;
  const int r = t - img * per_img;
  const int ty = r / p.tiles_x;
  y0 = ty * kTile;
  x0 = (r - ty * p.tiles_x) * kTile;
}

// ================================================================================================ stem
template <typename P>
__global__ void __launch_bounds__(kThreads, 1) stem_tc_kernel(const __grid_constant__ ConvEndsParams p) {
  using Stem = StemT<P>;
  extern __shared__ __align__(1024) uint8_t smem_ends[];
  const uint32_t base = ends_smem_base(smem_ends);
  uint8_t* const gen = smem_ends + (base - smem_u32(smem_ends));
  constexpr int S = Stem::kStages;
  const uint32_t full_bar = base + Stem::kBar, empty_bar = full_bar + 8 * S, w_bar = full_bar + 16 * S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total = p.n_img * p.tiles_x * p.tiles_y;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&p.a_map);
    prefetch_tensormap(&p.b_map);
    prefetch_tensormap(&p.d_map);
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 2);   // one arrival per consumer warpgroup
    }
    mbar_init(w_bar, 1);
    fence_barrier_init();
  }
  // the conversion of a page byte, as fp16(float(u8) / 255): the same expression for every byte, computed once.  An
  // fp16 page holds fp16(x) already, which for x = float(u8) / 255 is the same table entry.
  __half* const lut = reinterpret_cast<__half*>(gen + Stem::kLut);
  if constexpr (sizeof(P) == 1)
    for (int i = threadIdx.x; i < 256; i += kThreads) lut[i] = __float2half_rn(float(i) / 255.0f);
  __syncthreads();

  if (warp < 4) {
    // =============================== TMA producer
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(w_bar, Stem::kWBytes);
      for (int r = 0; r < 3; ++r) tma_load_2d(base + Stem::kW + r * 4096, &p.b_map, w_bar, r * 64, 0);
      int it = 0;
      for (int t = blockIdx.x; t < total; t += gridDim.x, ++it) {
        int img, y0, x0;
        ends_decode(p, t, img, y0, x0);
        const int stage = it % S;
        mbar_wait_relaxed(empty_bar + 8 * stage, ((it / S) & 1) ^ 1);
        mbar_arrive_expect_tx(full_bar + 8 * stage, Stem::kStageBytes);
        // page bytes of pixels 2*x0-2 .., rows 2*y0-2 ..: the zero fill beyond the page is the s2d padding
        tma_load_3d(base + Stem::kIn + stage * Stem::kStageStride, &p.a_map, full_bar + 8 * stage,
                    6 * x0 - 6 - Stem::kBoxSkip, 2 * y0 - 2, img);
      }
    }
    return;
  }

  // =============================== consumers
  const int wg = (warp >> 2) - 1;
  const int w4 = warp & 3, tid = threadIdx.x & 127;
  const bool leader = tid == 0;
  const uint32_t epi_bar = 1 + wg;
  const uint32_t s2d = base + Stem::kS2d + wg * Stem::kS2dBytes;
  uint8_t* const s2d_gen = gen + Stem::kS2d + wg * Stem::kS2dBytes;
  const uint32_t stg = base + Stem::kStg + wg * Stem::kStgBytes;
  const int q = lane >> 3, t4 = lane & 3;
  const int rr = (lane & 7) + 8 * (q & 1);   // the pixel (column of the tile) whose row address this lane gives
  float bias[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) bias[i] = p.bias[(i >> 1) * 8 + 2 * t4 + (i & 1)];
  mbar_wait(w_bar, 0);

  int it = 0;
  for (int t = blockIdx.x; t < total; t += gridDim.x, ++it) {
    int img, y0, x0;
    ends_decode(p, t, img, y0, x0);
    const int stage = it % S;
    mbar_wait(full_bar + 8 * stage, (it / S) & 1);
    // page -> fp16 space-to-depth tile of this warpgroup: s2d rows y0 + 8*wg - 1 .. +8, pixels x0-1 .. x0+18.  16-byte
    // chunk h of pixel X sits at chunk h ^ ((X >> 2) & 1), so that ldmatrix rows (8 consecutive pixels) hit 8 distinct
    // bank groups.
    {
      const P* in = reinterpret_cast<const P*>(gen + Stem::kIn + stage * Stem::kStageStride) + Stem::kBoxSkip;
      for (int px = tid; px < Stem::kS2dRows * Stem::kS2dCols; px += 128) {
        const int r = px / Stem::kS2dCols, c = px - r * Stem::kS2dCols;
        const P* b0 = in + (2 * (8 * wg + r)) * Stem::kBoxElems + 6 * c;
        const P* b1 = b0 + Stem::kBoxElems;
        // channels 0..5: (dy=0, dx=0, c), (dy=0, dx=1, c); 6..11: (dy=1, dx=0, c), (dy=1, dx=1, c); 12..15: 0
        uint4 lo, hi;
        __half2 h2[8];
        if constexpr (sizeof(P) == 1) {
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            h2[k] = __halves2half2(lut[b0[2 * k]], lut[b0[2 * k + 1]]);
            h2[3 + k] = __halves2half2(lut[b1[2 * k]], lut[b1[2 * k + 1]]);
          }
        } else {
          // element offsets 10 + 144 * row + 6 * c are even: 4-byte aligned pairs
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            h2[k] = reinterpret_cast<const __half2*>(b0)[k];
            h2[3 + k] = reinterpret_cast<const __half2*>(b1)[k];
          }
        }
        h2[6] = h2[7] = __floats2half2_rn(0.f, 0.f);
        memcpy(&lo, &h2[0], 16);
        memcpy(&hi, &h2[4], 16);
        const int sw = (c >> 2) & 1;
        uint4* dst = reinterpret_cast<uint4*>(s2d_gen + px * 32);
        dst[sw] = lo;
        dst[sw ^ 1] = hi;
      }
    }
    __syncwarp();
    named_barrier_sync(epi_bar, 128);   // the s2d tile is complete; the input stage is free
    if (leader) mbar_arrive(empty_bar + 8 * stage);

    // filter row r (tap dy = r - 1), window pixel j = K step.  Two A register sets: the fragments of row r + 1 load
    // while the MMAs of row r run.
    float acc[2][16] = {};
    uint32_t a[2][2][4][4];
    auto load_row = [&](int r, uint32_t (&set)[2][4][4]) {
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = rr + j;
          ldmatrix_x4(s2d + ((m * 4 + w4 + r) * Stem::kS2dCols + col) * 32 + 16 * ((q >> 1) ^ ((col >> 2) & 1)),
                      set[m][j]);
        }
    };
    load_row(0, a[0]);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const uint64_t bd = make_kmajor_desc(base + Stem::kW + r * 4096, 128);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int m = 0; m < 2; ++m) wgmma_n32_rs(acc[m], a[r & 1][m][j], bd + 2 * j, (r > 0 || j > 0) ? 1u : 0u);
      wgmma_commit();
      if (r < 2) {
        wgmma_wait<1>();   // row r - 1 has retired: its register set is free
        fence_a_set(a[(r + 1) & 1]);
        load_row(r + 1, a[(r + 1) & 1]);
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int m = 0; m < 2; ++m) wgmma_fence_regs(acc[m]);
    fence_a_set(a[0]);
    fence_a_set(a[1]);

    // ---- epilogue: bias + SiLU -> fp16 staging tile (64-byte swizzle of the store map) -> one TMA store
    if (leader) tma_store_wait_read();   // the previous tile's store has read the staging tile
    named_barrier_sync(epi_bar, 128);
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const uint32_t pixrow = uint32_t(m * 64 + w4 * 16 + (q & 1) * 8 + (lane & 7));
#pragma unroll
      for (int j = 0; j < 4; j += 2) {
        const uint32_t off = pixrow * 64 + uint32_t(j + (q >> 1)) * 16;
        const uint32_t addr = stg + (off ^ (((off >> 7) & 3) << 4));
        uint32_t rg[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int bi = (j + (i >> 1)) * 2;
          const float v0 = acc[m][j * 4 + 2 * i] + bias[bi], v1 = acc[m][j * 4 + 2 * i + 1] + bias[bi + 1];
          const __half2 o = __floats2half2_rn(__fdividef(v0, 1.0f + exp_neg_fast(v0)),
                                              __fdividef(v1, 1.0f + exp_neg_fast(v1)));
          memcpy(&rg[i], &o, 4);
        }
        stmatrix_x4(addr, rg);
      }
    }
    fence_proxy_async();
    named_barrier_sync(epi_bar, 128);
    if (leader) {
      tma_store_4d(&p.d_map, stg, 0, x0, y0 + 8 * wg, img);
      tma_store_commit();
    }
  }
  if (leader) tma_store_wait_all();
}

// ================================================================================================ seg tail
__global__ void __launch_bounds__(kThreads, 1) seg_tc_kernel(const __grid_constant__ ConvEndsParams p) {
  extern __shared__ __align__(1024) uint8_t smem_ends[];
  const uint32_t base = ends_smem_base(smem_ends);
  uint8_t* const gen = smem_ends + (base - smem_u32(smem_ends));
  constexpr int S = Seg::kStages;
  const uint32_t full_bar = base + Seg::kBar, empty_bar = full_bar + 8 * S, w_bar = full_bar + 16 * S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total = p.n_img * p.tiles_x * p.tiles_y;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&p.a_map);
    prefetch_tensormap(&p.b_map);
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 2);
    }
    mbar_init(w_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // =============================== TMA producer
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(w_bar, Seg::kWBytes);
      for (int tap = 0; tap < 9; ++tap) tma_load_2d(base + Seg::kW + tap * 1024, &p.b_map, w_bar, tap * 64, 0);
      int it = 0;
      for (int t = blockIdx.x; t < total; t += gridDim.x, ++it) {
        int img, y0, x0;
        ends_decode(p, t, img, y0, x0);
        const int stage = it % S;
        mbar_wait_relaxed(empty_bar + 8 * stage, ((it / S) & 1) ^ 1);
        mbar_arrive_expect_tx(full_bar + 8 * stage, Seg::kInBytes);
        tma_load_4d(base + Seg::kIn + stage * Seg::kStageBytes, &p.a_map, full_bar + 8 * stage, 0, x0 - 1, y0 - 1,
                    img);
      }
    }
    return;
  }

  // =============================== consumers
  const int wg = (warp >> 2) - 1;
  const int w4 = warp & 3, tid = threadIdx.x & 127;
  const bool leader = tid == 0;
  const uint32_t epi_bar = 1 + wg;
  float* const stg = reinterpret_cast<float*>(gen + Seg::kStg + wg * Seg::kStgBytes);
  const int q = lane >> 3, g = lane >> 2, t4 = lane & 3;
  const int rr = (lane & 7) + 8 * (q & 1);
  const int oh = 2 * p.gh, ow = 2 * p.gw;
  mbar_wait(w_bar, 0);

  int it = 0;
  for (int t = blockIdx.x; t < total; t += gridDim.x, ++it) {
    int img, y0, x0;
    ends_decode(p, t, img, y0, x0);
    const int stage = it % S;
    const uint32_t in = base + Seg::kIn + stage * Seg::kStageBytes;
    mbar_wait(full_bar + 8 * stage, (it / S) & 1);

    // tap (dy, dx) = (tap / 3 - 1, tap % 3 - 1).  Two A register sets: the fragments of tap + 1 load while the MMAs
    // of tap run.
    float acc[2][4] = {};
    uint32_t a[2][2][4][4];
    auto load_tap = [&](int tap, uint32_t (&set)[2][4][4]) {
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        // halo pixel of output (8*wg + 4*m + w4, rr) under this tap; 128-byte rows, chunk index ^ (pixel & 7)
        const int L = (8 * wg + 4 * m + w4 + tap / 3) * Seg::kHalo + rr + tap % 3;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          ldmatrix_x4(in + L * 128 + (((2 * ks + (q >> 1)) ^ (L & 7)) << 4), set[m][ks]);
      }
    };
    auto step = [&](int tap, uint32_t (&cur)[2][4][4], uint32_t (&nxt)[2][4][4]) {
      const uint64_t bd = make_kmajor_desc(base + Seg::kW + tap * 1024, 128);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int m = 0; m < 2; ++m) wgmma_n8_rs(acc[m], cur[m][ks], bd + 2 * ks, (tap > 0 || ks > 0) ? 1u : 0u);
      wgmma_commit();
      if (tap < 8) {
        wgmma_wait<1>();   // tap - 1 has retired: its register set is free
        fence_a_set(nxt);
        load_tap(tap + 1, nxt);
      }
    };
    load_tap(0, a[0]);
#pragma unroll
    for (int tap = 0; tap < 9; tap += 2) {
      step(tap, a[0], a[1]);
      if (tap + 1 < 9) step(tap + 1, a[1], a[0]);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int m = 0; m < 2; ++m) wgmma_fence_regs(acc[m]);
    fence_a_set(a[0]);
    fence_a_set(a[1]);
    // every warp of the warpgroup has retired its MMAs, so its ldmatrix reads of the stage are done
    __syncwarp();
    named_barrier_sync(epi_bar, 128);   // also: the previous tile's rows have been read out of the staging tile
    if (leader) mbar_arrive(empty_bar + 8 * stage);

    // ---- epilogue: columns 0..3 (lanes t4 = 0, 1) are the phases (py, px) = (t4, 0 / 1) -> sigmoid -> staged mask
    // rows 2*row + py of this warpgroup, then whole rows out
    if (t4 < 2) {
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = 4 * m + w4, col = g + 8 * h;
          const float s0 = 1.0f / (1.0f + expf(-acc[m][2 * h]));
          const float s1 = 1.0f / (1.0f + expf(-acc[m][2 * h + 1]));
          *reinterpret_cast<float2*>(stg + (2 * row + t4) * Seg::kStgPitch + 2 * col) = make_float2(s0, s1);
        }
    }
    named_barrier_sync(epi_bar, 128);
    {
      const int r = tid >> 3, c4 = tid & 7;   // 16 rows x 8 float4
      const float4 v = *reinterpret_cast<const float4*>(stg + r * Seg::kStgPitch + 4 * c4);
      const size_t o = (size_t(img) * oh + 2 * (y0 + 8 * wg) + r) * ow + 2 * x0 + 4 * c4;
      *reinterpret_cast<float4*>(p.mask_f32 + o) = v;
      *reinterpret_cast<uchar4*>(p.mask_u8 + o) =
          make_uchar4((uint8_t)(v.x * 255.0f), (uint8_t)(v.y * 255.0f), (uint8_t)(v.z * 255.0f), (uint8_t)(v.w * 255.0f));
    }
  }
}

// =========================================================================================
// host side

const char* conv_ends_plan_stem(ConvEndsPlan& plan, PFN_encodeTiled enc, const void* pages, bool f16_page, int n,
                                int ph, int pw, const void* w16, const float* bias, __half* dst, int dst_cstride,
                                int dst_coff, int cout, int act) {
  ConvEndsParams& p = plan.p;
  memset(&p, 0, sizeof(p));
  if (act != CTD_ACT_SILU) return "stem: the tensor-core stem fuses SiLU only";
  if (cout < 8 || cout > 32 || cout % 8) return "stem: output channels must be 8, 16, 24 or 32";
  if (ph % (2 * kTile) || pw % (2 * kTile)) return "stem: page sides must be multiples of 32";
  if (dst_coff % 8 || dst_cstride % 8) return "stem: destination slice must be 16-byte aligned";
  p.n_img = n;
  p.gh = ph / 2;
  p.gw = pw / 2;
  p.tiles_x = p.gw / kTile;
  p.tiles_y = p.gh / kTile;
  p.bias = bias;
  const cuuint32_t e1[3] = {1, 1, 1};
  {
    using Stem = StemT<uint8_t>;   // the box in elements is the same for both page types
    const cuuint64_t es = f16_page ? 2 : 1;
    const cuuint64_t dims[3] = {cuuint64_t(pw) * 3, cuuint64_t(ph), cuuint64_t(n)};
    const cuuint64_t str[2] = {cuuint64_t(pw) * 3 * es, cuuint64_t(pw) * 3 * ph * es};
    const cuuint32_t box[3] = {Stem::kBoxElems, Stem::kBoxRows, 1};
    if (enc(&p.a_map, f16_page ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 3,
            const_cast<void*>(pages), dims, str, box, e1, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return "stem: page tensor map";
  }
  {
    const cuuint64_t dims[2] = {192, 32};
    const cuuint64_t str[1] = {192 * 2};
    const cuuint32_t box[2] = {64, 32};
    if (enc(&p.b_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(w16), dims, str, box, e1,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return "stem: weight tensor map";
  }
  {
    // {cout, gw, gh, n} over the slice: TMA clips the neighbouring channels; boxes of 32 channels x 16 x 8 pixels
    const cuuint64_t px = cuuint64_t(dst_cstride) * 2;
    const cuuint64_t dims[4] = {cuuint64_t(cout), cuuint64_t(p.gw), cuuint64_t(p.gh), cuuint64_t(n)};
    const cuuint64_t str[3] = {px, px * p.gw, px * p.gw * p.gh};
    const cuuint32_t box[4] = {32, kTile, kTile / 2, 1};
    const cuuint32_t e4[4] = {1, 1, 1, 1};
    if (enc(&p.d_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, dst + dst_coff, dims, str, box, e4,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return "stem: destination tensor map";
  }
  const int total = n * p.tiles_x * p.tiles_y;
  plan.kind = f16_page ? CTD_END_STEM_F16 : CTD_END_STEM;
  plan.grid = dim3(unsigned(total < g_sms ? total : g_sms), 1, 1);
  plan.smem_bytes = f16_page ? StemT<__half>::kSmem : StemT<uint8_t>::kSmem;
  return nullptr;
}

const char* conv_ends_plan_seg(ConvEndsPlan& plan, PFN_encodeTiled enc, const __half* src, int src_cstride,
                               int src_coff, int src_c, int n, int gh, int gw, const void* w16, float* mask_f32,
                               uint8_t* mask_u8) {
  ConvEndsParams& p = plan.p;
  memset(&p, 0, sizeof(p));
  if (src_c != 64) return "seg tail: the tensor-core seg tail takes 64 input channels";
  if (gh % kTile || gw % kTile) return "seg tail: grid sides must be multiples of 16";
  if (src_coff % 8 || src_cstride % 8) return "seg tail: source slice must be 16-byte aligned";
  p.n_img = n;
  p.gh = gh;
  p.gw = gw;
  p.tiles_x = gw / kTile;
  p.tiles_y = gh / kTile;
  p.mask_f32 = mask_f32;
  p.mask_u8 = mask_u8;
  {
    const cuuint64_t cs = cuuint64_t(src_cstride) * 2;
    const cuuint64_t dims[4] = {64, cuuint64_t(gw), cuuint64_t(gh), cuuint64_t(n)};
    const cuuint64_t str[3] = {cs, cs * gw, cs * gw * gh};
    const cuuint32_t box[4] = {64, Seg::kHalo, Seg::kHalo, 1};
    const cuuint32_t e4[4] = {1, 1, 1, 1};
    if (enc(&p.a_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(src) + src_coff, dims, str, box, e4,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return "seg tail: input tensor map";
  }
  {
    const cuuint64_t dims[2] = {9 * 64, 16};
    const cuuint64_t str[1] = {9 * 64 * 2};
    const cuuint32_t box[2] = {64, 8};   // rows 0..7: the 4 phases and 4 zero rows (m64n8 MMAs)
    const cuuint32_t e2[2] = {1, 1};
    if (enc(&p.b_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(w16), dims, str, box, e2,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return "seg tail: weight tensor map";
  }
  const int total = n * p.tiles_x * p.tiles_y;
  plan.kind = CTD_END_SEG;
  plan.grid = dim3(unsigned(total < g_sms ? total : g_sms), 1, 1);
  plan.smem_bytes = Seg::kSmem;
  return nullptr;
}

cudaError_t conv_ends_init() {
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) g_sms = n;
  }
  cudaError_t e = cudaFuncSetAttribute(stem_tc_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       int(StemT<uint8_t>::kSmem));
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(stem_tc_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           int(StemT<__half>::kSmem));
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(seg_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(Seg::kSmem));
}

cudaError_t conv_ends_launch(const ConvEndsPlan& plan, cudaStream_t s) {
  if (plan.kind == CTD_END_STEM) stem_tc_kernel<uint8_t><<<plan.grid, kThreads, plan.smem_bytes, s>>>(plan.p);
  else if (plan.kind == CTD_END_STEM_F16) stem_tc_kernel<__half><<<plan.grid, kThreads, plan.smem_bytes, s>>>(plan.p);
  else if (plan.kind == CTD_END_SEG) seg_tc_kernel<<<plan.grid, kThreads, plan.smem_bytes, s>>>(plan.p);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

}  // namespace ctd
