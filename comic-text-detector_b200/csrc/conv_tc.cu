// wgmma implicit-GEMM convolution for sm_90a.
//
//   D[16*TH x BN] (fp32, registers) += A[16*TH x 16] * B[BN x 16]^T, K-major fp16 operands in 128B/64B/32B-swizzled
//   shared memory; the 16*TH rows are a 16xTH-pixel tile (TH = 8 or 16), the BN columns a slice of output channels
//
// Persistent, one CTA per SM, 384 threads: warpgroup 0 = TMA producer (one elected thread), warpgroups 1 and 2 =
// consumers, each owning TH/2 pixel rows of the tile (8*TH accumulator rows): per K = 16 step it issues TH/8 wgmma
// m64nBNk16 against the same B descriptor, and it runs the epilogue on its own accumulators.  At TH = 16 the producer
// warpgroup gives registers to the consumers (setmaxnreg 40 / 232: 128 accumulators per thread at BN = 128).  An
// mbarrier full/empty ring of operand stages sits between producer and consumers; each
// consumer keeps one wgmma group in flight and frees the stage of the previous group once that group has retired.
// Activations are 4-D TMA boxes over the NHWC buffers: out-of-bounds zero-fill IS the convolution padding, there is
// no im2col buffer; torch.cat inputs are K-concatenated from up to 3 tensor maps; stride 2 reads four parity maps;
// ConvTranspose 4x4 s2 p1 runs as 4 sub-pixel phases of 2x2 taps; Detect heads decode sigmoid / boxes in the epilogue.
// The fp16 NHWC epilogue (CONV, DECONV4) writes the warpgroup's tile into a swizzled staging buffer with stmatrix
// and one elected thread stores it with TMA through the destination map, so the store drains while the warpgroup
// runs the next tile's mainloop; an in-place residual is TMA-loaded into the same buffer at the start of the tile.
//
// Reference semantics: Conv.forward_fuse (models/yolov5/common.py:48-49), Bottleneck add (common.py:104),
// ConvTranspose2d+BN+ReLU (basemodel.py:26-28), Detect (yolo.py:23-44).
#include <cstdlib>
#include <cstring>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "kernels.h"
#include "ptx.cuh"

namespace ctd {

constexpr int kTileW = 16;     // tile width in grid pixels; the height TH (8 or 16) is a template parameter
constexpr int kThreads = 384;  // warpgroup 0 TMA, warpgroups 1-2 MMA + epilogue

// Shared memory per (BN, TH): stages x (A box of 16*TH rows + B box of BN rows, 128-byte rows in the worst case),
// then one fp16 staging tile of 8*TH pixels x BN channels per consumer warpgroup.
//   TH = 8:  BN 128: 5 x 32 KB + 2 x 16 KB | 64: 8 x 24 KB + 2 x 8 KB | 32: 10 x 20 KB + 2 x 4 KB | 16: 10 x 18 KB + 2 x 2 KB
//   TH = 16: BN 128: 3 x 48 KB + 2 x 32 KB | 64: 4 x 40 KB + 2 x 16 KB | 32: 5 x 36 KB + 2 x 8 KB | 16: 6 x 34 KB + 2 x 4 KB
template <int BN, int TH>
struct TcCfg {
  static constexpr int kABytes = TH * kTileW * 128;  // per stage (worst case 128-byte rows)
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStages = TH == 8 ? (BN >= 128 ? 5 : (BN >= 64 ? 8 : 10))
                                         : (BN >= 128 ? 3 : (BN >= 64 ? 4 : (BN >= 32 ? 5 : 6)));
  // staging: store boxes of kBoxN channels x 16 x TH/2 pixels, rows of kBoxN fp16 in the box's swizzle
  static constexpr int kBoxN = BN < 64 ? BN : 64;
  static constexpr int kBoxBytes = 8 * TH * kBoxN * 2;
  static constexpr int kStgBytes = (BN / kBoxN) * kBoxBytes;   // per consumer warpgroup
  static constexpr int kBiasFloats = 512;
  // 1024 bytes of alignment slack | operand ring | staging (2 warpgroups) | barriers (256 B) | bias
  static constexpr size_t kSmem = 1024 + size_t(kStages) * (kABytes + kBBytes) + 2 * kStgBytes + 256 + kBiasFloats * 4;
  static_assert(kSmem <= 227 * 1024, "conv_tc_kernel: shared memory");
  static_assert(kBoxBytes % 1024 == 0, "conv_tc_kernel: store boxes must keep the 1024-byte swizzle alignment");
};

template <int ACT>
__device__ __forceinline__ float apply_act(float v) {
  if constexpr (ACT == CTD_ACT_SILU) return __fdividef(v, 1.0f + exp_neg_fast(v));
  else if constexpr (ACT == CTD_ACT_LEAKY) return fmaxf(v, 0.1f * v);
  else if constexpr (ACT == CTD_ACT_RELU) return fmaxf(v, 0.f);
  else if constexpr (ACT == CTD_ACT_SIGMOID) return __fdividef(1.0f, 1.0f + exp_neg_fast(v));
  else return v;
}

// Split-fp16 mode: full-precision activation functions (expf / true division: the fast intrinsics above carry
// ~1e-6 relative error, 16 fp32 ulps, which the 1e-3 end-to-end budget of this mode cannot afford).
template <int ACT>
__device__ __forceinline__ float apply_act_precise(float v) {
  if constexpr (ACT == CTD_ACT_SILU) return v / (1.0f + expf(-v));
  else if constexpr (ACT == CTD_ACT_LEAKY) return fmaxf(v, 0.1f * v);
  else if constexpr (ACT == CTD_ACT_RELU) return fmaxf(v, 0.f);
  else if constexpr (ACT == CTD_ACT_SIGMOID) return 1.0f / (1.0f + expf(-v));
  else return v;
}

template <int BN>
__device__ __forceinline__ void wgmma_bn(float (&d)[BN / 2], uint64_t ad, uint64_t bd, uint32_t acc) {
  if constexpr (BN == 128) wgmma_n128(d, ad, bd, acc);
  else if constexpr (BN == 64) wgmma_n64(d, ad, bd, acc);
  else if constexpr (BN == 32) wgmma_n32(d, ad, bd, acc);
  else wgmma_n16(d, ad, bd, acc);
}

// fp16 epilogue of row block m of a consumer warpgroup: bias + activation (+ residual, already loaded into the
// staging tile) -> fp16, written into the staging tile in place.  One stmatrix x4 covers the 16 rows of this warp
// and 16 columns: matrix q holds rows 8*(q & 1) .. +7 and the column block j + (q >> 1), which are accumulators
// acc[4j + 2q], acc[4j + 2q + 1].  Rows of a box are kBoxN fp16 with the 32/64/128-byte swizzle of the tensor map (the
// 16-byte chunk index XOR address bits 7..9); eight consecutive rows then hit eight distinct chunk columns, so the
// stores are free of bank conflicts.
template <int BN, int TH, int ACT, bool RES>
__device__ __forceinline__ void stage_f16(const float (&acc)[BN / 2], const float* __restrict__ bias_s, uint32_t stg,
                                          int m, int warp4, int lane) {
  using Cfg = TcCfg<BN, TH>;
  constexpr uint32_t kRowBytes = Cfg::kBoxN * 2;
  const int q = lane >> 3;
  const uint32_t pixrow = uint32_t(m * 64 + warp4 * 16 + (q & 1) * 8 + (lane & 7));
#pragma unroll
  for (int j = 0; j < BN / 8; j += 2) {
    const int col = (j + (q >> 1)) * 8;   // first column of the matrix this lane addresses
    const uint32_t off = pixrow * kRowBytes + uint32_t(col % Cfg::kBoxN) * 2;
    const uint32_t addr = stg + uint32_t(col / Cfg::kBoxN) * Cfg::kBoxBytes +
                          (off ^ (((off >> 7) & (kRowBytes / 16 - 1)) << 4));
    uint32_t r[4];
    if constexpr (RES) ldmatrix_x4(addr, r);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = (j + (i >> 1)) * 8 + (lane & 3) * 2;
      float f0 = apply_act<ACT>(acc[j * 4 + 2 * i] + bias_s[c]);
      float f1 = apply_act<ACT>(acc[j * 4 + 2 * i + 1] + bias_s[c + 1]);
      if constexpr (RES) {
        __half2 h;
        memcpy(&h, &r[i], 4);
        const float2 rv = __half22float2(h);
        // __fadd_rn: never fused with the multiply of the fast division (one rounding each, as in the fp32 reference)
        f0 = __fadd_rn(f0, rv.x);
        f1 = __fadd_rn(f1, rv.y);
      }
      const __half2 o = __floats2half2_rn(f0, f1);
      memcpy(&r[i], &o, 4);
    }
    stmatrix_x4(addr, r);
  }
}

template <int ACT>
__device__ __forceinline__ void epi_pair_f32(float v0, float v1, const float* __restrict__ bias_s, int col,
                                             float* __restrict__ out, int ncols, bool residual) {
  if (col >= ncols) return;
  float f0 = apply_act_precise<ACT>(v0 + bias_s[col]);
  float f1 = apply_act_precise<ACT>(v1 + bias_s[col + 1]);
  if (col + 1 < ncols) {
    if (residual) {
      const float2 r = *reinterpret_cast<const float2*>(out + col);
      f0 += r.x;
      f1 += r.y;
    }
    *reinterpret_cast<float2*>(out + col) = make_float2(f0, f1);
  } else {
    if (residual) f0 += out[col];
    out[col] = f0;
  }
}

template <int BN, int ACT>
__device__ __forceinline__ void epilogue_f32(const float (&acc)[BN / 2], const float* __restrict__ bias_s,
                                             float* const (&out)[2], const bool (&valid)[2], int ncols, int lane,
                                             bool residual) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!valid[h]) continue;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      epi_pair_f32<ACT>(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1], bias_s, j * 8 + (lane & 3) * 2, out[h], ncols,
                        residual);
  }
}

template <int BN, int TH>
__global__ void __launch_bounds__(kThreads, 1) conv_tc_kernel(const __grid_constant__ ConvTcParams p) {
  using Cfg = TcCfg<BN, TH>;
  constexpr int MT = TH / 8;   // m64 row blocks per consumer warpgroup
  extern __shared__ __align__(1024) uint8_t smem_tc[];
  // the swizzled operand stages need 1024-byte alignment; the dynamic base is only guaranteed 16
  const uint32_t raw_base = smem_u32(smem_tc);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;
  uint8_t* const smem_gen = smem_tc + (smem_base - raw_base);
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + Cfg::kStages * Cfg::kABytes;
  const uint32_t stg_base = b_base + Cfg::kStages * Cfg::kBBytes;
  const uint32_t bar_base = stg_base + 2 * Cfg::kStgBytes;
  // barriers (8 B each): full[S] | empty[S] | residual[2] (one per consumer warpgroup)
  const uint32_t full_bar = bar_base, empty_bar = bar_base + 8 * Cfg::kStages, res_bar0 = bar_base + 16 * Cfg::kStages;
  float* bias_s = reinterpret_cast<float*>(smem_gen + (bar_base - smem_base) + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const ConvGeom& g = p.g;

  const int kb = p.kb_elems;
  const uint32_t row_bytes = kb * 2;
  const uint32_t stage_tx = uint32_t(TH * kTileW) * row_bytes + uint32_t(BN) * row_bytes;
  int kblocks_per_tap = 0;
  for (int s = 0; s < g.n_src; ++s) kblocks_per_tap += p.src_kblocks[s];
  const int n_terms = p.split ? 3 : 1;   // split-fp16 mode: (hi,hi) + (lo,hi) + (hi,lo) per K block
  const int its_per_tile = g.taps * kblocks_per_tap * n_terms;
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int n_nblk = g.cout_pad / BN;
  const int spatial_tiles = g.n_img * tiles_per_img;
  const int total_tiles = spatial_tiles * n_nblk * g.n_phase;

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < g.n_src; ++s)
      for (int q = 0; q < (g.in_stride == 2 ? 4 : 1); ++q) prefetch_tensormap(&p.a_map[s][q]);
    prefetch_tensormap(&p.b_map);
    if (p.dst != nullptr && !p.split)
      for (int ph = 0; ph < g.n_phase; ++ph) prefetch_tensormap(&p.d_map[ph]);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 2);   // one arrival per consumer warpgroup
    }
    mbar_init(res_bar0, 1);
    mbar_init(res_bar0 + 8, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < g.cout_pad && i < Cfg::kBiasFloats; i += kThreads) bias_s[i] = p.bias ? p.bias[i] : 0.f;
  __syncthreads();

  // tile index -> (spatial tile, phase, n block); n block varies fastest, then the DECONV4 phase, so that the CTAs
  // running concurrently share the A tile in L2.  The 4 phases of a deconvolution read the same input pixels, and
  // the four largest DECONV4 inputs of the benchmark (67-268 MB at 16 pages of 1024^2) exceed the 50 MB L2: with the
  // phase outermost, each phase's pass would read the whole input from HBM again.
  auto decode = [&](int t, int& phase, int& nblk, int& img, int& y0, int& x0) {
    nblk = t % n_nblk;
    const int r = t / n_nblk;
    phase = r % g.n_phase;
    const int sp = r / g.n_phase;
    img = sp / tiles_per_img;
    const int trem = sp - img * tiles_per_img;
    const int ty = trem / p.tiles_x;
    y0 = ty * TH;
    x0 = (trem - ty * p.tiles_x) * kTileW;
  };

  if (warp < 4) {
    // =============================== TMA producer (warpgroup 0) ===============================
    if constexpr (TH == 16) setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int it = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int phase, nblk, img, y0, x0;
        decode(t, phase, nblk, img, y0, x0);
        for (int tap = 0; tap < g.taps; ++tap) {
          const int dy = g.tap_dy[phase][tap], dx = g.tap_dx[phase][tap];
          const int q = p.tap_map[phase][tap];
          int kglob = tap * g.cin_total;
          for (int s = 0; s < g.n_src; ++s) {
            for (int cb = 0; cb < p.src_kblocks[s]; ++cb) {
              for (int term = 0; term < n_terms; ++term, ++it) {
                // term 0: A hi x B hi; 1: A lo x B hi; 2: A hi x B lo
                const int stage = it % Cfg::kStages;
                const uint32_t par = ((it / Cfg::kStages) & 1) ^ 1;
                mbar_wait_relaxed(empty_bar + 8 * stage, par);
                mbar_arrive_expect_tx(full_bar + 8 * stage, stage_tx);
                tma_load_4d(a_base + stage * Cfg::kABytes, &p.a_map[s][q], full_bar + 8 * stage, cb * kb, x0 + dx,
                            y0 + dy, img + (term == 1 ? p.split_img_off : 0));
                tma_load_2d(b_base + stage * Cfg::kBBytes, &p.b_map, full_bar + 8 * stage, kglob + cb * kb,
                            phase * g.cout_pad + nblk * BN + (term == 2 ? p.split_row_off : 0));
              }
            }
            kglob += g.src_c[s];
          }
        }
      }
    }
    return;
  }

  // =============================== consumers ====================================
  if constexpr (TH == 16) setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;                   // rows [64*MT*wg, 64*MT*(wg + 1)) of the tile
  const int wrow = ((warp & 3) << 4) + (lane >> 2);  // this thread's first fragment row within a 64-row block
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const uint64_t a_desc0 = make_kmajor_desc(a_base + uint32_t(wg * MT) * 64u * row_bytes, row_bytes);
  const uint64_t b_desc0 = make_kmajor_desc(b_base, row_bytes);
  const uint64_t a_mstep = (64u * row_bytes) >> 4;   // descriptor step from one 64-row block to the next
  const int ksteps = kb / 16;
  int stage = 0;
  uint32_t full_par = 0;
  constexpr int R = BN / 2;
  // fp16 NHWC destination (CONV, DECONV4): the epilogue stages the warpgroup's 8*TH x BN tile in shared memory
  // and one elected thread stores it with TMA while the warpgroup goes on to the next tile's mainloop
  const bool nhwc16 = p.dst != nullptr && !p.split;
  const bool res16 = nhwc16 && g.residual != 0;
  const uint32_t stg = stg_base + uint32_t(wg) * Cfg::kStgBytes;
  const uint32_t res_bar = res_bar0 + 8u * uint32_t(wg);
  const uint32_t epi_bar = 1 + wg;   // named barrier of this warpgroup's 128 threads (0 is __syncthreads)
  uint32_t res_par = 0;

  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    int phase, nblk, img, y0, x0;
    decode(t, phase, nblk, img, y0, x0);
    const int sy0 = y0 + wg * (TH / 2);   // first pixel row of this warpgroup's staging tile
    if (res16 && wg_leader) {
      // in-place residual: once the previous tile's store has read the staging tile, load this tile's residual box
      // into it, under the mainloop
      tma_store_wait_read();
      mbar_arrive_expect_tx(res_bar, Cfg::kStgBytes);
#pragma unroll
      for (int b = 0; b < BN / Cfg::kBoxN; ++b)
        tma_load_4d(stg + b * Cfg::kBoxBytes, &p.d_map[phase], res_bar, nblk * BN + b * Cfg::kBoxN, x0, sy0, img);
    }
    float acc[MT][R];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int i = 0; i < R; ++i) acc[m][i] = 0.f;

    bool split_done = false;
    if constexpr (BN <= 64 && TH == 8) {   // conv_tc_plan keeps split mode at 16x8 tiles
      if (p.split) {
        // Split-fp16 mode with PROMOTED accumulation.  The tensor core adds into its fp32 accumulator with
        // truncation: over the K/16 x 3 MMAs of a deep layer the one-sided errors add up to ~K/16 ulps.  So every
        // hi x hi MMA (K = 16) writes a FRESH accumulator that is added into `acc` in fp32 registers with
        // round-to-nearest; the cross terms (lo x hi, hi x lo: lo is stored scaled by kSplitLoScale, so they are
        // 2^-12 of the sum once unscaled and their truncation is 2^-36) accumulate in the tensor core as usual and
        // are unscaled and added last.
        float cross[R], tmp[R];
#pragma unroll
        for (int i = 0; i < R; ++i) cross[i] = 0.f;
        bool cross_started = false;
        for (int k_it = 0; k_it < its_per_tile; ++k_it) {
          mbar_wait(full_bar + 8 * stage, full_par);
          const uint64_t ad = a_desc0 + uint64_t(stage) * (Cfg::kABytes >> 4);
          const uint64_t bd = b_desc0 + uint64_t(stage) * (Cfg::kBBytes >> 4);
          if (k_it % 3 == 0) {
            for (int ks = 0; ks < ksteps; ++ks) {
              wgmma_fence();
              wgmma_bn<BN>(tmp, ad + 2 * ks, bd + 2 * ks, 0u);
              wgmma_commit();
              wgmma_wait<0>();
              wgmma_fence_regs(tmp);
#pragma unroll
              for (int i = 0; i < R; ++i) acc[0][i] = __fadd_rn(acc[0][i], tmp[i]);
            }
          } else {
            wgmma_fence();
            for (int ks = 0; ks < ksteps; ++ks)
              wgmma_bn<BN>(cross, ad + 2 * ks, bd + 2 * ks, (cross_started || ks > 0) ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(cross);
            cross_started = true;
          }
          if (wg_leader) mbar_arrive(empty_bar + 8 * stage);
          if (++stage == Cfg::kStages) { stage = 0; full_par ^= 1u; }
        }
#pragma unroll
        for (int i = 0; i < R; ++i) acc[0][i] = __fadd_rn(acc[0][i], cross[i] * kSplitLoUnscale);
        split_done = true;
      }
    }
    if (!split_done) {
      int prev = -1;
      for (int k_it = 0; k_it < its_per_tile; ++k_it) {
        mbar_wait(full_bar + 8 * stage, full_par);
        const uint64_t ad = a_desc0 + uint64_t(stage) * (Cfg::kABytes >> 4);
        const uint64_t bd = b_desc0 + uint64_t(stage) * (Cfg::kBBytes >> 4);
        wgmma_fence();
        // every row block m reads the same B box: an output element's K order does not depend on TH
        for (int ks = 0; ks < ksteps; ++ks)
#pragma unroll
          for (int m = 0; m < MT; ++m)
            wgmma_bn<BN>(acc[m], ad + m * a_mstep + 2 * ks, bd + 2 * ks, (k_it > 0 || ks > 0) ? 1u : 0u);
        wgmma_commit();
        // one group stays in flight: the previous group has retired, its stage goes back to the producer
        wgmma_wait<1>();
        if (prev >= 0 && wg_leader) mbar_arrive(empty_bar + 8 * prev);
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; full_par ^= 1u; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int m = 0; m < MT; ++m) wgmma_fence_regs(acc[m]);
      if (prev >= 0 && wg_leader) mbar_arrive(empty_bar + 8 * prev);
    }

    // ---------------------------------------------------------------- epilogue
    const float* bias_t = bias_s + nblk * BN;
    if (nhwc16) {
      if (res16) {
        mbar_wait(res_bar, res_par);
        res_par ^= 1u;
      } else {
        if (wg_leader) tma_store_wait_read();   // the previous tile's store has read the staging tile
        named_barrier_sync(epi_bar, 128);
      }
#define CTD_EPI(ACT)                                                                                   \
  _Pragma("unroll") for (int m = 0; m < MT; ++m) {                                                     \
    if (res16) stage_f16<BN, TH, ACT, true>(acc[m], bias_t, stg, m, warp & 3, lane);                   \
    else stage_f16<BN, TH, ACT, false>(acc[m], bias_t, stg, m, warp & 3, lane);                        \
  }
      switch (g.act) {
        case CTD_ACT_SILU: CTD_EPI(CTD_ACT_SILU) break;
        case CTD_ACT_LEAKY: CTD_EPI(CTD_ACT_LEAKY) break;
        case CTD_ACT_RELU: CTD_EPI(CTD_ACT_RELU) break;
        case CTD_ACT_SIGMOID: CTD_EPI(CTD_ACT_SIGMOID) break;
        default: CTD_EPI(CTD_ACT_NONE) break;
      }
#undef CTD_EPI
      // generic-proxy writes -> visible to the TMA (async proxy) store, then one thread stores the whole tile
      fence_proxy_async();
      named_barrier_sync(epi_bar, 128);
      if (wg_leader) {
#pragma unroll
        for (int b = 0; b < BN / Cfg::kBoxN; ++b)
          tma_store_4d(&p.d_map[phase], stg + b * Cfg::kBoxBytes, nblk * BN + b * Cfg::kBoxN, x0, sy0, img);
        tma_store_commit();
      }
      if (p.dst_map_cols < g.cout && p.dst_map_cols < (nblk + 1) * BN) {
        // columns [dst_map_cols, cout): within the last 16-byte granule of the slice, which the map leaves out
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = (wg * MT + m) * 64 + wrow + 8 * h;
            const int gy = y0 + row / kTileW, gx = x0 + row % kTileW;
            if (gy >= g.gh || gx >= g.gw) continue;
            const int oy = gy * g.out_mul + (phase >> 1), ox = gx * g.out_mul + (phase & 1);
            __half* out = p.dst + (size_t(img) * g.dst_h * g.dst_w + size_t(oy) * g.dst_w + ox) * g.dst_cstride +
                          g.dst_coff;
#pragma unroll
            for (int i = 0; i < R; ++i) {
              if (((i >> 1) & 1) != h) continue;
              const int c = (i >> 2) * 8 + (lane & 3) * 2 + (i & 1), col = nblk * BN + c;
              if (col < p.dst_map_cols || col >= g.cout) continue;
              float f;
              switch (g.act) {
                case CTD_ACT_SILU: f = apply_act<CTD_ACT_SILU>(acc[m][i] + bias_t[c]); break;
                case CTD_ACT_LEAKY: f = apply_act<CTD_ACT_LEAKY>(acc[m][i] + bias_t[c]); break;
                case CTD_ACT_RELU: f = apply_act<CTD_ACT_RELU>(acc[m][i] + bias_t[c]); break;
                case CTD_ACT_SIGMOID: f = apply_act<CTD_ACT_SIGMOID>(acc[m][i] + bias_t[c]); break;
                default: f = acc[m][i] + bias_t[c]; break;
              }
              if (res16) f = __fadd_rn(f, __half2float(out[col]));
              out[col] = __float2half_rn(f);
            }
          }
      }
      continue;
    }
    const int ph_y = phase >> 1, ph_x = phase & 1;
    const int ncols = g.cout - nblk * BN;   // columns of this N block that exist
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      int gy[2], gx[2];
      bool valid[2];
      size_t pix[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = (wg * MT + m) * 64 + wrow + 8 * h;
        gy[h] = y0 + row / kTileW;
        gx[h] = x0 + row % kTileW;
        valid[h] = gy[h] < g.gh && gx[h] < g.gw;
        const int oy = gy[h] * g.out_mul + ph_y, ox = gx[h] * g.out_mul + ph_x;
        pix[h] = valid[h] ? size_t(img) * g.dst_h * g.dst_w + size_t(oy) * g.dst_w + ox : 0;
      }
      if (p.dst == nullptr) {
        // Detect decode (yolo.py:36-44): columns = anchor*(5+nc) + o
        const int no = 5 + p.nc;
        float* rows = p.blks + (size_t(img) * p.blks_rows_per_img + p.level_row0) * no;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!valid[h]) continue;
#pragma unroll
          for (int i = 0; i < R; ++i) {
            if (((i >> 1) & 1) != h) continue;
            const int c = (i >> 2) * 8 + (lane & 3) * 2 + (i & 1);
            if (c >= ncols) continue;
            const int col = nblk * BN + c;
            const int a = col / no, o = col - a * no;
            const float s = 1.0f / (1.0f + expf(-(acc[m][i] + bias_t[c])));
            float r;
            if (o == 0) r = (s * 2.0f - 0.5f + float(gx[h])) * p.det_stride;
            else if (o == 1) r = (s * 2.0f - 0.5f + float(gy[h])) * p.det_stride;
            else if (o == 2) r = (s * 2.0f) * (s * 2.0f) * p.anchor_wh[2 * a];
            else if (o == 3) r = (s * 2.0f) * (s * 2.0f) * p.anchor_wh[2 * a + 1];
            else r = s;
            rows[(size_t(a) * g.gh * g.gw + size_t(gy[h]) * g.gw + gx[h]) * no + o] = r;
          }
        }
      } else {
        // split-fp16 mode: fp32 NHWC destination
        float* out32[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          out32[h] = reinterpret_cast<float*>(p.dst) + pix[h] * g.dst_cstride + g.dst_coff + nblk * BN;
        const bool res = g.residual != 0;
        switch (g.act) {
          case CTD_ACT_SILU: epilogue_f32<BN, CTD_ACT_SILU>(acc[m], bias_t, out32, valid, ncols, lane, res); break;
          case CTD_ACT_LEAKY: epilogue_f32<BN, CTD_ACT_LEAKY>(acc[m], bias_t, out32, valid, ncols, lane, res); break;
          case CTD_ACT_RELU: epilogue_f32<BN, CTD_ACT_RELU>(acc[m], bias_t, out32, valid, ncols, lane, res); break;
          case CTD_ACT_SIGMOID: epilogue_f32<BN, CTD_ACT_SIGMOID>(acc[m], bias_t, out32, valid, ncols, lane, res); break;
          default: epilogue_f32<BN, CTD_ACT_NONE>(acc[m], bias_t, out32, valid, ncols, lane, res); break;
        }
      }
    }
  }
  // the staging tiles must outlive the last TMA stores that read them
  if (nhwc16 && wg_leader) tma_store_wait_all();
}

// =========================================================================================
// host side

static const char* encode_map(PFN_encodeTiled enc, CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims,
                              const cuuint64_t* strides_bytes, const cuuint32_t* box, int kb_elems) {
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUtensorMapSwizzle sw = kb_elems == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                               : (kb_elems == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled failed";
}

// fp16 NHWC destination maps of the staged epilogue, one per phase: {cout & ~7, gw, gh, n_img} over the slice, so that
// TMA clips the padding columns (cout .. cout_pad), the neighbouring channels and the pixels beyond the grid (the
// innermost dimension is clipped in 16-byte units: the last cout % 8 columns are stored from registers).  A
// DECONV4 phase map starts at the phase's sub-pixel (ph_y, ph_x) and steps two destination pixels in x and y.  Boxes
// are min(BN, 64) channels x 16 x TH/2 pixels (one consumer warpgroup's half of the tile) in the swizzle of a K block
// of the same width.
static const char* encode_dst_maps(PFN_encodeTiled enc, ConvTcParams& p, const __half* dst, int bn, int th) {
  const ConvGeom& g = p.g;
  const int boxn = bn < 64 ? bn : 64;
  p.dst_map_cols = g.cout & ~7;
  if (p.dst_map_cols == 0) return "conv_tc: fp16 destination needs at least 8 output channels";
  const cuuint64_t px = cuuint64_t(g.dst_cstride) * 2;   // bytes per destination pixel
  for (int ph = 0; ph < g.n_phase; ++ph) {
    const int ph_y = ph >> 1, ph_x = ph & 1;
    const char* base = reinterpret_cast<const char*>(dst) + size_t(g.dst_coff) * 2 + (size_t(ph_y) * g.dst_w + ph_x) * px;
    cuuint64_t dims[4] = {cuuint64_t(p.dst_map_cols), cuuint64_t(g.gw), cuuint64_t(g.gh), cuuint64_t(g.n_img)};
    cuuint64_t str[3] = {px * g.out_mul, px * g.dst_w * g.out_mul, px * g.dst_w * g.dst_h};
    cuuint32_t box[4] = {cuuint32_t(boxn), kTileW, cuuint32_t(th / 2), 1};
    if (const char* e = encode_map(enc, &p.d_map[ph], base, 4, dims, str, box, boxn)) return e;
  }
  return nullptr;
}

static int g_num_sms = 132;

// N block: at most 128 output channels, so that a consumer warpgroup's 8*TH x BN fp32 accumulator fits in registers
// (64 per thread at TH = 8, 128 at TH = 16) next to the epilogue's addresses
static int pick_block_n(int cout_pad) {
  if (cout_pad >= 128 && cout_pad % 128 == 0) return 128;
  if (cout_pad % 64 == 0) return 64;
  if (cout_pad % 32 == 0) return 32;
  return 16;
}

template <int TH>
static size_t smem_for(int bn) {
  switch (bn) {
    case 128: return TcCfg<128, TH>::kSmem;
    case 64: return TcCfg<64, TH>::kSmem;
    case 32: return TcCfg<32, TH>::kSmem;
    default: return TcCfg<16, TH>::kSmem;
  }
}

const char* conv_tc_plan(ConvTcPlan& plan, PFN_encodeTiled enc, const ConvGeom& g, const void* const src_ptr[],
                         const int src_coff[], const void* w16, const float* bias, __half* dst, int split) {
  ConvTcParams& p = plan.p;
  memset(&p, 0, sizeof(p));
  p.g = g;
  p.split = split ? 1 : 0;
  p.split_img_off = g.n_img;
  p.split_row_off = g.n_phase * g.cout_pad;
  const int n_planes = split ? 2 : 1;   // hi | lo planes: images [0,n) | [n,2n) of the same buffer
  int kb = 64;
  for (int s = 0; s < g.n_src; ++s) {
    if (g.src_c[s] % 64 != 0 && kb > 32) kb = 32;
    if (g.src_c[s] % 32 != 0) kb = 16;
    if (g.src_c[s] % 16 != 0) return "conv_tc: source channels must be a multiple of 16";
    if (src_coff[s] % 8 != 0) return "conv_tc: source channel offset must be a multiple of 8";
  }
  if ((g.dst_coff % 8) != 0 || (g.dst_cstride % 8) != 0) return "conv_tc: destination slice must be 16-byte aligned";
  p.kb_elems = kb;
  for (int s = 0; s < g.n_src; ++s) p.src_kblocks[s] = g.src_c[s] / kb;
  p.tiles_x = (g.gw + kTileW - 1) / kTileW;
  int bn = pick_block_n(g.cout_pad);
  // small grids (the 1/32 and 1/64 layers): a narrower N block spreads the layer over more SMs
  const int tiles8 = g.n_img * p.tiles_x * ((g.gh + 7) / 8) * g.n_phase;   // 16x8 tiles per N block
  while (bn > 64 && tiles8 * (g.cout_pad / bn) <= g_num_sms / 2) bn /= 2;
  if (split && bn > 64) bn = 64;   // promoted accumulation keeps three BN/2-float fragments per thread in registers
  // 16x16 tiles (M = 256) read each weight box once per 256 pixels instead of 128.  Used for the fp16 NHWC-store ops
  // (CONV, DECONV4) whose layer still has a tile per SM at that size; split mode and Detect (dst == nullptr) stay at
  // 16x8.
  int th = 8;
  if (!split && dst != nullptr &&
      g.n_img * p.tiles_x * ((g.gh + 15) / 16) * g.n_phase * (g.cout_pad / bn) >= g_num_sms)
    th = 16;
  p.tiles_y = (g.gh + th - 1) / th;
  p.dst = dst;
  p.bias = bias;
  const int sh = g.src_h, sw = g.src_w;
  for (int s = 0; s < g.n_src; ++s) {
    const size_t cs = size_t(g.src_cstride[s]);
    const char* base = static_cast<const char*>(src_ptr[s]) + size_t(src_coff[s]) * 2;
    if (g.in_stride == 1) {
      cuuint64_t dims[4] = {cuuint64_t(g.src_c[s]), cuuint64_t(sw), cuuint64_t(sh), cuuint64_t(g.n_img * n_planes)};
      cuuint64_t str[3] = {cs * 2, cs * 2 * sw, cs * 2 * sw * sh};
      cuuint32_t box[4] = {cuuint32_t(kb), kTileW, cuuint32_t(th), 1};
      if (const char* e = encode_map(enc, &p.a_map[s][0], base, 4, dims, str, box, kb)) return e;
    } else {
      // parity views: pixel (2*yh+yp, 2*xh+xp)
      for (int q = 0; q < 4; ++q) {
        const int yp = q >> 1, xp = q & 1;
        cuuint64_t dims[4] = {cuuint64_t(g.src_c[s]), cuuint64_t(sw / 2), cuuint64_t(sh / 2), cuuint64_t(g.n_img * n_planes)};
        cuuint64_t str[3] = {cs * 2 * 2, cs * 2 * sw * 2, cs * 2 * sw * sh};
        cuuint32_t box[4] = {cuuint32_t(kb), kTileW, cuuint32_t(th), 1};
        const char* b2 = base + (size_t(yp) * sw + xp) * cs * 2;
        if (const char* e = encode_map(enc, &p.a_map[s][q], b2, 4, dims, str, box, kb)) return e;
      }
    }
  }
  // tap -> (parity map, offset in map coordinates)
  for (int ph = 0; ph < g.n_phase; ++ph)
    for (int t = 0; t < g.taps; ++t) {
      if (g.in_stride == 2) {
        // source pixel = 2*o + d, d in {-1,0,1}: d=-1 -> (h=o-1, parity 1); d=0 -> (o,0); d=1 -> (o,1)
        const int dy = g.tap_dy[ph][t], dx = g.tap_dx[ph][t];
        const int yp = dy != 0, xp = dx != 0;
        p.tap_map[ph][t] = int8_t(yp * 2 + xp);
        p.g.tap_dy[ph][t] = int8_t(dy < 0 ? -1 : 0);
        p.g.tap_dx[ph][t] = int8_t(dx < 0 ? -1 : 0);
      } else {
        p.tap_map[ph][t] = 0;
      }
    }
  plan.block_n = bn;
  plan.tile_h = th;
  if (dst != nullptr && !split)
    if (const char* e = encode_dst_maps(enc, p, dst, bn, th)) return e;
  if (split && ((g.dst_coff % 4) != 0 || (g.dst_cstride % 4) != 0 || (dst != nullptr && g.cout % 4 != 0)))
    return "conv_tc (split): fp32 destination slice must be 16-byte aligned";
  {
    cuuint64_t dims[2] = {cuuint64_t(g.k_total), cuuint64_t(g.n_phase) * cuuint64_t(g.cout_pad) * n_planes};
    cuuint64_t str[1] = {cuuint64_t(g.k_total) * 2};
    cuuint32_t box[2] = {cuuint32_t(kb), cuuint32_t(bn)};
    if (const char* e = encode_map(enc, &p.b_map, w16, 2, dims, str, box, kb)) return e;
  }
  {
    const int total_tiles = g.n_img * p.tiles_x * p.tiles_y * (g.cout_pad / bn) * g.n_phase;
    plan.grid = dim3(unsigned(total_tiles < g_num_sms ? total_tiles : g_num_sms), 1, 1);
  }
  if (g.cout_pad > 512) return "conv_tc: cout_pad > 512 not supported (bias staging)";
  plan.smem_bytes = th == 16 ? smem_for<16>(bn) : smem_for<8>(bn);
  return nullptr;
}

cudaError_t conv_tc_init() {
  cudaError_t e;
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) g_num_sms = n;
  }
#define CTD_SET(BN, TH)                                                                                       \
  e = cudaFuncSetAttribute(conv_tc_kernel<BN, TH>, cudaFuncAttributeMaxDynamicSharedMemorySize,               \
                           int(TcCfg<BN, TH>::kSmem));                                                        \
  if (e != cudaSuccess) return e;
  CTD_SET(128, 8) CTD_SET(64, 8) CTD_SET(32, 8) CTD_SET(16, 8)
  CTD_SET(128, 16) CTD_SET(64, 16) CTD_SET(32, 16) CTD_SET(16, 16)
#undef CTD_SET
  return cudaSuccess;
}

template <int TH>
static void launch_th(const ConvTcPlan& plan, cudaStream_t s) {
  switch (plan.block_n) {
    case 128: conv_tc_kernel<128, TH><<<plan.grid, kThreads, plan.smem_bytes, s>>>(plan.p); break;
    case 64: conv_tc_kernel<64, TH><<<plan.grid, kThreads, plan.smem_bytes, s>>>(plan.p); break;
    case 32: conv_tc_kernel<32, TH><<<plan.grid, kThreads, plan.smem_bytes, s>>>(plan.p); break;
    default: conv_tc_kernel<16, TH><<<plan.grid, kThreads, plan.smem_bytes, s>>>(plan.p); break;
  }
}

cudaError_t conv_tc_launch(const ConvTcPlan& plan, cudaStream_t s) {
  if (plan.tile_h == 16) launch_th<16>(plan, s);
  else launch_th<8>(plan, s);
  return cudaGetLastError();
}

}  // namespace ctd
