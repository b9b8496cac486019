// Batched strided page gather (ctd_submit_pages, ctd_submit_refine): every page of a batch that is already in device
// memory, laid out with any strides (a sub-window of a larger image, a permuted channels-first image), copied in one
// launch into the packed page buffer of the batch (u8 BGR [ih][iw][3] at the page's page_off), where the letterbox,
// refine_mask and the crop kernels read it; in the same launch, the batch's masks in device memory (u8 [ih][iw], any
// strides: a channel of a page) into its packed mask plane.  One CTA per row over the stacked rows of the gathered
// images, as backproject_batch_kernel.
#include <cuda_runtime.h>
#include <stdint.h>

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

}  // namespace

cudaError_t gather_pages_launch(const GatherPage* d_tab, int n, int total_rows, cudaStream_t s) {
  if (n < 1 || total_rows < 1) return cudaErrorInvalidValue;
  gather_pages_kernel<<<unsigned(total_rows), 256, 0, s>>>(d_tab, n);
  return cudaGetLastError();
}

}  // namespace ctd
