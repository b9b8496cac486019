// Host planner of the text-line crops (C ABI `ctd_region_plan`, include/ctd_b200.h): the geometry of the reference's
// `TextBlock.get_transformed_region` (utils/textblock.py:162-194) for many lines at once.
//
// The warp kernel (region.cu) rounds X0 * 32 / W to the nearest integer, and for the integer quads the detector emits
// that product lands on exact .5 ties, so a crop is bit-identical to cv2's only if the matrix it samples with is.  The
// planner therefore restates, in IEEE double and in OpenCV's operation order, each step that produces the matrix:
//   * the line expansion / clip and the size rule (python float arithmetic, `round` half to even);
//   * the vector norms as numpy computes them (OpenBLAS ddot: x0*x0, then x1*x1 fused into the sum);
//   * cv2.findHomography with 4 points, which never runs RANSAC: points converted to float32, the normalised DLT
//     (centroid + mean absolute deviation scaling), the 9x9 normal matrix, its eigenvector of smallest eigenvalue by
//     classical Jacobi rotations (largest off-diagonal pivot, scaled hypotenuse) as OpenCV's `eigen` runs them,
//     de-normalisation through two unfused 3x3 products and the scaling by 1 / H[2][2] (a multiply, so H[2][2] may
//     end up one ulp from 1, as in cv2's result);
//   * cv2.invert(M, DECOMP_LU) for 3x3, i.e. the adjugate over the cofactor-expanded determinant.
// Written from those algorithms' published descriptions; tests/test_cpu_regions.py compares every matrix with cv2's.
// Compiled with -ffp-contract=off (build.sh): a fused multiply-add anywhere except where written explicitly would
// change the matrices in the last bit.
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/ctd_b200.h"

namespace {

constexpr int kMaxSide = 32767;   // cv::remap's 16-bit coordinates (SHRT_MAX)

// the scaled hypotenuse OpenCV's Jacobi solver uses (not libm's hypot, which rounds differently)
inline double scaled_hypot(double a, double b) {
  a = fabs(a);
  b = fabs(b);
  if (a > b) {
    b /= a;
    return a * sqrt(1 + b * b);
  }
  if (b > 0) {
    a /= b;
    return b * sqrt(1 + a * a);
  }
  return 0;
}

// symmetric n x n eigen-decomposition by Jacobi rotations; on return W holds the eigenvalues in descending order and
// the rows of V the matching eigenvectors (A is destroyed)
void jacobi9(double* A, double* W, double* V) {
  const int n = 9;
  const double eps = DBL_EPSILON;
  int indR[9], indC[9];
  for (int i = 0; i < n; ++i) {
    for (int j = 0; j < n; ++j) V[i * n + j] = 0;
    V[i * n + i] = 1;
  }
  // indR[k]: column of the largest |A[k][m]|, m > k; indC[k]: row of the largest |A[m][k]|, m < k
  auto scan_row = [&](int k) {
    int m = k + 1;
    double mv = fabs(A[n * k + m]);
    for (int i = k + 2; i < n; ++i) {
      const double v = fabs(A[n * k + i]);
      if (mv < v) mv = v, m = i;
    }
    indR[k] = m;
  };
  auto scan_col = [&](int k) {
    int m = 0;
    double mv = fabs(A[k]);
    for (int i = 1; i < k; ++i) {
      const double v = fabs(A[n * i + k]);
      if (mv < v) mv = v, m = i;
    }
    indC[k] = m;
  };
  for (int k = 0; k < n; ++k) {
    W[k] = A[(n + 1) * k];
    if (k < n - 1) scan_row(k);
    if (k > 0) scan_col(k);
  }
  for (int iters = 0; iters < n * n * 30; ++iters) {
    int k = 0;
    double mv = fabs(A[indR[0]]);
    for (int i = 1; i < n - 1; ++i) {
      const double v = fabs(A[n * i + indR[i]]);
      if (mv < v) mv = v, k = i;
    }
    int l = indR[k];
    for (int i = 1; i < n; ++i) {
      const double v = fabs(A[n * indC[i] + i]);
      if (mv < v) mv = v, k = indC[i], l = i;
    }
    const double p = A[n * k + l];
    if (fabs(p) <= eps) break;
    const double y = (W[l] - W[k]) * 0.5;
    double t = fabs(y) + scaled_hypot(p, y);
    double s = scaled_hypot(p, t);
    const double c = t / s;
    s = p / s;
    t = (p / t) * p;
    if (y < 0) s = -s, t = -t;
    A[n * k + l] = 0;
    W[k] -= t;
    W[l] += t;
    auto rot = [&](double& v0, double& v1) {
      const double a0 = v0, b0 = v1;
      v0 = a0 * c - b0 * s;
      v1 = a0 * s + b0 * c;
    };
    for (int i = 0; i < k; ++i) rot(A[n * i + k], A[n * i + l]);
    for (int i = k + 1; i < l; ++i) rot(A[n * k + i], A[n * i + l]);
    for (int i = l + 1; i < n; ++i) rot(A[n * k + i], A[n * l + i]);
    for (int i = 0; i < n; ++i) rot(V[n * k + i], V[n * l + i]);
    for (int idx : {k, l}) {
      if (idx < n - 1) scan_row(idx);
      if (idx > 0) scan_col(idx);
    }
  }
  for (int k = 0; k < n - 1; ++k) {   // selection sort, descending
    int m = k;
    for (int i = k + 1; i < n; ++i)
      if (W[m] < W[i]) m = i;
    if (k != m) {
      std::swap(W[m], W[k]);
      for (int i = 0; i < n; ++i) std::swap(V[n * m + i], V[n * k + i]);
    }
  }
}

// D = A * B for 3x3 row-major matrices, each element summed left to right without fusing (OpenCV's small-matrix gemm)
void mul3(const double* A, const double* B, double* D) {
  double T[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) T[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
  for (int i = 0; i < 9; ++i) D[i] = T[i];
}

// cv::findHomography(src, dst, method, ...) for exactly 4 correspondences (points already float32): 0 when OpenCV
// returns an empty matrix (all x or all y of either set coincide)
int homography4(const float* M, const float* m, double* H) {
  const int count = 4;
  double cMx = 0, cMy = 0, cmx = 0, cmy = 0, sMx = 0, sMy = 0, smx = 0, smy = 0;
  for (int i = 0; i < count; ++i) {
    cmx += m[2 * i]; cmy += m[2 * i + 1];
    cMx += M[2 * i]; cMy += M[2 * i + 1];
  }
  cmx /= count; cmy /= count; cMx /= count; cMy /= count;
  for (int i = 0; i < count; ++i) {
    smx += fabs(m[2 * i] - cmx); smy += fabs(m[2 * i + 1] - cmy);
    sMx += fabs(M[2 * i] - cMx); sMy += fabs(M[2 * i + 1] - cMy);
  }
  if (fabs(smx) < DBL_EPSILON || fabs(smy) < DBL_EPSILON || fabs(sMx) < DBL_EPSILON || fabs(sMy) < DBL_EPSILON) return 0;
  smx = count / smx; smy = count / smy;
  sMx = count / sMx; sMy = count / sMy;
  const double invHnorm[9] = {1. / smx, 0, cmx, 0, 1. / smy, cmy, 0, 0, 1};
  const double Hnorm2[9] = {sMx, 0, -cMx * sMx, 0, sMy, -cMy * sMy, 0, 0, 1};
  double LtL[81] = {0};
  for (int i = 0; i < count; ++i) {
    const double x = (m[2 * i] - cmx) * smx, y = (m[2 * i + 1] - cmy) * smy;
    const double X = (M[2 * i] - cMx) * sMx, Y = (M[2 * i + 1] - cMy) * sMy;
    const double Lx[9] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y, -x};
    const double Ly[9] = {0, 0, 0, X, Y, 1, -y * X, -y * Y, -y};
    for (int j = 0; j < 9; ++j)
      for (int k = j; k < 9; ++k) LtL[9 * j + k] += Lx[j] * Lx[k] + Ly[j] * Ly[k];
  }
  for (int j = 0; j < 9; ++j)
    for (int k = 0; k < j; ++k) LtL[9 * j + k] = LtL[9 * k + j];
  double W[9], V[81];
  jacobi9(LtL, W, V);
  double H0[9];
  mul3(invHnorm, V + 72, H0);   // eigenvector of the smallest eigenvalue = last row
  mul3(H0, Hnorm2, H0);
  // scaled so that H[2][2] ~ 1, unless H[2][2] is within FLT_EPSILON of 0 (a degenerate quad): then left as it is
  const double scale = fabs(H0[8]) > FLT_EPSILON ? 1. / H0[8] : 1.;
  for (int i = 0; i < 9; ++i) H[i] = H0[i] * scale;
  return 1;
}

// cv::invert(M, DECOMP_LU) of a 3x3 double matrix; a singular matrix gives zeros (and cv's `false`)
void invert3(const double* m, double* out) {
  auto M = [&](int r, int c) { return m[3 * r + c]; };
  double d = M(0, 0) * (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) - M(0, 1) * (M(1, 0) * M(2, 2) - M(1, 2) * M(2, 0)) +
             M(0, 2) * (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0));
  if (d == 0.) {
    for (int i = 0; i < 9; ++i) out[i] = 0;
    return;
  }
  d = 1. / d;
  out[0] = (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) * d;
  out[1] = (M(0, 2) * M(2, 1) - M(0, 1) * M(2, 2)) * d;
  out[2] = (M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) * d;
  out[3] = (M(1, 2) * M(2, 0) - M(1, 0) * M(2, 2)) * d;
  out[4] = (M(0, 0) * M(2, 2) - M(0, 2) * M(2, 0)) * d;
  out[5] = (M(0, 2) * M(1, 0) - M(0, 0) * M(1, 2)) * d;
  out[6] = (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)) * d;
  out[7] = (M(0, 1) * M(2, 0) - M(0, 0) * M(2, 1)) * d;
  out[8] = (M(0, 0) * M(1, 1) - M(0, 1) * M(1, 0)) * d;
}

// norm of a 2-vector as numpy.linalg.norm returns it (sqrt of OpenBLAS's ddot: the second square fused into the sum)
inline double norm2(double a, double b) { return sqrt(fma(b, b, a * a)); }

// python's int(round(q)) for a finite q >= 0, as the rounded size of a crop side; -1 when the reference raises
// (q is inf or NaN)
inline int64_t py_round_size(double q) {
  if (!(q <= 1e18)) return -1;
  return int64_t(nearbyint(q));   // default rounding mode: half to even, like python's round
}

void plan_one(const ctd_region_line& L, int im_w, int im_h, int textheight, ctd_region& r) {
  double p[8];
  for (int i = 0; i < 8; ++i) p[i] = L.quad[i];
  if (L.language == 0 || (L.language == 2 && !L.vertical)) {
    const double e = L.font_size / 3;
    static const int sx[4] = {-1, 1, 1, -1}, sy[4] = {-1, -1, 1, 1};
    for (int i = 0; i < 4; ++i) {
      p[2 * i] += sx[i] < 0 ? -e : e;
      p[2 * i + 1] += sy[i] < 0 ? -e : e;
      // np.clip(a, 0, hi) = minimum(maximum(a, 0), hi)
      p[2 * i] = std::min(std::max(p[2 * i], 0.0), double(im_w));
      p[2 * i + 1] = std::min(std::max(p[2 * i + 1], 0.0), double(im_h));
    }
  }
  double mid[8];   // (src_pts[[1, 2, 3, 0]] + src_pts) / 2
  for (int i = 0; i < 4; ++i) {
    const int j = (i + 1) & 3;
    mid[2 * i] = (p[2 * j] + p[2 * i]) / 2;
    mid[2 * i + 1] = (p[2 * j + 1] + p[2 * i + 1]) / 2;
  }
  const double nv = norm2(mid[4] - mid[0], mid[5] - mid[1]);
  const double nh = norm2(mid[2] - mid[6], mid[3] - mid[7]);
  const double ratio = nv / nh;   // numpy: x / 0 = inf, 0 / 0 = nan (warnings, no exception)
  int64_t w, h;
  if (!L.vertical) {
    h = textheight;
    if (ratio == 0.0) { r.status = 1; return; }   // python float division by zero
    w = py_round_size(textheight / ratio);
  } else {
    w = textheight;
    h = py_round_size(textheight * ratio);
  }
  if (w < 0 || h < 0) { r.status = 1; return; }
  if (w >= kMaxSide || h >= kMaxSide) { r.status = 2; return; }
  r.rotate = L.vertical ? 1 : 0;
  float src[8], dst[8];
  for (int i = 0; i < 8; ++i) src[i] = float(p[i]);
  const float wm = float(w - 1), hm = float(h - 1);
  const float d[8] = {0, 0, wm, 0, wm, hm, 0, hm};
  for (int i = 0; i < 8; ++i) dst[i] = d[i];
  if (!homography4(src, dst, r.homography)) { r.status = 1; return; }
  invert3(r.homography, r.inverse);
  // cv2.warpPerspective with an empty dsize (a side rounded to 0) writes a page-sized image
  const int64_t ww = (w <= 0 || h <= 0) ? im_w : w, wh = (w <= 0 || h <= 0) ? im_h : h;
  r.out_h = int32_t(r.rotate ? ww : wh);
  r.out_w = int32_t(r.rotate ? wh : ww);
}

}  // namespace

extern "C" CTD_API int ctd_region_plan(const ctd_region_line* lines, int32_t n, int32_t im_w, int32_t im_h,
                                       int32_t textheight, ctd_region* out, size_t* total_bytes) {
  if (n < 0 || (n > 0 && (!lines || !out)) || !total_bytes) return CTD_E_INVALID;
  if (im_w < 1 || im_h < 1 || im_w >= kMaxSide || im_h >= kMaxSide || textheight < 2) return CTD_E_INVALID;
  size_t off = 0;
  for (int32_t i = 0; i < n; ++i) {
    ctd_region& r = out[i];
    r = ctd_region{};
    plan_one(lines[i], im_w, im_h, textheight, r);
    if (r.status != 0) {
      r.out_h = r.out_w = r.rotate = 0;
      for (int k = 0; k < 9; ++k) r.homography[k] = r.inverse[k] = 0;
    }
    r.offset = int64_t(off);
    off += size_t(r.out_h) * size_t(r.out_w) * 3;
  }
  *total_bytes = off;
  return CTD_OK;
}
