// Per-contour geometry of the DB post-processing (reference utils/db_utils.py:141-195):
//   get_mini_boxes  = cv2.minAreaRect -> cv2.boxPoints -> corner ordering          (176-195)
//   unclip          = shapely area/length -> pyclipper offset (JT_ROUND)            (168-174)
//   quantisation    = clip(round(x / w * dest_w), 0, dest_w) -> int16               (162-165)
// written as host+device inline functions so that the SAME code is unit-tested on the CPU against
// OpenCV (tests/test_cpu_geom.py builds tests/geom_host.cpp with g++) and runs inside the CUDA kernel
// (csrc/segrep.cu).  All float32 arithmetic goes through explicitly rounded, non-contracted ops
// (F_* macros) in the order OpenCV's rotating-calipers code performs them.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define CTD_HD __host__ __device__ __forceinline__
#else
#define CTD_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define F_MUL(a, b) __fmul_rn((a), (b))
#define F_ADD(a, b) __fadd_rn((a), (b))
#define F_SUB(a, b) __fsub_rn((a), (b))
#define F_DIV(a, b) __fdiv_rn((a), (b))
#define D_MUL(a, b) __dmul_rn((a), (b))
#define D_ADD(a, b) __dadd_rn((a), (b))
#define D_SUB(a, b) __dsub_rn((a), (b))
#define D_DIV(a, b) __ddiv_rn((a), (b))
#else
// host build uses -ffp-contract=off
#define F_MUL(a, b) ((float)((float)(a) * (float)(b)))
#define F_ADD(a, b) ((float)((float)(a) + (float)(b)))
#define F_SUB(a, b) ((float)((float)(a) - (float)(b)))
#define F_DIV(a, b) ((float)((float)(a) / (float)(b)))
#define D_MUL(a, b) ((double)(a) * (double)(b))
#define D_ADD(a, b) ((double)(a) + (double)(b))
#define D_SUB(a, b) ((double)(a) - (double)(b))
#define D_DIV(a, b) ((double)(a) / (double)(b))
#endif

namespace ctdgeom {

// Hull capacity for maps up to 2048^2 (ctd_seg_represent's limit).  A strictly convex lattice polygon's edges have
// pairwise distinct directions, so their primitive vectors are distinct; its edges' |dx| sum to twice its width and
// their |dy| to twice its height, so their L1 lengths sum to at most 4 * 2047 = 8188.  There are 4j nonzero integer
// vectors of L1 norm j: all 612 of norm <= 17 already sum to 7140, leaving room for at most 58 of norm 18 -- at most
// 670 vertices.  The monotone chain holds the closing vertex once more (671); 560-vertex polygons inside 1998^2 exist
// (tests/lattice_polygon.py).
constexpr int kMaxHull = 704;
constexpr int kMaxOffsetPts = 512; // vertices emitted by the round-join offset of a quad
constexpr double kPi = 3.141592653589793238;

struct IPt { int x, y; };
struct RRect { float cx, cy, w, h, angle; };

CTD_HD long long cross3(const IPt& o, const IPt& a, const IPt& b) {
  return (long long)(a.x - o.x) * (b.y - o.y) - (long long)(a.y - o.y) * (b.x - o.x);
}

// Andrew monotone chain over points sorted by (x, then y); strictly convex vertices; orientation
// cross > 0 in raw (x, y), i.e. the order cv2.convexHull(clockwise=False) emits; the output is rotated
// to start at the max-x (then max-y) vertex like OpenCV's Sklansky driver.  `pts` is overwritten.
// Returns the vertex count (<= cap), or -1 on overflow.
CTD_HD int hull_sorted(const IPt* pts, int n, IPt* hull, int cap) {
  if (n <= 0) return 0;
  int k = 0;
  for (int i = 0; i < n; ++i) {  // lower chain
    if (i > 0 && pts[i].x == pts[i - 1].x && pts[i].y == pts[i - 1].y) continue;
    while (k >= 2 && cross3(hull[k - 2], hull[k - 1], pts[i]) <= 0) --k;
    if (k >= cap) return -1;
    hull[k++] = pts[i];
  }
  const int lower = k + 1;
  for (int i = n - 2; i >= 0; --i) {  // upper chain
    if (pts[i].x == pts[i + 1].x && pts[i].y == pts[i + 1].y) continue;
    while (k >= lower && cross3(hull[k - 2], hull[k - 1], pts[i]) <= 0) --k;
    if (k >= cap) return -1;
    hull[k++] = pts[i];
  }
  if (k > 1) --k;  // last point repeats the first
  return k;
}

// rotate so that hull[0] is the max-x (ties: max-y) vertex
CTD_HD void hull_start_maxx(IPt* hull, int n, IPt* tmp) {
  if (n < 3) return;
  int s = 0;
  for (int i = 1; i < n; ++i)
    if (hull[i].x > hull[s].x || (hull[i].x == hull[s].x && hull[i].y > hull[s].y)) s = i;
  if (s == 0) return;
  for (int i = 0; i < n; ++i) tmp[i] = hull[(i + s) % n];
  for (int i = 0; i < n; ++i) hull[i] = tmp[i];
}

// OpenCV rotatingCalipers(CALIPERS_MINAREARECT) + minAreaRect wrapper, float32 arithmetic in OpenCV's
// order, followed by the angle normalisation of OpenCV >= 4.5 (angle in [-90, 0), width/height swapped
// accordingly).  hull: n >= 3 strictly convex vertices.  vect/inv: scratch of n entries each.
// first pass of minAreaRect: per-edge vectors / inverse lengths and the four extreme vertices (FIRST index of each
// extreme, like OpenCV's strict comparisons).  Element-wise work: the GPU runs it across the warp (segrep.cu).
struct MarExt { int left, bottom, right, top; };
CTD_HD void mar_edge(const IPt* hull, int n, int i, float* vx, float* vy, float* inv) {
  const int j = (i + 1 < n) ? i + 1 : 0;
  const float p0x = (float)hull[i].x, p0y = (float)hull[i].y, px = (float)hull[j].x, py = (float)hull[j].y;
  const double dx = (double)px - (double)p0x, dy = (double)py - (double)p0y;
  vx[i] = (float)dx;
  vy[i] = (float)dy;
  inv[i] = (float)D_DIV(1.0, sqrt(D_ADD(D_MUL(dx, dx), D_MUL(dy, dy))));
}
CTD_HD MarExt mar_prepass(const IPt* hull, int n, float* vx, float* vy, float* inv) {
  MarExt e{0, 0, 0, 0};
  float left_x, right_x, top_y, bottom_y;
  left_x = right_x = (float)hull[0].x;
  top_y = bottom_y = (float)hull[0].y;
  for (int i = 0; i < n; ++i) {
    const float p0x = (float)hull[i].x, p0y = (float)hull[i].y;
    if (p0x < left_x) { left_x = p0x; e.left = i; }
    if (p0x > right_x) { right_x = p0x; e.right = i; }
    if (p0y > top_y) { top_y = p0y; e.top = i; }
    if (p0y < bottom_y) { bottom_y = p0y; e.bottom = i; }
    mar_edge(hull, n, i, vx, vy, inv);
  }
  return e;
}

CTD_HD RRect mar_core(const IPt* hull, int n, const float* vx, const float* vy, const float* inv, MarExt ext) {
  const int left = ext.left, bottom = ext.bottom, right = ext.right, top = ext.top;
  float orientation = 0.f;
  {
    double ax = vx[n - 1], ay = vy[n - 1];
    for (int i = 0; i < n; ++i) {
      const double bx = vx[i], by = vy[i];
      const double convexity = D_SUB(D_MUL(ax, by), D_MUL(ay, bx));
      if (convexity != 0) {
        orientation = convexity > 0 ? 1.f : -1.f;
        break;
      }
      ax = bx;
      ay = by;
    }
  }
  float base_a = orientation, base_b = 0.f;
  int seq[4] = {bottom, right, top, left};
  float minarea = 3.402823466e+38f;
  int b_left = 0, b_bottom = 0;
  float b_a = 1.f, b_b = 0.f, b_w = 0.f, b_h = 0.f;
  for (int k = 0; k < n; ++k) {
    // OpenCV >= 4.5.2 (rotcalipers.cpp): the caliper side that meets its polygon edge first is found from the SIGN of
    // cross products of the four edge vectors rotated into a common frame (bottom: as is, right: 90 deg clockwise,
    // top: 180 deg, left: 90 deg counter-clockwise), not from float cosines -- exact for integer hull vertices
    float rvx[4], rvy[4];
    rvx[0] = vx[seq[0]];  rvy[0] = vy[seq[0]];
    rvx[1] = vy[seq[1]];  rvy[1] = -vx[seq[1]];
    rvx[2] = -vx[seq[2]]; rvy[2] = -vy[seq[2]];
    rvx[3] = -vy[seq[3]]; rvy[3] = vx[seq[3]];
    int main_element = 0;
    for (int i = 1; i < 4; ++i) {
      // firstVecIsRight(rot[i], rot[main]): rotate rot[i] 90 deg clockwise, dot with rot[main] < 0
      const float tx = rvy[i], ty = -rvx[i];
      if (F_ADD(F_MUL(tx, rvx[main_element]), F_MUL(ty, rvy[main_element])) < 0.f) main_element = i;
    }
    const int pindex = seq[main_element];
    const float lead_x = F_MUL(vx[pindex], inv[pindex]);
    const float lead_y = F_MUL(vy[pindex], inv[pindex]);
    switch (main_element) {
      case 0: base_a = lead_x; base_b = lead_y; break;
      case 1: base_a = lead_y; base_b = -lead_x; break;
      case 2: base_a = -lead_x; base_b = -lead_y; break;
      default: base_a = -lead_y; base_b = lead_x; break;
    }
    seq[main_element] += 1;
    if (seq[main_element] == n) seq[main_element] = 0;
    float dx = F_SUB((float)hull[seq[1]].x, (float)hull[seq[3]].x);
    float dy = F_SUB((float)hull[seq[1]].y, (float)hull[seq[3]].y);
    const float width = F_ADD(F_MUL(dx, base_a), F_MUL(dy, base_b));
    dx = F_SUB((float)hull[seq[2]].x, (float)hull[seq[0]].x);
    dy = F_SUB((float)hull[seq[2]].y, (float)hull[seq[0]].y);
    const float height = F_ADD(F_MUL(-dx, base_b), F_MUL(dy, base_a));
    const float area = F_MUL(width, height);
    if (area <= minarea) {
      minarea = area;
      b_left = seq[3];
      b_a = base_a;
      b_w = width;
      b_b = base_b;
      b_h = height;
      b_bottom = seq[0];
    }
  }
  const float A1 = b_a, B1 = b_b, A2 = -b_b, B2 = b_a;
  const float C1 = F_ADD(F_MUL(A1, (float)hull[b_left].x), F_MUL((float)hull[b_left].y, B1));
  const float C2 = F_ADD(F_MUL(A2, (float)hull[b_bottom].x), F_MUL((float)hull[b_bottom].y, B2));
  const float idet = F_DIV(1.f, F_SUB(F_MUL(A1, B2), F_MUL(A2, B1)));
  const float px = F_MUL(F_SUB(F_MUL(C1, B2), F_MUL(C2, B1)), idet);
  const float py = F_MUL(F_SUB(F_MUL(A1, C2), F_MUL(A2, C1)), idet);
  const float o1x = F_MUL(A1, b_w), o1y = F_MUL(B1, b_w), o2x = F_MUL(A2, b_h), o2y = F_MUL(B2, b_h);
  RRect r;
  r.cx = F_ADD(px, F_MUL(F_ADD(o1x, o2x), 0.5f));
  r.cy = F_ADD(py, F_MUL(F_ADD(o1y, o2y), 0.5f));
  r.w = (float)sqrt(D_ADD(D_MUL((double)o1x, (double)o1x), D_MUL((double)o1y, (double)o1y)));
  r.h = (float)sqrt(D_ADD(D_MUL((double)o2x, (double)o2x), D_MUL((double)o2y, (double)o2y)));
  // OpenCV 4.13 minAreaRect: the angle is formed in DOUBLE from the first side vector, brought into [-90, 0) by
  // quarter turns (each swaps width and height) and only then rounded to float -- pinned against cv2 on 20k random
  // hulls (tests/test_cpu_geom.py): f32(atan2(y, x) * 180 / pi - 90) for the first-quadrant vectors the calipers emit.
  double deg = D_DIV(D_MUL(atan2((double)o1y, (double)o1x), 180.0), kPi);
  int nsw = 0;
  while (deg >= 0) { deg = D_SUB(deg, 90.0); ++nsw; }
  while (deg < -90) { deg = D_ADD(deg, 90.0); ++nsw; }
  if (nsw & 1) { const float t = r.w; r.w = r.h; r.h = t; }
  const float ang = (float)deg;
  r.angle = ang;
  return r;
}

CTD_HD RRect min_area_rect(const IPt* hull, int n, float* vx, float* vy, float* inv) {
  const MarExt e = mar_prepass(hull, n, vx, vy, inv);
  return mar_core(hull, n, vx, vy, inv, e);
}

// cv2.boxPoints (RotatedRect::points)
CTD_HD void box_points(const RRect& r, float* px, float* py) {
  const double a_ = D_DIV(D_MUL((double)r.angle, kPi), 180.0);
  const float b = F_MUL((float)cos(a_), 0.5f);
  const float a = F_MUL((float)sin(a_), 0.5f);
  px[0] = F_SUB(F_SUB(r.cx, F_MUL(a, r.h)), F_MUL(b, r.w));
  py[0] = F_SUB(F_ADD(r.cy, F_MUL(b, r.h)), F_MUL(a, r.w));
  px[1] = F_SUB(F_ADD(r.cx, F_MUL(a, r.h)), F_MUL(b, r.w));
  py[1] = F_SUB(F_SUB(r.cy, F_MUL(b, r.h)), F_MUL(a, r.w));
  px[2] = F_SUB(F_MUL(2.f, r.cx), px[0]);
  py[2] = F_SUB(F_MUL(2.f, r.cy), py[0]);
  px[3] = F_SUB(F_MUL(2.f, r.cx), px[1]);
  py[3] = F_SUB(F_MUL(2.f, r.cy), py[1]);
}

// get_mini_boxes' ordering (db_utils.py:178-194): stable sort by x, then [TL, TR, BR, BL]
CTD_HD void order_mini_box(const float* px, const float* py, float* ox, float* oy) {
  int idx[4] = {0, 1, 2, 3};
  for (int i = 1; i < 4; ++i) {  // stable insertion sort by x
    const int v = idx[i];
    int j = i - 1;
    while (j >= 0 && px[idx[j]] > px[v]) { idx[j + 1] = idx[j]; --j; }
    idx[j + 1] = v;
  }
  int i1, i2, i3, i4;
  if (py[idx[1]] > py[idx[0]]) { i1 = 0; i4 = 1; } else { i1 = 1; i4 = 0; }
  if (py[idx[3]] > py[idx[2]]) { i2 = 2; i3 = 3; } else { i2 = 3; i3 = 2; }
  const int o[4] = {idx[i1], idx[i2], idx[i3], idx[i4]};
  for (int k = 0; k < 4; ++k) { ox[k] = px[o[k]]; oy[k] = py[o[k]]; }
}

CTD_HD long long clip_round(double v) { return v < 0 ? (long long)(v - 0.5) : (long long)(v + 0.5); }

// unclip (db_utils.py:168-174): GEOS ring area / length of the 4 float points, distance = area*ratio/length,
// Clipper 6.4.2 ClipperOffset(JT_ROUND, ET_CLOSEDPOLYGON, MiterLimit 2, ArcTolerance 0.25) of the
// points truncated to integers.  Emits the raw offset vertices (the trailing union only removes
// duplicate/collinear vertices, irrelevant for the convex hull taken next).  Returns the count.
CTD_HD int unclip_offset(const float* bx, const float* by, double ratio, IPt* out, int cap) {
  // --- GEOS Area::ofRingSigned / Length::ofLine on the closed ring
  double rx[5], ry[5];
  for (int i = 0; i < 4; ++i) { rx[i] = bx[i]; ry[i] = by[i]; }
  rx[4] = rx[0]; ry[4] = ry[0];
  const double x0 = rx[0];
  double p1y = ry[0], p2x = rx[1] - x0, p2y = ry[1], sum = 0.0, p1x;
  for (int i = 1; i < 4; ++i) {
    const double p0y = p1y;
    p1x = p2x; p1y = p2y;
    p2x = rx[i + 1] - x0; p2y = ry[i + 1];
    sum = D_ADD(sum, D_MUL(p1x, D_SUB(p0y, p2y)));
  }
  const double area = fabs(sum / 2.0);
  double len = 0.0;
  for (int i = 1; i < 5; ++i) {
    const double dx = rx[i] - rx[i - 1], dy = ry[i] - ry[i - 1];
    len = D_ADD(len, sqrt(D_ADD(D_MUL(dx, dx), D_MUL(dy, dy))));
  }
  const double delta = D_DIV(D_MUL(area, ratio), len);
  // --- ClipperOffset::AddPath (truncate to cInt, strip duplicates)
  long long cx[4], cy[4];
  int n = 0;
  long long tx[4], ty[4];
  for (int i = 0; i < 4; ++i) { tx[i] = (long long)bx[i]; ty[i] = (long long)by[i]; }
  int high = 3;
  while (high > 0 && tx[0] == tx[high] && ty[0] == ty[high]) --high;
  cx[0] = tx[0]; cy[0] = ty[0]; n = 1;
  for (int i = 1; i <= high; ++i)
    if (cx[n - 1] != tx[i] || cy[n - 1] != ty[i]) { cx[n] = tx[i]; cy[n] = ty[i]; ++n; }
  if (n < 3) return 0;
  // --- FixOrientations: Area(path) >= 0 else reverse
  {
    double a = 0;
    int j = n - 1;
    for (int i = 0; i < n; ++i) {
      a = D_ADD(a, D_MUL(D_ADD((double)cx[j], (double)cx[i]), D_SUB((double)cy[j], (double)cy[i])));
      j = i;
    }
    if (!(-a * 0.5 >= 0)) {
      for (int i = 0; i < n / 2; ++i) {
        long long t = cx[i]; cx[i] = cx[n - 1 - i]; cx[n - 1 - i] = t;
        t = cy[i]; cy[i] = cy[n - 1 - i]; cy[n - 1 - i] = t;
      }
    }
  }
  if (fabs(delta) < 1e-20) {
    int m = 0;
    for (int i = 0; i < n && m < cap; ++i) { out[m].x = (int)cx[i]; out[m].y = (int)cy[i]; ++m; }
    return m;
  }
  // --- DoOffset
  const double ad = fabs(delta);
  double y = 0.25 > ad * 0.25 ? ad * 0.25 : 0.25;  // ArcTolerance 0.25 vs |delta| * def_arc_tolerance
  double steps = D_DIV(kPi, acos(D_SUB(1.0, D_DIV(y, ad))));
  if (steps > ad * kPi) steps = ad * kPi;
  double m_sin = sin(D_DIV(2 * kPi, steps));
  const double m_cos = cos(D_DIV(2 * kPi, steps));
  const double steps_per_rad = D_DIV(steps, 2 * kPi);
  if (delta < 0.0) m_sin = -m_sin;
  double nx[4], ny[4];
  for (int j = 0; j < n; ++j) {
    const int j2 = (j + 1) % n;
    if (cx[j2] == cx[j] && cy[j2] == cy[j]) { nx[j] = 0; ny[j] = 0; continue; }
    double dx = (double)(cx[j2] - cx[j]), dy = (double)(cy[j2] - cy[j]);
    const double f = D_DIV(1.0, sqrt(D_ADD(D_MUL(dx, dx), D_MUL(dy, dy))));
    dx = D_MUL(dx, f);
    dy = D_MUL(dy, f);
    nx[j] = dy;
    ny[j] = -dx;
  }
  int m = 0;
#define CTD_EMIT(X, Y)                                 \
  do {                                                 \
    if (m < cap) { out[m].x = (int)(X); out[m].y = (int)(Y); } \
    ++m;                                               \
  } while (0)
  int k = n - 1;
  for (int j = 0; j < n; ++j) {
    double sin_a = D_SUB(D_MUL(nx[k], ny[j]), D_MUL(nx[j], ny[k]));
    bool done = false;
    if (fabs(D_MUL(sin_a, delta)) < 1.0) {
      const double cos_a = D_ADD(D_MUL(nx[k], nx[j]), D_MUL(ny[j], ny[k]));
      if (cos_a > 0) {
        CTD_EMIT(clip_round(D_ADD((double)cx[j], D_MUL(nx[k], delta))), clip_round(D_ADD((double)cy[j], D_MUL(ny[k], delta))));
        done = true;
      }
    } else if (sin_a > 1.0) sin_a = 1.0;
    else if (sin_a < -1.0) sin_a = -1.0;
    if (!done) {
      if (D_MUL(sin_a, delta) < 0) {
        CTD_EMIT(clip_round(D_ADD((double)cx[j], D_MUL(nx[k], delta))), clip_round(D_ADD((double)cy[j], D_MUL(ny[k], delta))));
        CTD_EMIT(cx[j], cy[j]);
        CTD_EMIT(clip_round(D_ADD((double)cx[j], D_MUL(nx[j], delta))), clip_round(D_ADD((double)cy[j], D_MUL(ny[j], delta))));
      } else {
        const double a = atan2(sin_a, D_ADD(D_MUL(nx[k], nx[j]), D_MUL(ny[k], ny[j])));
        long long st = clip_round(D_MUL(steps_per_rad, fabs(a)));
        if (st < 1) st = 1;
        double X = nx[k], Y = ny[k];
        for (long long i = 0; i < st; ++i) {
          CTD_EMIT(clip_round(D_ADD((double)cx[j], D_MUL(X, delta))), clip_round(D_ADD((double)cy[j], D_MUL(Y, delta))));
          const double X2 = X;
          X = D_SUB(D_MUL(X, m_cos), D_MUL(m_sin, Y));
          Y = D_ADD(D_MUL(X2, m_sin), D_MUL(Y, m_cos));
        }
        CTD_EMIT(clip_round(D_ADD((double)cx[j], D_MUL(nx[j], delta))), clip_round(D_ADD((double)cy[j], D_MUL(ny[j], delta))));
      }
    }
    k = j;
  }
#undef CTD_EMIT
  return m <= cap ? m : -1;
}

// simple in-place sort by (x, y) for the (small) offset point set
CTD_HD void sort_xy(IPt* p, int n) {
  for (int i = 1; i < n; ++i) {
    const IPt v = p[i];
    int j = i - 1;
    while (j >= 0 && (p[j].x > v.x || (p[j].x == v.x && p[j].y > v.y))) { p[j + 1] = p[j]; --j; }
    p[j + 1] = v;
  }
}

// np.round (half to even) on the float32 value, then clip (db_utils.py:162-163)
CTD_HD int16_t quantise(float v, int src_dim, int dst_dim) {
  float t = F_MUL(F_DIV(v, (float)src_dim), (float)dst_dim);
  float r = rintf(t);  // round-half-even in the default rounding mode
  if (r < 0.f) r = 0.f;
  if (r > (float)dst_dim) r = (float)dst_dim;
  return (int16_t)r;
}

// The per-contour chain after the first hull, in two stages so that the CUDA kernel can sort the offset
// points cooperatively in between.  Stage 1: get_mini_boxes + unclip -> number of offset points (0 = the
// contour is skipped: sside < 2 or a degenerate offset).  Stage 2 (points sorted by (x, y)): hull ->
// get_mini_boxes -> quantised int16 box.  hull/tmp: >= kMaxHull entries, off: >= kMaxOffsetPts, f*: >= kMaxHull.
CTD_HD int contour_stage1(IPt* hull, int nh, IPt* tmp, IPt* off, float* f0, float* f1, float* f2, double unclip_ratio) {
  if (nh < 3) return 0;  // minAreaRect of 1-2 points / collinear sets has a zero side -> sside < 2
  hull_start_maxx(hull, nh, tmp);
  const RRect r1 = min_area_rect(hull, nh, f0, f1, f2);
  const float sside = r1.w < r1.h ? r1.w : r1.h;
  if (sside < 2.f) return 0;
  float px[4], py[4], ox[4], oy[4];
  box_points(r1, px, py);
  order_mini_box(px, py, ox, oy);
  const int m = unclip_offset(ox, oy, unclip_ratio, off, kMaxOffsetPts);
  return m < 3 ? 0 : m;
}

CTD_HD bool contour_stage2(IPt* off, int m, IPt* hull, IPt* tmp, float* f0, float* f1, float* f2, int map_w, int map_h,
                           int dst_w, int dst_h, int16_t* box_out /*[8]*/) {
  const int nh2 = hull_sorted(off, m, hull, kMaxHull);
  if (nh2 < 3) return false;
  hull_start_maxx(hull, nh2, tmp);
  const RRect r2 = min_area_rect(hull, nh2, f0, f1, f2);
  float px[4], py[4], ox[4], oy[4];
  box_points(r2, px, py);
  order_mini_box(px, py, ox, oy);
  for (int k = 0; k < 4; ++k) {
    box_out[2 * k] = quantise(ox[k], map_w, dst_w);
    box_out[2 * k + 1] = quantise(oy[k], map_h, dst_h);
  }
  return true;
}

CTD_HD bool contour_to_box(IPt* hull, int nh, IPt* tmp, IPt* off, float* f0, float* f1, float* f2, int map_w, int map_h,
                           int dst_w, int dst_h, double unclip_ratio, int16_t* box_out /*[8]*/) {
  const int m = contour_stage1(hull, nh, tmp, off, f0, f1, f2, unclip_ratio);
  if (m == 0) return false;
  sort_xy(off, m);
  return contour_stage2(off, m, hull, tmp, f0, f1, f2, map_w, map_h, dst_w, dst_h, box_out);
}

}  // namespace ctdgeom
