// Host-side result assembly of the engine: text lines -> text blocks (native C++, C ABI `ctd_group_output`).
//
// Replaces the reference's `group_output` and its callees (utils/textblock.py:421-508 group_output, 302-342
// examine_textblk, 344-373 try_merge_textline, 375-388 merge_textlines, 390-419 split_textblk, 267-300
// sort_textblk_list, 87-106 adjust_bbox / sort_lines; utils/imgproc_utils.py:13-20 union_area).  The stage is a
// serial walk over <= 300 detector boxes and <= 1000 line quads per page whose float64 results are truncated to
// integers, so it runs on the host in IEEE double arithmetic with glibc's acos / sin / atan2 (SURVEY section 7): every
// sum the reference forms over line coordinates is a sum of half-integers and therefore exact in double, independent
// of numpy's reduction order or BLAS's use of FMA.
// shapely's `Polygon.intersects` (closed-set intersection of two quads) is an exact integer predicate here.
//
// Data model: a block is a struct of scalars plus a list of 4-point lines and a list of per-line distances (the
// reference's python lists / numpy arrays); the result is flattened into caller-provided arrays (ctd_b200.h).
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <array>
#include <vector>

#include "../../include/ctd_b200.h"

namespace {

typedef std::array<int64_t, 8> Quad;   // x0,y0 .. x3,y3

struct Block {
  int64_t xyxy[4] = {0, 0, 0, 0};
  std::vector<Quad> lines;
  std::vector<double> distance;
  int language = 2;
  bool vertical = false;
  double font_size = -1;
  int angle = 0;
  double vec[2] = {0, 0};
  double norm = -1;
  bool merged = false;
  bool font_is_float = false;   // python: font_size is an int until a merge averages it (json writes 23 vs 23.0)
  double weight = -1;
};

// ---- exact predicates on integer quads ----------------------------------------------------------------
inline int orient(const int64_t* a, const int64_t* b, const int64_t* c) {
  const int64_t v = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]);
  return (v > 0) - (v < 0);
}
inline bool in_box(const int64_t* a, const int64_t* b, const int64_t* p) {
  return std::min(a[0], b[0]) <= p[0] && p[0] <= std::max(a[0], b[0]) && std::min(a[1], b[1]) <= p[1] &&
         p[1] <= std::max(a[1], b[1]);
}
bool segments_touch(const int64_t* a, const int64_t* b, const int64_t* c, const int64_t* d) {
  const int o1 = orient(a, b, c), o2 = orient(a, b, d), o3 = orient(c, d, a), o4 = orient(c, d, b);
  if (o1 != o2 && o3 != o4) return true;
  return (o1 == 0 && in_box(a, b, c)) || (o2 == 0 && in_box(a, b, d)) || (o3 == 0 && in_box(c, d, a)) ||
         (o4 == 0 && in_box(c, d, b));
}
bool inside_or_on(const int64_t* p, const Quad& q) {
  bool inside = false;
  for (int i = 0; i < 4; ++i) {
    const int64_t* a = &q[2 * i];
    const int64_t* b = &q[2 * ((i + 1) & 3)];
    if (orient(a, b, p) == 0 && in_box(a, b, p)) return true;
    if ((a[1] > p[1]) != (b[1] > p[1])) {
      const int64_t t = (b[0] - a[0]) * (p[1] - a[1]) - (p[0] - a[0]) * (b[1] - a[1]);
      if (t != 0 && ((t > 0) == (b[1] > a[1]))) inside = !inside;
    }
  }
  return inside;
}
// closed-set intersection of two simple quads (what shapely's Polygon.intersects answers for valid rings)
bool quads_intersect(const Quad& a, const Quad& b) {
  int64_t ax0 = a[0], ax1 = a[0], ay0 = a[1], ay1 = a[1], bx0 = b[0], bx1 = b[0], by0 = b[1], by1 = b[1];
  for (int i = 1; i < 4; ++i) {
    ax0 = std::min(ax0, a[2 * i]); ax1 = std::max(ax1, a[2 * i]);
    ay0 = std::min(ay0, a[2 * i + 1]); ay1 = std::max(ay1, a[2 * i + 1]);
    bx0 = std::min(bx0, b[2 * i]); bx1 = std::max(bx1, b[2 * i]);
    by0 = std::min(by0, b[2 * i + 1]); by1 = std::max(by1, b[2 * i + 1]);
  }
  if (ax1 < bx0 || bx1 < ax0 || ay1 < by0 || by1 < ay0) return false;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j)
      if (segments_touch(&a[2 * i], &a[2 * ((i + 1) & 3)], &b[2 * j], &b[2 * ((j + 1) & 3)])) return true;
  return inside_or_on(&a[0], b) || inside_or_on(&b[0], a);
}

// ---- numpy / python semantics ---------------------------------------------------------------------------
// python slice bounds a[lo:hi] on an axis of length n
inline void py_slice(int64_t& lo, int64_t& hi, int64_t n) {
  if (lo < 0) lo = std::max<int64_t>(lo + n, 0);
  if (hi < 0) hi = std::max<int64_t>(hi + n, 0);
  lo = std::min(lo, n);
  hi = std::min(hi, n);
  if (hi < lo) hi = lo;
}
// mask[y1:y2, x1:x2].mean() / 255  (NaN for an empty slice, like numpy)
double mask_score(const uint8_t* mask, int im_w, int im_h, int64_t x1, int64_t y1, int64_t x2, int64_t y2) {
  py_slice(y1, y2, im_h);
  py_slice(x1, x2, im_w);
  const int64_t cnt = (y2 - y1) * (x2 - x1);
  if (cnt <= 0) return NAN;
  uint64_t sum = 0;
  for (int64_t y = y1; y < y2; ++y) {
    const uint8_t* r = mask + size_t(y) * im_w;
    uint64_t s = 0;
    for (int64_t x = x1; x < x2; ++x) s += r[x];
    sum += s;
  }
  return double(sum) / double(cnt) / 255.0;
}
// imgproc_utils.py:13-20 (the INTERSECTION area; -1 when the boxes are disjoint)
inline int64_t union_area(const int64_t* a, const int64_t* b) {
  const int64_t x1 = std::max(a[0], b[0]), y1 = std::max(a[1], b[1]);
  const int64_t x2 = std::min(a[2], b[2]), y2 = std::min(a[3], b[3]);
  if (y2 < y1 || x2 < x1) return -1;
  return (y2 - y1) * (x2 - x1);
}
inline double py_round(double v) { return nearbyint(v); }   // round-half-even (default FP environment)

void adjust_bbox(Block& b, bool with_bbox) {   // textblock.py:87-98
  int64_t lo_x = INT64_MAX, lo_y = INT64_MAX, hi_x = INT64_MIN, hi_y = INT64_MIN;
  for (const Quad& q : b.lines)
    for (int i = 0; i < 4; ++i) {
      lo_x = std::min(lo_x, q[2 * i]); hi_x = std::max(hi_x, q[2 * i]);
      lo_y = std::min(lo_y, q[2 * i + 1]); hi_y = std::max(hi_y, q[2 * i + 1]);
    }
  if (with_bbox) {
    b.xyxy[0] = std::min(lo_x, b.xyxy[0]); b.xyxy[1] = std::min(lo_y, b.xyxy[1]);
    b.xyxy[2] = std::max(hi_x, b.xyxy[2]); b.xyxy[3] = std::max(hi_y, b.xyxy[3]);
  } else {
    b.xyxy[0] = lo_x; b.xyxy[1] = lo_y; b.xyxy[2] = hi_x; b.xyxy[3] = hi_y;
  }
}

// examine_textblk (textblock.py:302-342): reading direction, angle, font size, distance of every line to the origin
void examine(Block& b, int im_w, int /*im_h*/, bool sort) {
  const size_t n = b.lines.size();
  double v[2] = {0, 0}, h[2] = {0, 0};
  std::vector<double> cx(n), cy(n);
  for (size_t i = 0; i < n; ++i) {
    const Quad& q = b.lines[i];
    double mx[4], my[4];
    for (int k = 0; k < 4; ++k) {   // middle_pnts = (lines[:, [1,2,3,0]] + lines) / 2
      mx[k] = (double(q[2 * ((k + 1) & 3)]) + double(q[2 * k])) / 2;
      my[k] = (double(q[2 * ((k + 1) & 3) + 1]) + double(q[2 * k + 1])) / 2;
    }
    v[0] += mx[2] - mx[0]; v[1] += my[2] - my[0];
    h[0] += mx[1] - mx[3]; h[1] += my[1] - my[3];
    cx[i] = (double(q[0]) + double(q[4])) / 2;
    cy[i] = (double(q[1]) + double(q[5])) / 2;
  }
  const double norm_v = sqrt(v[0] * v[0] + v[1] * v[1]), norm_h = sqrt(h[0] * h[0] + h[1] * h[1]);
  const bool vertical = b.language == 1 ? norm_v > norm_h : norm_v > norm_h * 2;
  double pv[2], pn, ox, font;
  if (vertical) {
    pv[0] = v[0]; pv[1] = v[1]; pn = norm_v; ox = double(im_w);   // vertical text is read right to left
    font = py_round(norm_h / double(n));
  } else {
    pv[0] = h[0]; pv[1] = h[1]; pn = norm_h; ox = 0;
    font = py_round(norm_v / double(n));
  }
  int angle = int(atan2(pv[1], pv[0]) / M_PI * 180);
  b.distance.resize(n);
  for (size_t i = 0; i < n; ++i) {
    const double dx = cx[i] - ox, dy = cy[i];
    const double d = sqrt(dx * dx + dy * dy);
    const double rad = acos((dx * pv[0] + dy * pv[1]) / (d * pn));
    b.distance[i] = fabs(sin(rad) * d);
  }
  if (vertical) angle -= 90;
  if (abs(angle) < 3) angle = 0;
  b.angle = angle;
  b.font_size = font;
  b.vertical = vertical;
  b.vec[0] = pv[0]; b.vec[1] = pv[1];
  b.norm = pn;
  if (sort) {   // sort_lines (textblock.py:100-105): argsort of the distances, NaN last
    std::vector<int> idx(n);
    for (size_t i = 0; i < n; ++i) idx[i] = int(i);
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int c) {
      const double da = b.distance[a], dc = b.distance[c];
      if (isnan(da)) return false;
      if (isnan(dc)) return true;
      return da < dc;
    });
    std::vector<Quad> l2(n);
    std::vector<double> d2(n);
    for (size_t i = 0; i < n; ++i) { l2[i] = b.lines[idx[i]]; d2[i] = b.distance[idx[i]]; }
    b.lines.swap(l2);
    b.distance.swap(d2);
  }
}

// try_merge_textline (textblock.py:344-373)
bool try_merge(Block& a, Block& o) {
  if (o.merged) return false;
  const double fntsize_tol = 1.3, distance_tol = 2;
  const double div = a.font_size / o.font_size;
  const double n1 = double(a.lines.size()), n2 = double(o.lines.size());
  const double avg = (a.font_size * n1 + o.font_size * n2) / (n1 + n2);
  const double prod = a.vec[0] * o.vec[0] + a.vec[1] * o.vec[1];
  const double sum[2] = {a.vec[0] + o.vec[0], a.vec[1] + o.vec[1]};
  const double cosv = prod / a.norm / o.norm;
  const double gap = o.distance.back() - a.distance.back();
  const Quad& la = a.lines.back();
  const Quad& lo = o.lines.back();
  const double px = double(lo[0] - la[0]), py = double(lo[1] - la[1]);
  const double gap_p1 = sqrt(px * px + py * py);
  if (!quads_intersect(la, lo)) {
    if (div > fntsize_tol || 1 / div > fntsize_tol) return false;
    if (fabs(cosv) < 0.866) return false;   // cos 30
    if (gap > distance_tol * avg || gap_p1 > avg * 2.5) return false;
  }
  a.lines.push_back(o.lines.front());
  a.vec[0] = sum[0]; a.vec[1] = sum[1];
  a.angle = int(py_round(atan2(sum[1], sum[0]) * (180.0 / M_PI)));
  if (a.vertical) a.angle -= 90;
  a.norm = sqrt(sum[0] * sum[0] + sum[1] * sum[1]);
  a.distance.push_back(o.distance.back());
  a.font_size = avg;
  a.font_is_float = true;
  o.merged = true;
  return true;
}

// merge_textlines (textblock.py:375-388)
void merge_scattered(std::vector<Block>& blks, std::vector<Block>& out) {
  if (blks.size() < 2) {
    for (Block& b : blks) out.push_back(std::move(b));
    return;
  }
  std::stable_sort(blks.begin(), blks.end(), [](const Block& a, const Block& c) { return a.distance[0] < c.distance[0]; });
  std::vector<size_t> kept;
  for (size_t i = 0; i < blks.size(); ++i) {
    if (blks[i].merged) continue;
    for (size_t j = i + 1; j < blks.size(); ++j) try_merge(blks[i], blks[j]);
    kept.push_back(i);
  }
  for (size_t i : kept) {
    adjust_bbox(blks[i], false);
    out.push_back(std::move(blks[i]));
  }
}

// split_textblk (textblock.py:390-419); returns true when the block was split into several
bool split_block(Block& blk, std::vector<Block>& parts) {
  const double font_size = blk.font_size;
  const Quad first = blk.lines[0];
  // lines.sort(key = |line[0] - l0[0]|): python's sort is stable; the distances keep their old order
  std::vector<double> key(blk.lines.size());
  for (size_t i = 0; i < blk.lines.size(); ++i) {
    const double dx = double(blk.lines[i][0] - first[0]), dy = double(blk.lines[i][1] - first[1]);
    key[i] = sqrt(dx * dx + dy * dy);
  }
  std::vector<int> idx(blk.lines.size());
  for (size_t i = 0; i < idx.size(); ++i) idx[i] = int(i);
  std::stable_sort(idx.begin(), idx.end(), [&](int a, int c) { return key[a] < key[c]; });
  std::vector<Quad> lines(blk.lines.size());
  for (size_t i = 0; i < idx.size(); ++i) lines[i] = blk.lines[idx[i]];
  blk.lines = lines;
  const double tol = font_size * 2;
  Block cur = blk;
  cur.lines.assign(1, first);
  parts.clear();
  parts.push_back(cur);
  for (size_t j = 0; j + 1 < lines.size(); ++j) {
    const Quad& prev = lines[j];
    const Quad& line = lines[j + 1];
    bool split = false;
    if (!quads_intersect(prev, line)) {
      const double d = fabs(blk.distance[j + 1] - blk.distance[j]);
      if (d > tol) {
        split = true;
      } else if (blk.vertical && abs(blk.angle) < 15) {
        if (parts.back().lines.size() > 1 || d > font_size)
          split = double(llabs(prev[1] - line[1])) > font_size;
      }
    }
    if (split) {
      Block nb = parts.back();
      nb.lines.assign(1, line);
      parts.push_back(nb);
    } else {
      parts.back().lines.push_back(line);
    }
  }
  if (parts.size() > 1) {
    for (Block& p : parts) adjust_bbox(p, false);
    return true;
  }
  return false;
}

// sort_textblk_list (textblock.py:267-300): 4 x 3 reading grid, right to left when Japanese blocks dominate
void reading_order(std::vector<Block>& blks, int im_w_i, int im_h_i) {
  if (blks.empty()) return;
  size_t n_ja = 0;
  for (const Block& b : blks) n_ja += b.language == 1;
  const bool flip = double(n_ja) > double(blks.size()) / 2;
  const double full_w = im_w_i, im_h = im_h_i;
  double im_w = im_w_i;
  const bool halved = im_w_i > im_h_i;
  if (halved) im_w /= 2;
  const double gy = 4, gx = 3;
  const double area = im_h * im_w;
  for (Block& b : blks) {
    double cx = double(b.xyxy[0] + b.xyxy[2]) / 2;
    if (flip) cx = halved ? full_w - cx : im_w - cx;
    const int32_t col = int32_t(cx / im_w * gx);
    const double cy = double(b.xyxy[1] + b.xyxy[3]) / 2;
    const int32_t row = int32_t(cy / im_h * gy);
    const double cell = double(row) * gx + double(col);
    double w = cell * area + 1.2 * (cx - double(col) * im_w / gx) + (cy - double(row) * im_h / gy);
    if (halved && col >= 3) w += area * gy * gx;
    b.weight = w;
  }
  std::stable_sort(blks.begin(), blks.end(), [](const Block& a, const Block& c) { return a.weight < c.weight; });
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------
extern "C" int ctd_group_output(const int32_t* blk_xyxy, const int32_t* blk_cls, int32_t n_blk, const int32_t* lines,
                                int32_t n_lines, int32_t im_w, int32_t im_h, const uint8_t* mask, int32_t sort_blklist,
                                ctd_block* blocks_out, int32_t blocks_cap, int32_t* lines_out, int32_t lines_cap,
                                double* dist_out, int32_t dist_cap, int32_t* n_blocks_out) {
  if (!n_blocks_out || n_blk < 0 || n_lines < 0 || im_w < 1 || im_h < 1 || (n_blk > 0 && (!blk_xyxy || !blk_cls)) ||
      (n_lines > 0 && !lines))
    return CTD_E_INVALID;
  *n_blocks_out = 0;
  std::vector<Block> blk_list, loose_hor, loose_ver, final_list;
  blk_list.resize(size_t(n_blk));
  for (int i = 0; i < n_blk; ++i) {
    for (int k = 0; k < 4; ++k) blk_list[i].xyxy[k] = blk_xyxy[4 * i + k];
    const int c = blk_cls[i];
    blk_list[i].language = (c >= 0 && c <= 2) ? c : 2;
  }
  // step 1: every line goes to the detector box covering most of it, or becomes a scattered line
  const double bbox_score_thresh = 0.4, mask_score_thresh = 0.1;
  for (int li = 0; li < n_lines; ++li) {
    Quad q;
    for (int k = 0; k < 8; ++k) q[k] = lines[8 * li + k];
    int64_t bx1 = q[0], bx2 = q[0], by1 = q[1], by2 = q[1];
    for (int k = 1; k < 4; ++k) {
      bx1 = std::min(bx1, q[2 * k]); bx2 = std::max(bx2, q[2 * k]);
      by1 = std::min(by1, q[2 * k + 1]); by2 = std::max(by2, q[2 * k + 1]);
    }
    const int64_t lbox[4] = {bx1, by1, bx2, by2};
    const double line_area = double((by2 - by1) * (bx2 - bx1));
    double best = -1;
    int best_i = -1;
    for (int j = 0; j < n_blk; ++j) {
      const double score = double(union_area(blk_list[j].xyxy, lbox)) / line_area;   // +-inf / NaN when the area is 0
      if (best < score) { best = score; best_i = j; }
    }
    if (best > bbox_score_thresh) {
      blk_list[best_i].lines.push_back(q);
      continue;
    }
    if (mask != nullptr && mask_score(mask, im_w, im_h, bx1, by1, bx2, by2) < mask_score_thresh) continue;
    Block single;
    single.xyxy[0] = bx1; single.xyxy[1] = by1; single.xyxy[2] = bx2; single.xyxy[3] = by2;
    single.lines.push_back(q);
    examine(single, im_w, im_h, false);
    (single.vertical ? loose_ver : loose_hor).push_back(std::move(single));
  }
  // step 2: per detector box -- drop empty boxes over little mask, measure, split manga columns at distance gaps
  for (Block& blk : blk_list) {
    if (blk.lines.empty()) {
      const int64_t* b = blk.xyxy;
      if (mask != nullptr && mask_score(mask, im_w, im_h, b[0], b[1], b[2], b[3]) < mask_score_thresh) continue;
      blk.lines.push_back(Quad{b[0], b[1], b[2], b[1], b[2], b[3], b[0], b[3]});   // xywh2xyxypoly
    }
    examine(blk, im_w, im_h, true);
    const bool want_split = blk.lines.size() > 1 && (blk.language == 1 || blk.vertical);
    std::vector<Block> parts;
    bool did_split = false;
    if (want_split) did_split = split_block(blk, parts);
    else parts.push_back(blk);
    if (!did_split)
      for (Block& p : parts) adjust_bbox(p, true);
    for (Block& p : parts) final_list.push_back(std::move(p));
  }
  // step 3: merge the scattered lines, then order the page
  merge_scattered(loose_hor, final_list);
  merge_scattered(loose_ver, final_list);
  if (sort_blklist) reading_order(final_list, im_w, im_h);
  for (Block& b : final_list) {
    if (b.language == 0 && !b.vertical) {
      if (b.lines.empty()) continue;
      const int expand = std::max(int(b.font_size * 0.1), 2);
      const double rad = double(b.angle) * (M_PI / 180.0);
      static const int sgn[4][2] = {{-1, -1}, {1, -1}, {1, 1}, {-1, 1}};
      for (Quad& q : b.lines)
        for (int k = 0; k < 4; ++k) {
          double x = double(q[2 * k]) + double(sgn[k][0]) * sin(rad) * double(expand);
          double y = double(q[2 * k + 1]) + double(sgn[k][1]) * cos(rad) * double(expand);
          x = std::min(std::max(x, 0.0), double(im_w - 1));
          y = std::min(std::max(y, 0.0), double(im_h - 1));
          q[2 * k] = int64_t(x);
          q[2 * k + 1] = int64_t(y);
        }
      b.font_size += expand;
    }
  }
  // flatten
  size_t tl = 0, td = 0;
  for (const Block& b : final_list) { tl += b.lines.size(); td += b.distance.size(); }
  *n_blocks_out = int32_t(final_list.size());
  if (int64_t(final_list.size()) > blocks_cap || int64_t(tl) > lines_cap || int64_t(td) > dist_cap) return CTD_E_CAPACITY;
  if ((!blocks_out && !final_list.empty()) || (!lines_out && tl) || (!dist_out && td)) return CTD_E_INVALID;
  size_t lo = 0, d0 = 0;
  for (size_t i = 0; i < final_list.size(); ++i) {
    const Block& b = final_list[i];
    ctd_block& o = blocks_out[i];
    for (int k = 0; k < 4; ++k) o.xyxy[k] = int32_t(b.xyxy[k]);
    o.language = b.language;
    o.vertical = b.vertical ? 1 : 0;
    o.angle = b.angle;
    o.merged = b.merged ? 1 : 0;
    o.font_is_float = b.font_is_float ? 1 : 0;
    o.n_lines = int32_t(b.lines.size());
    o.line_off = int32_t(lo);
    o.n_dist = int32_t(b.distance.size());
    o.dist_off = int32_t(d0);
    o.font_size = b.font_size;
    o.vec[0] = b.vec[0]; o.vec[1] = b.vec[1];
    o.norm = b.norm;
    o.weight = b.weight;
    for (const Quad& q : b.lines) {
      for (int k = 0; k < 8; ++k) lines_out[8 * lo + k] = int32_t(q[k]);
      ++lo;
    }
    for (double d : b.distance) dist_out[d0++] = d;
  }
  return CTD_OK;
}
