// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_orb.cpp header for the rules).
//
// CPU restatement of the reference's line-feature extraction path:
//   LINEextractor::operator()             src/LineExtractor.cpp:26-93
//   LSDDetector::detect / detectImpl      opencv_contrib line_descriptor (not vendored); spec copy
//                                         Thirdparty/line_descriptor/src/LSDDetector_custom.cpp:56-215
//   cv::createLineSegmentDetector()       OpenCV imgproc lsd.cpp (not vendored): restated from the published LSD
//                                         algorithm (von Gioi et al.) as OpenCV implements it, defaults
//                                         REFINE_STD, scale 0.8, sigma_scale 0.6, quant 2, ang_th 22.5, density 0.7,
//                                         1024 bins.  PINNED end-to-end against cv2 4.13 (tests/test_oracle_line.py
//                                         + tests/golden/lsd_cv2_*.npz): identical segment lists.
//   BinaryDescriptor::compute (LBD)       spec copy Thirdparty/line_descriptor/src/binary_descriptor_custom.cpp
//                                         :74-116 (band pairs), :217-259 (weights), :350-398 (blur+Sobel),
//                                         :539-687 (computeImpl), :1026-1372 (computeLBD)
// Parity status: LSD PINNED end to end to cv2 4.13; LBD, the KeyLine conversion and LINEextractor's selection are PARITY
// UNPINNED (opencv_contrib's line_descriptor is not installed; they follow the vendored spec copy line by line).
// Seed ordering: OpenCV 4.13's ll_angle orders the pixels by gradient bin such that equal bins keep row-major pixel
// order (a stable ordering).  order_mode 1 (the default, std::stable_sort) reproduces cv2's segment lists exactly and is
// what the GPU path implements; order_mode 0 (an unstable std::sort on the same records) is kept only to show that it
// does NOT reproduce cv2.  See DESIGN.md §2.
// Other fixed choices: the KeyLine that LineExtractor.cpp:64 appends through resize() is value-initialised
// (all zero) here — in the reference its fields are indeterminate; lines of equal response keep detection order
// (the reference's std::sort is unstable there too); 0 detected lines -> 1 zero KeyLine (the reference reads
// _keylines[-1]).

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {
const double NOTDEF = -1024.0, M_3_2_PI_ = (3 * 3.14159265358979323846) / 2, M_2__PI_ = 2 * 3.14159265358979323846;
const double DEG_TO_RADS = 3.14159265358979323846 / 180;
const double PI_ = 3.14159265358979323846;
const uint8_t USED = 1, NOTUSED = 0;

inline int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) { if (p < 0) p = -p; else p = 2 * (n - 1) - p; }
  return p;
}
float fast_atan2(float y, float x) {  // cv::fastAtan2 (pinned in tests/test_oracle_orb.py)
  const float k = (float)(180.0 / 3.14159265358979323846);
  const float p1 = 0.9997878412794807f * k, p3 = -0.3258083974640975f * k;
  const float p5 = 0.1555786518463281f * k, p7 = -0.04432655554792128f * k;
  float ax = std::fabs(x), ay = std::fabs(y), a, c, c2;
  if (ax >= ay) { c = ay / (ax + (float)DBL_EPSILON); c2 = c * c; a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c; }
  else { c = ax / (ay + (float)DBL_EPSILON); c2 = c * c; a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c; }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}
void blur_sep_u8(const uint8_t* src, int w, int h, uint8_t* dst, const int* taps, int ksize) {  // 8.8 fixed point
  int r = ksize / 2;
  std::vector<uint16_t> tmp((size_t)w * h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      int s = 0;
      for (int k = -r; k <= r; k++) s += src[(size_t)y * w + reflect101(x + k, w)] * taps[k + r];
      tmp[(size_t)y * w + x] = (uint16_t)s;
    }
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      uint32_t s = 0;
      for (int k = -r; k <= r; k++) s += (uint32_t)tmp[(size_t)reflect101(y + k, h) * w + x] * taps[k + r];
      dst[(size_t)y * w + x] = (uint8_t)((s + 32768u) >> 16);
    }
}
// cv::resize(..., fx=fy=0.8, INTER_LINEAR_EXACT) for 8U: source coordinate (d+0.5)*1.25-0.5, 8-bit weights
void resize_08_exact(const uint8_t* src, int sw, int sh, std::vector<uint8_t>& dst, int& dw, int& dh) {
  dw = (int)lrint(sw * 0.8); dh = (int)lrint(sh * 0.8);
  dst.assign((size_t)dw * dh, 0);
  std::vector<int> xo(dw), xf(dw), yo(dh), yf(dh);
  auto coef = [](int s, int d, std::vector<int>& o, std::vector<int>& f) {
    for (int i = 0; i < d; i++) {
      double fx = (i + 0.5) * 1.25 - 0.5;
      int si = (int)std::floor(fx);
      double fr = fx - si;
      if (si < 0) { si = 0; fr = 0; }
      if (si >= s - 1) { si = s - 1; fr = 0; }
      o[i] = si; f[i] = (int)std::floor(fr * 256 + 0.5);
    }
  };
  coef(sw, dw, xo, xf); coef(sh, dh, yo, yf);
  std::vector<int> h0(dw), h1(dw);
  for (int y = 0; y < dh; y++) {
    const uint8_t* r0 = src + (size_t)yo[y] * sw;
    const uint8_t* r1 = src + (size_t)std::min(yo[y] + 1, sh - 1) * sw;
    for (int x = 0; x < dw; x++) {
      int a = xo[x], b = std::min(xo[x] + 1, sw - 1);
      h0[x] = r0[a] * (256 - xf[x]) + r0[b] * xf[x];
      h1[x] = r1[a] * (256 - xf[x]) + r1[b] * xf[x];
      dst[(size_t)y * dw + x] = (uint8_t)((h0[x] * (256 - yf[y]) + h1[x] * yf[y] + 32768) >> 16);
    }
  }
}

// ---------------------------------------------------------------------------------------------- LSD
struct RegionPoint { int x, y; double angle, modgrad; };
struct Rect { double x1, y1, x2, y2, width, x, y, theta, dx, dy, prec, p; };
struct NormPoint { int px, py, norm; };

thread_local long g_stat[8] = {0};  // debug statistics: region_grow calls, points added, regions >= min size, refine regrows, ...

// what region_grow adds to its float sums per pixel: lsd.cpp's  sumdx += cos(float(angle))  read three ways
enum { kAddCosf = 0, kAddCosRounded = 1, kAddCosDouble = 2 };

struct Lsd {
  int w = 0, h = 0, order_mode = 0, addend = kAddCosf;
  std::vector<uint8_t> scaled, used;
  std::vector<double> angles, modgrad;
  std::vector<NormPoint> ordered;

  static inline double dist(double x1, double y1, double x2, double y2) { return std::sqrt((x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1)); }
  static inline double distSq(double x1, double y1, double x2, double y2) { return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1); }
  static inline double angle_diff_signed(double a, double b) {
    double diff = a - b;
    while (diff <= -PI_) diff += M_2__PI_;
    while (diff > PI_) diff -= M_2__PI_;
    return diff;
  }
  static inline double angle_diff(double a, double b) { return std::fabs(angle_diff_signed(a, b)); }

  void ll_angle(double threshold, unsigned n_bins) {
    angles.assign((size_t)w * h, NOTDEF);
    modgrad.assign((size_t)w * h, 0.0);
    double max_grad = -1;
    for (int y = 0; y < h - 1; ++y)
      for (int x = 0; x < w - 1; ++x) {
        const uint8_t* r = &scaled[(size_t)y * w];
        const uint8_t* n = &scaled[(size_t)(y + 1) * w];
        int DA = n[x + 1] - r[x], BC = r[x + 1] - n[x];
        int gx = DA + BC, gy = DA - BC;
        double norm = std::sqrt((gx * gx + gy * gy) / 4.0);
        modgrad[(size_t)y * w + x] = norm;
        if (norm <= threshold) angles[(size_t)y * w + x] = NOTDEF;
        else {
          angles[(size_t)y * w + x] = fast_atan2(float(gx), float(-gy)) * DEG_TO_RADS;
          if (norm > max_grad) max_grad = norm;
        }
      }
    double bin_coef = (max_grad > 0) ? double(n_bins - 1) / max_grad : 0;
    ordered.clear();
    ordered.reserve((size_t)w * h);
    for (int y = 0; y < h - 1; ++y)
      for (int x = 0; x < w - 1; ++x) {
        NormPoint p;
        p.px = x; p.py = y; p.norm = int(modgrad[(size_t)y * w + x] * bin_coef);
        ordered.push_back(p);
      }
    auto cmp = [](const NormPoint& a, const NormPoint& b) { return a.norm > b.norm; };
    if (order_mode == 0) std::sort(ordered.begin(), ordered.end(), cmp);
    else std::stable_sort(ordered.begin(), ordered.end(), cmp);
  }

  inline bool isAligned(int x, int y, double theta, double prec) const {
    if (x < 0 || y < 0 || x >= w || y >= h) return false;
    const double a = angles[(size_t)y * w + x];
    if (a == NOTDEF) return false;
    double n_theta = theta - a;
    if (n_theta < 0) n_theta = -n_theta;
    if (n_theta > M_3_2_PI_) { n_theta -= M_2__PI_; if (n_theta < 0) n_theta = -n_theta; }
    return n_theta <= prec;
  }

  void region_grow(int sx, int sy, std::vector<RegionPoint>& reg, double& reg_angle, double prec) {
    reg.clear();
    g_stat[0]++;
    RegionPoint seed;
    seed.x = sx; seed.y = sy;
    reg_angle = angles[(size_t)sy * w + sx];
    seed.angle = reg_angle; seed.modgrad = modgrad[(size_t)sy * w + sx];
    reg.push_back(seed);
    float sumdx = float(std::cos(reg_angle)), sumdy = float(std::sin(reg_angle));
    used[(size_t)sy * w + sx] = USED;
    for (size_t i = 0; i < reg.size(); i++) {
      const int rx = reg[i].x, ry = reg[i].y;
      int xx_min = std::max(rx - 1, 0), xx_max = std::min(rx + 1, w - 1);
      int yy_min = std::max(ry - 1, 0), yy_max = std::min(ry + 1, h - 1);
      for (int yy = yy_min; yy <= yy_max; ++yy)
        for (int xx = xx_min; xx <= xx_max; ++xx) {
          uint8_t& is_used = used[(size_t)yy * w + xx];
          if (is_used != USED && isAligned(xx, yy, reg_angle, prec)) {
            const double angle = angles[(size_t)yy * w + xx];
            is_used = USED;
            RegionPoint rp;
            rp.x = xx; rp.y = yy; rp.modgrad = modgrad[(size_t)yy * w + xx]; rp.angle = angle;
            reg.push_back(rp);
            g_stat[1]++;
            // lsd.cpp adds cos(float(angle)), sin(float(angle)).  kAddCosf (the default): <cmath>'s float overloads, libm's cosf /
            // sinf; kAddCosRounded: the fp64 functions rounded to fp32; kAddCosDouble: ::cos(double) added in fp64 to the float sum.
            // They differ in the last bit on 1.3 % of the gradients; tests/test_oracle_lsd_knife_edge.py holds cv2 to kAddCosf on
            // images where the three give different segment lists (tools/gen_lsd_knife_edge.py)
            const float af = float(angle);
            if (addend == kAddCosf) { sumdx += cosf(af); sumdy += sinf(af); }
            else if (addend == kAddCosRounded) { sumdx += float(std::cos(double(af))); sumdy += float(std::sin(double(af))); }
            else { sumdx = float(double(sumdx) + std::cos(double(af))); sumdy = float(double(sumdy) + std::sin(double(af))); }
            reg_angle = fast_atan2(sumdy, sumdx) * DEG_TO_RADS;
          }
        }
    }
  }

  double get_theta(const std::vector<RegionPoint>& reg, double x, double y, double reg_angle, double prec) const {
    double Ixx = 0.0, Iyy = 0.0, Ixy = 0.0;
    for (size_t i = 0; i < reg.size(); ++i) {
      const double regx = reg[i].x, regy = reg[i].y, weight = reg[i].modgrad;
      double dx = regx - x, dy = regy - y;
      Ixx += dy * dy * weight;
      Iyy += dx * dx * weight;
      Ixy -= dx * dy * weight;
    }
    double lambda = 0.5 * (Ixx + Iyy - std::sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
    double theta = (std::fabs(Ixx) > std::fabs(Iyy)) ? double(fast_atan2(float(lambda - Ixx), float(Ixy)))
                                                     : double(fast_atan2(float(Ixy), float(lambda - Iyy)));
    theta *= DEG_TO_RADS;
    if (angle_diff(theta, reg_angle) > prec) theta += PI_;
    return theta;
  }

  void region2rect(const std::vector<RegionPoint>& reg, double reg_angle, double prec, double p, Rect& rec) const {
    double x = 0, y = 0, sum = 0;
    for (size_t i = 0; i < reg.size(); ++i) {
      const double weight = reg[i].modgrad;
      x += double(reg[i].x) * weight;
      y += double(reg[i].y) * weight;
      sum += weight;
    }
    x /= sum; y /= sum;
    double theta = get_theta(reg, x, y, reg_angle, prec);
    double dx = std::cos(theta), dy = std::sin(theta);
    double l_min = 0, l_max = 0, w_min = 0, w_max = 0;
    for (size_t i = 0; i < reg.size(); ++i) {
      double regdx = double(reg[i].x) - x, regdy = double(reg[i].y) - y;
      double l = regdx * dx + regdy * dy;
      double ww = -regdx * dy + regdy * dx;
      if (l > l_max) l_max = l; else if (l < l_min) l_min = l;
      if (ww > w_max) w_max = ww; else if (ww < w_min) w_min = ww;
    }
    rec.x1 = x + l_min * dx; rec.y1 = y + l_min * dy;
    rec.x2 = x + l_max * dx; rec.y2 = y + l_max * dy;
    rec.width = w_max - w_min;
    rec.x = x; rec.y = y; rec.theta = theta; rec.dx = dx; rec.dy = dy; rec.prec = prec; rec.p = p;
    if (rec.width < 1.0) rec.width = 1.0;
  }

  bool reduce_region_radius(std::vector<RegionPoint>& reg, double reg_angle, double prec, double p, Rect& rec,
                            double density, double density_th) {
    double xc = double(reg[0].x), yc = double(reg[0].y);
    double radSq1 = distSq(xc, yc, rec.x1, rec.y1), radSq2 = distSq(xc, yc, rec.x2, rec.y2);
    double radSq = radSq1 > radSq2 ? radSq1 : radSq2;
    while (density < density_th) {
      radSq *= 0.75 * 0.75;
      for (size_t i = 0; i < reg.size(); ++i) {
        if (distSq(xc, yc, double(reg[i].x), double(reg[i].y)) > radSq) {
          used[(size_t)reg[i].y * w + reg[i].x] = NOTUSED;
          std::swap(reg[i], reg[reg.size() - 1]);
          reg.pop_back();
          --i;
        }
      }
      if (reg.size() < 2) return false;
      region2rect(reg, reg_angle, prec, p, rec);
      density = double(reg.size()) / (dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
    }
    return true;
  }

  bool refine(std::vector<RegionPoint>& reg, double reg_angle, double prec, double p, Rect& rec, double density_th) {
    double density = double(reg.size()) / (dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
    if (density >= density_th) return true;
    double xc = double(reg[0].x), yc = double(reg[0].y);
    const double ang_c = reg[0].angle;
    double sum = 0, s_sum = 0;
    int n = 0;
    for (size_t i = 0; i < reg.size(); ++i) {
      used[(size_t)reg[i].y * w + reg[i].x] = NOTUSED;
      if (dist(xc, yc, reg[i].x, reg[i].y) < rec.width) {
        double ang_d = angle_diff_signed(reg[i].angle, ang_c);
        sum += ang_d; s_sum += ang_d * ang_d; ++n;
      }
    }
    double mean_angle = sum / double(n);
    g_stat[3]++;
    double tau = 2.0 * std::sqrt((s_sum - 2.0 * mean_angle * sum) / double(n) + mean_angle * mean_angle);
    region_grow(reg[0].x, reg[0].y, reg, reg_angle, tau);
    if (reg.size() < 2) return false;
    region2rect(reg, reg_angle, prec, p, rec);
    density = double(reg.size()) / (dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
    if (density < density_th) return reduce_region_radius(reg, reg_angle, prec, p, rec, density, density_th);
    return true;
  }

  // cv::LineSegmentDetector::detect on an 8-bit image -> Vec4f list.  scale1: the detector made with scale 1.0, which grows
  // regions on the image itself (no blur, no resize)
  void detect(const uint8_t* img, int iw, int ih, std::vector<float>& lines, bool scale1 = false) {
    const double ANG_TH = 22.5, QUANT = 2.0, SCALE = scale1 ? 1.0 : 0.8, DENSITY_TH = 0.7;
    const unsigned N_BINS = 1024;
    const double prec = PI_ * ANG_TH / 180, p = ANG_TH / 180, rho = QUANT / std::sin(prec);
    if (scale1) {
      scaled.assign(img, img + (size_t)iw * ih); w = iw; h = ih;
    } else {
      std::vector<uint8_t> g((size_t)iw * ih);
      static const int taps[7] = {0, 4, 56, 136, 56, 4, 0};  // GaussianBlur 7x7, sigma 0.6/0.8 = 0.75, 8.8 fixed point
      blur_sep_u8(img, iw, ih, g.data(), taps, 7);
      resize_08_exact(g.data(), iw, ih, scaled, w, h);
    }
    ll_angle(rho, N_BINS);
    const double LOG_NT = 5 * (std::log10(double(w)) + std::log10(double(h))) / 2 + std::log10(11.0);
    const size_t min_reg_size = size_t(-LOG_NT / std::log10(p));
    used.assign((size_t)w * h, NOTUSED);
    std::vector<RegionPoint> reg;
    lines.clear();
    for (size_t i = 0; i < ordered.size(); ++i) {
      const int px = ordered[i].px, py = ordered[i].py;
      if (used[(size_t)py * w + px] == NOTUSED && angles[(size_t)py * w + px] != NOTDEF) {
        double reg_angle;
        region_grow(px, py, reg, reg_angle, prec);
        if (reg.size() == 1) g_stat[4]++;
        if (reg.size() <= 3) g_stat[5]++;
        if (reg.size() < min_reg_size) continue;
        g_stat[2]++;
        Rect rec;
        region2rect(reg, reg_angle, prec, p, rec);
        if (!refine(reg, reg_angle, prec, p, rec, DENSITY_TH)) continue;
        rec.x1 += 0.5; rec.y1 += 0.5; rec.x2 += 0.5; rec.y2 += 0.5;
        rec.x1 /= SCALE; rec.y1 /= SCALE; rec.x2 /= SCALE; rec.y2 /= SCALE; rec.width /= SCALE;
        lines.push_back(float(rec.x1)); lines.push_back(float(rec.y1));
        lines.push_back(float(rec.x2)); lines.push_back(float(rec.y2));
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------- KeyLine + LBD
struct KeyLine {  // 17 fields, 68 bytes: cv::line_descriptor::KeyLine layout (descriptor_custom.hpp:105-174)
  float angle; int class_id; int octave; float ptx, pty; float response; float size;
  float startPointX, startPointY, endPointX, endPointY;
  float sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
  float lineLength; int numOfPixels;
};
static_assert(sizeof(KeyLine) == 68, "KeyLine layout");

// LSDDetector::detectImpl for numOctaves = 1, scale = 1 (LineExtractor passes (int)1.2 = 1): KeyLines from segments
void make_keylines(const std::vector<float>& lines, int iw, int ih, const uint8_t* mask, std::vector<KeyLine>& kls) {
  kls.clear();
  int class_counter = -1;
  for (size_t k = 0; k + 3 < lines.size(); k += 4) {
    float e[4] = {lines[k], lines[k + 1], lines[k + 2], lines[k + 3]};
    if (e[0] < 0) e[0] = 0;
    if (e[0] >= iw) e[0] = (float)iw - 1.0f;
    if (e[2] < 0) e[2] = 0;
    if (e[2] >= iw) e[2] = (float)iw - 1.0f;
    if (e[1] < 0) e[1] = 0;
    if (e[1] >= ih) e[1] = (float)ih - 1.0f;
    if (e[3] < 0) e[3] = 0;
    if (e[3] >= ih) e[3] = (float)ih - 1.0f;
    KeyLine kl;
    const float octaveScale = 1.0f;  // pow((float)scale, 0)
    kl.startPointX = e[0] * octaveScale; kl.startPointY = e[1] * octaveScale;
    kl.endPointX = e[2] * octaveScale; kl.endPointY = e[3] * octaveScale;
    kl.sPointInOctaveX = e[0]; kl.sPointInOctaveY = e[1]; kl.ePointInOctaveX = e[2]; kl.ePointInOctaveY = e[3];
    kl.lineLength = (float)std::sqrt(std::pow((double)(e[0] - e[2]), 2) + std::pow((double)(e[1] - e[3]), 2));
    // cv::LineIterator(img, Point2f, Point2f).count, 8-connected, end-points rounded half-to-even
    int x0 = (int)lrintf(e[0]), y0 = (int)lrintf(e[1]), x1 = (int)lrintf(e[2]), y1 = (int)lrintf(e[3]);
    kl.numOfPixels = std::max(std::abs(x1 - x0), std::abs(y1 - y0)) + 1;
    // atan2(float, float) resolves to <cmath>'s float overload: libm's atan2f (nm -u of the reference object: atan2f), not the
    // rounded fp64 function (they differ by one ulp on ~16 % of the lines)
    kl.angle = atan2f(kl.endPointY - kl.startPointY, kl.endPointX - kl.startPointX);
    kl.class_id = ++class_counter;
    kl.octave = 0;
    kl.size = (kl.endPointX - kl.startPointX) * (kl.endPointY - kl.startPointY);
    kl.response = kl.lineLength / (float)std::max(iw, ih);
    kl.ptx = (kl.endPointX + kl.startPointX) / 2; kl.pty = (kl.endPointY + kl.startPointY) / 2;
    kls.push_back(kl);
  }
  if (mask) {
    for (size_t i = 0; i < kls.size(); i++) {
      const KeyLine& kl = kls[i];
      if (mask[(size_t)(int)kl.startPointY * iw + (int)kl.startPointX] == 0 &&
          mask[(size_t)(int)kl.endPointY * iw + (int)kl.endPointX] == 0) {
        kls.erase(kls.begin() + i);
        i--;
      }
    }
  }
}

static const int kCombinations[32][2] = {
    {0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {0, 6}, {1, 2}, {1, 3}, {1, 4}, {1, 5}, {1, 6}, {2, 3}, {2, 4}, {2, 5}, {2, 6}, {2, 7},
    {2, 8}, {3, 4}, {3, 5}, {3, 6}, {3, 7}, {3, 8}, {4, 5}, {4, 6}, {4, 7}, {4, 8}, {5, 6}, {5, 7}, {5, 8}, {6, 7}, {6, 8}, {7, 8}};
const int NUM_OF_BANDS = 9, WIDTH_OF_BAND = 7;

struct Lbd {
  int w, h;
  std::vector<int16_t> dx, dy;
  double gaussCoefL[21], gaussCoefG[63];
  Lbd() {
    double u = (WIDTH_OF_BAND * 3 - 1) / 2;           // integer division as in the reference: 10
    double sigma = (WIDTH_OF_BAND * 2 + 1) / 2;       // 7
    double invsigma2 = -1 / (2 * sigma * sigma);
    for (int i = 0; i < WIDTH_OF_BAND * 3; i++) { double dis = i - u; gaussCoefL[i] = std::exp(dis * dis * invsigma2); }
    u = (NUM_OF_BANDS * WIDTH_OF_BAND - 1) / 2;      // 31
    sigma = u;
    invsigma2 = -1 / (2 * sigma * sigma);
    for (int i = 0; i < NUM_OF_BANDS * WIDTH_OF_BAND; i++) { double dis = i - u; gaussCoefG[i] = std::exp(dis * dis * invsigma2); }
  }
  void prepare(const uint8_t* img, int iw, int ih) {  // GaussianBlur 5x5 sigma 1 + Sobel 3x3 -> int16
    w = iw; h = ih;
    std::vector<uint8_t> b((size_t)w * h);
    static const int t5[5] = {14, 62, 104, 62, 14};
    blur_sep_u8(img, w, h, b.data(), t5, 5);
    dx.assign((size_t)w * h, 0); dy.assign((size_t)w * h, 0);
    sobel3(b.data(), w, h, dx.data(), dy.data());
  }
  // cv::Sobel(src 8U, dst 16S, 1, 0, 3) and (0, 1, 3), BORDER_REFLECT_101 (binary_descriptor_custom.cpp:395-396)
  static void sobel3(const uint8_t* b, int w, int h, int16_t* dx, int16_t* dy) {
    for (int y = 0; y < h; y++)
      for (int x = 0; x < w; x++) {
        int xm = reflect101(x - 1, w), xp = reflect101(x + 1, w), ym = reflect101(y - 1, h), yp = reflect101(y + 1, h);
        auto P = [&](int xx, int yy) { return (int)b[(size_t)yy * w + xx]; };
        dx[(size_t)y * w + x] = (int16_t)((P(xp, ym) - P(xm, ym)) + 2 * (P(xp, y) - P(xm, y)) + (P(xp, yp) - P(xm, yp)));
        dy[(size_t)y * w + x] = (int16_t)((P(xm, yp) - P(xm, ym)) + 2 * (P(x, yp) - P(x, ym)) + (P(xp, yp) - P(xp, ym)));
      }
  }
  // computeLBD for one line (octave 0) + binary conversion; desVec72 (optional) receives the float descriptor
  void describe(const KeyLine& kl, uint8_t* out32, float* desVec72) const {
    const short heightOfLSP = (short)(WIDTH_OF_BAND * NUM_OF_BANDS);
    float pS[8][NUM_OF_BANDS];  // pgdL, ngdL, pgdL2, ngdL2, pgdO, ngdO, pgdO2, ngdO2
    memset(pS, 0, sizeof(pS));
    const short realWidth = (short)w, imageWidth = (short)(w - 1), imageHeight = (short)(h - 1);
    const short lengthOfLSP = (short)kl.numOfPixels;
    const short halfHeight = (heightOfLSP - 1) / 2, halfWidth = (lengthOfLSP - 1) / 2;
    const float midX = (float)(0.5 * (kl.sPointInOctaveX + kl.ePointInOctaveX));
    const float midY = (float)(0.5 * (kl.sPointInOctaveY + kl.ePointInOctaveY));
    float dL[2], dO[2];
    sincosf(kl.angle, &dL[1], &dL[0]);   // cos / sin of a float: libm's float functions (the reference object calls sincosf)
    dO[0] = -dL[1]; dO[1] = dL[0];
    float sCorX0 = -dL[0] * halfWidth + dL[1] * halfHeight + midX;
    float sCorY0 = -dL[1] * halfWidth - dL[0] * halfHeight + midY;
    for (short hID = 0; hID < heightOfLSP; hID++) {
      float sCorX = sCorX0, sCorY = sCorY0;
      float pgdL = 0, ngdL = 0, pgdO = 0, ngdO = 0;
      for (short wID = 0; wID < lengthOfLSP; wID++) {
        short t = (short)roundf(sCorX);
        short xCor = (t < 0) ? 0 : (t > imageWidth) ? imageWidth : t;
        t = (short)roundf(sCorY);
        short yCor = (t < 0) ? 0 : (t > imageHeight) ? imageHeight : t;
        short ddx = dx[(size_t)yCor * realWidth + xCor], ddy = dy[(size_t)yCor * realWidth + xCor];
        float gDL = ddx * dL[0] + ddy * dL[1];
        float gDO = ddx * dO[0] + ddy * dO[1];
        if (gDL > 0) pgdL += gDL; else ngdL -= gDL;
        if (gDO > 0) pgdO += gDO; else ngdO -= gDO;
        sCorX += dL[0]; sCorY += dL[1];
      }
      sCorX0 -= dL[1]; sCorY0 += dL[0];
      float c = (float)gaussCoefG[hID];
      pgdL = c * pgdL; ngdL = c * ngdL;
      float pgdL2 = pgdL * pgdL, ngdL2 = ngdL * ngdL;
      pgdO = c * pgdO; ngdO = c * ngdO;
      float pgdO2 = pgdO * pgdO, ngdO2 = ngdO * ngdO;
      const float rs[8] = {pgdL, ngdL, pgdL2, ngdL2, pgdO, ngdO, pgdO2, ngdO2};
      auto add = [&](short band, float cg) {
        pS[0][band] += cg * rs[0]; pS[1][band] += cg * rs[1];
        pS[2][band] += cg * cg * rs[2]; pS[3][band] += cg * cg * rs[3];
        pS[4][band] += cg * rs[4]; pS[5][band] += cg * rs[5];
        pS[6][band] += cg * cg * rs[6]; pS[7][band] += cg * cg * rs[7];
      };
      short bandID = (short)(hID / WIDTH_OF_BAND);
      add(bandID, (float)gaussCoefL[hID % WIDTH_OF_BAND + WIDTH_OF_BAND]);
      bandID--;
      if (bandID >= 0) add(bandID, (float)gaussCoefL[hID % WIDTH_OF_BAND + 2 * WIDTH_OF_BAND]);
      bandID = bandID + 2;
      if (bandID < NUM_OF_BANDS) add(bandID, (float)gaussCoefL[hID % WIDTH_OF_BAND]);
    }
    float des[72];
    const float invN2 = (float)(1.0 / (WIDTH_OF_BAND * 2.0)), invN3 = (float)(1.0 / (WIDTH_OF_BAND * 3.0));
    for (short b = 0; b < NUM_OF_BANDS; b++) {
      float invN = (b == 0 || b == NUM_OF_BANDS - 1) ? invN2 : invN3, temp;
      short d = b * 8;
      temp = pS[0][b] * invN; des[d] = temp; des[d + 4] = sqrtf(pS[2][b] * invN - temp * temp);
      temp = pS[1][b] * invN; des[d + 1] = temp; des[d + 5] = sqrtf(pS[3][b] * invN - temp * temp);
      temp = pS[4][b] * invN; des[d + 2] = temp; des[d + 6] = sqrtf(pS[6][b] * invN - temp * temp);
      temp = pS[5][b] * invN; des[d + 3] = temp; des[d + 7] = sqrtf(pS[7][b] * invN - temp * temp);
    }
    float tempM = 0, tempS = 0;
    for (int i = 0; i < 72; i += 8) {
      tempM += des[i] * des[i]; tempM += des[i + 1] * des[i + 1]; tempM += des[i + 2] * des[i + 2]; tempM += des[i + 3] * des[i + 3];
      tempS += des[i + 4] * des[i + 4]; tempS += des[i + 5] * des[i + 5]; tempS += des[i + 6] * des[i + 6]; tempS += des[i + 7] * des[i + 7];
    }
    tempM = 1 / sqrtf(tempM); tempS = 1 / sqrtf(tempS);
    for (int i = 0; i < 72; i += 8) {
      des[i] *= tempM; des[i + 1] *= tempM; des[i + 2] *= tempM; des[i + 3] *= tempM;
      des[i + 4] *= tempS; des[i + 5] *= tempS; des[i + 6] *= tempS; des[i + 7] *= tempS;
    }
    for (int i = 0; i < 72; i++) if (des[i] > 0.4) des[i] = (float)0.4;
    float temp = 0;
    for (int i = 0; i < 72; i++) temp += des[i] * des[i];
    temp = 1 / sqrtf(temp);
    for (int i = 0; i < 72; i++) des[i] = des[i] * temp;
    if (desVec72) memcpy(desVec72, des, sizeof(des));
    for (int comb = 0; comb < 32; comb++) {
      const float* f1 = &des[8 * kCombinations[comb][0]];
      const float* f2 = &des[8 * kCombinations[comb][1]];
      uint8_t r = 0;
      for (int i = 0; i < 8; i++) if (f1[i] > f2[i]) r += (uint8_t)(1 << i);
      out32[comb] = r;
    }
  }
};
}  // namespace

extern "C" {
void oracle_lsd_stats(long* out, int reset) { for (int i = 0; i < 8; i++) { out[i] = g_stat[i]; if (reset) g_stat[i] = 0; } }
// cv::createLineSegmentDetector()->detect(img): returns number of segments; lines receives 4 floats each
int oracle_lsd_detect(const uint8_t* img, int w, int h, int order_mode, float* lines, int cap) {
  Lsd l;
  l.order_mode = order_mode;
  std::vector<float> v;
  l.detect(img, w, h, v);
  int n = (int)v.size() / 4;
  memcpy(lines, v.data(), sizeof(float) * 4 * std::min(n, cap));
  return n;
}
// the same with scale 1.0 (cv::createLineSegmentDetector(LSD_REFINE_STD, 1.0)): regions grown on the image itself; addend:
// what region_grow adds to its sums (kAddCosf, the default, kAddCosRounded or kAddCosDouble)
int oracle_lsd_detect_scale1(const uint8_t* img, int w, int h, int addend, float* lines, int cap) {
  if (addend < kAddCosf || addend > kAddCosDouble) return -1;
  Lsd l;
  l.order_mode = 1;
  l.addend = addend;
  std::vector<float> v;
  l.detect(img, w, h, v, true);
  int n = (int)v.size() / 4;
  memcpy(lines, v.data(), sizeof(float) * 4 * std::min(n, cap));
  return n;
}
// intermediate taps for stage-level parity tests: scaled image, gradient magnitude, angle
int oracle_lsd_stages(const uint8_t* img, int w, int h, uint8_t* scaled, double* modgrad, double* angles, int* sw, int* sh) {
  Lsd l;
  std::vector<uint8_t> g((size_t)w * h);
  static const int taps[7] = {0, 4, 56, 136, 56, 4, 0};
  blur_sep_u8(img, w, h, g.data(), taps, 7);
  resize_08_exact(g.data(), w, h, l.scaled, l.w, l.h);
  l.ll_angle(2.0 / std::sin(PI_ * 22.5 / 180), 1024);
  *sw = l.w; *sh = l.h;
  if (scaled) memcpy(scaled, l.scaled.data(), l.scaled.size());
  if (modgrad) memcpy(modgrad, l.modgrad.data(), l.modgrad.size() * 8);
  if (angles) memcpy(angles, l.angles.data(), l.angles.size() * 8);
  return 0;
}
// LBD for given KeyLines (68-byte records)
void oracle_lbd_compute(const uint8_t* img, int w, int h, const void* keylines, int n, uint8_t* desc, float* desvec) {
  Lbd lbd;
  lbd.prepare(img, w, h);
  const KeyLine* k = (const KeyLine*)keylines;
  for (int i = 0; i < n; i++) lbd.describe(k[i], desc + 32 * i, desvec ? desvec + 72 * i : nullptr);
}
// the Sobel pair alone, on an image that is already blurred (the primitive behind the OpenCV stand-in of oracle/shim/)
void oracle_sobel3_u8(const uint8_t* img, int w, int h, int16_t* dx, int16_t* dy) { Lbd::sobel3(img, w, h, dx, dy); }
void oracle_lbd_sobel(const uint8_t* img, int w, int h, int16_t* dx, int16_t* dy) {
  Lbd lbd;
  lbd.prepare(img, w, h);
  memcpy(dx, lbd.dx.data(), (size_t)w * h * 2); memcpy(dy, lbd.dy.data(), (size_t)w * h * 2);
}
// LINEextractor::operator()(image, mask, keylines, descriptors, lineVec2d); returns the number of KeyLines
int oracle_line_extract(const uint8_t* img, int w, int h, const uint8_t* mask, int nfeatures, double min_line_length,
                        int order_mode, void* keylines_out, uint8_t* desc_out, double* linefunc_out, int cap) {
  Lsd l;
  l.order_mode = order_mode;
  std::vector<float> segs;
  l.detect(img, w, h, segs);
  std::vector<KeyLine> kls;
  make_keylines(segs, w, h, mask, kls);
  std::stable_sort(kls.begin(), kls.end(), [](const KeyLine& a, const KeyLine& b) { return a.response > b.response; });
  int total, index;
  if ((int)kls.size() > nfeatures) { total = nfeatures; index = nfeatures; }
  else { total = (int)kls.size(); index = (int)kls.size(); }
  if (total > 0 && kls[total - 1].lineLength < min_line_length) {
    for (int i = 0; i < total - 1; i++)
      if (kls[i].lineLength >= min_line_length && kls[i + 1].lineLength < min_line_length) { index = i; break; }
  }
  KeyLine zero;
  memset(&zero, 0, sizeof(zero));
  kls.resize(index + 1, zero);
  for (int i = 0; i < index + 1; i++) kls[i].class_id = i;
  int n = (int)kls.size();
  if (n > cap) return -1;
  Lbd lbd;
  lbd.prepare(img, w, h);
  KeyLine* out = (KeyLine*)keylines_out;
  for (int i = 0; i < n; i++) {
    out[i] = kls[i];
    lbd.describe(kls[i], desc_out + 32 * i, nullptr);
    const double sx = kls[i].startPointX, sy = kls[i].startPointY, ex = kls[i].endPointX, ey = kls[i].endPointY;
    double lx = sy * 1.0 - 1.0 * ey, ly = 1.0 * ex - sx * 1.0, lz = sx * ey - sy * ex;  // sp x ep
    double nn = std::sqrt(lx * lx + ly * ly);
    linefunc_out[3 * i] = lx / nn; linefunc_out[3 * i + 1] = ly / nn; linefunc_out[3 * i + 2] = lz / nn;
  }
  return n;
}
}
