// The demo's landmark, pose and wireframe overlays drawn into whole frames (include/dad3d.h "overlays"): draw_points over
// draw_landmarks / draw_3d_landmarks (demo_utils.py:22-47), draw_pose (demo_utils.py:68-94) into each box's crop view,
// draw_mesh (demo_utils.py:50-65), and calculate_rpy (model_training/model/flame.py:238-264) for every head.
//
// The raster restates the cv2 calls the demo makes (cv2 4.13.0; tests/overlay_model.py is the model, pinned against the
// binary; tests/wireframe_model.py for LineAA): the midpoint filled circle, the clipped 8-connected line iterator, the
// anti-aliased line, and for thickness >= 2 the segment clipped to the area grown by the thickness, a 16-bit fixed-point
// quad (outline by the fixed-point line, inside by the convex scan-line fill) and two cap circles.  All of it is integer work in cv2's own int64 / double expressions; fp64 values use
// explicit _rn intrinsics so nvcc cannot contract them into an fma.
#include <climits>
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"

namespace dad3d {
namespace {

constexpr int kXYShift = 16;
constexpr long long kXYOne = 1LL << kXYShift;
constexpr int kPoseInts = DAD3D_POSE_RECORD_INTS;

// ---------------------------------------------------------------------------------------------------------- primitives
// Everything draws into a clip area of w x h pixels (the frame, or a box's crop view) through Plot::operator()(x, y),
// which the caller only invokes for 0 <= x < w, 0 <= y < h.

template <class Plot>
__device__ void hspan(long long y, long long x0, long long x1, long long w, long long h, Plot& plot) {
  if (y < 0 || y >= h) return;
  x0 = max(x0, 0LL);
  x1 = min(x1, w - 1);
  for (long long x = x0; x <= x1; ++x) plot(x, y);
}

// cv::Circle with fill (drawing.cpp, LINE_8, shift 0): spans of rows c +- dy over [c - dx, c + dx] and rows c +- dx over
// [c - dy, c + dy] along the integer midpoint recurrence.
template <class Plot>
__device__ void fill_circle(long long cx, long long cy, int r, long long w, long long h, Plot& plot) {
  int err = 0, dx = r, dy = 0, plus = 1, minus = 2 * r - 1;
  while (dx >= dy) {
    if (cx - dx < w && cx + dx >= 0 && cy - dx < h && cy + dx >= 0) {
      hspan(cy - dy, cx - dx, cx + dx, w, h, plot);
      hspan(cy + dy, cx - dx, cx + dx, w, h, plot);
      hspan(cy - dx, cx - dy, cx + dy, w, h, plot);
      hspan(cy + dx, cx - dy, cx + dy, w, h, plot);
    }
    ++dy;
    err += plus;
    plus += 2;
    const int m = (err <= 0) - 1;
    err -= minus & m;
    dx += m;
    minus -= m & 2;
  }
}

// cv::clipLine over int64 points and a w x h area; false when nothing is left.  The second point's correction uses the
// first point as already corrected, as cv2 does.
__device__ bool clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
  if (w <= 0 || h <= 0) return false;
  const long long right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += __double2ll_rz(__ddiv_rn(__dmul_rn(static_cast<double>(a - y1), static_cast<double>(x2 - x1)),
                                     static_cast<double>(y2 - y1)));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += __double2ll_rz(__ddiv_rn(__dmul_rn(static_cast<double>(a - y2), static_cast<double>(x2 - x1)),
                                     static_cast<double>(y2 - y1)));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += __double2ll_rz(__ddiv_rn(__dmul_rn(static_cast<double>(a - x1), static_cast<double>(y2 - y1)),
                                       static_cast<double>(x2 - x1)));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += __double2ll_rz(__ddiv_rn(__dmul_rn(static_cast<double>(a - x2), static_cast<double>(y2 - y1)),
                                       static_cast<double>(x2 - x1)));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// cv2.line, thickness 1, LINE_8: cv::LineIterator(8-connected, left to right) over the clipped segment.
template <class Plot>
__device__ void thin_line(long long x1, long long y1, long long x2, long long y2, long long w, long long h, Plot& plot) {
  if (!(x1 >= 0 && x1 < w && x2 >= 0 && x2 < w && y1 >= 0 && y1 < h && y2 >= 0 && y2 < h) &&
      !clip_line(w, h, x1, y1, x2, y2))
    return;
  long long dx = x2 - x1, dy = y2 - y1, sx = 1, sy = 1;
  if (dx < 0) {
    dx = -dx;
    dy = -dy;
    long long t = x1; x1 = x2; x2 = t;
    t = y1; y1 = y2; y2 = t;
  }
  if (dy < 0) {
    dy = -dy;
    sy = -1;
  }
  const bool vert = dy > dx;
  if (vert) {
    const long long t = dx; dx = dy; dy = t;
  }
  long long err = dx - (dy + dy);
  const long long plus = dx + dx, minus = -(dy + dy);
  long long x = x1, y = y1;
  for (long long i = 0; i <= dx; ++i) {
    plot(x, y);
    const bool minor = err < 0;
    err += minus + (minor ? plus : 0);
    if (vert) {
      y += sy;
      if (minor) x += sx;
    } else {
      x += sx;
      if (minor) y += sy;
    }
  }
}

// cv2's fixed-point Line2 (16-bit fraction): the outline of a thick segment's quad.
template <class Plot>
__device__ void line2(long long x1, long long y1, long long x2, long long y2, long long w, long long h, Plot& plot) {
  if (!clip_line(w << kXYShift, h << kXYShift, x1, y1, x2, y2)) return;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long j = dx < 0 ? -1 : 0, ax = (dx ^ j) - j;
  const long long i = dy < 0 ? -1 : 0, ay = (dy ^ i) - i;
  long long x_step, y_step, ecount;
  const bool horiz = ax > ay;
  if (horiz) {
    dy = (dy ^ j) - j;
    if (j) {
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    x_step = kXYOne;
    y_step = (dy * kXYOne) / (ax | 1);
    ecount = (x2 - x1) >> kXYShift;
  } else {
    dx = (dx ^ i) - i;
    if (i) {
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    x_step = (dx * kXYOne) / (ay | 1);
    y_step = kXYOne;
    ecount = (y2 - y1) >> kXYShift;
  }
  x1 += kXYOne >> 1;
  y1 += kXYOne >> 1;
  auto put = [&](long long x, long long y) {
    if (x >= 0 && x < w && y >= 0 && y < h) plot(x, y);
  };
  put((x2 + (kXYOne >> 1)) >> kXYShift, (y2 + (kXYOne >> 1)) >> kXYShift);
  if (horiz) {
    x1 >>= kXYShift;
    for (; ecount >= 0; --ecount, ++x1, y1 += y_step) put(x1, y1 >> kXYShift);
  } else {
    y1 >>= kXYShift;
    for (; ecount >= 0; --ecount, x1 += x_step, ++y1) put(x1 >> kXYShift, y1);
  }
}

// cv::FillConvexPoly for 4 points, shift 16, LINE_8: the outline, then the two-edge scan-line fill.
template <class Plot>
__device__ void fill_quad(const long long (&vx)[4], const long long (&vy)[4], long long w, long long h, Plot& plot) {
  constexpr int npts = 4;
  const long long delta = kXYOne >> 1;
  long long xmin = vx[0], xmax = vx[0], ymin = vy[0], ymax = vy[0];
  int imin = 0;
  long long px = vx[npts - 1], py = vy[npts - 1];
  for (int k = 0; k < npts; ++k) {
    if (vy[k] < ymin) {
      ymin = vy[k];
      imin = k;
    }
    ymax = max(ymax, vy[k]);
    xmax = max(xmax, vx[k]);
    xmin = min(xmin, vx[k]);
    line2(px, py, vx[k], vy[k], w, h, plot);
    px = vx[k];
    py = vy[k];
  }
  xmin = (xmin + delta) >> kXYShift;
  xmax = (xmax + delta) >> kXYShift;
  ymin = (ymin + delta) >> kXYShift;
  ymax = (ymax + delta) >> kXYShift;
  if (xmax < 0 || ymax < 0 || xmin >= w || ymin >= h) return;
  ymax = min(ymax, h - 1);
  int e_idx[2] = {imin, imin}, e_di[2] = {1, npts - 1};
  long long e_ye[2] = {ymin, ymin}, e_x[2] = {-kXYOne, -kXYOne}, e_dx[2] = {0, 0};
  int edges = npts;
  long long y = ymin;
  do {
    for (int k = 0; k < 2; ++k) {
      if (y >= e_ye[k]) {
        int idx0 = e_idx[k], di = e_di[k];
        int idx = idx0 + di;
        if (idx >= npts) idx -= npts;
        for (; edges-- > 0;) {
          const long long ty = (vy[idx] + delta) >> kXYShift;
          if (ty > y) {
            const long long xs = vx[idx0], xe = vx[idx];
            e_ye[k] = ty;
            e_dx[k] = ((xe - xs) * 2 + (ty - y)) / (2 * (ty - y));
            e_x[k] = xs;
            e_idx[k] = idx;
            break;
          }
          idx0 = idx;
          idx += di;
          if (idx >= npts) idx -= npts;
        }
      }
    }
    if (edges < 0) break;
    if (y >= 0) {
      const int left = e_x[0] > e_x[1] ? 1 : 0;
      const long long xx1 = (e_x[left] + delta) >> kXYShift;
      const long long xx2 = (e_x[1 - left] + delta) >> kXYShift;
      if (xx2 >= 0 && xx1 < w) hspan(y, xx1, xx2, w, h, plot);
    }
    e_x[0] += e_dx[0];
    e_x[1] += e_dx[1];
  } while (++y <= ymax);
}

// cv2.line(img, p0, p1, color, t, LINE_8) in a w x h area, t >= 1.
template <class Plot>
__device__ void segment(long long x0, long long y0, long long x1, long long y1, int t, long long w, long long h, Plot& plot) {
  if (t <= 1) {
    thin_line(x0, y0, x1, y1, w, h, plot);
    return;
  }
  x0 += t; y0 += t; x1 += t; y1 += t;                 // clipped to the area grown by t on every side first
  if (!clip_line(w + 2 * t, h + 2 * t, x0, y0, x1, y1)) return;
  x0 -= t; y0 -= t; x1 -= t; y1 -= t;
  const long long P0x = x0 * kXYOne, P0y = y0 * kXYOne, P1x = x1 * kXYOne, P1y = y1 * kXYOne;
  const double dx = __dmul_rn(static_cast<double>(P0x - P1x), 1.0 / kXYOne);
  const double dy = __dmul_rn(static_cast<double>(P1y - P0y), 1.0 / kXYOne);
  double r = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  const long long tt = static_cast<long long>(t) << (kXYShift - 1);
  if (fabs(r) > 2.220446049250313e-16) {
    r = __ddiv_rn(__dadd_rn(static_cast<double>(tt), (t & 1) ? 0.5 * kXYOne : 0.0), __dsqrt_rn(r));
    const long long dpx = __double2ll_rn(__dmul_rn(dy, r)), dpy = __double2ll_rn(__dmul_rn(dx, r));
    const long long qx[4] = {P0x + dpx, P0x - dpx, P1x - dpx, P1x + dpx};
    const long long qy[4] = {P0y + dpy, P0y - dpy, P1y - dpy, P1y + dpy};
    fill_quad(qx, qy, w, h, plot);
  }
  const int rad = static_cast<int>((tt + (kXYOne >> 1)) >> kXYShift);
  fill_circle(x0, y0, rad, w, h, plot);
  fill_circle(x1, y1, rad, w, h, plot);
}

// ---------------------------------------------------------------------------------------------------------- points
struct PointPlot {
  uint8_t* img;          // the frame
  long long W;
  uint8_t c0, c1, c2;
  __device__ void operator()(long long x, long long y) const {
    uint8_t* p = img + (y * W + x) * 3;
    p[0] = c0;
    p[1] = c1;
    p[2] = c2;
  }
};

__device__ __forceinline__ bool to_int32(double v, long long& out) {
  if (!(v > -2147483649.0 && v < 2147483648.0)) return false;     // NaN, inf, or outside int32 after truncation
  out = __double2ll_rz(v);
  return true;
}

// grid.x covers the L points, grid.y strides over heads
__global__ void overlay_points_kernel(const void* __restrict__ src, int is_float, int R, int n_src, int ncomp,
                                      const int64_t* __restrict__ index, int L, const dad3d_roi* __restrict__ rois,
                                      int radius, uint8_t c0, uint8_t c1, uint8_t c2, uint8_t* __restrict__ frames, int F,
                                      int H, int W) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  for (int r = blockIdx.y; r < R; r += gridDim.y) {
    const dad3d_roi q = rois[r];
    if (!q.valid || q.frame < 0 || q.frame >= F) continue;
    const long long v = index ? index[l] : l;
    if (v < 0 || v >= n_src) continue;
    const size_t off = (static_cast<size_t>(r) * n_src + static_cast<size_t>(v)) * ncomp;
    long long x, y;
    if (is_float) {
      const float* p = static_cast<const float*>(src) + off;
      if (!to_int32(static_cast<double>(p[0]), x) || !to_int32(static_cast<double>(p[1]), y)) continue;
    } else {
      const int64_t* p = static_cast<const int64_t*>(src) + off;
      x = p[0];
      y = p[1];
      if (x < INT32_MIN || x > INT32_MAX || y < INT32_MIN || y > INT32_MAX) continue;
    }
    PointPlot plot{frames + static_cast<size_t>(q.frame) * H * W * 3, W, c0, c1, c2};
    fill_circle(x, y, radius, W, H, plot);
  }
}

// ---------------------------------------------------------------------------------------------------------- pose
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }

// torch's CPU kernels: |x| = sqrt(fma(x2, x2, fma(x1, x1, x0 * x0))); cross_i = fma(a_j, b_k, -(a_k * b_j))
__device__ void normalize3(const float (&a)[3], float (&o)[3]) {     // F.normalize: x / max(|x|, 1e-12)
  float n = __fsqrt_rn(__fmaf_rn(a[2], a[2], __fmaf_rn(a[1], a[1], fmul(a[0], a[0]))));
  n = n < 1e-12f ? 1e-12f : n;                                       // NaN stays NaN, as clamp_min
  for (int i = 0; i < 3; ++i) o[i] = __fdiv_rn(a[i], n);
}

__device__ void cross3(const float (&a)[3], const float (&b)[3], float (&o)[3]) {
  o[0] = __fmaf_rn(a[1], b[2], -fmul(a[2], b[1]));
  o[1] = __fmaf_rn(a[2], b[0], -fmul(a[0], b[2]));
  o[2] = __fmaf_rn(a[0], b[1], -fmul(a[1], b[0]));
}

__device__ double py_mod(double a, double b) {                       // numpy's float remainder (sign of the divisor)
  double m = fmod(a, b);
  if (m != 0.0) {
    if ((b < 0) != (m < 0)) m = __dadd_rn(m, b);
  } else {
    m = copysign(0.0, b);
  }
  return m;
}

__device__ long long floor_div(long long a, long long b) {
  long long q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
  return q;
}

__device__ double limit_angle(double angle) {                        // flame.py:239-251 with pi = 180
  const double pi = 180.0;
  if (angle < -pi) {
    const long long k = -2 * floor_div(static_cast<long long>(__ddiv_rn(angle, pi)), 2);
    angle = __dadd_rn(angle, __dmul_rn(static_cast<double>(k), pi));
  }
  if (angle > pi) {
    const long long k = 2 * floor_div(static_cast<long long>(__ddiv_rn(angle, pi)) + 1, 2);
    angle = __dsub_rn(angle, __dmul_rn(static_cast<double>(k), pi));
  }
  return angle;
}

// cv2.arrowedLine's tip points (tipLength 0.1) for the segment p1 -> p2.
__device__ void arrow_tips(long long x1, long long y1, long long x2, long long y2, int* out) {
  const double ddx = static_cast<double>(x1 - x2), ddy = static_cast<double>(y1 - y2);
  const double tip = __dmul_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(ddx, ddx), __dmul_rn(ddy, ddy))), 0.1);
  const double ang = atan2(__dsub_rn(static_cast<double>(y1), static_cast<double>(y2)),
                           __dsub_rn(static_cast<double>(x1), static_cast<double>(x2)));
  const double qp = __dadd_rn(ang, M_PI / 4), qm = __dsub_rn(ang, M_PI / 4);
  out[0] = __double2int_rn(__dadd_rn(static_cast<double>(x2), __dmul_rn(tip, cos(qp))));
  out[1] = __double2int_rn(__dadd_rn(static_cast<double>(y2), __dmul_rn(tip, sin(qp))));
  out[2] = __double2int_rn(__dadd_rn(static_cast<double>(x2), __dmul_rn(tip, cos(qm))));
  out[3] = __double2int_rn(__dadd_rn(static_cast<double>(y2), __dmul_rn(tip, sin(qm))));
}

// The orthogonal polar factor U V^T of a nearly orthogonal 3x3 matrix, in fp64: scipy's from_matrix replaces a matrix whose
// Gram matrix is not the identity to 1e-12 by U V^T of its SVD (always the case for one built from fp32 vectors, which is
// ~1e-7 off).  Newton's iteration X <- (X + X^-T) / 2, with X^-T = cofactor(X) / det(X), converges quadratically from such
// a start: three steps take 1e-7 to the fp64 rounding level (~1e-15 of LAPACK's U V^T).
__device__ void polar_factor(double (&m)[3][3]) {
  for (int it = 0; it < 3; ++it) {
    double c[3][3];
    for (int i = 0; i < 3; ++i) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
      for (int j = 0; j < 3; ++j) {
        const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        c[i][j] = __dsub_rn(__dmul_rn(m[i1][j1], m[i2][j2]), __dmul_rn(m[i1][j2], m[i2][j1]));
      }
    }
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(m[0][0], c[0][0]), __dmul_rn(m[0][1], c[0][1])),
                                 __dmul_rn(m[0][2], c[0][2]));
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) m[i][j] = __dmul_rn(__dadd_rn(m[i][j], __ddiv_rn(c[i][j], det)), 0.5);
  }
}

__global__ void pose_geometry_kernel(const float* __restrict__ params, int R, int P, int ri,
                                     const dad3d_roi* __restrict__ rois, double* __restrict__ rpy_out,
                                     int32_t* __restrict__ pose_out, float* __restrict__ rot_out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  // rot_mat_from_6dof (model/utils.py:92-101), fp32 in torch's order; columns b1, b2, b3
  const float* v = params + static_cast<size_t>(r) * P + ri;
  const float vx[3] = {v[0], v[1], v[2]}, vy[3] = {v[3], v[4], v[5]};
  float b1[3], b2[3], b3[3], c[3];
  normalize3(vx, b1);
  cross3(b1, vy, c);
  normalize3(c, b3);
  cross3(b1, b3, c);
  for (int i = 0; i < 3; ++i) b2[i] = -c[i];
  if (rot_out) {                                                     // R row-major: R[i][0..2] = b1[i], b2[i], b3[i]
    float* o = rot_out + static_cast<size_t>(r) * 9;
    for (int i = 0; i < 3; ++i) {
      o[3 * i + 0] = b1[i];
      o[3 * i + 1] = b2[i];
      o[3 * i + 2] = b3[i];
    }
  }
  // Rotation.from_matrix(R^T) (scipy 1.18): m's rows are b1, b2, b3; its polar factor, then Markley's quaternion
  double m[3][3];
  for (int i = 0; i < 3; ++i) {
    m[0][i] = b1[i];
    m[1][i] = b2[i];
    m[2][i] = b3[i];
  }
  polar_factor(m);
  const double tr = __dadd_rn(__dadd_rn(m[0][0], m[1][1]), m[2][2]);
  const double dec[4] = {m[0][0], m[1][1], m[2][2], tr};
  int choice = 0;
  for (int k = 1; k < 4; ++k)
    if (dec[k] > dec[choice] || (isnan(dec[k]) && !isnan(dec[choice]))) choice = k;
  double qv[4];
  if (choice == 0) {
    qv[0] = __dadd_rn(__dsub_rn(1.0, tr), __dmul_rn(2.0, m[0][0])); qv[1] = __dadd_rn(m[1][0], m[0][1]);
    qv[2] = __dadd_rn(m[2][0], m[0][2]); qv[3] = __dsub_rn(m[2][1], m[1][2]);
  } else if (choice == 1) {
    qv[0] = __dadd_rn(m[1][0], m[0][1]); qv[1] = __dadd_rn(__dsub_rn(1.0, tr), __dmul_rn(2.0, m[1][1]));
    qv[2] = __dadd_rn(m[2][1], m[1][2]); qv[3] = __dsub_rn(m[0][2], m[2][0]);
  } else if (choice == 2) {
    qv[0] = __dadd_rn(m[2][0], m[0][2]); qv[1] = __dadd_rn(m[2][1], m[1][2]);
    qv[2] = __dadd_rn(__dsub_rn(1.0, tr), __dmul_rn(2.0, m[2][2])); qv[3] = __dsub_rn(m[1][0], m[0][1]);
  } else {
    qv[0] = __dsub_rn(m[2][1], m[1][2]); qv[1] = __dsub_rn(m[0][2], m[2][0]);
    qv[2] = __dsub_rn(m[1][0], m[0][1]); qv[3] = __dadd_rn(1.0, tr);
  }
  const double qn = __dsqrt_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(qv[0], qv[0]), __dmul_rn(qv[1], qv[1])),
                                                   __dmul_rn(qv[2], qv[2])), __dmul_rn(qv[3], qv[3])));
  for (int k = 0; k < 4; ++k) qv[k] = __ddiv_rn(qv[k], qn);
  // as_euler("xyz"): extrinsic Tait-Bryan, i, j, k = 0, 1, 2, sign +1
  const double a = __dsub_rn(qv[3], qv[1]), b = __dadd_rn(qv[0], qv[2]);
  const double cc = __dadd_rn(qv[1], qv[3]), d = __dsub_rn(qv[2], qv[0]);
  const double half_sum = atan2(b, a), half_diff = atan2(d, cc);
  const double mid = __dmul_rn(2.0, atan2(hypot(cc, d), hypot(a, b)));
  double first, third;
  if (fabs(mid) <= 1e-7) {
    first = __dmul_rn(2.0, half_sum);
    third = 0.0;
  } else if (fabs(__dsub_rn(mid, M_PI)) <= 1e-7) {
    first = __dmul_rn(-2.0, half_diff);
    third = 0.0;
  } else {
    first = __dsub_rn(half_sum, half_diff);
    third = __dadd_rn(half_sum, half_diff);
  }
  const double ang_rad[3] = {first, __dsub_rn(mid, M_PI / 2), third};
  double ang[3];
  for (int k = 0; k < 3; ++k)
    ang[k] = __dmul_rn(__dsub_rn(py_mod(__dadd_rn(ang_rad[k], M_PI), 2 * M_PI), M_PI), 180.0 / M_PI);
  const double roll = limit_angle(ang[2]), pitch = limit_angle(__dsub_rn(ang[0], 180.0)), yaw = limit_angle(ang[1]);
  if (rpy_out) {
    rpy_out[3 * r + 0] = roll;
    rpy_out[3 * r + 1] = pitch;
    rpy_out[3 * r + 2] = yaw;
  }
  if (!pose_out) return;
  // draw_pose (demo_utils.py:68-94) in the crop view of the box
  int32_t* rec = pose_out + static_cast<size_t>(r) * kPoseInts;
  const dad3d_roi q = rois[r];
  const int w = q.w, h = q.h;
  const int tdx = w / 2, tdy = h / 2, size = h / 10;
  const int t = __double2int_rz(__dmul_rn(static_cast<double>(h), 0.005));
  const double rr = __ddiv_rn(__dmul_rn(roll, M_PI), 180.0);
  const double rp = __ddiv_rn(__dmul_rn(pitch, M_PI), 180.0);
  const double ry = -__ddiv_rn(__dmul_rn(yaw, M_PI), 180.0);
  const double cy = cos(ry), sy = sin(ry), cr = cos(rr), sr = sin(rr), cp = cos(rp), sp = sin(rp);
  const double sz = static_cast<double>(size), fx = static_cast<double>(tdx), fy = static_cast<double>(tdy);
  const double vals[6] = {
      __dadd_rn(__dmul_rn(sz, __dmul_rn(cy, cr)), fx),
      __dadd_rn(__dmul_rn(sz, __dadd_rn(__dmul_rn(cp, sr), __dmul_rn(__dmul_rn(cr, sp), sy))), fy),
      __dadd_rn(__dmul_rn(sz, __dmul_rn(-cy, sr)), fx),
      __dadd_rn(__dmul_rn(sz, __dsub_rn(__dmul_rn(cp, cr), __dmul_rn(__dmul_rn(sp, sy), sr))), fy),
      __dadd_rn(__dmul_rn(sz, sy), fx),
      __dadd_rn(__dmul_rn(sz, __dmul_rn(-cy, sp)), fy)};
  bool finite = true;
  for (int k = 0; k < 6; ++k) finite = finite && isfinite(vals[k]) && fabs(vals[k]) < 1e9;
  for (int k = 0; k < kPoseInts; ++k) rec[k] = 0;
  rec[0] = (q.valid && t >= 1 && finite) ? 1 : 0;                   // cv2.arrowedLine refuses thickness 0
  rec[1] = q.frame;
  rec[2] = q.x;
  rec[3] = q.y;
  rec[4] = w;
  rec[5] = h;
  rec[6] = t;
  rec[8] = tdx;
  rec[9] = tdy;
  if (!finite) return;
  for (int k = 0; k < 3; ++k) {
    const int ex = __double2int_rz(vals[2 * k]), ey = __double2int_rz(vals[2 * k + 1]);   // Python int(): truncation
    rec[10 + 6 * k] = ex;
    rec[11 + 6 * k] = ey;
    arrow_tips(tdx, tdy, ex, ey, rec + 12 + 6 * k);
  }
}

struct KeyPlot {
  int* key;              // the frame's key plane
  long long x0, y0;      // the crop's origin in the frame
  long long W, H;
  int value;
  __device__ void operator()(long long x, long long y) const {   // (x, y) lies in the crop; only frame pixels are marked
    const long long fx = x0 + x, fy = y0 + y;
    if (fx >= 0 && fx < W && fy >= 0 && fy < H) atomicMax(key + fy * W + fx, value);
  }
};

// one thread per (box, arrow, segment): pass 1 of the pose raster
__global__ void pose_raster_kernel(const int32_t* __restrict__ pose, int R, int* __restrict__ key, int F, int H, int W) {
  const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= 9LL * R) return;
  const int r = static_cast<int>(g / 9), s = static_cast<int>(g % 9), k = s / 3, part = s % 3;
  const int32_t* rec = pose + static_cast<size_t>(r) * kPoseInts;
  if (!rec[0] || rec[1] < 0 || rec[1] >= F) return;
  const int x = rec[2], y = rec[3], w = rec[4], h = rec[5], t = rec[6];
  const int* a = rec + 10 + 6 * k;                                   // end, tip 1, tip 2
  const long long ex = a[0], ey = a[1];
  const long long sx = part == 0 ? rec[8] : a[2 * part], sy = part == 0 ? rec[9] : a[2 * part + 1];
  KeyPlot plot{key + static_cast<size_t>(rec[1]) * H * W, x, y, W, H, 3 * r + k + 1};
  segment(sx, sy, ex, ey, t, w, h, plot);
}

__global__ void pose_resolve_kernel(const int* __restrict__ key, size_t n, uint8_t* __restrict__ frames) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int v = key[i];
    if (v <= 0) continue;
    const int k = (v - 1) % 3;                                      // arrows: red, green, blue
    uint8_t* p = frames + 3 * i;
    p[0] = k == 2 ? 255 : 0;
    p[1] = k == 1 ? 255 : 0;
    p[2] = k == 0 ? 255 : 0;
  }
}

// ---------------------------------------------------------------------------------------------------------- wireframes
// draw_mesh (demo_utils.py:50-65): cv2.line(img, p, q, EDGE_COLOR, 1, LINE_AA) per edge in order, i.e. cv2's LineAA.  Its
// blends do not commute, so every pixel must see its (box, edge) stamps in order.  A tile CTA owns its pixels in registers
// and walks the boxes, then each box's edges in chunks of blockDim, in order; a walk stamps a pixel at most once, so each
// pixel folds its stamps in exactly cv2's order.  No fragment arena: memory is [R, 5] ints whatever the heads look like.

constexpr int kMeshTile = 32;                          // tile side in pixels
constexpr int kMeshThreads = 256;
constexpr int kMeshPix = kMeshTile * kMeshTile / kMeshThreads;
constexpr int kMeshMargin = 3;                         // covers the 3-pixel stamp and the step one past the second end
constexpr int kMeshWsInts = DAD3D_MESH_WS_INTS;

__constant__ int c_slope_corr[32] = {181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
                                     203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254};
__constant__ int c_filter[64] = {168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
                                 254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
                                 158, 149, 140, 131, 122, 114, 105, 97,  89,  82,  75,  68,  62,  56,  50,  45,
                                 40,  36,  32,  28,  25,  22,  19,  16,  14,  12,  11,  9,   8,   7,   5,   5};

// One LineAA walk: step k = 0..count visits major coordinate m0 + k at minor position minor0 + k * step (16.16).
struct MeshWalk {
  long long minor0, step;
  int m0, count;
  uint16_t ep[9];                                      // the end-point table, indexed min(k, 2) * 3 + min(count - k, 2)
  uint8_t x_major;
};

// LineAA's set-up (drawing.cpp) for integer end points in a w x h image; false when clipLine leaves nothing.
__device__ bool line_aa_walk(long long x1, long long y1, long long x2, long long y2, long long w, long long h,
                             MeshWalk& o) {
  x1 *= kXYOne; y1 *= kXYOne; x2 *= kXYOne; y2 *= kXYOne;
  if (!clip_line(w << kXYShift, h << kXYShift, x1, y1, x2, y2)) return false;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long j = dx < 0 ? -1 : 0, ax = (dx ^ j) - j;
  const long long i = dy < 0 ? -1 : 0, ay = (dy ^ i) - i;
  long long e1, e2;
  o.x_major = ax > ay;
  if (o.x_major) {
    dy = (dy ^ j) - j;
    if (j) {
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    o.step = (dy * kXYOne) / (ax | 1);
    x2 += kXYOne;
    o.count = static_cast<int>((x2 >> kXYShift) - (x1 >> kXYShift));
    y1 += ((o.step * -(x1 & (kXYOne - 1))) >> kXYShift) + (kXYOne >> 1);
    o.m0 = static_cast<int>(x1 >> kXYShift);
    o.minor0 = y1;
    e1 = x1; e2 = x2;
  } else {
    dx = (dx ^ i) - i;
    if (i) {
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    o.step = (dx * kXYOne) / (ay | 1);
    y2 += kXYOne;
    o.count = static_cast<int>((y2 >> kXYShift) - (y1 >> kXYShift));
    x1 += ((o.step * -(y1 & (kXYOne - 1))) >> kXYShift) + (kXYOne >> 1);
    o.m0 = static_cast<int>(y1 >> kXYShift);
    o.minor0 = x1;
    e1 = y1; e2 = y2;
  }
  int slope = static_cast<int>((o.step >> (kXYShift - 5)) & 0x3f);
  slope ^= o.step < 0 ? 0x3f : 0;
  slope = (slope & 0x20) ? 0x100 : c_slope_corr[slope];
  const int fi = static_cast<int>((e1 >> (kXYShift - 7)) & 0x78), fj = static_cast<int>((e2 >> (kXYShift - 7)) & 0x78);
  const int t0 = slope << 7, t1 = ((0x78 - fi) | 4) * slope, t2 = (fj | 4) * slope;
  o.ep[0] = 0;
  o.ep[8] = static_cast<uint16_t>(slope);
  o.ep[1] = o.ep[3] = static_cast<uint16_t>(((((fj - fi) & 0x78) | 4) * slope >> 8) & 0x1ff);
  o.ep[2] = static_cast<uint16_t>((t1 >> 8) & 0x1ff);
  o.ep[4] = static_cast<uint16_t>(((((fj - fi) + 0x80) | 4) * slope >> 8) & 0x1ff);
  o.ep[5] = static_cast<uint16_t>(((t1 + t0) >> 8) & 0x1ff);
  o.ep[6] = static_cast<uint16_t>((t2 >> 8) & 0x1ff);
  o.ep[7] = static_cast<uint16_t>(((t2 + t0) >> 8) & 0x1ff);
  return true;
}

// Per-box pass, one CTA per box: ws[r] = (frame if the box draws, else -1; then the pixel box x0, y0, x1, y1 that its
// stamps can touch, clipped to the frame).  A box draws when its record is valid and every end point of every edge is
// finite and fits int32 after truncation (cv2 raises otherwise, and draw_mesh has no output) -- and it touches the frame.
__global__ void mesh_box_kernel(const float* __restrict__ verts, int nv, int ncomp, const int32_t* __restrict__ edges,
                                int E, const dad3d_roi* __restrict__ rois, int F, int H, int W, int32_t* __restrict__ ws) {
  const int r = blockIdx.x;
  __shared__ long long s_box[4];
  if (threadIdx.x == 0) {
    s_box[0] = s_box[1] = LLONG_MAX;
    s_box[2] = s_box[3] = LLONG_MIN;
  }
  __syncthreads();
  long long x0 = LLONG_MAX, y0 = LLONG_MAX, x1 = LLONG_MIN, y1 = LLONG_MIN;
  bool ok = true;
  const float* v = verts + static_cast<size_t>(r) * nv * ncomp;
  for (int e = threadIdx.x; e < 2 * E && ok; e += blockDim.x) {
    const int idx = edges[e];
    long long x, y;
    if (idx < 0 || idx >= nv || !to_int32(static_cast<double>(v[static_cast<size_t>(idx) * ncomp]), x) ||
        !to_int32(static_cast<double>(v[static_cast<size_t>(idx) * ncomp + 1]), y)) {
      ok = false;
      break;
    }
    x0 = min(x0, x); x1 = max(x1, x);
    y0 = min(y0, y); y1 = max(y1, y);
  }
  const bool all_ok = __syncthreads_and(ok);
  if (x0 <= x1) {
    atomicMin(&s_box[0], x0); atomicMin(&s_box[1], y0);
    atomicMax(&s_box[2], x1); atomicMax(&s_box[3], y1);
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const dad3d_roi q = rois[r];
  const long long bx0 = max(s_box[0] - kMeshMargin, 0LL), by0 = max(s_box[1] - kMeshMargin, 0LL);
  const long long bx1 = min(s_box[2] + kMeshMargin, W - 1LL), by1 = min(s_box[3] + kMeshMargin, H - 1LL);
  const bool draw = q.valid && q.frame >= 0 && q.frame < F && all_ok && E > 0 && bx0 <= bx1 && by0 <= by1;
  int32_t* o = ws + static_cast<size_t>(r) * kMeshWsInts;
  o[0] = draw ? q.frame : -1;
  o[1] = draw ? static_cast<int32_t>(bx0) : 0;
  o[2] = draw ? static_cast<int32_t>(by0) : 0;
  o[3] = draw ? static_cast<int32_t>(bx1) : -1;
  o[4] = draw ? static_cast<int32_t>(by1) : -1;
}

// Exclusive position of this thread's flag among the block's set flags, in thread order; *total = their count.
__device__ __forceinline__ int block_compact(bool flag, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) s_warp[warp] = __popc(m);
  __syncthreads();
  int base = 0, n = 0;
  for (int k = 0; k < kMeshThreads / 32; ++k) {
    base += k < warp ? s_warp[k] : 0;
    n += s_warp[k];
  }
  *total = n;
  return base + __popc(m & ((1u << lane) - 1u));
}

// Tile pass: one CTA per (frame, kMeshTile^2 tile); each thread holds kMeshPix pixels of it in registers.
__global__ void __launch_bounds__(kMeshThreads) mesh_tile_kernel(
    const float* __restrict__ verts, int nv, int ncomp, const int32_t* __restrict__ edges, int E, int R,
    const int32_t* __restrict__ ws, int c0, int c1, int c2, uint8_t* __restrict__ frames, int H, int W, int tiles_x,
    int tiles_y) {
  __shared__ MeshWalk s_walk[kMeshThreads];
  __shared__ int s_box[kMeshThreads];
  __shared__ int s_warp[kMeshThreads / 32];
  __shared__ int s_filter[64];
  if (threadIdx.x < 64) s_filter[threadIdx.x] = c_filter[threadIdx.x];
  const long long t = blockIdx.x;
  const int f = static_cast<int>(t / (static_cast<long long>(tiles_x) * tiles_y));
  const int rem = static_cast<int>(t % (static_cast<long long>(tiles_x) * tiles_y));
  const int tx0 = (rem % tiles_x) * kMeshTile, ty0 = (rem / tiles_x) * kMeshTile;
  const int tx1 = min(tx0 + kMeshTile, W) - 1, ty1 = min(ty0 + kMeshTile, H) - 1;
  uint8_t* img = frames + static_cast<size_t>(f) * H * W * 3;
  int px[kMeshPix], py[kMeshPix], col[kMeshPix][3];
#pragma unroll
  for (int p = 0; p < kMeshPix; ++p) {
    const int l = threadIdx.x + p * kMeshThreads;
    px[p] = tx0 + l % kMeshTile;
    py[p] = ty0 + l / kMeshTile;
    if (px[p] <= tx1 && py[p] <= ty1) {
      const uint8_t* q = img + (static_cast<size_t>(py[p]) * W + px[p]) * 3;
      col[p][0] = q[0]; col[p][1] = q[1]; col[p][2] = q[2];
    } else {
      px[p] = -1;                                      // outside the frame: cv2 never stamps it
    }
  }
  bool dirty = false;
  for (int rb = 0; rb < R; rb += kMeshThreads) {       // the boxes that touch this tile, in order
    const int r = rb + threadIdx.x;
    bool hit = false;
    if (r < R) {
      const int32_t* b = ws + static_cast<size_t>(r) * kMeshWsInts;
      hit = b[0] == f && b[1] <= tx1 && b[3] >= tx0 && b[2] <= ty1 && b[4] >= ty0;
    }
    int nbox;
    const int pos = block_compact(hit, s_warp, &nbox);
    if (hit) s_box[pos] = r;
    __syncthreads();
    for (int bi = 0; bi < nbox; ++bi) {
      const float* v = verts + static_cast<size_t>(s_box[bi]) * nv * ncomp;
      for (int eb = 0; eb < E; eb += kMeshThreads) {   // the box's edges that touch the tile, in order
        const int e = eb + threadIdx.x;
        bool keep = false;
        MeshWalk wk;
        if (e < E) {
          const int a = edges[2 * static_cast<size_t>(e)], b = edges[2 * static_cast<size_t>(e) + 1];
          // the box draws, so both ends are finite and fit int32
          const long long ax = __float2ll_rz(v[static_cast<size_t>(a) * ncomp]);
          const long long ay = __float2ll_rz(v[static_cast<size_t>(a) * ncomp + 1]);
          const long long bx = __float2ll_rz(v[static_cast<size_t>(b) * ncomp]);
          const long long by = __float2ll_rz(v[static_cast<size_t>(b) * ncomp + 1]);
          keep = min(ax, bx) - kMeshMargin <= tx1 && max(ax, bx) + kMeshMargin >= tx0 &&
                 min(ay, by) - kMeshMargin <= ty1 && max(ay, by) + kMeshMargin >= ty0 &&
                 line_aa_walk(ax, ay, bx, by, W, H, wk);
          if (keep) {                                  // the steps inside the tile's major range touch its minor range?
            const int lo = wk.x_major ? tx0 : ty0, hi = wk.x_major ? tx1 : ty1;
            const int mlo = wk.x_major ? ty0 : tx0, mhi = wk.x_major ? ty1 : tx1;
            const long long k0 = max(0LL, static_cast<long long>(lo) - wk.m0);
            const long long k1 = min(static_cast<long long>(wk.count), static_cast<long long>(hi) - wk.m0);
            if (k0 > k1) {
              keep = false;
            } else {
              const long long ya = (wk.minor0 + k0 * wk.step) >> kXYShift, yb = (wk.minor0 + k1 * wk.step) >> kXYShift;
              keep = min(ya, yb) - 1 <= mhi && max(ya, yb) + 1 >= mlo;
            }
          }
        }
        int n;
        const int wpos = block_compact(keep, s_warp, &n);
        if (keep) s_walk[wpos] = wk;
        __syncthreads();
        for (int q = 0; q < n; ++q) {
          const MeshWalk& w = s_walk[q];
#pragma unroll
          for (int p = 0; p < kMeshPix; ++p) {
            if (px[p] < 0) continue;
            const long long k = static_cast<long long>(w.x_major ? px[p] : py[p]) - w.m0;
            if (k < 0 || k > w.count) continue;
            const long long y = w.minor0 + k * w.step;
            const int o = (w.x_major ? py[p] : px[p]) - (static_cast<int>(y >> kXYShift) - 1);
            if (o < 0 || o > 2) continue;
            const int dist = static_cast<int>((y >> (kXYShift - 5)) & 31);
            const int fidx = o == 0 ? dist + 32 : (o == 1 ? dist : 63 - dist);
            const int ei = static_cast<int>(min(k, 2LL) * 3 + min(static_cast<long long>(w.count) - k, 2LL));
            const int al = (w.ep[ei] * s_filter[fidx] >> 8) & 0xff;
            const int cc[3] = {c0, c1, c2};
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {           // cv2 applies the blend twice
              int x = col[p][ch];
              x += ((cc[ch] - x) * al + 127) >> 8;
              x += ((cc[ch] - x) * al + 127) >> 8;
              col[p][ch] = x;
            }
            dirty = true;
          }
        }
        __syncthreads();
      }
    }
    __syncthreads();
  }
  if (!dirty) return;
#pragma unroll
  for (int p = 0; p < kMeshPix; ++p) {
    if (px[p] < 0) continue;
    uint8_t* q = img + (static_cast<size_t>(py[p]) * W + px[p]) * 3;
    q[0] = static_cast<uint8_t>(col[p][0]);
    q[1] = static_cast<uint8_t>(col[p][1]);
    q[2] = static_cast<uint8_t>(col[p][2]);
  }
}

}  // namespace
}  // namespace dad3d

extern "C" int dad3d_overlay_mesh(const float* vertices_d, int32_t R, int32_t nv, int32_t ncomp, const int32_t* edges_d,
                                  int32_t E, const dad3d_roi* rois_d, const uint8_t* color_h, int32_t* ws_d,
                                  uint8_t* frames_d, int32_t F, int32_t H, int32_t W, dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(R >= 0 && E >= 0, "R, E");
  if (R == 0 || E == 0) return DAD3D_OK;
  DAD3D_REQUIRE(vertices_d && edges_d && rois_d && color_h && ws_d && frames_d, "null pointer");
  DAD3D_REQUIRE(nv > 0 && (ncomp == 2 || ncomp == 3) && F > 0 && H > 0 && W > 0 && E <= INT32_MAX / 2, "sizes");
  const long long tiles_x = (W + kMeshTile - 1) / kMeshTile, tiles_y = (H + kMeshTile - 1) / kMeshTile;
  const long long tiles = tiles_x * tiles_y * F;
  DAD3D_REQUIRE(tiles <= INT32_MAX, "too many tiles");
  auto s = reinterpret_cast<cudaStream_t>(stream);
  mesh_box_kernel<<<R, 256, 0, s>>>(vertices_d, nv, ncomp, edges_d, E, rois_d, F, H, W, ws_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  mesh_tile_kernel<<<static_cast<unsigned>(tiles), kMeshThreads, 0, s>>>(
      vertices_d, nv, ncomp, edges_d, E, R, ws_d, color_h[0], color_h[1], color_h[2], frames_d, H, W,
      static_cast<int>(tiles_x), static_cast<int>(tiles_y));
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

extern "C" int dad3d_pose_geometry(const float* params_d, int32_t R, int32_t num_params, int32_t rotation_index,
                                   const dad3d_roi* rois_d, double* rpy_d, int32_t* pose_d, float* rot_d,
                                   dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(R >= 0, "R");
  if (R == 0) return DAD3D_OK;
  DAD3D_REQUIRE(params_d, "null pointer");
  DAD3D_REQUIRE(rotation_index >= 0 && rotation_index + 6 <= num_params, "rotation index");
  DAD3D_REQUIRE((pose_d == nullptr) == (rois_d == nullptr), "pose_d and rois_d go together");
  DAD3D_REQUIRE(rpy_d || pose_d || rot_d, "nothing to write");
  pose_geometry_kernel<<<ceil_div(R, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      params_d, R, num_params, rotation_index, rois_d, rpy_d, pose_d, rot_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

extern "C" int dad3d_overlay_points(const void* points_d, int32_t is_float, int32_t R, int32_t n_src, int32_t ncomp,
                                    const int64_t* index_d, int32_t L, const dad3d_roi* rois_d, int32_t radius,
                                    const uint8_t* color_h, uint8_t* frames_d, int32_t F, int32_t H, int32_t W,
                                    dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(R >= 0 && L >= 0, "R, L");
  if (R == 0 || L == 0) return DAD3D_OK;
  DAD3D_REQUIRE(points_d && rois_d && frames_d && color_h, "null pointer");
  DAD3D_REQUIRE(n_src > 0 && ncomp >= 2 && radius >= 0 && F > 0 && H > 0 && W > 0, "sizes");
  DAD3D_REQUIRE(index_d || L <= n_src, "L > n_src without an index");
  dim3 grid(ceil_div(L, 128), R < 65535 ? R : 65535);
  overlay_points_kernel<<<grid, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      points_d, is_float ? 1 : 0, R, n_src, ncomp, index_d, L, rois_d, radius, color_h[0], color_h[1], color_h[2],
      frames_d, F, H, W);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

extern "C" int dad3d_overlay_pose(const int32_t* pose_d, int32_t R, int32_t* key_ws_d, uint8_t* frames_d, int32_t F,
                                  int32_t H, int32_t W, dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(R >= 0, "R");
  if (R == 0) return DAD3D_OK;
  DAD3D_REQUIRE(pose_d && key_ws_d && frames_d, "null pointer");
  DAD3D_REQUIRE(F > 0 && H > 0 && W > 0 && R <= (INT32_MAX - 3) / 3, "sizes");
  auto s = reinterpret_cast<cudaStream_t>(stream);
  const size_t n = static_cast<size_t>(F) * H * W;
  DAD3D_CUDA_OK(cudaMemsetAsync(key_ws_d, 0, n * sizeof(int32_t), s));
  const long long threads = 9LL * R;
  pose_raster_kernel<<<static_cast<unsigned>((threads + 127) / 128), 128, 0, s>>>(pose_d, R, key_ws_d, F, H, W);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  const size_t blocks = (n + 255) / 256;
  pose_resolve_kernel<<<static_cast<unsigned>(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, s>>>(key_ws_d, n, frames_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}
