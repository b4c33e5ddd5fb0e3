// Per-pixel arithmetic of the letter-box pre-processing, shared by preprocess_kernel (whole images, preprocess.cu) and
// preprocess_rois_kernel (crops of whole frames, roi.cu): the reference's albumentations pipeline
//   LongestMaxSize(256, cv2.INTER_LINEAR on uint8) -> PadIfNeeded(256, 256, constant 0, centred) -> Normalize(imagenet)
//   -> HWC->CHW   (predictor.py:195-203, :85-89).
// The bilinear resize restates OpenCV's 8-bit fixed-point path bit-exactly (11-bit coefficients, horizontal taps clamped
// with zeroed fraction, vertical taps clamped by row index only, two-step rounded vertical blend); the normalisation
// uses the same two fp32 roundings as albumentations (subtract mean*255, multiply by 1/(std*255)).
#pragma once
#include <cstdint>

namespace dad3d {

// Where one source image (or crop) lands in the S x S letter-box.  H, W: the source's size, which is where bilinear taps
// clamp; nh, nw: its resized size; top, left: the PadIfNeeded offsets; scale_x/y: cv::resize's 1 / (new / old).
struct LetterboxGeom {
  int H, W, nh, nw, top, left, do_resize;
  double scale_x, scale_y;
};

__device__ __forceinline__ void lin_coeff(int d, double scale, int n_src, bool clamp_frac, int* s0, int* s1, int* a0, int* a1) {
  float f = static_cast<float>((static_cast<double>(d) + 0.5) * scale - 0.5);
  int s = static_cast<int>(floorf(f));
  f -= static_cast<float>(s);
  if (clamp_frac) {                         // cv::resize horizontal pass: out-of-range taps collapse onto the border pixel
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n_src - 1) { f = 0.f; s = n_src - 1; }
  }
  int c0 = __float2int_rn((1.f - f) * 2048.f);     // saturate_cast<short>(float): round half to even
  int c1 = __float2int_rn(f * 2048.f);
  c0 = max(-32768, min(32767, c0));
  c1 = max(-32768, min(32767, c1));
  *a0 = c0;
  *a1 = c1;
  *s0 = max(0, min(n_src - 1, s));                  // vertical pass: rows are clamped, the fraction is kept
  *s1 = max(0, min(n_src - 1, s + 1));
}

// uint8 RGB value of letter-box pixel (x, y); img points at the source's first pixel and its rows are `pitch` bytes apart.
// Pixels outside the resized image are the constant-0 padding (img is not read).
__device__ __forceinline__ void letterbox_pixel(const uint8_t* __restrict__ img, size_t pitch, const LetterboxGeom& g, int x,
                                                int y, int v[3]) {
  v[0] = v[1] = v[2] = 0;
  const int dx = x - g.left, dy = y - g.top;
  if (dx < 0 || dx >= g.nw || dy < 0 || dy >= g.nh) return;
  if (!g.do_resize) {
    const uint8_t* s = img + static_cast<size_t>(dy) * pitch + static_cast<size_t>(dx) * 3;
    v[0] = s[0]; v[1] = s[1]; v[2] = s[2];
    return;
  }
  int sx0, sx1, ax0, ax1, sy0, sy1, ay0, ay1;
  lin_coeff(dx, g.scale_x, g.W, true, &sx0, &sx1, &ax0, &ax1);
  lin_coeff(dy, g.scale_y, g.H, false, &sy0, &sy1, &ay0, &ay1);
  const uint8_t* r0 = img + static_cast<size_t>(sy0) * pitch;
  const uint8_t* r1 = img + static_cast<size_t>(sy1) * pitch;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = r0[sx0 * 3 + c] * ax0 + r0[sx1 * 3 + c] * ax1;
    const int h1 = r1[sx0 * 3 + c] * ax0 + r1[sx1 * 3 + c] * ax1;
    const int r = ((((ay0 * (h0 >> 4)) >> 16) + ((ay1 * (h1 >> 4)) >> 16) + 2) >> 2);
    v[c] = max(0, min(255, r));
  }
}

// Normalise and store pixel (x, y) into a [3,S,S] fp32 plane set.
__device__ __forceinline__ void store_normalised(float* __restrict__ out, int S, int x, int y, const int v[3],
                                                 const float mean[3], const float inv_std[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c)
    out[(static_cast<size_t>(c) * S + y) * S + x] = __fmul_rn(__fsub_rn(static_cast<float>(v[c]), mean[c]), inv_std[c]);
}

}  // namespace dad3d
