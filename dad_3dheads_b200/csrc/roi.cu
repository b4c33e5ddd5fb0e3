// Heads from boxes in whole frames (include/dad3d.h "heads from boxes"): crop geometry, letter-box pre-processing of the
// crops read in place from the frames, and the read-back of the encoder's outputs into frame pixels.  Every value that
// depends on a box is computed here on the device, so a captured graph replays correctly with new boxes.
// Arithmetic that restates the reference's float64 / fp32 expressions uses explicit _rn intrinsics: nvcc would otherwise
// contract a - b * c into an fma, which rounds once where numpy and torch round twice.
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"
#include "letterbox.cuh"

namespace dad3d {

struct Extend {
  double left, right, top, bottom;
};

__global__ void roi_setup_kernel(const int32_t* __restrict__ boxes, const int32_t* __restrict__ frame_index, int R, int F,
                                 int H, int W, int S, Extend e, dad3d_roi* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const double bx = boxes[4 * r], by = boxes[4 * r + 1], bw = boxes[4 * r + 2], bh = boxes[4 * r + 3];
  // extend_bbox (data/utils.py:73-100): float64, then astype(int32) truncates toward zero
  long long x = __double2int_rz(__dsub_rn(bx, __dmul_rn(bw, e.left)));
  long long y = __double2int_rz(__dsub_rn(by, __dmul_rn(bh, e.top)));
  const long long w = __double2int_rz(__dmul_rn(bw, __dadd_rn(__dadd_rn(1.0, e.right), e.left)));
  const long long h = __double2int_rz(__dmul_rn(bh, __dadd_rn(__dadd_rn(1.0, e.top), e.bottom)));
  // ensure_bbox_boundaries (data/utils.py:103-115): x2 from the CLIPPED x1 plus the original w
  x = min(max(0LL, x), static_cast<long long>(W));
  y = min(max(0LL, y), static_cast<long long>(H));
  const long long x2 = min(max(0LL, x + w), static_cast<long long>(W));
  const long long y2 = min(max(0LL, y + h), static_cast<long long>(H));
  dad3d_roi q;
  q.x = static_cast<int>(x);
  q.y = static_cast<int>(y);
  q.w = static_cast<int>(x2 - x);
  q.h = static_cast<int>(y2 - y);
  q.frame = frame_index ? frame_index[r] : 0;
  q.valid = q.frame >= 0 && q.frame < F && q.w > 0 && q.h > 0;
  q.new_h = q.new_w = 0;
  q.scale = 1.0;
  if (q.valid) {                                     // FaceMeshPredictor._get_paddings (predictor.py:117-123)
    q.scale = __ddiv_rn(static_cast<double>(S), static_cast<double>(max(q.h, q.w)));
    q.new_h = static_cast<int>(rint(__dmul_rn(static_cast<double>(q.h), q.scale)));    // py3round: half to even
    q.new_w = static_cast<int>(rint(__dmul_rn(static_cast<double>(q.w), q.scale)));
    if (q.new_h < 1 || q.new_w < 1) {
      q.valid = 0;
      q.new_h = q.new_w = 0;
      q.scale = 1.0;
    }
  }
  q.pre_top = q.new_h < S ? (S - q.new_h) / 2 : 0;           // PadIfNeeded centring
  q.pre_left = q.new_w < S ? (S - q.new_w) / 2 : 0;
  const int side = max(q.new_h, q.new_w);                      // calculate_paddings (model/utils.py:71-77)
  q.post_top = (side - q.new_h) / 2;
  q.post_left = (side - q.new_w) / 2;
  if (!q.valid) q.pre_top = q.pre_left = q.post_top = q.post_left = 0;
  q.inv_scale_x = q.valid ? __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(q.new_w), q.w)) : 1.0;   // cv::resize
  q.inv_scale_y = q.valid ? __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(q.new_h), q.h)) : 1.0;
  out[r] = q;
}

// blockIdx.z = ROI; frames [F,H,W,3] uint8 -> out [R,3,S,S] fp32
__global__ void preprocess_rois_kernel(const uint8_t* __restrict__ frames, int H, int W, const dad3d_roi* __restrict__ rois,
                                       int S, float mean0, float mean1, float mean2, float inv0, float inv1, float inv2,
                                       float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= S || y >= S) return;
  const dad3d_roi q = rois[blockIdx.z];
  LetterboxGeom g;
  g.H = q.h; g.W = q.w; g.nh = q.new_h; g.nw = q.new_w; g.top = q.pre_top; g.left = q.pre_left;
  g.do_resize = (q.new_h != q.h || q.new_w != q.w) ? 1 : 0;
  g.scale_x = q.inv_scale_x; g.scale_y = q.inv_scale_y;
  const size_t pitch = static_cast<size_t>(W) * 3;
  const uint8_t* img = q.valid ? frames + (static_cast<size_t>(q.frame) * H + q.y) * pitch + static_cast<size_t>(q.x) * 3
                               : nullptr;        // invalid: new_h = new_w = 0, every pixel is padding and img is not read
  int v[3];
  letterbox_pixel(img, pitch, g, x, y, v);
  const float mean[3] = {mean0, mean1, mean2}, inv_std[3] = {inv0, inv1, inv2};
  store_normalised(out + static_cast<size_t>(blockIdx.z) * 3 * S * S, S, x, y, v, mean, inv_std);
}

// one block per head
__global__ void readjust_rois_kernel(const float* params, const float* __restrict__ lms,
                                     const dad3d_roi* __restrict__ rois, int P, int L, int si, int ti, int S,
                                     float* params_out, int64_t* __restrict__ points) {
  const int r = blockIdx.x;
  const dad3d_roi q = rois[r];
  const float scale = __double2float_rn(q.scale);       // torch rounds the Python-float scale to the tensor's fp32
  const float Sf = static_cast<float>(S);
  const float* p_in = params + static_cast<size_t>(r) * P;
  float* p_out = params_out + static_cast<size_t>(r) * P;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    float v = p_in[i];
    if (i == si) {                                      // readjust_3dmm_to_the_input_image (predictor.py:154-176)
      v = __fsub_rn(__fdiv_rn(__fadd_rn(v, 1.f), scale), 1.f);
    } else if (i == ti + 2) {
      v = 0.f;                                          // reprojected_vertices zeroes translation z in place
    } else if (i == ti || i == ti + 1) {
      const bool is_x = i == ti;
      const float pad = __fdiv_rn(__fmul_rn(static_cast<float>(is_x ? q.post_left : q.post_top), 2.f), Sf);
      v = __fsub_rn(__fdiv_rn(__fsub_rn(__fadd_rn(v, 1.f), pad), scale), 1.f);
      const float off = __fdiv_rn(__fmul_rn(static_cast<float>(is_x ? q.x : q.y), 2.f), Sf);   // crop -> frame
      v = __fadd_rn(v, off);
    }
    p_out[i] = v;
  }
  const float* l_in = lms + static_cast<size_t>(r) * L * 2;
  int64_t* pts = points + static_cast<size_t>(r) * L * 2;
  for (int j = threadIdx.x; j < 2 * L; j += blockDim.x) {
    const bool is_x = (j & 1) == 0;
    const float l = fminf(fmaxf(__fmul_rn(l_in[j], 256.f), 0.f), 256.f);         // fp32 (predictor.py:108,128)
    const double d = __ddiv_rn(__dsub_rn(static_cast<double>(l), static_cast<double>(is_x ? q.post_left : q.post_top)),
                               q.scale);                                             // float64 (predictor.py:144-150)
    pts[j] = static_cast<int64_t>(d) + (is_x ? q.x : q.y);
  }
}

}  // namespace dad3d

extern "C" int dad3d_roi_setup(const int32_t* boxes_d, const int32_t* frame_index_d, int32_t R, int32_t F, int32_t H, int32_t W,
                               int32_t img_size, const double* extend_h, dad3d_roi* rois_d, dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(R >= 0, "R");
  if (R == 0) return DAD3D_OK;
  DAD3D_REQUIRE(boxes_d && rois_d && extend_h, "null pointer");
  DAD3D_REQUIRE(F > 0 && H > 0 && W > 0 && img_size > 0, "sizes");
  const Extend e{extend_h[0], extend_h[1], extend_h[2], extend_h[3]};
  roi_setup_kernel<<<ceil_div(R, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(boxes_d, frame_index_d, R, F, H, W,
                                                                                        img_size, e, rois_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

extern "C" int dad3d_preprocess_rois(const uint8_t* frames_d, int32_t H, int32_t W, const dad3d_roi* rois_d, int32_t R,
                                     int32_t img_size, const float* mean255_h, const float* inv_std255_h, float* out_d,
                                     dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(R >= 0 && R <= 65535, "R (at most 65535 ROIs per call)");
  if (R == 0) return DAD3D_OK;
  DAD3D_REQUIRE(frames_d && rois_d && out_d && mean255_h && inv_std255_h, "null pointer");
  DAD3D_REQUIRE(H > 0 && W > 0 && img_size > 0, "sizes");
  dim3 block(32, 8), grid(ceil_div(img_size, 32), ceil_div(img_size, 8), R);
  preprocess_rois_kernel<<<grid, block, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      frames_d, H, W, rois_d, img_size, mean255_h[0], mean255_h[1], mean255_h[2], inv_std255_h[0], inv_std255_h[1],
      inv_std255_h[2], out_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

extern "C" int dad3d_readjust_rois(const float* params_d, const float* landmarks_d, const dad3d_roi* rois_d, int32_t R,
                                   int32_t num_params, int32_t num_landmarks, int32_t scale_index, int32_t translation_index,
                                   int32_t img_size, float* params_out_d, int64_t* points_d, dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(R >= 0, "R");
  if (R == 0) return DAD3D_OK;
  DAD3D_REQUIRE(params_d && landmarks_d && rois_d && params_out_d && points_d, "null pointer");
  DAD3D_REQUIRE(num_params > 0 && num_landmarks > 0 && img_size > 0, "sizes");
  DAD3D_REQUIRE(scale_index >= 0 && scale_index < num_params && translation_index >= 0 &&
                    translation_index + 3 <= num_params, "scale / translation index");
  readjust_rois_kernel<<<R, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(params_d, landmarks_d, rois_d, num_params,
                                                                              num_landmarks, scale_index, translation_index,
                                                                              img_size, params_out_d, points_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}
