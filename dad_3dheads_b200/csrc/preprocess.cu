// Device-side image pre-processing (SURVEY §8f "next" row 2): the letter-box of letterbox.cuh in one kernel per image batch:
// uint8 RGB [H,W,3] (device) -> fp32 [3,S,S] slot of the encoder's input batch.
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"
#include "letterbox.cuh"

namespace dad3d {

struct PreParams {
  LetterboxGeom g;
  int S;
  float mean[3], inv_std[3];
};

// blockIdx.z = image of a same-sized batch ([B,H,W,3] uint8 -> [B,3,S,S] fp32); a single image is the B = 1 case
__global__ void preprocess_kernel(const uint8_t* __restrict__ img, PreParams p, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= p.S || y >= p.S) return;
  img += static_cast<size_t>(blockIdx.z) * p.g.H * p.g.W * 3;
  out += static_cast<size_t>(blockIdx.z) * 3 * p.S * p.S;
  int v[3];
  letterbox_pixel(img, static_cast<size_t>(p.g.W) * 3, p.g, x, y, v);
  store_normalised(out, p.S, x, y, v, p.mean, p.inv_std);
}

}  // namespace dad3d

extern "C" int dad3d_preprocess(const uint8_t* image_d, int32_t H, int32_t W, int32_t new_h, int32_t new_w, int32_t img_size,
                                const float* mean255_h, const float* inv_std255_h, float* out_d, dad3d_stream stream) {
  return dad3d_preprocess_batch(image_d, 1, H, W, new_h, new_w, img_size, mean255_h, inv_std255_h, out_d, stream);
}

extern "C" int dad3d_preprocess_batch(const uint8_t* images_d, int32_t B, int32_t H, int32_t W, int32_t new_h, int32_t new_w,
                                      int32_t img_size, const float* mean255_h, const float* inv_std255_h, float* out_d,
                                      dad3d_stream stream) {
  using namespace dad3d;
  if (B == 0) return DAD3D_OK;
  const uint8_t* image_d = images_d;
  DAD3D_REQUIRE(B > 0 && B <= 65535, "batch");
  DAD3D_REQUIRE(image_d && out_d && mean255_h && inv_std255_h, "null pointer");
  DAD3D_REQUIRE(H > 0 && W > 0 && new_h > 0 && new_w > 0 && new_h <= img_size && new_w <= img_size, "sizes");
  PreParams p;
  p.g.H = H; p.g.W = W; p.g.nh = new_h; p.g.nw = new_w; p.S = img_size;
  p.g.top = new_h < img_size ? static_cast<int>((img_size - new_h) / 2.0) : 0;     // PadIfNeeded centring
  p.g.left = new_w < img_size ? static_cast<int>((img_size - new_w) / 2.0) : 0;
  p.g.do_resize = (new_h != H || new_w != W) ? 1 : 0;
  p.g.scale_x = 1.0 / (static_cast<double>(new_w) / W);                             // cv::resize: 1 / inv_scale_x
  p.g.scale_y = 1.0 / (static_cast<double>(new_h) / H);
  for (int c = 0; c < 3; ++c) { p.mean[c] = mean255_h[c]; p.inv_std[c] = inv_std255_h[c]; }
  dim3 block(32, 8), grid(ceil_div(img_size, 32), ceil_div(img_size, 8), B);
  preprocess_kernel<<<grid, block, 0, reinterpret_cast<cudaStream_t>(stream)>>>(image_d, p, out_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}
