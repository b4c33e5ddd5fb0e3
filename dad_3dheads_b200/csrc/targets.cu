// Training targets (include/dad3d.h "training targets"): what the reference's FlameDataset computes per item after the crop
// (model_training/data/flame_dataset.py:115-200), for a whole batch on the device.
// The projection and keypoint chain restates numpy's float32 expressions in an explicit operation order with _rn
// intrinsics, so tests/targets_model.py can restate it bit for bit: nvcc would otherwise contract a * b + c into an fma
// where numpy rounds twice.  The reference's 4x4 matmuls go through BLAS sgemm, whose order and fma use depend on the host
// CPU and the BLAS build; the kernel takes the order of OpenBLAS's x86 kernels (an fma chain over k), which is what numpy
// runs on common hosts, but no order matches every BLAS.
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"

namespace dad3d {

// row r of the float32 product m @ [x, y, z, w] (m row-major 4x4): one product, then an fma per term in k order -- the
// order OpenBLAS's x86 sgemm kernels take for numpy's float32 matmul
__device__ __forceinline__ float mat_row(const float* m, int r, float x, float y, float z, float w) {
  const float* q = m + 4 * r;
  return __fmaf_rn(q[3], w, __fmaf_rn(q[2], z, __fmaf_rn(q[1], y, __fmul_rn(q[0], x))));
}

// _load_mesh (flame_dataset.py:115-128): world_homo = model_view @ [v, 1]
__device__ __forceinline__ float4 to_world(const float* mv, const float* v) {
  const float x = v[0], y = v[1], z = v[2];
  return make_float4(mat_row(mv, 0, x, y, z, 1.f), mat_row(mv, 1, x, y, z, 1.f), mat_row(mv, 2, x, y, z, 1.f),
                     mat_row(mv, 3, x, y, z, 1.f));
}

struct HeadGeom {
  int crop_x, crop_y, frame_h, w, h, pre_left, pre_top;
  float scale;                    // fp32(img_size / max(h, w)): numpy rounds the Python-float scale to the keypoint's fp32
};

// _project_vertices_onto_image (flame_dataset.py:130-141) -> crop pixels: fp32 P @ X, divide by w, fp32 height - y, then
// `-= (x, y)` of the crop, which numpy computes in float64 (float32 array minus an int32 array) and stores as float32.
__device__ __forceinline__ float2 project(const float* P, float4 X, const HeadGeom& g) {
  const float cx = mat_row(P, 0, X.x, X.y, X.z, X.w), cy = mat_row(P, 1, X.x, X.y, X.z, X.w);
  const float cw = mat_row(P, 3, X.x, X.y, X.z, X.w);
  const float px = __fdiv_rn(cx, cw);
  const float py = __fsub_rn(static_cast<float>(g.frame_h), __fdiv_rn(cy, cw));
  return make_float2(__double2float_rn(__dsub_rn(static_cast<double>(px), static_cast<double>(g.crop_x))),
                     __double2float_rn(__dsub_rn(static_cast<double>(py), static_cast<double>(g.crop_y))));
}

// albumentations 1.0.0 keypoint path under numpy 2 / NEP 50: LongestMaxSize x * s and PadIfNeeded + pad, each in fp32
__device__ __forceinline__ float2 to_network(float2 p, const HeadGeom& g) {
  return make_float2(__fadd_rn(__fmul_rn(p.x, g.scale), static_cast<float>(g.pre_left)),
                     __fadd_rn(__fmul_rn(p.y, g.scale), static_cast<float>(g.pre_top)));
}

// one CTA per head
__global__ void __launch_bounds__(256) targets_kernel(const float* __restrict__ verts, const float* __restrict__ model_view,
                                                      const float* __restrict__ projection, const int32_t* __restrict__ origins,
                                                      const dad3d_roi* __restrict__ rois, int V,
                                                      const int32_t* __restrict__ lm_index, const int32_t* __restrict__ lm_tri,
                                                      const float* __restrict__ lm_bary, int C, int S,
                                                      float* __restrict__ keypoints, float* __restrict__ landmarks,
                                                      float* __restrict__ landmarks_norm, uint8_t* __restrict__ presence) {
  __shared__ float mats[32];
  const int b = blockIdx.x;
  if (threadIdx.x < 32)
    mats[threadIdx.x] = threadIdx.x < 16 ? model_view[b * 16 + threadIdx.x] : projection[b * 16 + threadIdx.x - 16];
  __syncthreads();
  const float* mv = mats;
  const float* P = mats + 16;
  const dad3d_roi q = rois[b];
  HeadGeom g;
  g.crop_x = origins[3 * b];
  g.crop_y = origins[3 * b + 1];
  g.frame_h = origins[3 * b + 2];
  g.w = q.w;
  g.h = q.h;
  g.pre_left = q.pre_left;
  g.pre_top = q.pre_top;
  g.scale = __double2float_rn(q.scale);
  const float* v_b = verts + static_cast<size_t>(b) * V * 3;
  float2* kp = reinterpret_cast<float2*>(keypoints) + static_cast<size_t>(b) * V;
  for (int i = threadIdx.x; i < V; i += blockDim.x) kp[i] = to_network(project(P, to_world(mv, v_b + 3 * i), g), g);
  for (int l = threadIdx.x; l < C; l += blockDim.x) {
    float4 X;
    if (lm_tri) {
      // get_68_landmarks (data/utils.py:120-206) on world_homo[..., :3]: torch's fp32 sum of three products, left to right,
      // then [lm, 1]
      float acc[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float4 w = to_world(mv, v_b + 3 * lm_tri[3 * l + k]);
        const float bk = lm_bary[3 * l + k];
        const float t[3] = {__fmul_rn(w.x, bk), __fmul_rn(w.y, bk), __fmul_rn(w.z, bk)};
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] = k == 0 ? t[c] : __fadd_rn(acc[c], t[c]);
      }
      X = make_float4(acc[0], acc[1], acc[2], 1.f);
    } else {
      X = to_world(mv, v_b + 3 * lm_index[l]);      // world_homo[indices]: the computed w is kept
    }
    const float2 c = project(P, X, g);
    // _get_2d_landmarks_w_presence (flame_dataset.py:166-170): strictly inside the crop, before any resize
    const bool in = c.x > 0.f && c.x < static_cast<float>(g.w) && c.y > 0.f && c.y < static_cast<float>(g.h);
    const float2 n = to_network(c, g);
    const size_t o = static_cast<size_t>(b) * C + l;
    reinterpret_cast<float2*>(landmarks)[o] = n;
    reinterpret_cast<float2*>(landmarks_norm)[o] =
        make_float2(__fdiv_rn(n.x, static_cast<float>(S)), __fdiv_rn(n.y, static_cast<float>(S)));
    presence[o] = in ? 1 : 0;
  }
}

// numpy's float32 floor division (npy_divmodf), then int(): the heat-map cell of one coordinate.  false when int() would
// raise (not finite); cells far outside the plane are clamped to +-2^24, where every window is already empty.
__device__ __forceinline__ bool heat_cell(float p, float stride, int* cell) {
  if (!isfinite(p)) return false;
  const float mod = fmodf(p, stride);
  float div = __fdiv_rn(__fsub_rn(p, mod), stride);
  if (mod != 0.f && ((stride < 0.f) != (mod < 0.f))) div = __fsub_rn(div, 1.f);
  float fl = 0.f;
  if (div != 0.f) {
    fl = floorf(div);
    if (__fsub_rn(div, fl) > 0.5f) fl = __fadd_rn(fl, 1.f);
  }
  *cell = static_cast<int>(fminf(fmaxf(fl, -16777216.f), 16777216.f));
  return true;
}

// Python's slice bound normalisation for a sequence of length n
__device__ __forceinline__ int slice_bound(int i, int n) { return i < 0 ? max(i + n, 0) : min(i, n); }

// draw_gaussian (data/utils.py:51-70) along one axis: the plane range [h0, h0 + n) takes window entries [g0, g0 + n)
struct Span {
  int h0, g0, n;
};

__device__ __forceinline__ Span window_span(int c, int r, int S, int D) {
  const int lo = min(c, r), hi = min(S - c, r + 1);
  const int hs = slice_bound(c - lo, S), he = slice_bound(c + hi, S);
  const int gs = slice_bound(r - lo, D), ge = slice_bound(r + hi, D);
  Span s;
  s.h0 = hs;
  s.g0 = gs;
  s.n = he - hs == ge - gs ? max(he - hs, 0) : 0;    // both ranges have one length for every cell (swept in the tests)
  return s;
}

struct Window {
  Span x, y;
};

__device__ __forceinline__ uint32_t heat_byte(int yy, int xx, const Window& w, const uint8_t* __restrict__ table, int D) {
  const int dy = yy - w.y.h0, dx = xx - w.x.h0;
  if (static_cast<unsigned>(dy) < static_cast<unsigned>(w.y.n) && static_cast<unsigned>(dx) < static_cast<unsigned>(w.x.n))
    return __ldg(&table[(w.y.g0 + dy) * D + w.x.g0 + dx]);
  return 0u;
}

// one CTA per plane: every byte of the plane is written, the aligned body with 16-byte stores
__global__ void __launch_bounds__(256) heatmap_kernel(const float* __restrict__ landmarks, const uint8_t* __restrict__ presence,
                                                      int S, float stride, const uint8_t* __restrict__ table, int radius,
                                                      uint8_t* __restrict__ out) {
  const size_t p = blockIdx.x;
  const int D = 2 * radius + 1;
  Window w;
  w.x.n = w.y.n = 0;
  int cx, cy;
  const float2 lm = reinterpret_cast<const float2*>(landmarks)[p];
  if (presence[p] && heat_cell(lm.x, stride, &cx) && heat_cell(lm.y, stride, &cy)) {
    w.x = window_span(cx, radius, S, D);
    w.y = window_span(cy, radius, S, D);
    if (w.x.n == 0 || w.y.n == 0) w.x.n = w.y.n = 0;
  }
  const int n = S * S;
  uint8_t* plane = out + p * static_cast<size_t>(n);
  const int head = min(n, static_cast<int>((16u - (reinterpret_cast<uintptr_t>(plane) & 15u)) & 15u));
  const int body = (n - head) / 16;
  for (int i = threadIdx.x; i < head; i += blockDim.x) plane[i] = heat_byte(i / S, i % S, w, table, D);
  uint4* vec = reinterpret_cast<uint4*>(plane + head);
  for (int j = threadIdx.x; j < body; j += blockDim.x) {
    const int i0 = head + 16 * j;
    int yy = i0 / S, xx = i0 - yy * S;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (w.y.n > 0 && (i0 + 15) / S >= w.y.h0 && yy < w.y.h0 + w.y.n) {
      uint32_t word[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        word[k >> 2] |= heat_byte(yy, xx, w, table, D) << (8 * (k & 3));
        if (++xx == S) {
          xx = 0;
          ++yy;
        }
      }
      v = make_uint4(word[0], word[1], word[2], word[3]);
    }
    vec[j] = v;
  }
  for (int i = head + 16 * body + threadIdx.x; i < n; i += blockDim.x) plane[i] = heat_byte(i / S, i % S, w, table, D);
}

}  // namespace dad3d

extern "C" int dad3d_training_targets(const float* vertices_d, const float* model_view_d, const float* projection_d,
                                      const int32_t* origins_d, const dad3d_roi* rois_d, int32_t B, int32_t V,
                                      const int32_t* lm_index_d, const int32_t* lm_tri_d, const float* lm_bary_d, int32_t C,
                                      int32_t img_size, float* keypoints_d, float* landmarks_d, float* landmarks_norm_d,
                                      uint8_t* presence_d, dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(B >= 0, "B");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(vertices_d && model_view_d && projection_d && origins_d && rois_d && keypoints_d && landmarks_d &&
                    landmarks_norm_d && presence_d, "null pointer");
  DAD3D_REQUIRE(V > 0 && C > 0 && img_size > 0, "sizes");
  DAD3D_REQUIRE((lm_index_d != nullptr) != (lm_tri_d != nullptr), "exactly one of lm_index_d and lm_tri_d");
  DAD3D_REQUIRE(!lm_tri_d || lm_bary_d, "lm_tri_d needs lm_bary_d");
  targets_kernel<<<B, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(vertices_d, model_view_d, projection_d, origins_d,
                                                                        rois_d, V, lm_index_d, lm_tri_d, lm_bary_d, C,
                                                                        img_size, keypoints_d, landmarks_d, landmarks_norm_d,
                                                                        presence_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

extern "C" int dad3d_heatmap_targets(const float* landmarks_d, const uint8_t* presence_d, int32_t planes, int32_t S,
                                     int32_t stride, const uint8_t* table_d, int32_t radius, uint8_t* out_d,
                                     dad3d_stream stream) {
  using namespace dad3d;
  DAD3D_REQUIRE(planes >= 0, "planes");
  if (planes == 0) return DAD3D_OK;
  DAD3D_REQUIRE(landmarks_d && presence_d && table_d && out_d, "null pointer");
  DAD3D_REQUIRE(S > 0 && S <= 32768 && stride > 0 && radius >= 0 && radius <= 1024, "sizes");
  heatmap_kernel<<<planes, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(landmarks_d, presence_d, S,
                                                                             static_cast<float>(stride), table_d, radius,
                                                                             out_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}
