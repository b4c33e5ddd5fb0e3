// The demo's UV texture of every boxed head (inference/uv_texture.py:21-47) in two kernels per call.
//
// uv_normals_kernel: one thread per (head, vertex) -> the z component of psbody's Mesh.estimate_vertex_normals: the face
//   normals cross(v[f1] - v[f0], v[f2] - v[f0]) summed over the vertex's faces in ascending face index (the rows of
//   faces_by_vertex(as_sparse_matrix=True) times the dense normals, as scipy's csr_matvecs sums them), divided by
//   sqrt((nx^2 + ny^2) + nz^2), a norm of 0 replaced by 1.
// uv_texels_kernel: one thread per (head, output texel) -> the texel's 3 bytes: the barycentric point and normal z of the
//   texel's table entry, the back-face test, rint, the strict bounds test and the copy of the source pixel; 0 for texels
//   without an entry, rejected texels and invalid heads.
// All arithmetic is fp64, as psbody's float64 Mesh.v; every operation is an explicit __d*_rn, so nothing is contracted and the
// kernels equal tests/uv_model.py bit for bit.  Texels are distinct in the table, so no two threads write one byte.

#include <climits>
#include <cstdint>
#include <vector>

#include "../../include/dad3d.h"
#include "common.h"

struct dad3d_uv {
  int32_t S = 0, V = 0, NF = 0, device = 0;
  int32_t* vid_d = nullptr;        // [S*S, 3] vertex ids of each texel's entry; -1 in slot 0: no entry
  double* bary_d = nullptr;        // [S*S, 3] its barycentrics
  int32_t* faces_d = nullptr;      // [NF, 3]
  int32_t* row_d = nullptr;        // [V + 1] CSR rows: where each vertex's faces start
  int32_t* col_d = nullptr;        // [nnz] face ids, ascending within a row
  double* mult_d = nullptr;        // [nnz] how many times the face lists the vertex (the CSR's summed 1.0 entries)
};

namespace dad3d {
namespace {

constexpr int kNormalThreads = 128;
constexpr int kTexelThreads = 256;

__device__ __forceinline__ double3 vtx(const float* __restrict__ v, int i) {
  return make_double3(static_cast<double>(v[3 * i]), static_cast<double>(v[3 * i + 1]),
                      static_cast<double>(v[3 * i + 2]));
}

__device__ __forceinline__ bool head_ok(const uint8_t* valid, const int32_t* frame_index, int r, int F, int* frame) {
  const int f = frame_index ? frame_index[r] : 0;
  *frame = f;
  return (!valid || valid[r]) && f >= 0 && f < F;
}

__global__ void __launch_bounds__(kNormalThreads)
uv_normals_kernel(const float* __restrict__ verts, int V, const uint8_t* __restrict__ valid,
                  const int32_t* __restrict__ frame_index, int F, const int32_t* __restrict__ faces,
                  const int32_t* __restrict__ row, const int32_t* __restrict__ col, const double* __restrict__ mult,
                  double* __restrict__ nz_out) {
  const int i = blockIdx.x * kNormalThreads + threadIdx.x;
  const int r = blockIdx.y;
  int frame;
  if (i >= V || !head_ok(valid, frame_index, r, F, &frame)) return;
  const float* v = verts + static_cast<size_t>(r) * V * 3;
  double sx = 0.0, sy = 0.0, sz = 0.0;
  for (int e = row[i]; e < row[i + 1]; ++e) {
    const int f = col[e];
    const double3 p0 = vtx(v, faces[3 * f]), p1 = vtx(v, faces[3 * f + 1]), p2 = vtx(v, faces[3 * f + 2]);
    const double ax = __dsub_rn(p1.x, p0.x), ay = __dsub_rn(p1.y, p0.y), az = __dsub_rn(p1.z, p0.z);
    const double bx = __dsub_rn(p2.x, p0.x), by = __dsub_rn(p2.y, p0.y), bz = __dsub_rn(p2.z, p0.z);
    const double nx = __dsub_rn(__dmul_rn(ay, bz), __dmul_rn(az, by));
    const double ny = __dsub_rn(__dmul_rn(az, bx), __dmul_rn(ax, bz));
    const double nz = __dsub_rn(__dmul_rn(ax, by), __dmul_rn(ay, bx));
    const double m = mult[e];
    sx = __dadd_rn(sx, __dmul_rn(m, nx));
    sy = __dadd_rn(sy, __dmul_rn(m, ny));
    sz = __dadd_rn(sz, __dmul_rn(m, nz));
  }
  double norm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx, sx), __dmul_rn(sy, sy)), __dmul_rn(sz, sz)));
  if (norm == 0.0) norm = 1.0;
  nz_out[static_cast<size_t>(r) * V + i] = __ddiv_rn(sz, norm);
}

__global__ void __launch_bounds__(kTexelThreads)
uv_texels_kernel(const float* __restrict__ verts, int V, const uint8_t* __restrict__ valid,
                 const int32_t* __restrict__ frame_index, const uint8_t* __restrict__ frames, int F, int H, int W,
                 const int32_t* __restrict__ vid, const double* __restrict__ bary, const double* __restrict__ nz_all,
                 int SS, uint8_t* __restrict__ out) {
  const int t = blockIdx.x * kTexelThreads + threadIdx.x;
  const int r = blockIdx.y;
  if (t >= SS) return;
  uint8_t c0 = 0, c1 = 0, c2 = 0;
  int frame;
  const int a = vid[3 * t];
  if (a >= 0 && head_ok(valid, frame_index, r, F, &frame)) {
    const int b = vid[3 * t + 1], c = vid[3 * t + 2];
    const double b0 = bary[3 * t], b1 = bary[3 * t + 1], b2 = bary[3 * t + 2];
    const double* nz = nz_all + static_cast<size_t>(r) * V;
    // n_dot_view = -pixel_3d_normals[:, 2] (uv_texture.py:36); NaN passes, as `n_dot_view[i] < 0.0` is False
    const double n_dot_view = -__dadd_rn(__dadd_rn(__dmul_rn(nz[a], b0), __dmul_rn(nz[b], b1)), __dmul_rn(nz[c], b2));
    if (!(n_dot_view < 0.0)) {
      const float* v = verts + static_cast<size_t>(r) * V * 3;
      const double px = __dadd_rn(__dadd_rn(__dmul_rn(static_cast<double>(v[3 * a]), b0),
                                            __dmul_rn(static_cast<double>(v[3 * b]), b1)),
                                  __dmul_rn(static_cast<double>(v[3 * c]), b2));
      const double py = __dadd_rn(__dadd_rn(__dmul_rn(static_cast<double>(v[3 * a + 1]), b0),
                                            __dmul_rn(static_cast<double>(v[3 * b + 1]), b1)),
                                  __dmul_rn(static_cast<double>(v[3 * c + 1]), b2));
      // np.round(., 0) is rint (half to even).  On the rounded doubles the strict bounds test equals the reference's test
      // on .astype(int): NaN, infinities and |x| >= 2^63 (INT64_MIN there) fail it either way.
      const double x = rint(px), y = rint(py);
      if (x > 0.0 && x < static_cast<double>(W) && y > 0.0 && y < static_cast<double>(H)) {
        const uint8_t* src = frames + ((static_cast<size_t>(frame) * H + static_cast<int>(y)) * W + static_cast<int>(x)) * 3;
        c0 = src[0];
        c1 = src[1];
        c2 = src[2];
      }
    }
  }
  uint8_t* dst = out + (static_cast<size_t>(r) * SS + t) * 3;
  dst[0] = c0;
  dst[1] = c1;
  dst[2] = c2;
}

int uv_upload(dad3d_uv* h, const std::vector<int32_t>& vid, const std::vector<double>& bary, const int32_t* faces_h,
              const int32_t* row_h, const int32_t* col_h, const std::vector<double>& mult) {
  auto up = [](auto** dst, const void* src, size_t bytes) -> cudaError_t {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(dst), bytes);
    return e != cudaSuccess ? e : cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice);
  };
  const size_t nnz = mult.size();
  DAD3D_CUDA_OK(up(&h->vid_d, vid.data(), vid.size() * 4));
  DAD3D_CUDA_OK(up(&h->bary_d, bary.data(), bary.size() * 8));
  DAD3D_CUDA_OK(up(&h->faces_d, faces_h, static_cast<size_t>(h->NF) * 3 * 4));
  DAD3D_CUDA_OK(up(&h->row_d, row_h, (static_cast<size_t>(h->V) + 1) * 4));
  DAD3D_CUDA_OK(up(&h->col_d, col_h, nnz * 4));
  DAD3D_CUDA_OK(up(&h->mult_d, mult.data(), nnz * 8));
  return DAD3D_OK;
}

}  // namespace
}  // namespace dad3d

using namespace dad3d;

extern "C" {

void dad3d_uv_destroy(dad3d_uv* h) {
  if (!h) return;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->device);
  for (void* p : {static_cast<void*>(h->vid_d), static_cast<void*>(h->bary_d), static_cast<void*>(h->faces_d),
                  static_cast<void*>(h->row_d), static_cast<void*>(h->col_d), static_cast<void*>(h->mult_d)})
    if (p) cudaFree(p);
  cudaSetDevice(prev);
  delete h;
}

int dad3d_uv_create(dad3d_uv** out, int32_t img_size, const int32_t* texel_h, const int32_t* vertex_ids_h,
                    const double* bary_h, int32_t T, const int32_t* faces_h, int32_t NF, const int32_t* csr_row_h,
                    const int32_t* csr_col_h, int32_t V, int32_t device) {
  DAD3D_REQUIRE(out && faces_h && csr_row_h && (T == 0 || (texel_h && vertex_ids_h && bary_h)), "null pointer");
  *out = nullptr;
  DAD3D_REQUIRE(img_size >= 1 && img_size <= 16384, "img_size outside [1, 16384]");
  DAD3D_REQUIRE(T >= 0 && NF >= 1 && V >= 1, "T, NF, V");
  const int64_t SS = static_cast<int64_t>(img_size) * img_size;
  std::vector<int32_t> vid(static_cast<size_t>(SS) * 3, -1);
  std::vector<double> bary(static_cast<size_t>(SS) * 3, 0.0);
  for (int32_t e = 0; e < T; ++e) {
    const int32_t t = texel_h[e];
    DAD3D_REQUIRE(t >= 0 && t < SS, "texel outside the image");
    DAD3D_REQUIRE(vid[3 * static_cast<size_t>(t)] < 0, "duplicate texel");
    for (int k = 0; k < 3; ++k) {
      const int32_t i = vertex_ids_h[3 * static_cast<size_t>(e) + k];
      DAD3D_REQUIRE(i >= 0 && i < V, "vertex id outside [0, V)");
      vid[3 * static_cast<size_t>(t) + k] = i;
      bary[3 * static_cast<size_t>(t) + k] = bary_h[3 * static_cast<size_t>(e) + k];
    }
  }
  for (int64_t k = 0; k < 3LL * NF; ++k) DAD3D_REQUIRE(faces_h[k] >= 0 && faces_h[k] < V, "face vertex outside [0, V)");
  DAD3D_REQUIRE(csr_row_h[0] == 0, "csr_row[0] != 0");
  for (int32_t i = 0; i < V; ++i) DAD3D_REQUIRE(csr_row_h[i + 1] >= csr_row_h[i], "csr_row not ascending");
  const int32_t nnz = csr_row_h[V];
  DAD3D_REQUIRE(nnz == 0 || csr_col_h, "null pointer");
  // the CSR must be faces_by_vertex: each row the vertex's distinct faces, ascending; the multiplicity comes from the face
  std::vector<double> mult(static_cast<size_t>(nnz));
  int64_t listed = 0;
  for (int32_t i = 0; i < V; ++i)
    for (int32_t e = csr_row_h[i]; e < csr_row_h[i + 1]; ++e) {
      const int32_t f = csr_col_h[e];
      DAD3D_REQUIRE(f >= 0 && f < NF, "csr face outside [0, NF)");
      DAD3D_REQUIRE(e == csr_row_h[i] || csr_col_h[e - 1] < f, "csr row not strictly ascending");
      const int m = (faces_h[3 * f] == i) + (faces_h[3 * f + 1] == i) + (faces_h[3 * f + 2] == i);
      DAD3D_REQUIRE(m > 0, "csr lists a face that does not hold the vertex");
      mult[e] = m;
      listed += m;
    }
  DAD3D_REQUIRE(listed == 3LL * NF, "csr misses a face of a vertex");
  int prev = 0;
  DAD3D_CUDA_OK(cudaGetDevice(&prev));
  DAD3D_CUDA_OK(cudaSetDevice(device));
  dad3d_uv* h = new dad3d_uv;
  h->S = img_size; h->V = V; h->NF = NF; h->device = device;
  const int rc = uv_upload(h, vid, bary, faces_h, csr_row_h, csr_col_h, mult);
  cudaSetDevice(prev);
  if (rc != DAD3D_OK) {
    dad3d_uv_destroy(h);
    return rc;
  }
  *out = h;
  return DAD3D_OK;
}

size_t dad3d_uv_workspace_bytes(const dad3d_uv* h, int32_t R) {
  if (!h || R < 0) return 0;
  return static_cast<size_t>(R) * h->V * sizeof(double);
}

int dad3d_uv_texture(const dad3d_uv* h, const float* vertices_d, int32_t R, const uint8_t* valid_d, const uint8_t* frames_d,
                     int32_t F, int32_t H, int32_t W, const int32_t* frame_index_d, uint8_t* out_d, void* workspace_d,
                     size_t workspace_bytes, dad3d_stream stream_) {
  DAD3D_REQUIRE(h, "null handle");
  DAD3D_REQUIRE(R >= 0 && R <= 65535, "R outside [0, 65535]");
  DAD3D_REQUIRE(F >= 1 && H >= 1 && W >= 1, "F, H, W");
  if (R == 0) return DAD3D_OK;
  DAD3D_REQUIRE(vertices_d && frames_d && out_d && workspace_d, "null pointer");
  DAD3D_REQUIRE(workspace_bytes >= dad3d_uv_workspace_bytes(h, R), "workspace too small");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  double* nz = static_cast<double*>(workspace_d);
  const int SS = h->S * h->S;
  uv_normals_kernel<<<dim3(ceil_div(h->V, kNormalThreads), R), kNormalThreads, 0, stream>>>(
      vertices_d, h->V, valid_d, frame_index_d, F, h->faces_d, h->row_d, h->col_d, h->mult_d, nz);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  uv_texels_kernel<<<dim3(ceil_div(SS, kTexelThreads), R), kTexelThreads, 0, stream>>>(
      vertices_d, h->V, valid_d, frame_index_d, frames_d, F, H, W, h->vid_d, h->bary_d, nz, SS, out_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // extern "C"
