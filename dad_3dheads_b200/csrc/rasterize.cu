// Z-buffer rasteriser and vertex normals on the GPU (SURVEY §8f row 4): the reference's Sim3DR native component
// (Sim3DR/lib/rasterize_kernel.cpp:158-292 `_rasterize`, :158-236 `_get_normal`; callers inference/pncc_estimator.py:16-43,
// Sim3DR/Sim3DR.py:8-29).  BIT-EXACT with the reference's sequential C++ loop:
//   * every floating-point operation is issued in the reference's order with round-to-nearest intrinsics (no FMA contraction:
//     the reference's build has none), so barycentric weights, depths and colours are the same bits;
//   * the sequential z-test "if (p_depth > depth_buffer[pix])" over triangles in index order = per pixel the maximum depth, ties
//     won by the LOWEST triangle index: one 64-bit atomicMax on (orderable(depth) << 32 | ~index) per covered pixel, then a
//     per-pixel resolve pass that shades the winner.  alpha must be 1 (what Sim3DR.rasterize passes; blending with alpha < 1 is
//     order-dependent).
//   * both passes run over a batch of heads that share one triangle list and colour table (PNCC, depth and triangle-index
//     maps of a whole predict_batch); each head has its own key words, so a head's result does not depend on the batch.
//     dad3d_rasterize is the one-head call.
//   * with a head -> image map (dad3d_rasterize_frames) several heads share one image's key words: the key's low word is
//     ~(head * ntri + triangle), so one atomicMax keeps the nearest surface and, on an exact tie, the lower (head, triangle)
//     pair -- the reference's loop over the union mesh of the image's heads in head order.  Pass 2 then runs over
//     (pixel, image) and decodes head and triangle from the winner.  Without a map, image = head and the low word is ~triangle.
//   * vertex normals accumulate the un-normalised face normals of the incident triangles in ascending triangle order (caller-built
//     CSR adjacency), the order of the reference's scatter loop.
//   * lit meshes (Sim3DR/lighting.py:23-71 RenderPipeline): light_kernel computes each head's per-vertex light in the
//     reference's float32 order (the power correctly rounded), and pass 2 takes per-head colour tables (a colour stride).
// Integer / float HBM-bound work; no tensor cores.
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"

namespace dad3d {

__device__ __forceinline__ float rmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float radd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float rsub(float a, float b) { return __fsub_rn(a, b); }

// get_point_weight (rasterize_kernel.cpp:52-82), operation for operation
__device__ __forceinline__ void point_weight(float* w, float px, float py, float p0x, float p0y, float p1x, float p1y, float p2x,
                                             float p2y) {
  const float v0x = rsub(p2x, p0x), v0y = rsub(p2y, p0y);
  const float v1x = rsub(p1x, p0x), v1y = rsub(p1y, p0y);
  const float v2x = rsub(px, p0x), v2y = rsub(py, p0y);
  const float dot00 = radd(rmul(v0x, v0x), rmul(v0y, v0y));
  const float dot01 = radd(rmul(v0x, v1x), rmul(v0y, v1y));
  const float dot02 = radd(rmul(v0x, v2x), rmul(v0y, v2y));
  const float dot11 = radd(rmul(v1x, v1x), rmul(v1y, v1y));
  const float dot12 = radd(rmul(v1x, v2x), rmul(v1y, v2y));
  const float den = rsub(rmul(dot00, dot11), rmul(dot01, dot01));
  const float inv = (den == 0.f) ? 0.f : __fdiv_rn(1.0f, den);
  const float u = rmul(rsub(rmul(dot11, dot02), rmul(dot01, dot12)), inv);
  const float v = rmul(rsub(rmul(dot00, dot12), rmul(dot01, dot02)), inv);
  w[0] = rsub(rsub(1.0f, u), v);
  w[1] = v;
  w[2] = u;
}

__device__ __forceinline__ unsigned int orderable(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct TriSetup {
  float p0x, p0y, d0, p1x, p1y, d1, p2x, p2y, d2;
  int i0, i1, i2;
};
__device__ __forceinline__ TriSetup load_tri(const float* __restrict__ v, const int* __restrict__ t, int i) {
  TriSetup s;
  s.i0 = t[3 * i]; s.i1 = t[3 * i + 1]; s.i2 = t[3 * i + 2];
  s.p0x = v[3 * s.i0]; s.p0y = v[3 * s.i0 + 1]; s.d0 = v[3 * s.i0 + 2];
  s.p1x = v[3 * s.i1]; s.p1y = v[3 * s.i1 + 1]; s.d1 = v[3 * s.i1 + 2];
  s.p2x = v[3 * s.i2]; s.p2y = v[3 * s.i2 + 1]; s.d2 = v[3 * s.i2 + 2];
  return s;
}

// pass 1: one thread per (triangle, head) walks the triangle's bounding box.  Heads run along grid y, strided by gridDim.y so
// that batches past the 65 535 grid-y limit loop; every head offset is 64-bit.  image_of_head (NULL: head b draws into image
// b) sends a head's keys to its image; a head mapped outside [0, n_images) draws nothing.
__global__ void raster_tri_kernel(const float* __restrict__ verts, int nv, int batch, const int* __restrict__ tris, int ntri,
                                  int h, int w, int negate_z, const int* __restrict__ image_of_head, int n_images,
                                  const float* __restrict__ depth_in, unsigned long long* __restrict__ key) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ntri) return;
  const long long hw = static_cast<long long>(h) * w;
  for (int b = blockIdx.y; b < batch; b += gridDim.y) {
    const int img = image_of_head ? image_of_head[b] : b;
    if (img < 0 || img >= n_images) continue;
    // the tie-break word: the triangle, or with a map the (head, triangle) pair, which the caller keeps below 2^32 - 1
    const unsigned int rank = image_of_head ? static_cast<unsigned int>(b) * static_cast<unsigned int>(ntri) +
                                                  static_cast<unsigned int>(i)
                                            : static_cast<unsigned int>(i);
    TriSetup s = load_tri(verts + static_cast<long long>(b) * nv * 3, tris, i);
    if (negate_z) { s.d0 = -s.d0; s.d1 = -s.d1; s.d2 = -s.d2; }
    const int x_min = max(static_cast<int>(ceilf(fminf(s.p0x, fminf(s.p1x, s.p2x)))), 0);
    const int x_max = min(static_cast<int>(floorf(fmaxf(s.p0x, fmaxf(s.p1x, s.p2x)))), w - 1);
    const int y_min = max(static_cast<int>(ceilf(fminf(s.p0y, fminf(s.p1y, s.p2y)))), 0);
    const int y_max = min(static_cast<int>(floorf(fmaxf(s.p0y, fmaxf(s.p1y, s.p2y)))), h - 1);
    if (x_max < x_min || y_max < y_min) continue;
    const float* dh = depth_in ? depth_in + img * hw : nullptr;
    unsigned long long* kh = key + img * hw;
    for (int y = y_min; y <= y_max; ++y)
      for (int x = x_min; x <= x_max; ++x) {
        float wt[3];
        point_weight(wt, static_cast<float>(x), static_cast<float>(y), s.p0x, s.p0y, s.p1x, s.p1y, s.p2x, s.p2y);
        if (wt[2] > 0 && wt[1] > 0 && wt[0] > 0) {
          const float d = radd(radd(rmul(wt[0], s.d0), rmul(wt[1], s.d1)), rmul(wt[2], s.d2));
          const int pix = y * w + x;
          if (d > (dh ? dh[pix] : -1e8f)) {                       // Sim3DR.py:22 initialises the buffer to -1e8
            // d + 0 maps -0 to +0 (and nothing else): the sequential z-test sees -0 and +0 as a tie, the lower index keeps it
            const unsigned long long k = (static_cast<unsigned long long>(orderable(radd(d, 0.0f))) << 32) |
                                         static_cast<unsigned long long>(0xFFFFFFFFu - rank);
            atomicMax(&kh[pix], k);
          }
        }
      }
  }
}

// pass 2: one thread per (pixel, image) shades the winning triangle; tri_index gets the winner or -1 in depth-buffer rows.
// mapped != 0: the key names (head, triangle) as head * ntri + triangle, and head_index gets the head or -1.  Head b's
// colours start at colors + b * color_stride (0: every head shares one table).
__global__ void raster_resolve_kernel(const float* __restrict__ verts, int nv, int n_images, const int* __restrict__ tris,
                                      int ntri, int mapped, const float* __restrict__ colors, long long color_stride, int h,
                                      int w, int c, int reverse, int negate_z, const unsigned long long* __restrict__ key,
                                      unsigned char* __restrict__ image, float* __restrict__ depth, int* __restrict__ tri_index,
                                      int* __restrict__ head_index) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const long long hw = static_cast<long long>(h) * w;
  if (pix >= hw) return;
  const int y = pix / w, x = pix - y * w;
  const int yo = reverse ? (h - 1 - y) : y;
  for (int m = blockIdx.y; m < n_images; m += gridDim.y) {
    const long long at = m * hw + pix;
    const unsigned long long k = key[at];
    const unsigned int rank = 0xFFFFFFFFu - static_cast<unsigned int>(k & 0xFFFFFFFFull);
    const int b = k == 0ull ? -1 : (mapped ? static_cast<int>(rank / static_cast<unsigned int>(ntri)) : m);
    const int i = k == 0ull ? -1 : (mapped ? static_cast<int>(rank - static_cast<unsigned int>(b) * ntri)
                                           : static_cast<int>(rank));
    if (tri_index) tri_index[at] = i;
    if (head_index) head_index[at] = b;
    if (i < 0) continue;
    const float* vh = verts + static_cast<long long>(b) * nv * 3;
    TriSetup s = load_tri(vh, tris, i);
    if (negate_z) { s.d0 = -s.d0; s.d1 = -s.d1; s.d2 = -s.d2; }
    float wt[3];
    point_weight(wt, static_cast<float>(x), static_cast<float>(y), s.p0x, s.p0y, s.p1x, s.p1y, s.p2x, s.p2y);
    if (depth) depth[at] = radd(radd(rmul(wt[0], s.d0), rmul(wt[1], s.d1)), rmul(wt[2], s.d2));
    if (!image) continue;
    unsigned char* px = image + (m * hw + static_cast<long long>(yo) * w + x) * c;
    const float* col = colors + b * color_stride;                     // the winning head's colours (stride 0: one table)
    for (int ch = 0; ch < c; ++ch) {
      const float pc = radd(radd(rmul(wt[0], col[c * s.i0 + ch]), rmul(wt[1], col[c * s.i1 + ch])), rmul(wt[2], col[c * s.i2 + ch]));
      // (unsigned char)((1 - alpha) * image + alpha * 255 * p_color) with alpha = 1
      const float old = static_cast<float>(px[ch]);
      const float val = radd(rmul(rsub(1.0f, 1.0f), old), rmul(rmul(1.0f, 255.0f), pc));
      px[ch] = static_cast<unsigned char>(static_cast<int>(val));
    }
  }
}

// the normal of vertex i (_get_normal): un-normalised face normals of its incident triangles, added in ascending triangle
// order, then divided by their length (1e-6 when it is not positive).  negate_z reads -z (exact: negation commutes with
// rounding).
__device__ __forceinline__ void vertex_normal(const float* __restrict__ v, const int* __restrict__ t,
                                              const int* __restrict__ adj_off, const int* __restrict__ adj_tri, int i,
                                              bool negate_z, float n[3]) {
  float nx = 0.f, ny = 0.f, nz = 0.f;
  for (int e = adj_off[i]; e < adj_off[i + 1]; ++e) {
    const int tr = adj_tri[e];
    const int a = t[3 * tr], b = t[3 * tr + 1], c = t[3 * tr + 2];
    const float za = negate_z ? -v[3 * a + 2] : v[3 * a + 2];
    const float zb = negate_z ? -v[3 * b + 2] : v[3 * b + 2];
    const float zc = negate_z ? -v[3 * c + 2] : v[3 * c + 2];
    const float v1x = rsub(v[3 * b], v[3 * a]), v1y = rsub(v[3 * b + 1], v[3 * a + 1]), v1z = rsub(zb, za);
    const float v2x = rsub(v[3 * c], v[3 * a]), v2y = rsub(v[3 * c + 1], v[3 * a + 1]), v2z = rsub(zc, za);
    nx = radd(nx, rsub(rmul(v1y, v2z), rmul(v1z, v2y)));
    ny = radd(ny, rsub(rmul(v1z, v2x), rmul(v1x, v2z)));
    nz = radd(nz, rsub(rmul(v1x, v2y), rmul(v1y, v2x)));
  }
  float det = __fsqrt_rn(radd(radd(rmul(nx, nx), rmul(ny, ny)), rmul(nz, nz)));
  if (det <= 0) det = 1e-6f;
  n[0] = __fdiv_rn(nx, det);
  n[1] = __fdiv_rn(ny, det);
  n[2] = __fdiv_rn(nz, det);
}

// one thread per vertex
__global__ void vertex_normal_kernel(const float* __restrict__ v, const int* __restrict__ t, const int* __restrict__ adj_off,
                                     const int* __restrict__ adj_tri, int nver, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nver) return;
  vertex_normal(v, t, adj_off, adj_tri, i, false, out + 3 * i);
}

// ---- lighting (Sim3DR/lighting.py:37-63) ----------------------------------------------------------------------------------

// np.clip(x, 0, 1): max(x, 0) then min(., 1), each "a > b ? a : b" with a NaN kept (so clip(-0) = +0 and NaN stays)
__device__ __forceinline__ float clip01(float x) {
  if (x != x) return x;
  const float t = x > 0.f ? x : 0.f;
  return t < 1.f ? t : 1.f;
}
// np.min / np.max reductions propagate NaN
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || a < b) ? a : b; }
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || a > b) ? a : b; }

// x ** e correctly rounded to float32, e in [0, 16]: the product in double-double (error below 2^-100 relative), then one
// rounding; a double-double that is exactly a float32 midpoint is resolved by the sign of its low part.
__device__ __forceinline__ float pow_cr(float x, int e) {
  if (e == 0) return 1.0f;
  if (!isfinite(x) || x == 0.f) {                        // zeros, infinities and NaN: the plain product has the exact result
    float r = x;
    for (int k = 1; k < e; ++k) r = __fmul_rn(r, x);
    return r;
  }
  const double xd = x;
  double hi = xd, lo = 0.0;
  for (int k = 1; k < e; ++k) {                          // (hi, lo) *= x
    const double p = __dmul_rn(hi, xd);
    const double err = __fma_rn(lo, xd, __fma_rn(hi, xd, -p));
    hi = __dadd_rn(p, err);
    lo = __dsub_rn(err, __dsub_rn(hi, p));
  }
  const float f = __double2float_rn(hi);
  if (!isfinite(hi) || lo == 0.0 || static_cast<double>(f) == hi) return f;
  // hi lies strictly between f and its neighbour g on hi's side; only an exact midpoint can round the wrong way
  const float g = nextafterf(f, hi > static_cast<double>(f) ? INFINITY : -INFINITY);
  const double mid = 0.5 * (static_cast<double>(f) + static_cast<double>(g));
  if (hi != mid) return f;
  return ((g > f) == (lo > 0.0)) ? g : f;
}

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? nan_max(v, u) : nan_min(v, u);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = red[0];
  for (int k = 1; k < nw; ++k) v = is_max ? nan_max(v, red[k]) : nan_min(v, red[k]);
  return v;
}

// one CTA per head (heads along grid x, strided): the head's per-axis min / max, then every vertex's normal and light.
// norm_vertices (lighting.py:9-14) needs only those six values: its steps round monotonically, so the global max of
// v - min is max_a (max_a - min_a), and the per-axis max after "/ M * 2" is that of the per-axis max.
__global__ void __launch_bounds__(256) light_kernel(const float* __restrict__ verts, int nv, int batch,
                                                    const int* __restrict__ tris, const int* __restrict__ adj_off,
                                                    const int* __restrict__ adj_tri, int negate_z, dad3d_lighting L,
                                                    float* __restrict__ light_out) {
  __shared__ float red[32];
  for (int b = blockIdx.x; b < batch; b += gridDim.x) {
    const float* v = verts + static_cast<long long>(b) * nv * 3;
    float* out = light_out + static_cast<long long>(b) * nv * 3;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = threadIdx.x; i < nv; i += blockDim.x)
      for (int a = 0; a < 3; ++a) {
        const float x = (a == 2 && negate_z) ? -v[3 * i + 2] : v[3 * i + a];
        lo[a] = nan_min(lo[a], x);
        hi[a] = nan_max(hi[a], x);
      }
    for (int a = 0; a < 3; ++a) {
      lo[a] = block_reduce(lo[a], false, red);
      hi[a] = block_reduce(hi[a], true, red);
    }
    float span[3], half_top[3];
    for (int a = 0; a < 3; ++a) span[a] = rsub(hi[a], lo[a]);                       // max(v - min) per axis
    const float M = nan_max(nan_max(span[0], span[1]), span[2]);                    // vertices.max()
    for (int a = 0; a < 3; ++a) half_top[a] = __fdiv_rn(rmul(__fdiv_rn(span[a], M), 2.f), 2.f);   // max(0) / 2

    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
      float n[3];
      vertex_normal(v, tris, adj_off, adj_tri, i, negate_z != 0, n);
      float vn[3], light[3] = {0.f, 0.f, 0.f};
      for (int a = 0; a < 3; ++a) {
        const float x = (a == 2 && negate_z) ? -v[3 * i + 2] : v[3 * i + a];
        vn[a] = rsub(rmul(__fdiv_rn(rsub(x, lo[a]), M), 2.f), half_top[a]);
      }
      if (L.intensity_ambient > 0)
        for (int a = 0; a < 3; ++a) light[a] = radd(light[a], rmul(L.intensity_ambient, L.color_ambient[a]));
      if (L.intensity_directional > 0) {
        float dir[3];
        for (int a = 0; a < 3; ++a) dir[a] = rsub(L.light_pos[a], vn[a]);
        float len = __fsqrt_rn(radd(radd(rmul(dir[0], dir[0]), rmul(dir[1], dir[1])), rmul(dir[2], dir[2])));
        for (int a = 0; a < 3; ++a) dir[a] = __fdiv_rn(dir[a], len);
        const float cs = radd(radd(rmul(n[0], dir[0]), rmul(n[1], dir[1])), rmul(n[2], dir[2]));
        const float cc = clip01(cs);
        for (int a = 0; a < 3; ++a)
          light[a] = radd(light[a], rmul(L.intensity_directional, rmul(L.color_directional[a], cc)));
        if (L.intensity_specular > 0) {
          float v2v[3];
          for (int a = 0; a < 3; ++a) v2v[a] = rsub(L.view_pos[a], vn[a]);
          len = __fsqrt_rn(radd(radd(rmul(v2v[0], v2v[0]), rmul(v2v[1], v2v[1])), rmul(v2v[2], v2v[2])));
          const float two_cos = rmul(2.f, cs);
          float spe = 0.f;
          for (int a = 0; a < 3; ++a) {
            const float refl = rsub(rmul(two_cos, n[a]), dir[a]);
            const float p = pow_cr(rmul(__fdiv_rn(v2v[a], len), refl), L.specular_exp);
            spe = a == 0 ? p : radd(spe, p);
          }
          spe = cs != 0.f ? clip01(spe) : 0.f;
          for (int a = 0; a < 3; ++a)
            light[a] = radd(light[a], rmul(rmul(L.intensity_specular, L.color_directional[a]), clip01(spe)));
        }
      }
      for (int a = 0; a < 3; ++a) out[3 * i + a] = clip01(light[a]);
    }
  }
}

}  // namespace dad3d

using namespace dad3d;

extern "C" {

}  // extern "C"

namespace {

// both entries: `batch` heads drawn into `n_images` images; image_of_head_d NULL is the identity map (n_images = batch)
int rasterize_mapped(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d, int32_t ntri,
                     const float* colors_d, long long color_stride, int32_t c, int32_t h, int32_t w, int32_t reverse,
                     int32_t negate_z, const int32_t* image_of_head_d, int32_t n_images, uint8_t* image_d, float* depth_d,
                     int32_t* tri_index_d, int32_t* head_index_d, unsigned long long* key_ws_d, dad3d_stream stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const size_t hw = static_cast<size_t>(h) * w;
  if (n_images == 0) return DAD3D_OK;
  if (batch == 0 || ntri == 0) {                     // nothing covers any pixel: image and depth stay, the indices are all -1
    if (tri_index_d) DAD3D_CUDA_OK(cudaMemsetAsync(tri_index_d, 0xFF, sizeof(int32_t) * hw * n_images, stream));
    if (head_index_d) DAD3D_CUDA_OK(cudaMemsetAsync(head_index_d, 0xFF, sizeof(int32_t) * hw * n_images, stream));
    return DAD3D_OK;
  }
  DAD3D_CUDA_OK(cudaMemsetAsync(key_ws_d, 0, sizeof(unsigned long long) * hw * n_images, stream));
  const unsigned int gy = static_cast<unsigned int>(batch < 65535 ? batch : 65535);
  raster_tri_kernel<<<dim3((ntri + 127) / 128, gy), 128, 0, stream>>>(vertices_d, nv, batch, triangles_d, ntri, h, w,
                                                                       negate_z, image_of_head_d, n_images, depth_d,
                                                                       key_ws_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  const unsigned int gm = static_cast<unsigned int>(n_images < 65535 ? n_images : 65535);
  raster_resolve_kernel<<<dim3(static_cast<unsigned int>((hw + 255) / 256), gm), 256, 0, stream>>>(
      vertices_d, nv, n_images, triangles_d, ntri, image_of_head_d ? 1 : 0, colors_d, color_stride, h, w, c, reverse, negate_z,
      key_ws_d, image_d, depth_d, tri_index_d, head_index_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int launch_light(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d, const int32_t* adj_offsets_d,
                 const int32_t* adj_triangles_d, int32_t negate_z, const dad3d_lighting& lighting, float* light_d,
                 cudaStream_t stream) {
  if (batch == 0) return DAD3D_OK;
  const unsigned int gx = static_cast<unsigned int>(batch < 65535 ? batch : 65535);
  light_kernel<<<gx, 256, 0, stream>>>(vertices_d, nv, batch, triangles_d, adj_offsets_d, adj_triangles_d, negate_z, lighting,
                                       light_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // namespace

extern "C" {

int dad3d_light_batch(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d,
                      const int32_t* adj_offsets_d, const int32_t* adj_triangles_d, int32_t negate_z, dad3d_lighting lighting,
                      float* light_d, dad3d_stream stream) {
  DAD3D_REQUIRE((vertices_d && triangles_d && adj_offsets_d && adj_triangles_d && light_d) || batch == 0, "null pointer");
  DAD3D_REQUIRE(batch >= 0 && nv > 0 && static_cast<long long>(nv) * 3 < (1ll << 31), "shape");
  DAD3D_REQUIRE(lighting.specular_exp >= 0 && lighting.specular_exp <= 16, "specular_exp must be an integer in [0, 16]");
  return launch_light(vertices_d, nv, batch, triangles_d, adj_offsets_d, adj_triangles_d, negate_z, lighting, light_d,
                      reinterpret_cast<cudaStream_t>(stream));
}

int dad3d_render_lit(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d, int32_t ntri,
                     const int32_t* adj_offsets_d, const int32_t* adj_triangles_d, int32_t negate_z, dad3d_lighting lighting,
                     const int32_t* image_of_head_d, int32_t n_images, int32_t h, int32_t w, float* light_ws_d,
                     uint8_t* image_d, unsigned long long* key_ws_d, dad3d_stream stream) {
  DAD3D_REQUIRE(((vertices_d && adj_offsets_d && adj_triangles_d && light_ws_d) || batch == 0) && (triangles_d || ntri == 0) &&
                    image_d && key_ws_d,
                "null pointer");
  DAD3D_REQUIRE(batch >= 0 && nv > 0 && ntri >= 0 && h > 0 && w > 0 && static_cast<long long>(h) * w < (1ll << 31) &&
                    static_cast<long long>(nv) * 3 < (1ll << 31) && (!image_of_head_d || n_images >= 0),
                "shape");
  DAD3D_REQUIRE(lighting.specular_exp >= 0 && lighting.specular_exp <= 16, "specular_exp must be an integer in [0, 16]");
  DAD3D_REQUIRE(!image_of_head_d || static_cast<unsigned long long>(batch) * static_cast<unsigned long long>(ntri) <=
                                        0xFFFFFFFEull,
                "batch * ntri exceeds 2^32 - 2");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (ntri > 0) {                                       // without triangles nothing is drawn and the light is not needed
    const int rc = launch_light(vertices_d, nv, batch, triangles_d, adj_offsets_d, adj_triangles_d, negate_z, lighting,
                                light_ws_d, st);
    if (rc != DAD3D_OK) return rc;
  }
  return rasterize_mapped(vertices_d, nv, batch, triangles_d, ntri, light_ws_d, static_cast<long long>(nv) * 3, 3, h, w, 0,
                          negate_z, image_of_head_d, image_of_head_d ? n_images : batch, image_d, nullptr, nullptr, nullptr,
                          key_ws_d, stream);
}

int dad3d_rasterize_batch(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d, int32_t ntri,
                          const float* colors_d, int32_t c, int32_t h, int32_t w, int32_t reverse, int32_t negate_z,
                          uint8_t* image_d, float* depth_d, int32_t* tri_index_d, unsigned long long* key_ws_d,
                          dad3d_stream stream) {
  DAD3D_REQUIRE(vertices_d && (triangles_d || ntri == 0) && key_ws_d, "null pointer");
  DAD3D_REQUIRE(!image_d || colors_d, "image_d needs colors_d");
  DAD3D_REQUIRE(batch >= 0 && nv > 0 && ntri >= 0 && h > 0 && w > 0 && c > 0 && static_cast<long long>(h) * w < (1ll << 31),
                "shape");
  return rasterize_mapped(vertices_d, nv, batch, triangles_d, ntri, colors_d, 0, c, h, w, reverse, negate_z, nullptr, batch,
                          image_d, depth_d, tri_index_d, nullptr, key_ws_d, stream);
}

int dad3d_rasterize_frames(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d, int32_t ntri,
                           const float* colors_d, int32_t c, const int32_t* image_of_head_d, int32_t n_images, int32_t h,
                           int32_t w, int32_t negate_z, uint8_t* image_d, float* depth_d, int32_t* tri_index_d,
                           int32_t* head_index_d, unsigned long long* key_ws_d, dad3d_stream stream) {
  DAD3D_REQUIRE(((vertices_d && image_of_head_d) || batch == 0) && (triangles_d || ntri == 0) && key_ws_d, "null pointer");
  DAD3D_REQUIRE(!image_d || colors_d, "image_d needs colors_d");
  DAD3D_REQUIRE(batch >= 0 && nv > 0 && ntri >= 0 && n_images >= 0 && h > 0 && w > 0 && c > 0 &&
                    static_cast<long long>(h) * w < (1ll << 31),
                "shape");
  // the key's low word holds ~(head * ntri + triangle): every pair must stay below 2^32 - 1
  DAD3D_REQUIRE(static_cast<unsigned long long>(batch) * static_cast<unsigned long long>(ntri) <= 0xFFFFFFFEull,
                "batch * ntri exceeds 2^32 - 2");
  return rasterize_mapped(vertices_d, nv, batch, triangles_d, ntri, colors_d, 0, c, h, w, 0, negate_z, image_of_head_d, n_images,
                          image_d, depth_d, tri_index_d, head_index_d, key_ws_d, stream);
}

int dad3d_rasterize(const float* vertices_d, const int32_t* triangles_d, const float* colors_d, int32_t ntri, uint8_t* image_d,
                    float* depth_d, unsigned long long* key_ws_d, int32_t h, int32_t w, int32_t c, int32_t reverse,
                    dad3d_stream stream) {
  DAD3D_REQUIRE(vertices_d && triangles_d && colors_d && image_d && depth_d && key_ws_d, "null pointer");
  // nv only sets the stride between heads, which one head never uses: 1 stands in for the vertex count this call lacks
  return dad3d_rasterize_batch(vertices_d, 1, 1, triangles_d, ntri, colors_d, c, h, w, reverse, 0, image_d, depth_d, nullptr,
                               key_ws_d, stream);
}

int dad3d_vertex_normals(const float* vertices_d, const int32_t* triangles_d, const int32_t* adj_offsets_d,
                         const int32_t* adj_triangles_d, int32_t nver, float* normals_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(vertices_d && triangles_d && adj_offsets_d && adj_triangles_d && normals_d, "null pointer");
  DAD3D_REQUIRE(nver >= 0, "shape");
  if (nver == 0) return DAD3D_OK;
  vertex_normal_kernel<<<(nver + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      vertices_d, triangles_d, adj_offsets_d, adj_triangles_d, nver, normals_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // extern "C"
