// GPU kernels for the DAD-3DHeads benchmark evaluator's hot spots (SURVEY §8f row 1):
//   dad3d_eval_chamfer   one-directional chamfer term  mean_i min_j |a_i - b_j|^2   (dad_3dheads_benchmark/utils.py:122-140:
//                        kaolin chamfer_distance(gt_face, aligned_pred, w1 = 1, w2 = 0))
//   dad3d_eval_zn        Z_n ordinal-depth accuracy exactly as benchmark.py:110-138 computes it (including its index
//                        selection: column-wise argsort of the gt distance matrix, columns 1..n)
//   dad3d_eval_align     pred * scale @ rotation + translation over all vertices (utils.py:178-197, the per-vertex python loop)
// All batched over heads; HBM-bound / latency-bound integer-and-float work, no tensor cores.
#include <cfloat>
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"

namespace dad3d {

// one block per (head, chunk of a); b is streamed through shared memory in tiles
__global__ void __launch_bounds__(256)
chamfer_kernel(const float* __restrict__ a, int na, const float* __restrict__ b, int nb, float* __restrict__ partial) {
  __shared__ float sb[3 * 1024];
  const int head = blockIdx.y;
  const float* A = a + static_cast<size_t>(head) * na * 3;
  const float* Bp = b + static_cast<size_t>(head) * nb * 3;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float ax = 0.f, ay = 0.f, az = 0.f;
  if (i < na) { ax = A[3 * i]; ay = A[3 * i + 1]; az = A[3 * i + 2]; }
  float best = FLT_MAX;
  for (int j0 = 0; j0 < nb; j0 += 1024) {
    const int n = min(1024, nb - j0);
    __syncthreads();
    for (int t = threadIdx.x; t < 3 * n; t += blockDim.x) sb[t] = Bp[3 * j0 + t];
    __syncthreads();
    for (int j = 0; j < n; ++j) {
      const float dx = ax - sb[3 * j], dy = ay - sb[3 * j + 1], dz = az - sb[3 * j + 2];
      best = fminf(best, fmaf(dx, dx, fmaf(dy, dy, dz * dz)));
    }
  }
  // block sum of the per-point minima
  float v = (i < na) ? best : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __shared__ float ws[8];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += ws[w];
    atomicAdd(&partial[head], s / static_cast<float>(na));
  }
}

// Z_n: one block per (head, j); sorts (distance to point j+1, index) of all K points with an in-shared-memory bitonic sort
// (K <= 4096), then for every i compares the depth order of (i, order[i]) in gt and pred.
constexpr int kZnMax = 4096;
__global__ void __launch_bounds__(1024)
zn_kernel(const float* __restrict__ pred, const float* __restrict__ gt, int K, int top_k, float* __restrict__ out) {
  __shared__ float key[kZnMax];
  __shared__ int val[kZnMax];
  const int head = blockIdx.y, j = blockIdx.x;
  const float* G = gt + static_cast<size_t>(head) * K * 3;
  const float* P = pred + static_cast<size_t>(head) * K * 3;
  const int c = j + 1;                                  // benchmark.py:126: columns 1..top_k of the column-sorted index matrix
  const float cx = G[3 * c], cy = G[3 * c + 1], cz = G[3 * c + 2];
  const float cn = fmaf(cx, cx, fmaf(cy, cy, cz * cz));
  for (int k = threadIdx.x; k < kZnMax; k += blockDim.x) {
    if (k < K) {
      // torch.cdist (p = 2, > 25 points) evaluates |a|^2 + |b|^2 - 2 a.b, clamps at 0 and takes the square root
      const float x = G[3 * k], y = G[3 * k + 1], z = G[3 * k + 2];
      const float n2 = fmaf(x, x, fmaf(y, y, z * z));
      const float d2 = fmaxf(n2 + cn - 2.0f * fmaf(x, cx, fmaf(y, cy, z * cz)), 0.f);
      key[k] = (k == c) ? 0.f : sqrtf(d2);
      val[k] = k;
    } else {
      key[k] = FLT_MAX;
      val[k] = k;
    }
  }
  __syncthreads();
  for (int size = 2; size <= kZnMax; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < kZnMax / 2; t += blockDim.x) {
        const int lo = (t / stride) * 2 * stride + (t % stride);
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const float kl = key[lo], kh = key[hi];
        const int vl = val[lo], vh = val[hi];
        const bool gt_ = (kl > kh) || (kl == kh && vl > vh);      // ties broken by index (stable order)
        if (gt_ == up) { key[lo] = kh; key[hi] = kl; val[lo] = vh; val[hi] = vl; }
      }
      __syncthreads();
    }
  }
  int agree = 0;
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    const int nb = val[i];                               // the i-th nearest point of point c -- what benchmark.py:131-134 indexes
    const bool g = G[3 * i + 2] >= G[3 * nb + 2];
    const bool p = P[3 * i + 2] >= P[3 * nb + 2];
    agree += (g == p) ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) agree += __shfl_xor_sync(0xffffffffu, agree, o);
  __shared__ int ws[32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = agree;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < 32; ++w) s += ws[w];
    atomicAdd(&out[head], static_cast<float>(s) / (static_cast<float>(K) * static_cast<float>(top_k)));
  }
}

__global__ void align_kernel(const float* __restrict__ v, int nv, int B, const float* __restrict__ scale,
                             const float* __restrict__ rot, const float* __restrict__ trans, float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(B) * nv) return;
  const int h = static_cast<int>(i / nv);
  const float x = v[3 * i], y = v[3 * i + 1], z = v[3 * i + 2];
  const float* R = rot + 9 * h;                           // row-vector convention: out = s * (v @ R) + t
  const float s = scale[h];
#pragma unroll
  for (int c = 0; c < 3; ++c) out[3 * i + c] = fmaf(s, fmaf(x, R[c], fmaf(y, R[3 + c], z * R[6 + c])), trans[3 * h + c]);
}

// both batched kernels put the head on grid.y, which holds at most 65535 blocks: larger batches run in slices of heads
constexpr int32_t kMaxGridY = 65535;

}  // namespace dad3d

using namespace dad3d;

extern "C" {

int dad3d_eval_chamfer(const float* a_d, int32_t na, const float* b_d, int32_t nb, int32_t B, float* out_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(a_d && b_d && out_d, "null pointer");
  DAD3D_REQUIRE(na > 0 && nb > 0 && B >= 0, "shape");
  if (B == 0) return DAD3D_OK;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DAD3D_CUDA_OK(cudaMemsetAsync(out_d, 0, sizeof(float) * B, stream));
  for (int32_t h0 = 0; h0 < B; h0 += kMaxGridY) {
    const int32_t n = B - h0 < kMaxGridY ? B - h0 : kMaxGridY;
    chamfer_kernel<<<dim3((na + 255) / 256, n), 256, 0, stream>>>(a_d + static_cast<size_t>(h0) * na * 3, na,
                                                                  b_d + static_cast<size_t>(h0) * nb * 3, nb, out_d + h0);
    count_launch();
    DAD3D_CUDA_OK(cudaGetLastError());
  }
  return DAD3D_OK;
}

int dad3d_eval_zn(const float* pred_d, const float* gt_d, int32_t K, int32_t B, int32_t top_k, float* out_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(pred_d && gt_d && out_d, "null pointer");
  DAD3D_REQUIRE(K > top_k && K <= kZnMax && top_k >= 1 && B >= 0, "K must be in (top_k, 4096]");
  if (B == 0) return DAD3D_OK;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DAD3D_CUDA_OK(cudaMemsetAsync(out_d, 0, sizeof(float) * B, stream));
  for (int32_t h0 = 0; h0 < B; h0 += kMaxGridY) {
    const int32_t n = B - h0 < kMaxGridY ? B - h0 : kMaxGridY;
    const size_t off = static_cast<size_t>(h0) * K * 3;
    zn_kernel<<<dim3(top_k, n), 1024, 0, stream>>>(pred_d + off, gt_d + off, K, top_k, out_d + h0);
    count_launch();
    DAD3D_CUDA_OK(cudaGetLastError());
  }
  return DAD3D_OK;
}

int dad3d_eval_align(const float* verts_d, int32_t nv, int32_t B, const float* scale_d, const float* rot_d, const float* trans_d,
                     float* out_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(verts_d && scale_d && rot_d && trans_d && out_d, "null pointer");
  DAD3D_REQUIRE(nv > 0 && B >= 0, "shape");
  const long long total = static_cast<long long>(B) * nv;
  if (total == 0) return DAD3D_OK;
  align_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      verts_d, nv, B, scale_d, rot_d, trans_d, out_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // extern "C"
