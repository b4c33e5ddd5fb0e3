// The reference's training-step metrics (FlameLightningModel._step_fn, train/flame_lightning_model.py:299-357):
//   soft IoU of the heat-map                          metrics/iou.py:15-31
//   keypoint NME and "failure rate" (share of heads   metrics/keypoints.py:19-52, on the 2D landmarks, the reprojected
//   whose error is below threshold * norm)            face vertices and normalize_to_cube of the 3D face vertices
// Memory-bound reductions.  Per-plane / per-head partial results, then one single-CTA reduction in a fixed order (fp64 sums,
// integer counts), so values are bit-reproducible and no head's record depends on another head.  No floating-point atomics
// and nothing that synchronises with the host: a step's launches capture in a CUDA graph.
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"
#include "reductions.cuh"

namespace dad3d {

struct KpGroups {
  dad3d_kp_group g[DAD3D_METRIC_MAX_GROUPS];
};

struct Thresholds {
  float v[DAD3D_METRIC_MAX_THRESHOLDS];
};

// keypoint j of head b: prediction fp32(fp32(p * pred_scale) * m), target fp32(fp32(t * m) * target_scale), m the presence
// (1 without one) -- with m = 1 and unit scales both are p and t exactly
__device__ __forceinline__ void kp_operands(const dad3d_kp_group& G, int b, int j, float (&p)[3], float (&t)[3]) {
  const long long r = G.index_d ? G.index_d[j] : j;
  const float* pp = G.pred_d + b * G.pred_stride + r * G.k;
  const float* tp = G.target_d + b * G.target_stride + r * G.k;
  const float m = G.presence_d ? static_cast<float>(G.presence_d[b * G.presence_stride + j]) : 1.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p[c] = c < G.k ? __fmul_rn(__fmul_rn(pp[c], G.pred_scale), m) : 0.f;
    t[c] = c < G.k ? __fmul_rn(__fmul_rn(tp[c], m), G.target_scale) : 0.f;
  }
}

// |d|_2 with one rounding per step: d0 d0, then an fma per further coordinate
__device__ __forceinline__ float dist(const float (&d)[3], int k) {
  float s = __fmul_rn(d[0], d[0]);
  s = fmaf(d[1], d[1], s);
  if (k == 3) s = fmaf(d[2], d[2], s);
  return sqrtf(s);
}

// One block per (head, group): records [B, G, 2] = (err, norm).
__global__ void __launch_bounds__(kThreads)
keypoint_errors_kernel(const KpGroups gs, int G, float* __restrict__ records) {
  __shared__ float smf[kWarps];
  __shared__ Ext sme[kWarps * 6];
  const int b = blockIdx.x / G, g = blockIdx.x % G;
  const dad3d_kp_group& P = gs.g[g];
  const int n = P.n, K = P.k;
  float a[1] = {0.f};
  if (!P.normalize) {
    for (int j = threadIdx.x; j < n; j += kThreads) {
      float p[3], t[3], d[3];
      kp_operands(P, b, j, p, t);
#pragma unroll
      for (int c = 0; c < 3; ++c) d[c] = __fsub_rn(p[c], t[c]);
      a[0] += dist(d, K);
    }
  } else {
    // normalize_to_cube of prediction (k < 3) and target (k >= 3): min, then max of v - min, then the overall max of the
    // centred values; only values matter here, so the selected positions are not kept
    Ext lo[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) lo[k] = ext_init<false>();
    for (int j = threadIdx.x; j < n; j += kThreads) {
      float p[3], t[3];
      kp_operands(P, b, j, p, t);
#pragma unroll
      for (int c = 0; c < 3; ++c) { take<false>(lo[c], p[c], j); take<false>(lo[3 + c], t[c], j); }
    }
    block_ext<false, 6>(lo, sme);
    Ext hi[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) hi[k] = ext_init<true>();
    for (int j = threadIdx.x; j < n; j += kThreads) {
      float p[3], t[3];
      kp_operands(P, b, j, p, t);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        take<true>(hi[c], __fsub_rn(p[c], lo[c].v), j);
        take<true>(hi[3 + c], __fsub_rn(t[c], lo[3 + c].v), j);
      }
    }
    block_ext<true, 6>(hi, sme);
    float half[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) half[k] = 0.5f * hi[k].v;
    Ext top[2] = {ext_init<true>(), ext_init<true>()};
    for (int j = threadIdx.x; j < n; j += kThreads) {
      float p[3], t[3];
      kp_operands(P, b, j, p, t);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (c < K) {
          take<true>(top[0], centred(p[c], lo[c].v, half[c]), j * 3 + c);
          take<true>(top[1], centred(t[c], lo[3 + c].v, half[3 + c]), j * 3 + c);
        }
    }
    block_ext<true, 2>(top, sme);
    const float M = top[0].v, tM = top[1].v;
    for (int j = threadIdx.x; j < n; j += kThreads) {
      float p[3], t[3], d[3];
      kp_operands(P, b, j, p, t);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        d[c] = __fsub_rn(centred(p[c], lo[c].v, half[c]) / M, centred(t[c], lo[3 + c].v, half[3 + c]) / tM);
      a[0] += dist(d, K);
    }
  }
  block_sum<1>(a, smf);
  if (threadIdx.x == 0) {
    float norm = 2.f;
    if (P.box_w_d) {
      // torch.sqrt(bbox[:, 2] * bbox[:, 3]): the int32 product wraps, then it is rounded to fp32
      const uint32_t w = static_cast<uint32_t>(P.box_w_d[b * P.box_stride]);
      const uint32_t h = static_cast<uint32_t>(P.box_h_d[b * P.box_stride]);
      norm = sqrtf(static_cast<float>(static_cast<int32_t>(w * h)));
    }
    float* r = records + 2 * (static_cast<size_t>(b) * G + g);
    r[0] = a[0] / static_cast<float>(n);
    r[1] = norm;
  }
}

// fp64 sum over the block in a fixed order (per-thread strided sums, warp butterflies, warps in order); every thread gets it
__device__ __forceinline__ double block_dsum(double x, double* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = x;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < kWarps; ++i) s += sm[i];
  return s;
}

__device__ __forceinline__ int block_isum(int x, int* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = x;
  __syncthreads();
  int s = 0;
  for (int i = 0; i < kWarps; ++i) s += sm[i];
  return s;
}

__global__ void __launch_bounds__(kThreads)
metrics_reduce_kernel(const float* __restrict__ stats, int planes, float eps, const float* __restrict__ rec, int B, int G,
                      float nme_scale, int below, const Thresholds thr, int T, double weight, float* __restrict__ values,
                      float* __restrict__ per_head, double* __restrict__ epoch, float* __restrict__ epoch_values) {
  __shared__ double smd[kWarps];
  __shared__ int smi[kWarps];
  int nv = 0;
  if (stats) {
    double acc = 0.0;
    for (int p = threadIdx.x; p < planes; p += kThreads) {
      const float* st = stats + 4 * static_cast<size_t>(p);
      acc += static_cast<double>(__fadd_rn(st[0], eps) / iou_den(st[0], st[1], st[2], eps));
    }
    acc = block_dsum(acc, smd);
    if (threadIdx.x == 0) values[0] = static_cast<float>(acc / planes);
    nv = 1;
  }
  for (int g = 0; g < G; ++g) {
    double acc = 0.0;
    int cnt[DAD3D_METRIC_MAX_THRESHOLDS] = {0, 0, 0, 0};
    for (int b = threadIdx.x; b < B; b += kThreads) {
      const float* r = rec + 2 * (static_cast<size_t>(b) * G + g);
      const float err = r[0], norm = r[1];
      const float q = err / norm;
      if (per_head) per_head[static_cast<size_t>(b) * G + g] = q;
      acc += static_cast<double>(q);
#pragma unroll
      for (int t = 0; t < DAD3D_METRIC_MAX_THRESHOLDS; ++t) {
        const float bound = __fmul_rn(thr.v[t], norm);
        if (t < T) cnt[t] += below ? (err < bound) : (err > bound);
      }
    }
    acc = block_dsum(acc, smd);
    int tot[DAD3D_METRIC_MAX_THRESHOLDS];
#pragma unroll
    for (int t = 0; t < DAD3D_METRIC_MAX_THRESHOLDS; ++t) tot[t] = block_isum(cnt[t], smi);
    if (threadIdx.x == 0) {
      values[nv] = __fmul_rn(static_cast<float>(acc / B), nme_scale);
      for (int t = 0; t < T; ++t) values[nv + 1 + t] = static_cast<float>(tot[t]) / static_cast<float>(B);
    }
    nv += 1 + T;
  }
  if (epoch && threadIdx.x == 0) {
    for (int i = 0; i < nv; ++i) epoch[i] += static_cast<double>(values[i]) * weight;
    epoch[nv] += weight;
    for (int i = 0; i < nv; ++i) epoch_values[i] = static_cast<float>(epoch[i] / epoch[nv]);
  }
}

template <bool LOGITS>
void iou_stats_launch(const float* x_d, const void* t_d, bool u8, int planes, int hw, float* stats_d, cudaStream_t s) {
  if (u8)
    iou_forward_kernel<LOGITS, uint8_t><<<planes, kThreads, 0, s>>>(x_d, static_cast<const uint8_t*>(t_d), hw, stats_d);
  else
    iou_forward_kernel<LOGITS, float><<<planes, kThreads, 0, s>>>(x_d, static_cast<const float*>(t_d), hw, stats_d);
}

}  // namespace dad3d

using namespace dad3d;

extern "C" {

int dad3d_iou_stats(const float* x_d, const void* t_d, int32_t target_u8, int32_t logits, int32_t planes, int32_t hw,
                    float* stats_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(x_d && t_d && stats_d, "null pointer");
  DAD3D_REQUIRE(planes >= 1 && hw >= 1, "shape");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (logits)
    iou_stats_launch<true>(x_d, t_d, target_u8 != 0, planes, hw, stats_d, stream);
  else
    iou_stats_launch<false>(x_d, t_d, target_u8 != 0, planes, hw, stats_d, stream);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_keypoint_errors(const dad3d_kp_group* groups_h, int32_t G, int32_t B, float* records_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(groups_h && records_d, "null pointer");
  DAD3D_REQUIRE(G >= 1 && G <= DAD3D_METRIC_MAX_GROUPS, "G must be 1 to DAD3D_METRIC_MAX_GROUPS");
  DAD3D_REQUIRE(B >= 1 && static_cast<long long>(B) * G <= INT_MAX, "B out of range");
  KpGroups gs = {};
  for (int g = 0; g < G; ++g) {
    const dad3d_kp_group& P = groups_h[g];
    DAD3D_REQUIRE(P.pred_d && P.target_d, "null pointer");
    DAD3D_REQUIRE(P.k == 2 || P.k == 3, "k must be 2 or 3");
    DAD3D_REQUIRE(P.n >= 1, "a group needs at least one keypoint");
    DAD3D_REQUIRE((P.box_w_d == nullptr) == (P.box_h_d == nullptr), "box widths and heights come together");
    gs.g[g] = P;
  }
  keypoint_errors_kernel<<<B * G, kThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(gs, G, records_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_metrics_reduce(const float* stats_d, int32_t planes, float eps, const float* records_d, int32_t B, int32_t G,
                         float nme_scale, int32_t below, const float* thresholds_h, int32_t n_thresholds, double weight,
                         float* values_d, float* per_head_d, double* epoch_d, float* epoch_values_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(values_d, "null pointer");
  DAD3D_REQUIRE(stats_d || records_d, "nothing to reduce");
  DAD3D_REQUIRE(!stats_d || planes >= 1, "planes");
  DAD3D_REQUIRE(!records_d || (G >= 1 && G <= DAD3D_METRIC_MAX_GROUPS && B >= 1), "G, B");
  DAD3D_REQUIRE(n_thresholds >= 0 && n_thresholds <= DAD3D_METRIC_MAX_THRESHOLDS && (n_thresholds == 0 || thresholds_h),
                "thresholds");
  DAD3D_REQUIRE((epoch_d == nullptr) == (epoch_values_d == nullptr), "epoch_d and epoch_values_d come together");
  Thresholds thr = {};
  for (int t = 0; t < n_thresholds; ++t) thr.v[t] = thresholds_h[t];
  metrics_reduce_kernel<<<1, kThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      stats_d, planes, eps, records_d, B, records_d ? G : 0, nme_scale, below, thr, n_thresholds, weight, values_d,
      per_head_d, epoch_d, epoch_values_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // extern "C"
