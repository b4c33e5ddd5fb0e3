// Device pieces shared by the training losses (loss.cu) and the training metrics (metrics.cu): deterministic block
// reductions, normalize_to_cube's centring (model/utils.py:55-68), and the per-plane soft-IoU statistics.
#pragma once
#include <climits>
#include <cstdint>

namespace dad3d {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// ---- deterministic block reductions (256 threads; every thread gets the result) -------------------------------------
template <int N>
__device__ __forceinline__ void block_sum(float (&x)[N], float* sm /* [kWarps * N] */) {
#pragma unroll
  for (int k = 0; k < N; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x[k] += __shfl_xor_sync(0xffffffffu, x[k], o);
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) sm[w * N + k] = x[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; ++k) {
    float s = 0.f;
    for (int i = 0; i < kWarps; ++i) s += sm[i * N + k];
    x[k] = s;
  }
}

// (value, index) pairs: the extreme value, first index on ties -- the index torch's min / max over a dimension return.
// A NaN never wins a comparison, so it cannot be selected; a head whose values are all NaN keeps the sentinel index.
struct Ext {
  float v;
  int i;
};
template <bool MAX>
__device__ __forceinline__ bool beats(float a, int ia, float b, int ib) {
  return (MAX ? a > b : a < b) || (a == b && ia < ib);
}
template <bool MAX>
__device__ __forceinline__ void take(Ext& e, float v, int i) {
  if (beats<MAX>(v, i, e.v, e.i)) e = {v, i};
}
template <bool MAX, int N>
__device__ __forceinline__ void block_ext(Ext (&x)[N], Ext* sm /* [kWarps * N] */) {
#pragma unroll
  for (int k = 0; k < N; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float v = __shfl_xor_sync(0xffffffffu, x[k].v, o);
      const int i = __shfl_xor_sync(0xffffffffu, x[k].i, o);
      take<MAX>(x[k], v, i);
    }
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) sm[w * N + k] = x[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; ++k) {
    Ext e = sm[k];
    for (int i = 1; i < kWarps; ++i) take<MAX>(e, sm[i * N + k].v, sm[i * N + k].i);
    x[k] = e;
  }
}

template <bool MAX>
__device__ __forceinline__ Ext ext_init() { return {MAX ? -INFINITY : INFINITY, INT_MAX}; }

// normalize_to_cube before its final division: (v - min) - 0.5 * max(v - min), with half = 0.5 * max(v - min)
__device__ __forceinline__ float centred(float v, float mn, float half) { return __fsub_rn(__fsub_rn(v, mn), half); }

// ---- soft-IoU statistics per (b, c) plane -----------------------------------------------------------------------------
constexpr float kIouEps = 1e-6f;

// sigmoid(x) and sigmoid'(x) = s (1 - s) = q / (1 + q)^2 with q = exp(-|x|): no cancellation in 1 - s, no overflow
__device__ __forceinline__ void sigmoid2(float x, float& s, float& ds) {
  const float q = expf(-fabsf(x));
  const float r = 1.f / (1.f + q);
  s = x >= 0.f ? r : q * r;
  ds = q * r * r;
}

// (T + S) - I + eps: the reference's denominator
__device__ __forceinline__ float iou_den(float I, float T, float S, float eps = kIouEps) {
  return __fadd_rn(__fsub_rn(__fadd_rn(T, S), I), eps);
}

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// a target element as fp32: itself, or a uint8 heat-map byte as uint8_to_float32 makes it (x.div(255.0), model/flame.py:
// 232-236: fp32(u) / 255 rounded once)
__device__ __forceinline__ float target_value(float t) { return t; }
__device__ __forceinline__ float target_value(uint8_t u) { return static_cast<float>(u) / 255.f; }
__device__ __forceinline__ float4 load4(const float* p, int i) { return reinterpret_cast<const float4*>(p)[i]; }
__device__ __forceinline__ float4 load4(const uint8_t* p, int i) {
  const uchar4 u = reinterpret_cast<const uchar4*>(p)[i];
  return make_float4(target_value(u.x), target_value(u.y), target_value(u.z), target_value(u.w));
}

// One block per (b, c) plane: stats [P, 4] = (I = sum s t, T = sum t^2, S = sum s^2, iou = (I + eps) / (T + S - I + eps)),
// s = sigmoid(x) for LOGITS, else x itself (probabilities).
template <bool LOGITS, typename T>
__global__ void __launch_bounds__(kThreads)
iou_forward_kernel(const float* __restrict__ x, const T* __restrict__ t, int hw, float* __restrict__ stats) {
  __shared__ float sm[kWarps * 3];
  const size_t base = static_cast<size_t>(blockIdx.x) * hw;
  const float* xp = x + base;
  const T* tp = t + base;
  float a[3] = {0.f, 0.f, 0.f};
  auto add = [&](float xv, float tv) {
    float s = xv;
    if constexpr (LOGITS) {
      float ds;
      sigmoid2(xv, s, ds);
    }
    a[0] = fmaf(s, tv, a[0]);
    a[1] = fmaf(tv, tv, a[1]);
    a[2] = fmaf(s, s, a[2]);
  };
  if ((hw & 3) == 0 && aligned16(xp) && (reinterpret_cast<uintptr_t>(tp) & (4 * sizeof(T) - 1)) == 0) {
    const float4* x4 = reinterpret_cast<const float4*>(xp);
#pragma unroll 4
    for (int i = threadIdx.x; i < (hw >> 2); i += kThreads) {
      const float4 xv = x4[i], tv = load4(tp, i);
      add(xv.x, tv.x); add(xv.y, tv.y); add(xv.z, tv.z); add(xv.w, tv.w);
    }
  } else {
    for (int i = threadIdx.x; i < hw; i += kThreads) add(xp[i], target_value(tp[i]));
  }
  block_sum<3>(a, sm);
  if (threadIdx.x == 0) {
    float* st = stats + 4 * static_cast<size_t>(blockIdx.x);
    st[0] = a[0]; st[1] = a[1]; st[2] = a[2];
    st[3] = __fadd_rn(a[0], kIouEps) / iou_den(a[0], a[1], a[2]);
  }
}

}  // namespace dad3d
