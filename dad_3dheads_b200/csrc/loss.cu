// The reference's training losses (config/loss/train_loss.yaml) and their gradients:
//   heat-map IoU                 losses/keypoint_losses.py:5-31
//   landmarks with visibility    losses/landmarks_loss_w_visibility.py:10-26
//   vertex-subset losses         losses/vertices_3d_loss.py:30-48 (normalize_to_cube, model/utils.py:55-68) and
//                                losses/reprojection_loss.py:22-46, over the index sets of utils.py:108-117
// Memory-bound elementwise and reduction work.  Forward and backward are separate kernels; every reduction is a per-plane /
// per-head partial sum followed by one sum in a fixed order (no floating-point atomics), so results are bit-reproducible and
// one head's values never reach another head's gradient.  Backward kernels read the incoming loss gradient from device
// memory: nothing here synchronises with the host, so forward and backward can be captured in a CUDA graph.
#include <climits>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/dad3d.h"
#include "common.h"
#include "reductions.cuh"

struct dad3d_vsub {
  int32_t S = 0, V = 0, E = 0, device = 0;
  int32_t* idx_d = nullptr;        // [E] the sets' vertex indices, concatenated in set order
  int32_t* off_d = nullptr;        // [S + 1] where each set starts in idx_d
  int32_t* ent_set_d = nullptr;    // [E] set of each entry
  int32_t* inv_off_d = nullptr;    // [V + 1] per vertex, where its entries start in inv_ent_d
  int32_t* inv_ent_d = nullptr;    // [E] entries of each vertex, ascending (= set order, then position)
  float* w_d = nullptr;            // [S] set weights
};

namespace dad3d {

// ---- criteria (nn.L1Loss / nn.MSELoss / nn.SmoothL1Loss(beta = 1) before their mean) ------------------------------------
// Every fp32 and fp64 site nvcc could contract is written with an explicit rounding, in the form nvcc already chose (the
// SASS is unchanged), so tests/loss_model.py can restate each kernel exactly.
__device__ __forceinline__ float crit_value(int crit, float d) {
  const float a = fabsf(d);
  if (crit == DAD3D_LOSS_L1) return a;
  if (crit == DAD3D_LOSS_L2) return __fmul_rn(d, d);
  return a < 1.f ? __fmul_rn(__fmul_rn(0.5f, d), d) : __fsub_rn(a, 0.5f);
}

// acc + crit_value(crit, d): l2's square is fused into the sum; the other criteria round their value, then the sum
__device__ __forceinline__ float crit_accum(int crit, float d, float acc) {
  const float a = fabsf(d);
  if (crit == DAD3D_LOSS_L1) return __fadd_rn(acc, a);
  if (crit == DAD3D_LOSS_L2) return __fmaf_rn(d, d, acc);
  return __fadd_rn(acc, a < 1.f ? __fmul_rn(__fmul_rn(0.5f, d), d) : __fsub_rn(a, 0.5f));
}

__device__ __forceinline__ float crit_grad(int crit, float d) {
  const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
  if (crit == DAD3D_LOSS_L1) return sg;
  if (crit == DAD3D_LOSS_L2) return __fadd_rn(d, d);      // 2 d, exact
  return fabsf(d) < 1.f ? d : sg;
}

// ---- finalize: out = bias + sum_s coef_s * sum_b x[b * ld + s * sld], in fp64, in a fixed order ----------------------
// coef_s = scale * w[s] / |set s| for the vertex-subset losses (w, off given), else scale.
__global__ void __launch_bounds__(kThreads)
finalize_kernel(const float* __restrict__ x, int B, int S, long long ld, int sld, const float* __restrict__ w,
                const int32_t* __restrict__ off, double scale, double bias, float* __restrict__ out) {
  __shared__ double sm[kWarps];
  double total = bias;
  for (int s = 0; s < S; ++s) {
    double acc = 0.0;
    for (int b = threadIdx.x; b < B; b += kThreads)
      acc = __dadd_rn(acc, static_cast<double>(x[b * ld + static_cast<long long>(s) * sld]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    double sum = 0.0;
    for (int i = 0; i < kWarps; ++i) sum = __dadd_rn(sum, sm[i]);
    const double coef = w ? __dmul_rn(scale, static_cast<double>(w[s])) / static_cast<double>(off[s + 1] - off[s]) : scale;
    total = __fma_rn(coef, sum, total);
  }
  if (threadIdx.x == 0) *out = static_cast<float>(total);
}

// ---- heat-map IoU ---------------------------------------------------------------------------------------------------
// The forward's per-plane statistics are iou_forward_kernel<true, float> (reductions.cuh), shared with the metrics.
// d loss / d x = -g / P * (t D - N (2 s - t)) / D^2 * s (1 - s),  N = I + eps, D = T + S - I + eps
__global__ void __launch_bounds__(kThreads)
iou_backward_kernel(const float* __restrict__ x, const float* __restrict__ t, int hw, int P, const float* __restrict__ stats,
                    const float* __restrict__ grad_out, float* __restrict__ gx) {
  const size_t base = static_cast<size_t>(blockIdx.x) * hw;
  const float* xp = x + base;
  const float* tp = t + base;
  float* gp = gx + base;
  const float* st = stats + 4 * static_cast<size_t>(blockIdx.x);
  const float N = __fadd_rn(st[0], kIouEps), D = iou_den(st[0], st[1], st[2]);
  const float coef = -*grad_out / (static_cast<float>(P) * D * D);
  auto grad = [&](float xv, float tv) {
    float s, ds;
    sigmoid2(xv, s, ds);
    return __fmul_rn(__fmul_rn(coef, __fmaf_rn(tv, D, -__fmul_rn(N, __fsub_rn(__fadd_rn(s, s), tv)))), ds);
  };
  if ((hw & 3) == 0 && aligned16(xp) && aligned16(tp) && aligned16(gp)) {
    const float4* x4 = reinterpret_cast<const float4*>(xp);
    const float4* t4 = reinterpret_cast<const float4*>(tp);
    float4* g4 = reinterpret_cast<float4*>(gp);
#pragma unroll 4
    for (int i = threadIdx.x; i < (hw >> 2); i += kThreads) {
      const float4 xv = x4[i], tv = t4[i];
      g4[i] = make_float4(grad(xv.x, tv.x), grad(xv.y, tv.y), grad(xv.z, tv.z), grad(xv.w, tv.w));
    }
  } else {
    for (int i = threadIdx.x; i < hw; i += kThreads) gp[i] = grad(xp[i], tp[i]);
  }
}

// ---- landmarks with visibility: criterion(p * mp, t * mt), mean over B N 2 ---------------------------------------------
__global__ void lmk_forward_kernel(const float* __restrict__ p, const float* __restrict__ pm, const float* __restrict__ t,
                                   const float* __restrict__ tm, int B, int N, int crit, float* __restrict__ partial) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double acc = 0.0;
  for (int n = 0; n < N; ++n) {
    const size_t i = static_cast<size_t>(b) * N + n;
    const float mp = pm[i], mt = tm[i];
#pragma unroll
    for (int c = 0; c < 2; ++c) acc += crit_value(crit, __fmaf_rn(p[2 * i + c], mp, -__fmul_rn(t[2 * i + c], mt)));
  }
  partial[b] = static_cast<float>(acc);
}

__global__ void lmk_backward_kernel(const float* __restrict__ p, const float* __restrict__ pm, const float* __restrict__ t,
                                    const float* __restrict__ tm, int B, int N, int crit, const float* __restrict__ grad_out,
                                    float* __restrict__ gp) {
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= 2LL * B * N) return;
  const long long i = e >> 1;
  const float scale = *grad_out / (2.f * static_cast<float>(B) * static_cast<float>(N));
  const float mp = pm[i];
  gp[e] = __fmul_rn(__fmul_rn(scale, crit_grad(crit, __fmaf_rn(p[e], mp, -__fmul_rn(t[e], tm[i])))), mp);
}

// ---- vertex-subset losses ---------------------------------------------------------------------------------------------
// Per (head, set) record, DAD3D_VSUB_RECORD_FLOATS words.  With normalisation, for prediction (p) and target (t):
// mn = min over the set per coordinate, half = 0.5 * max(v - mn) per coordinate, M = max over (vertex, coordinate) of
// (v - mn) - half (first in vertex-then-coordinate order on ties, as max(-1) then max(-2) select), and the positions that
// won each reduction.  u = ((v - mn) - half) / M is normalize_to_cube's output.  The forward also stores the g-free sums the
// backward needs: sco = sum c'(u - w) u, sg[c] = sum_n c'(u - w)[n, c].
struct VsubRec {
  float loss;
  float mn[3], half[3], M;
  float tmn[3], thalf[3], tM;
  int32_t amin[3], amax[3], nstar, cstar;
  float sco, sg[3];
};
static_assert(sizeof(VsubRec) <= DAD3D_VSUB_RECORD_FLOATS * sizeof(float), "record size");

// one block per (head, set)
template <int K, bool NORM>
__global__ void __launch_bounds__(kThreads)
vsub_forward_kernel(const float* __restrict__ v, const float* __restrict__ t, int V, const int32_t* __restrict__ idx,
                    const int32_t* __restrict__ off, int S, int crit, float* __restrict__ rec) {
  __shared__ float smf[kWarps * 5];
  __shared__ Ext sme[kWarps * 2 * K];
  const int b = blockIdx.x / S, s = blockIdx.x % S;
  const int j0 = off[s], n = off[s + 1] - j0;
  const int32_t* I = idx + j0;
  const float* vb = v + static_cast<size_t>(b) * V * K;
  const float* tb = t + static_cast<size_t>(b) * V * K;
  VsubRec* R = reinterpret_cast<VsubRec*>(rec + static_cast<size_t>(blockIdx.x) * DAD3D_VSUB_RECORD_FLOATS);
  if constexpr (!NORM) {
    float a[1] = {0.f};
    for (int j = threadIdx.x; j < n; j += kThreads) {
      const size_t q = static_cast<size_t>(I[j]) * K;
#pragma unroll
      for (int c = 0; c < K; ++c) a[0] = crit_accum(crit, vb[q + c] - tb[q + c], a[0]);
    }
    block_sum<1>(a, smf);
    if (threadIdx.x == 0) R->loss = a[0];
  } else {
    // pass 1: per-coordinate minima (with the winning position for the prediction)
    Ext lo[2 * K];
#pragma unroll
    for (int k = 0; k < 2 * K; ++k) lo[k] = ext_init<false>();
    for (int j = threadIdx.x; j < n; j += kThreads) {
      const size_t q = static_cast<size_t>(I[j]) * K;
#pragma unroll
      for (int c = 0; c < K; ++c) { take<false>(lo[c], vb[q + c], j); take<false>(lo[K + c], tb[q + c], j); }
    }
    block_ext<false, 2 * K>(lo, sme);
    // pass 2: per-coordinate maxima of v - mn
    Ext hi[2 * K];
#pragma unroll
    for (int k = 0; k < 2 * K; ++k) hi[k] = ext_init<true>();
    for (int j = threadIdx.x; j < n; j += kThreads) {
      const size_t q = static_cast<size_t>(I[j]) * K;
#pragma unroll
      for (int c = 0; c < K; ++c) {
        take<true>(hi[c], __fsub_rn(vb[q + c], lo[c].v), j);
        take<true>(hi[K + c], __fsub_rn(tb[q + c], lo[K + c].v), j);
      }
    }
    block_ext<true, 2 * K>(hi, sme);
    float half[2 * K];
#pragma unroll
    for (int k = 0; k < 2 * K; ++k) half[k] = 0.5f * hi[k].v;
    // pass 3: the overall maximum of the centred values, first in (position, coordinate) order
    Ext top[2] = {ext_init<true>(), ext_init<true>()};
    for (int j = threadIdx.x; j < n; j += kThreads) {
      const size_t q = static_cast<size_t>(I[j]) * K;
#pragma unroll
      for (int c = 0; c < K; ++c) {
        take<true>(top[0], centred(vb[q + c], lo[c].v, half[c]), j * K + c);
        take<true>(top[1], centred(tb[q + c], lo[K + c].v, half[K + c]), j * K + c);
      }
    }
    block_ext<true, 2>(top, sme);
    const float M = top[0].v, tM = top[1].v;
    // pass 4: criterion sum and the backward's g-free sums
    float a[2 + K];
#pragma unroll
    for (int k = 0; k < 2 + K; ++k) a[k] = 0.f;
    for (int j = threadIdx.x; j < n; j += kThreads) {
      const size_t q = static_cast<size_t>(I[j]) * K;
#pragma unroll
      for (int c = 0; c < K; ++c) {
        const float u = centred(vb[q + c], lo[c].v, half[c]) / M;
        const float w = centred(tb[q + c], lo[K + c].v, half[K + c]) / tM;
        const float d = u - w;
        const float cd = crit_grad(crit, d);
        a[0] = crit_accum(crit, d, a[0]);
        a[1] = fmaf(cd, u, a[1]);
        a[2 + c] += cd;
      }
    }
    block_sum<2 + K>(a, smf);
    if (threadIdx.x == 0) {
      R->loss = a[0];
      R->M = M;
      R->tM = tM;
      R->sco = a[1];
      R->nstar = top[0].i == INT_MAX ? -1 : top[0].i / K;
      R->cstar = top[0].i == INT_MAX ? -1 : top[0].i % K;
      for (int c = 0; c < 3; ++c) {
        const bool in = c < K;
        R->mn[c] = in ? lo[c].v : 0.f;
        R->tmn[c] = in ? lo[K + c].v : 0.f;
        R->half[c] = in ? half[c] : 0.f;
        R->thalf[c] = in ? half[K + c] : 0.f;
        R->amin[c] = in ? lo[c].i : -1;
        R->amax[c] = in ? hi[c].i : -1;
        R->sg[c] = in ? a[2 + c] : 0.f;
      }
    }
  }
}

// One thread per (head, vertex): the sum, over the vertex's entries in set order, of each entry's gradient; zero for a
// vertex in no set.  Normalised: with G = coef c'(u - w), coef = g w_s / (B |set| K),
//   d/dv = G / M                                       every entry
//        + dM,   dM = -coef sco / M                    the entry and coordinate that gave M
//        + A_c,  A_c = -0.5 (coef sg[c] / M + [c == c*] dM)   the entries that gave max(v - mn) and min(v), coordinate c
// (the chain rule through v / M, v - 0.5 max(v), v - min(v), routing each reduction's gradient to its selected entry).
template <int K, bool NORM>
__global__ void __launch_bounds__(kThreads)
vsub_backward_kernel(const float* __restrict__ v, const float* __restrict__ t, int B, int V, dad3d_vsub h_, int crit,
                     const float* __restrict__ rec, const float* __restrict__ grad_out, float* __restrict__ gv) {
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<long long>(B) * V) return;
  const int b = static_cast<int>(e / V), vtx = static_cast<int>(e % V);
  const float g = *grad_out;
  const size_t q = static_cast<size_t>(e) * K;
  float x[K], y[K], acc[K];
#pragma unroll
  for (int c = 0; c < K; ++c) { x[c] = v[q + c]; y[c] = t[q + c]; acc[c] = 0.f; }
  for (int k = h_.inv_off_d[vtx]; k < h_.inv_off_d[vtx + 1]; ++k) {
    const int ent = h_.inv_ent_d[k];
    const int s = h_.ent_set_d[ent];
    const int pos = ent - h_.off_d[s];
    const int n = h_.off_d[s + 1] - h_.off_d[s];
    const float coef = g * (h_.w_d[s] / (static_cast<float>(B) * static_cast<float>(n) * static_cast<float>(K)));
    const VsubRec* R = reinterpret_cast<const VsubRec*>(rec + (static_cast<size_t>(b) * h_.S + s) * DAD3D_VSUB_RECORD_FLOATS);
    if constexpr (NORM) {
      const float M = R->M;
      const float dM = -coef * R->sco / M;
#pragma unroll
      for (int c = 0; c < K; ++c) {
        const float u = centred(x[c], R->mn[c], R->half[c]) / M;
        const float w = centred(y[c], R->tmn[c], R->thalf[c]) / R->tM;
        float d = coef * crit_grad(crit, u - w) / M;
        const float A = -0.5f * (coef * R->sg[c] / M + (c == R->cstar ? dM : 0.f));
        if (pos == R->nstar && c == R->cstar) d += dM;
        if (pos == R->amax[c]) d += A;
        if (pos == R->amin[c]) d += A;
        acc[c] += d;
      }
    } else {
#pragma unroll
      for (int c = 0; c < K; ++c) acc[c] = __fmaf_rn(coef, crit_grad(crit, x[c] - y[c]), acc[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < K; ++c) gv[q + c] = acc[c];
}

template <int K, bool NORM>
int vsub_launch(const dad3d_vsub* h, const float* v_d, const float* t_d, int32_t B, int32_t crit, float* rec_d,
                const float* grad_out_d, float* grad_d, float* loss_d, cudaStream_t stream) {
  if (grad_d == nullptr) {
    vsub_forward_kernel<K, NORM><<<B * h->S, kThreads, 0, stream>>>(v_d, t_d, h->V, h->idx_d, h->off_d, h->S, crit, rec_d);
    count_launch();
    DAD3D_CUDA_OK(cudaGetLastError());
    finalize_kernel<<<1, kThreads, 0, stream>>>(rec_d, B, h->S, static_cast<long long>(h->S) * DAD3D_VSUB_RECORD_FLOATS,
                                                DAD3D_VSUB_RECORD_FLOATS, h->w_d, h->off_d, 1.0 / (static_cast<double>(B) * K),
                                                0.0, loss_d);
  } else {
    const long long n = static_cast<long long>(B) * h->V;
    vsub_backward_kernel<K, NORM><<<static_cast<unsigned>((n + kThreads - 1) / kThreads), kThreads, 0, stream>>>(
        v_d, t_d, B, h->V, *h, crit, rec_d, grad_out_d, grad_d);
  }
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int vsub_run(const dad3d_vsub* h, const float* v_d, const float* t_d, int32_t B, int32_t K, int32_t normalize, int32_t crit,
             float* rec_d, const float* grad_out_d, float* grad_d, float* loss_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(h && v_d && t_d && rec_d, "null pointer");
  DAD3D_REQUIRE(K == 2 || K == 3, "K must be 2 or 3");
  DAD3D_REQUIRE(crit >= DAD3D_LOSS_L1 && crit <= DAD3D_LOSS_SMOOTH_L1, "criterion");
  DAD3D_REQUIRE(B >= 1 && static_cast<long long>(B) * h->S <= INT_MAX && static_cast<long long>(B) * h->V * K <= INT_MAX,
                "B out of range");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (K == 3) return normalize ? vsub_launch<3, true>(h, v_d, t_d, B, crit, rec_d, grad_out_d, grad_d, loss_d, stream)
                               : vsub_launch<3, false>(h, v_d, t_d, B, crit, rec_d, grad_out_d, grad_d, loss_d, stream);
  return normalize ? vsub_launch<2, true>(h, v_d, t_d, B, crit, rec_d, grad_out_d, grad_d, loss_d, stream)
                   : vsub_launch<2, false>(h, v_d, t_d, B, crit, rec_d, grad_out_d, grad_d, loss_d, stream);
}

}  // namespace dad3d

using namespace dad3d;

extern "C" {

int dad3d_iou_forward(const float* x_d, const float* t_d, int32_t planes, int32_t hw, float* stats_d, float* loss_d,
                      dad3d_stream stream_) {
  DAD3D_REQUIRE(x_d && t_d && stats_d && loss_d, "null pointer");
  DAD3D_REQUIRE(planes >= 1 && hw >= 1, "shape");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  iou_forward_kernel<true, float><<<planes, kThreads, 0, stream>>>(x_d, t_d, hw, stats_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  finalize_kernel<<<1, kThreads, 0, stream>>>(stats_d + 3, planes, 1, 4, 0, nullptr, nullptr, -1.0 / planes, 1.0, loss_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_iou_backward(const float* x_d, const float* t_d, int32_t planes, int32_t hw, const float* stats_d,
                       const float* grad_out_d, float* grad_x_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(x_d && t_d && stats_d && grad_out_d && grad_x_d, "null pointer");
  DAD3D_REQUIRE(planes >= 1 && hw >= 1, "shape");
  iou_backward_kernel<<<planes, kThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(x_d, t_d, hw, planes, stats_d,
                                                                                        grad_out_d, grad_x_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_landmarks_forward(const float* p_d, const float* p_presence_d, const float* t_d, const float* t_presence_d,
                            int32_t B, int32_t N, int32_t criterion, float* partial_d, float* loss_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(p_d && p_presence_d && t_d && t_presence_d && partial_d && loss_d, "null pointer");
  DAD3D_REQUIRE(B >= 1 && N >= 1 && 2LL * B * N <= INT_MAX, "shape");
  DAD3D_REQUIRE(criterion >= DAD3D_LOSS_L1 && criterion <= DAD3D_LOSS_SMOOTH_L1, "criterion");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  lmk_forward_kernel<<<ceil_div(B, 128), 128, 0, stream>>>(p_d, p_presence_d, t_d, t_presence_d, B, N, criterion, partial_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  finalize_kernel<<<1, kThreads, 0, stream>>>(partial_d, B, 1, 1, 0, nullptr, nullptr, 1.0 / (2.0 * B * N), 0.0, loss_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_landmarks_backward(const float* p_d, const float* p_presence_d, const float* t_d, const float* t_presence_d,
                             int32_t B, int32_t N, int32_t criterion, const float* grad_out_d, float* grad_p_d,
                             dad3d_stream stream_) {
  DAD3D_REQUIRE(p_d && p_presence_d && t_d && t_presence_d && grad_out_d && grad_p_d, "null pointer");
  DAD3D_REQUIRE(B >= 1 && N >= 1 && 2LL * B * N <= INT_MAX, "shape");
  DAD3D_REQUIRE(criterion >= DAD3D_LOSS_L1 && criterion <= DAD3D_LOSS_SMOOTH_L1, "criterion");
  lmk_backward_kernel<<<ceil_div(2 * B * N, kThreads), kThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      p_d, p_presence_d, t_d, t_presence_d, B, N, criterion, grad_out_d, grad_p_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

void dad3d_vsub_destroy(dad3d_vsub* h) {
  if (!h) return;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->device);
  for (void* p : {static_cast<void*>(h->idx_d), static_cast<void*>(h->off_d), static_cast<void*>(h->ent_set_d),
                  static_cast<void*>(h->inv_off_d), static_cast<void*>(h->inv_ent_d), static_cast<void*>(h->w_d)})
    if (p) cudaFree(p);
  cudaSetDevice(prev);
  delete h;
}

static int vsub_upload(dad3d_vsub* h, const std::vector<int32_t>& idx, const std::vector<int32_t>& off,
                       const std::vector<int32_t>& ent_set, const std::vector<int32_t>& inv_off,
                       const std::vector<int32_t>& inv_ent, const float* weights_h) {
  auto up = [](auto** dst, const void* src, size_t bytes) -> cudaError_t {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(dst), bytes);
    return e != cudaSuccess ? e : cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice);
  };
  DAD3D_CUDA_OK(up(&h->idx_d, idx.data(), idx.size() * 4));
  DAD3D_CUDA_OK(up(&h->off_d, off.data(), off.size() * 4));
  DAD3D_CUDA_OK(up(&h->ent_set_d, ent_set.data(), ent_set.size() * 4));
  DAD3D_CUDA_OK(up(&h->inv_off_d, inv_off.data(), inv_off.size() * 4));
  DAD3D_CUDA_OK(up(&h->inv_ent_d, inv_ent.data(), inv_ent.size() * 4));
  DAD3D_CUDA_OK(up(&h->w_d, weights_h, static_cast<size_t>(h->S) * 4));
  return DAD3D_OK;
}

int dad3d_vsub_create(dad3d_vsub** out, const int32_t* indices_h, const int32_t* offsets_h, const float* weights_h, int32_t S,
                      int32_t V, int32_t device) {
  DAD3D_REQUIRE(out && indices_h && offsets_h && weights_h, "null pointer");
  DAD3D_REQUIRE(S >= 1 && V >= 1 && offsets_h[0] == 0, "S, V, offsets[0]");
  *out = nullptr;
  for (int32_t s = 0; s < S; ++s) DAD3D_REQUIRE(offsets_h[s + 1] > offsets_h[s], "every set needs at least one index");
  const int32_t E = offsets_h[S];
  for (int32_t e = 0; e < E; ++e) DAD3D_REQUIRE(indices_h[e] >= 0 && indices_h[e] < V, "index outside [0, V)");
  std::vector<int32_t> idx(indices_h, indices_h + E), off(offsets_h, offsets_h + S + 1), ent_set(E), inv_off(V + 1, 0),
      inv_ent(E);
  for (int32_t s = 0; s < S; ++s)
    for (int32_t e = off[s]; e < off[s + 1]; ++e) ent_set[e] = s;
  for (int32_t e = 0; e < E; ++e) ++inv_off[idx[e] + 1];
  for (int32_t v = 0; v < V; ++v) inv_off[v + 1] += inv_off[v];
  std::vector<int32_t> fill(inv_off.begin(), inv_off.end() - 1);
  for (int32_t e = 0; e < E; ++e) inv_ent[fill[idx[e]]++] = e;       // ascending entries per vertex
  int prev = 0;
  DAD3D_CUDA_OK(cudaGetDevice(&prev));
  DAD3D_CUDA_OK(cudaSetDevice(device));
  dad3d_vsub* h = new dad3d_vsub;
  h->S = S; h->V = V; h->E = E; h->device = device;
  const int rc = vsub_upload(h, idx, off, ent_set, inv_off, inv_ent, weights_h);
  cudaSetDevice(prev);
  if (rc != DAD3D_OK) {
    dad3d_vsub_destroy(h);
    return rc;
  }
  *out = h;
  return DAD3D_OK;
}

int dad3d_vsub_forward(const dad3d_vsub* h, const float* v_d, const float* t_d, int32_t B, int32_t K, int32_t normalize,
                       int32_t criterion, float* records_d, float* loss_d, dad3d_stream stream) {
  DAD3D_REQUIRE(loss_d, "null pointer");
  return vsub_run(h, v_d, t_d, B, K, normalize, criterion, records_d, nullptr, nullptr, loss_d, stream);
}

int dad3d_vsub_backward(const dad3d_vsub* h, const float* v_d, const float* t_d, int32_t B, int32_t K, int32_t normalize,
                        int32_t criterion, const float* records_d, const float* grad_out_d, float* grad_v_d,
                        dad3d_stream stream) {
  DAD3D_REQUIRE(grad_out_d && grad_v_d, "null pointer");
  return vsub_run(h, v_d, t_d, B, K, normalize, criterion, const_cast<float*>(records_d), grad_out_d, grad_v_d, nullptr,
                  stream);
}

}  // extern "C"
