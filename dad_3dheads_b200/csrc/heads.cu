// DAD-3DNet's three ClassificationHeads (flame_regression.py:45-59) and their epilogue (:96-100), forward and weight
// gradients, for training the heads over a frozen backbone.  Weights are packed: w1 [1536, 2048] (shape | pose | landmarks
// rows of logit_image.0), b1 [1536], w2 [549, 512] (rows 0-402 shape, 403-412 pose, 413-548 landmarks; row r reads the
// 512-wide hidden block of its head), b2 [549].
//
// All arithmetic is fp32 on the CUDA cores.  Every sum runs in a fixed order (tests/heads_model.py restates each one), and
// there are no floating-point atomics, so results are bit-reproducible.  The weights change every step, so they are read as
// they are rather than packed for the tile engine; the products are small (at B = 64 the first layer is 0.40 GFLOP).
//
// Launches:  forward   gemm (f w1^T, split over K) -> hidden (sum splits + b1, relu, dropout) -> gemm (d w2^T per head,
//                      split over K) -> output (sum splits + b2, tanh * limit | identity | relu)
//            backward  dout (do and db2) -> gemm (dw2 and dd per head, one launch) -> dhidden (dh and db1) -> gemm (dw1)
#include <algorithm>
#include <cstdint>

#include "../../include/dad3d.h"
#include "common.h"

namespace dad3d {
namespace {

constexpr int kFeat = 2048, kHid = 512, kHidAll = 1536, kOut = 549, kShape = 403, kParams = 413, kLms = 136;
constexpr int kMaskWords = kHidAll / 32;          // 48: dropout keep bits of one row
constexpr int kOutWords = (kOut + 31) / 32;       // 18: o > 0 bits of one row
constexpr int kHeadRows[3] = {kShape, kParams - kShape, kLms};
constexpr int kFc1Splits = 8, kFc2Splits = 4;     // K = 2048 and 512 in chunks of 256 and 128
constexpr int kTile = 64, kTk = 16, kThreads = 256;
constexpr int kMaxProblems = 6;

// C(m, n) = sum_k A(m, k) B(k, n) over k in [s * kchunk, min(K, (s + 1) * kchunk)) for split s = blockIdx.y, one fma per
// k in increasing order from 0.f, stored to c + s * split_stride.  A(m, k) = a[m * sam + k * sak], B(k, n) = b[k * sbk +
// n * sbn], C(m, n) = c[m * ldc + n].
struct GemmProblem {
  const float* a;
  long long sam, sak;
  const float* b;
  long long sbk, sbn;
  float* c;
  long long ldc, split_stride;
  int M, N, K, kchunk, tiles_n, tile0;    // tile0: first flat tile index of this problem in the launch
};
struct GemmBatch {
  GemmProblem p[kMaxProblems];
  int count;
};

// 64 x 64 output tile per CTA; thread (tm, tn) owns rows tm + 16 i and columns tn + 16 j, i, j < 4.  Operands stage through
// shared memory 16 k at a time; out-of-range elements stage as 0, and fma(0, 0, acc) == acc for an acc that starts at +0.
__global__ void __launch_bounds__(kThreads) heads_gemm_kernel(const __grid_constant__ GemmBatch g) {
  int t = blockIdx.x, pi = 0;
  while (pi + 1 < g.count && t >= g.p[pi + 1].tile0) ++pi;
  const GemmProblem& P = g.p[pi];
  const int kb = blockIdx.y * P.kchunk;
  if (kb >= P.K) return;
  const int ke = min(P.K, kb + P.kchunk);
  t -= P.tile0;
  const int m0 = (t / P.tiles_n) * kTile, n0 = (t % P.tiles_n) * kTile;
  __shared__ float As[kTk][kTile + 1], Bs[kTk][kTile + 1];
  const int tid = threadIdx.x, tm = tid >> 4, tn = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = kb; k0 < ke; k0 += kTk) {
#pragma unroll
    for (int i = 0; i < kTile * kTk / kThreads; ++i) {
      const int e = tid + i * kThreads;
      // the unit-stride index runs fastest, so the loads coalesce
      const int am = P.sak == 1 ? e / kTk : e % kTile, ak = P.sak == 1 ? e % kTk : e / kTile;
      const int bn = P.sbk == 1 ? e / kTk : e % kTile, bk = P.sbk == 1 ? e % kTk : e / kTile;
      const int gm = m0 + am, gak = k0 + ak, gn = n0 + bn, gbk = k0 + bk;
      As[ak][am] = (gm < P.M && gak < ke) ? __ldg(P.a + gm * P.sam + gak * P.sak) : 0.f;
      Bs[bk][bn] = (gn < P.N && gbk < ke) ? __ldg(P.b + gbk * P.sbk + gn * P.sbn) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kTk; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[k][tm + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[k][tn + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = __fmaf_rn(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* c = P.c + blockIdx.y * P.split_stride;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gm = m0 + tm + 16 * i, gn = n0 + tn + 16 * j;
      if (gm < P.M && gn < P.N) c[gm * P.ldc + gn] = acc[i][j];
    }
}

// Philox4x32-10 (Salmon et al., SC'11; Random123's philox4x32 with 10 rounds)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// Block of 8 warps over 32 columns: warp w takes rows w, w + 8, ... of column blockIdx.x * 32 + lane.  A column sum over the
// rows runs per warp in row order from 0.f, then over the 8 warps in order.
__device__ __forceinline__ float column_total(float part, float (*red)[32]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  red[w][lane] = part;
  __syncthreads();
  float s = red[0][lane];
#pragma unroll
  for (int i = 1; i < 8; ++i) s = __fadd_rn(s, red[i][lane]);
  return s;
}

// h = relu(sum of the split partials + b1); dropout keep bit from Philox4x32-10 at key = seed, counter = (*counter_d, row
// * 1536 + column, 0): kept iff fp32(word0 >> 8) * 2^-24 < keep; d = kept ? h * scale : 0
__global__ void __launch_bounds__(kThreads) heads_hidden_kernel(const float* __restrict__ part, int B, const float* __restrict__ b1,
                                                           int train, float keep, float scale, uint64_t seed,
                                                           const unsigned long long* __restrict__ counter, float* __restrict__ h,
                                                           float* __restrict__ d, uint32_t* __restrict__ mask) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * 32 + lane;
  const int b = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (b >= B) return;                                                  // whole warps
  const long long i = static_cast<long long>(b) * kHidAll + n;
  float s = part[i];
#pragma unroll
  for (int sp = 1; sp < kFc1Splits; ++sp) s = __fadd_rn(s, part[sp * static_cast<long long>(B) * kHidAll + i]);
  const float hv = fmaxf(__fadd_rn(s, b1[n]), 0.f);
  bool kept = true;
  if (train) {
    const unsigned long long ctr = *counter;
    const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32),
                                             static_cast<uint32_t>(i), 0u),
                                  make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
    kept = __fmul_rn(static_cast<float>(r.x >> 8), 0x1p-24f) < keep;
  }
  h[i] = hv;
  d[i] = kept ? __fmul_rn(hv, scale) : 0.f;
  const uint32_t bits = __ballot_sync(0xffffffffu, kept);
  if (lane == 0) mask[b * kMaskWords + blockIdx.x] = bits;
}

// o = sum of the split partials + b2 -> params [B,413] = [tanh(o) * limit | o], landmarks [B,136] = relu(o); y = tanh(o)
// [B,403] and the o > 0 bits of every column [B,18] are kept for the backward.  Advances *counter after a training step.
__global__ void __launch_bounds__(kThreads) heads_output_kernel(const float* __restrict__ part, int B, const float* __restrict__ b2,
                                                           float limit, float* __restrict__ params, float* __restrict__ landmarks,
                                                           float* __restrict__ y, uint32_t* __restrict__ obits,
                                                           unsigned long long* __restrict__ counter) {
  const int lane = threadIdx.x & 31, r = blockIdx.x * 32 + lane;
  const int b = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (counter && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *counter += 1;
  if (b >= B) return;
  float o = 0.f;
  if (r < kOut) {
    const long long i = static_cast<long long>(b) * kOut + r;
    o = part[i];
#pragma unroll
    for (int sp = 1; sp < kFc2Splits; ++sp) o = __fadd_rn(o, part[sp * static_cast<long long>(B) * kOut + i]);
    o = __fadd_rn(o, b2[r]);
    if (r < kShape) {
      const float t = tanhf(o);
      y[b * kShape + r] = t;
      params[b * kParams + r] = __fmul_rn(t, limit);
    } else if (r < kParams) {
      params[b * kParams + r] = o;
    } else {
      landmarks[b * kLms + r - kParams] = fmaxf(o, 0.f);
    }
  }
  const uint32_t bits = __ballot_sync(0xffffffffu, r < kOut && o > 0.f);
  if (lane == 0) obits[b * kOutWords + blockIdx.x] = bits;
}

// do [B,549]: shape fp32(dparams * limit) * fma(-y, y, 1) (torch's tanh_backward, contracted as on the CPU), pose dparams,
// landmarks dlandmarks * [o > 0]; db2 = column sums of do
__global__ void __launch_bounds__(kThreads) heads_dout_kernel(const float* __restrict__ dparams, const float* __restrict__ dlms,
                                                         int B, float limit, const float* __restrict__ y,
                                                         const uint32_t* __restrict__ obits, float* __restrict__ dout,
                                                         float* __restrict__ db2) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, r = blockIdx.x * 32 + lane;
  float acc = 0.f;
  if (r < kOut)
    for (int b = threadIdx.x >> 5; b < B; b += 8) {
      float g;
      if (r < kShape) {
        const float t = y[b * kShape + r];
        g = __fmul_rn(__fmul_rn(dparams[b * kParams + r], limit), __fmaf_rn(-t, t, 1.f));
      } else if (r < kParams) {
        g = dparams[b * kParams + r];
      } else {
        g = (obits[b * kOutWords + blockIdx.x] >> lane) & 1u ? dlms[b * kLms + r - kParams] : 0.f;
      }
      dout[b * kOut + r] = g;
      acc = __fadd_rn(acc, g);
    }
  const float s = column_total(acc, red);
  if (threadIdx.x < 32 && r < kOut) db2[r] = s;
}

// dh = (kept and h > 0) ? dd * scale : 0 (dropout's then relu's backward); db1 = column sums of dh
__global__ void __launch_bounds__(kThreads) heads_dhidden_kernel(const float* __restrict__ dd, int B, const float* __restrict__ h,
                                                            const uint32_t* __restrict__ mask, float scale,
                                                            float* __restrict__ dh, float* __restrict__ db1) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, n = blockIdx.x * 32 + lane;
  float acc = 0.f;
  for (int b = threadIdx.x >> 5; b < B; b += 8) {
    const long long i = static_cast<long long>(b) * kHidAll + n;
    const bool kept = (mask[b * kMaskWords + blockIdx.x] >> lane) & 1u;
    const float g = kept && h[i] > 0.f ? __fmul_rn(dd[i], scale) : 0.f;
    dh[i] = g;
    acc = __fadd_rn(acc, g);
  }
  const float s = column_total(acc, red);
  if (threadIdx.x < 32) db1[n] = s;
}

void add_problem(GemmBatch& g, GemmProblem p, int* tiles) {
  p.tiles_n = ceil_div(p.N, kTile);
  p.tile0 = *tiles;
  *tiles += ceil_div(p.M, kTile) * p.tiles_n;
  g.p[g.count++] = p;
}

void launch_gemm(const GemmBatch& g, int tiles, int splits, cudaStream_t stream) {
  heads_gemm_kernel<<<dim3(static_cast<unsigned>(tiles), static_cast<unsigned>(splits)), kThreads, 0, stream>>>(g);
  count_launch();
}

// workspace: the forward's split partials, or the backward's do, dd and dh
size_t fwd_ws_floats(int B) { return static_cast<size_t>(B) * (kFc1Splits * kHidAll + kFc2Splits * kOut); }
size_t bwd_ws_floats(int B) { return static_cast<size_t>(B) * (kOut + 2 * kHidAll); }

// torch's dropout arithmetic for a Python float p: scale fp32(1 / (1 - p)) and keep probability fp32(1 - p), both from fp64
float dropout_scale(int train, double p) { return train ? static_cast<float>(1.0 / (1.0 - p)) : 1.f; }

// ceil(B / 8) rows of 8 on gridDim.y (at most 65535) in the hidden and output kernels
constexpr int kMaxBatch = 8 * 65535;

}  // namespace
}  // namespace dad3d

using namespace dad3d;

extern "C" {

size_t dad3d_heads_workspace_bytes(int32_t B) {
  if (B <= 0) return 0;
  return std::max(fwd_ws_floats(B), bwd_ws_floats(B)) * sizeof(float);
}

int dad3d_heads_forward(const float* features_d, int32_t B, const float* w1_d, const float* b1_d, const float* w2_d,
                        const float* b2_d, float limit, int32_t train, double p, uint64_t seed,
                        unsigned long long* counter_d, float* params_d, float* landmarks_d, float* h_d, float* d_d,
                        uint32_t* mask_d, float* y_d, uint32_t* obits_d, void* workspace_d, size_t workspace_bytes,
                        dad3d_stream stream_) {
  DAD3D_REQUIRE(B >= 1 && B <= kMaxBatch, "B must be in [1, 524280]");
  DAD3D_REQUIRE(features_d && w1_d && b1_d && w2_d && b2_d && params_d && landmarks_d && h_d && d_d && mask_d && y_d &&
                    obits_d && workspace_d,
                "null pointer");
  DAD3D_REQUIRE(!train || counter_d, "training needs counter_d");
  DAD3D_REQUIRE(!train || (p >= 0.0 && p < 1.0), "dropout p must be in [0, 1)");
  DAD3D_REQUIRE(workspace_bytes >= dad3d_heads_workspace_bytes(B), "workspace too small");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  float* part1 = static_cast<float*>(workspace_d);
  float* part2 = part1 + static_cast<size_t>(kFc1Splits) * B * kHidAll;
  const long long rows = B;

  GemmBatch g1 = {};
  int tiles = 0;
  add_problem(g1, {features_d, kFeat, 1, w1_d, 1, kFeat, part1, kHidAll, rows * kHidAll, B, kHidAll, kFeat,
                   kFeat / kFc1Splits},
              &tiles);
  launch_gemm(g1, tiles, kFc1Splits, stream);

  const float keep = static_cast<float>(1.0 - p);
  heads_hidden_kernel<<<dim3(kMaskWords, static_cast<unsigned>(ceil_div(B, 8))), kThreads, 0, stream>>>(
      part1, B, b1_d, train, keep, dropout_scale(train, p), seed, counter_d, h_d, d_d, mask_d);
  count_launch();

  GemmBatch g2 = {};
  tiles = 0;
  for (int hd = 0, r0 = 0; hd < 3; r0 += kHeadRows[hd++])
    add_problem(g2, {d_d + hd * kHid, kHidAll, 1, w2_d + static_cast<size_t>(r0) * kHid, 1, kHid, part2 + r0, kOut,
                     rows * kOut, B, kHeadRows[hd], kHid, kHid / kFc2Splits},
                &tiles);
  launch_gemm(g2, tiles, kFc2Splits, stream);

  heads_output_kernel<<<dim3(kOutWords, static_cast<unsigned>(ceil_div(B, 8))), kThreads, 0, stream>>>(
      part2, B, b2_d, limit, params_d, landmarks_d, y_d, obits_d, train ? counter_d : nullptr);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_heads_backward(const float* dparams_d, const float* dlandmarks_d, const float* features_d, int32_t B,
                         const float* w2_d, float limit, int32_t train, double p, const float* h_d, const float* d_d,
                         const uint32_t* mask_d, const float* y_d, const uint32_t* obits_d, float* dw1_d, float* db1_d,
                         float* dw2_d, float* db2_d, void* workspace_d, size_t workspace_bytes, dad3d_stream stream_) {
  DAD3D_REQUIRE(B >= 1 && B <= kMaxBatch, "B must be in [1, 524280]");
  DAD3D_REQUIRE(dparams_d && dlandmarks_d && features_d && w2_d && h_d && d_d && mask_d && y_d && obits_d && dw1_d &&
                    db1_d && dw2_d && db2_d && workspace_d,
                "null pointer");
  DAD3D_REQUIRE(!train || (p >= 0.0 && p < 1.0), "dropout p must be in [0, 1)");
  DAD3D_REQUIRE(workspace_bytes >= dad3d_heads_workspace_bytes(B), "workspace too small");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  float* dout = static_cast<float*>(workspace_d);
  float* dd = dout + static_cast<size_t>(B) * kOut;
  float* dh = dd + static_cast<size_t>(B) * kHidAll;

  heads_dout_kernel<<<kOutWords, kThreads, 0, stream>>>(dparams_d, dlandmarks_d, B, limit, y_d, obits_d, dout, db2_d);
  count_launch();

  // per head: dw2 rows = do^T d over the batch, and dd block = do w2 over the head's rows; one launch
  GemmBatch g = {};
  int tiles = 0;
  for (int hd = 0, r0 = 0; hd < 3; r0 += kHeadRows[hd++]) {
    add_problem(g, {dout + r0, 1, kOut, d_d + hd * kHid, kHidAll, 1, dw2_d + static_cast<size_t>(r0) * kHid, kHid, 0,
                    kHeadRows[hd], kHid, B, B},
                &tiles);
    add_problem(g, {dout + r0, kOut, 1, w2_d + static_cast<size_t>(r0) * kHid, kHid, 1, dd + hd * kHid, kHidAll, 0, B,
                    kHid, kHeadRows[hd], kHeadRows[hd]},
                &tiles);
  }
  launch_gemm(g, tiles, 1, stream);

  heads_dhidden_kernel<<<kMaskWords, kThreads, 0, stream>>>(dd, B, h_d, mask_d, dropout_scale(train, p), dh, db1_d);
  count_launch();

  GemmBatch g1 = {};
  tiles = 0;
  add_problem(g1, {dh, 1, kHidAll, features_d, kFeat, 1, dw1_d, kFeat, 0, kHidAll, kFeat, B, B}, &tiles);
  launch_gemm(g1, tiles, 1, stream);
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // extern "C"
