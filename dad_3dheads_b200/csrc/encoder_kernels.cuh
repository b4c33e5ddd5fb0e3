// Device code of the DAD-3DNet encoder (everything that is not the wgmma tile engine itself):
//   EpiConvT           fused conv epilogue: folded-BN bias, residual add / gate multiply, ReLU, split into pieces
//   stem_conv_kernel   7x7/2 conv (Cin = 3) + folded BN + ReLU, fp32 CUDA cores, NCHW fp32 image -> NHWC fp32 (DAD3D_STEM_SIMT=1)
//   stem_s2d_kernel    2x2 space-to-depth + piece split of the image: the stem runs on the tile engine as a 4x4 conv
//   stem_pool_kernel   3x3/2 max-pool + split into pieces
//   bifpn_fuse_kernel  fast-normalised weighted sum of 2-3 maps with nearest resampling (BiFPN node input)
//   fusion_concat_kernel  [x | sigmoid(bilinear_align_corners(heatmap)) | p5] channel concat (FusionLayer input)
//   gap_kernel         global average pool
//   head_finalize_kernel  tanh*3 / identity / relu on the MLP outputs -> 3DMM params + 2D landmarks
// Activations are NHWC with channels padded to a multiple of 64 and stored as P "piece" planes of bf16
// (x = p0 + p1 + p2, see tile_gemm.cuh); plane p starts at base + p * plane_elems.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "tile_gemm.cuh"

namespace dad3d {

// ------------------------------------------------------------------------------------------------ piece helpers
// Two 16-bit piece formats (EpiConvT<F16>::kBf16): bf16 (x = p0 + p1 + p2, 8 + 8 + 8 mantissa bits, fp32 exponent range) and
// fp16 (x = hi + lo, 11 + 11 bits; |x| saturates at 65504 and the lo piece goes subnormal below |x| = 2^-3, leaving an
// absolute representation error <= 2^-25).
__device__ __forceinline__ uint16_t bf16_bits(float x) { return __bfloat16_as_ushort(__float2bfloat16_rn(x)); }
__device__ __forceinline__ float bf16_to_f32(uint16_t b) { return __uint_as_float(static_cast<uint32_t>(b) << 16); }

// one piece of the pair (a, b): returns the packed 16-bit pieces (a low, b high) and leaves the exact remainders in a, b
template <bool F16>
__device__ __forceinline__ uint32_t split_pair(float& a, float& b) {
  uint32_t w;
  if constexpr (F16) {
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(w) : "f"(b), "f"(a));
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w));
    a -= f.x;
    b -= f.y;
  } else {
    const uint16_t lo = bf16_bits(a), hi = bf16_bits(b);
    a -= bf16_to_f32(lo);
    b -= bf16_to_f32(hi);
    w = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
  }
  return w;
}
template <bool F16>
__device__ __forceinline__ void add_pair(uint32_t w, float& a, float& b) {
  if constexpr (F16) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w));
    a += f.x;
    b += f.y;
  } else {
    a += __uint_as_float(w << 16);
    b += __uint_as_float(w & 0xffff0000u);
  }
}

struct ActView {            // read-only view of a piece tensor
  const uint16_t* base;
  long long plane;          // elements per plane
  int planes;
  int C;                    // channel stride (padded channel count)
  int fp16;                 // piece format: 0 bf16, 1 fp16
};
__device__ __forceinline__ float act_load(const ActView& a, long long off) {
  float s = 0.f;
  for (int p = a.planes - 1; p >= 0; --p) {                                                    // small pieces first
    const uint16_t h = __ldg(a.base + p * a.plane + off);
    s += a.fp16 ? __half2float(__ushort_as_half(h)) : bf16_to_f32(h);
  }
  return s;
}
// 8 consecutive channels (16 B per plane); every plane's load is issued before the first one is consumed
__device__ __forceinline__ void act_load8(const ActView& a, long long off, float (&v)[8]) {
  uint4 q[3];
#pragma unroll
  for (int p = 0; p < 3; ++p)
    if (p < a.planes) q[p] = __ldg(reinterpret_cast<const uint4*>(a.base + p * a.plane + off));
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
#pragma unroll
  for (int pp = 0; pp < 3; ++pp) {
    const int p = 2 - pp;                                        // small pieces first
    if (p < a.planes) {
      const uint32_t w[4] = {q[p].x, q[p].y, q[p].z, q[p].w};
      if (a.fp16) {
#pragma unroll
        for (int j = 0; j < 4; ++j) add_pair<true>(w[j], v[2 * j], v[2 * j + 1]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) add_pair<false>(w[j], v[2 * j], v[2 * j + 1]);
      }
    }
  }
}
__device__ __forceinline__ void act_store8(uint16_t* base, long long plane, int planes, int fp16, long long off,
                                           const float (&v)[8]) {
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = v[j];
  for (int p = 0; p < planes; ++p) {
    uint32_t w[4];
    if (fp16) {
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = split_pair<true>(r[2 * j], r[2 * j + 1]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = split_pair<false>(r[2 * j], r[2 * j + 1]);
    }
    *reinterpret_cast<uint4*>(base + p * plane + off) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// ------------------------------------------------------------------------------------------------ conv epilogue
struct EpiConvParams {
    const float* bias;        // [Cout_pad] folded BN shift / conv bias
    const float* scale;       // [Cout_pad] per-output-channel 2^-s that undoes the weight scaling (fp16 pieces only)
    int relu;
    int res_mode;             // 0 none, 1 add before ReLU, 2 multiply after bias (FusionLayer gate); same pixel indexing
    ActView res;              // as the output.  (ResUnit / BiFPN residual adds normally ride the K axis instead.)
    int up2;                  // store every output pixel to the 2x2 block it covers in a [N, 2H, 2W, C] tensor (nearest
                              // up-sampling fused into the store: maps.c are 5-D parity views, see make_plan)
    int parity;               // 1 + 2a + b: this launch computes the output pixels (2i + a, 2j + b) of a [N, 2H, 2W, C] tensor
                              // (tile grid = the half-resolution grid) and stores them through the same 5-D view
    uint16_t* out;            // piece planes [planes][pix][ld_out]; may be null when only out_f32 is wanted
    long long out_plane;
    int out_planes;
    int ld_out;
    float* out_f32;           // optional fp32 copy [pix][ld_f32]
    int ld_f32;
};

template <bool F16>
struct EpiConvT {
  static constexpr int kBf16 = F16 ? 0 : 1;       // operand format of the tile engine
  static constexpr bool kFragment = true;         // piece outputs (ep.out != nullptr) run on the register fragments
  struct State {};
  using Params = EpiConvParams;
  // fp32-only outputs (heat-map, MLP logits): direct vector stores of this thread's row
  static __device__ __forceinline__ void run_f32(const Params& ep, const EpiCtx& c) {
    int cb, ce;
    epi_chunk_range(*c.g, c.grp, &cb, &ce);
    for (int ch = cb; ch < ce; ++ch) {
      float x[32];
      const bool tail16 = ch * 32 + 32 > c.g->block_n;            // 16-column last chunk (block_n = 80)
      if (tail16) epi_load16<0>(c, ch * 32, x);
      else epi_load32<0>(c, ch * 32, x);
      if (!c.valid) continue;
      const int col = c.col0 + ch * 32;
      float4* d = reinterpret_cast<float4*>(ep.out_f32 + c.pix * ep.ld_f32 + col);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (tail16 && j >= 4) break;
        const float4 b = __ldg(reinterpret_cast<const float4*>(ep.bias + col) + j);
        float4 o;
        if constexpr (F16) {
          const float4 sc = __ldg(reinterpret_cast<const float4*>(ep.scale + col) + j);
          o = make_float4(fmaf(x[4 * j], sc.x, b.x), fmaf(x[4 * j + 1], sc.y, b.y), fmaf(x[4 * j + 2], sc.z, b.z),
                          fmaf(x[4 * j + 3], sc.w, b.w));
        } else {
          o = make_float4(x[4 * j] + b.x, x[4 * j + 1] + b.y, x[4 * j + 2] + b.z, x[4 * j + 3] + b.w);
        }
        if (ep.relu) {
          o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
        }
        d[j] = o;
      }
    }
  }

  // Piece outputs: the fragment epilogue.  Each thread holds rows r0, r0 + 8 of its warp's 16 tile rows and the column
  // pairs 8j + 2(lane & 3) of the wgmma accumulators; per element, in this order: acc0 + acc1, folded-BN scale and bias,
  // residual add or gate multiply, ReLU, split into 16-bit pieces.  Columns go in chunks of 32: per piece plane a chunk is
  // one 1 KiB staging tile (16 rows x 64 B, TMA SWIZZLE_64B pattern: 16-byte chunk index XOR ((row >> 1) & 3), written
  // bank-conflict free with 32-bit stores) and one TMA store of the warp's 16-row box.
  template <int BN>
  static __device__ __forceinline__ void run_frag(const Params& ep, FragCtx& f, const float (&a0)[BN / 2],
                                                  const float (&a1)[BN / 2], bool two) {
    const int q = f.lane & 3;
#pragma unroll
    for (int ch = 0; ch < BN / 32; ++ch) {
      float x[16];                                     // the chunk's values: x[4 jj + 2 hr + e] = a0[4 (4 ch + jj) + 2 hr + e]
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * ch + jj;
        const int col = f.col0 + 8 * j + 2 * q;
        const float2 b = __ldg(reinterpret_cast<const float2*>(ep.bias + col));
        float2 sc = make_float2(1.f, 1.f);
        if constexpr (F16) sc = __ldg(reinterpret_cast<const float2*>(ep.scale + col));
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          float& x0 = x[4 * jj + 2 * hr];
          float& x1 = x[4 * jj + 2 * hr + 1];
          x0 = a0[4 * j + 2 * hr];
          x1 = a0[4 * j + 2 * hr + 1];
          if (two) { x0 += a1[4 * j + 2 * hr]; x1 += a1[4 * j + 2 * hr + 1]; }
          if constexpr (F16) {
            x0 = fmaf(x0, sc.x, b.x); x1 = fmaf(x1, sc.y, b.y);
          } else {
            x0 += b.x; x1 += b.y;
          }
          if (ep.res_mode != 0) {
            // residual / gate operand at the same pixel and channels, pieces summed smallest first
            uint32_t w[3] = {0u, 0u, 0u};
            if (f.valid[hr]) {
              const uint16_t* src = ep.res.base + f.pix[hr] * ep.res.C + col;
#pragma unroll
              for (int p = 0; p < 3; ++p)
                if (p < ep.res.planes) w[p] = __ldg(reinterpret_cast<const uint32_t*>(src + p * ep.res.plane));
            }
            float r0 = 0.f, r1 = 0.f;
#pragma unroll
            for (int pp = 0; pp < 3; ++pp)
              if (2 - pp < ep.res.planes) add_pair<F16>(w[2 - pp], r0, r1);
            if (ep.res_mode == 1) { x0 += r0; x1 += r1; }
            else { x0 *= r0; x1 *= r1; }
          }
          if (ep.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        }
      }
      const int col = f.col0 + 32 * ch;
      for (int p = 0; p < ep.out_planes; ++p) {
        uint8_t* tile = f.stage + ((f.store_seq++ & 3) << 10);
        if (f.lane == 0) ptx::bulk_wait_read<3>();      // the store that last used this tile has read it
        __syncwarp();
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int row = (f.lane >> 2) + 8 * hr;
            const uint32_t w = split_pair<F16>(x[4 * jj + 2 * hr], x[4 * jj + 2 * hr + 1]);
            *reinterpret_cast<uint32_t*>(tile + row * 64 + ((jj ^ ((row >> 1) & 3)) << 4) + 4 * q) = w;
          }
        ptx::fence_proxy_async_smem();
        __syncwarp();
        if (f.lane == 0) {
          if (ep.up2) {
            const int row0 = f.bn0 * f.g->Ho + f.bh0;   // merged (image, row) coordinate of the 5-D parity view
#pragma unroll
            for (int ab = 0; ab < 4; ++ab) ptx::tma_store_5d(&f.maps->c[p], tile, col, ab & 1, f.bw0, ab >> 1, row0);
          } else if (ep.parity) {
            ptx::tma_store_5d(&f.maps->c[p], tile, col, (ep.parity - 1) & 1, f.bw0, (ep.parity - 1) >> 1,
                              f.bn0 * f.g->Ho + f.bh0);
          } else {
            ptx::tma_store_4d(&f.maps->c[p], tile, col, f.bw0, f.bh0, f.bn0);
          }
          ptx::bulk_commit();
        }
      }
    }
  }

  // fp32 outputs only (ep.out == nullptr; piece outputs take run_frag)
  static __device__ __forceinline__ void prefetch(const Params&, EpiCtx&, State&) {}
  static __device__ __forceinline__ void run(const Params& ep, EpiCtx& c, State&) { run_f32(ep, c); }
};
using EpiConv = EpiConvT<false>;      // bf16 pieces
using EpiConvH = EpiConvT<true>;      // fp16 hi/lo pieces, per-channel weight scale undone in the epilogue

// ------------------------------------------------------------------------------------------------ stem
// 7x7 stride-2 pad-3 conv, 3 -> 64 channels, BN folded, ReLU.  in: NCHW fp32 [B,3,H,W]; out: NHWC fp32 [B,H/2,W/2,64].
// Block = 16x16 output pixels, 256 threads.  Thread = 4 horizontally adjacent pixels x 16 output channels (warp-uniform
// channel group, so weight reads are shared-memory broadcasts); per (channel, filter row) the 13 input values the 4 pixels
// need are loaded once and reused across the 7 filter columns.
constexpr int kStemTile = 16;
constexpr int kStemPatch = kStemTile * 2 + 5;    // 37
constexpr int kStemSmemBytes = (147 * 64 + 3 * kStemPatch * (kStemPatch + 1)) * 4;
__global__ void __launch_bounds__(256, 2)
stem_conv_kernel(const float* __restrict__ img, const float* __restrict__ w /*[147][64]*/, const float* __restrict__ bias,
                 int H, int W, float* __restrict__ out) {
  extern __shared__ float stem_smem[];            // kStemSmemBytes of dynamic shared memory
  float* s_w = stem_smem;                                                       // [147][64]
  float (*s_in)[kStemPatch][kStemPatch + 1] =
      reinterpret_cast<float (*)[kStemPatch][kStemPatch + 1]>(stem_smem + 147 * 64);   // [3][37][38]
  const int Ho = H / 2, Wo = W / 2;
  const int b = blockIdx.z;
  const int oy0 = blockIdx.y * kStemTile, ox0 = blockIdx.x * kStemTile;
  const int t = threadIdx.x;
  for (int i = t; i < 147 * 64; i += 256) s_w[i] = __ldg(&w[i]);
  const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
  for (int i = t; i < 3 * kStemPatch * kStemPatch; i += 256) {
    const int c = i / (kStemPatch * kStemPatch);
    const int rem = i - c * kStemPatch * kStemPatch;
    const int py = rem / kStemPatch, px = rem - py * kStemPatch;
    const int iy = iy0 + py, ix = ix0 + px;
    float val = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) val = __ldg(&img[((static_cast<size_t>(b) * 3 + c) * H + iy) * W + ix]);
    s_in[c][py][px] = val;
  }
  __syncthreads();
  const int warp = t >> 5, lane = t & 31;
  const int cg = warp & 3;                         // 16-channel group, warp-uniform
  const int quad = (warp >> 2) * 32 + lane;        // 0..63: 4 quads per tile row
  const int ty = quad >> 2, qx = quad & 3;
  float2 acc[4][8];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[p][o] = make_float2(0.f, 0.f);
  for (int c = 0; c < 3; ++c)
#pragma unroll 1
    for (int ky = 0; ky < 7; ++ky) {
      float in[13];
      const float* irow = &s_in[c][ty * 2 + ky][qx * 8];
#pragma unroll
      for (int k = 0; k < 13; ++k) in[k] = irow[k];
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float4* wr = reinterpret_cast<const float4*>(&s_w[((c * 7 + ky) * 7 + kx) * 64 + cg * 16]);
        const float4 q0 = wr[0], q1 = wr[1], q2 = wr[2], q3 = wr[3];
        const float2 wv[8] = {make_float2(q0.x, q0.y), make_float2(q0.z, q0.w), make_float2(q1.x, q1.y),
                              make_float2(q1.z, q1.w), make_float2(q2.x, q2.y), make_float2(q2.z, q2.w),
                              make_float2(q3.x, q3.y), make_float2(q3.z, q3.w)};
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float xs = in[2 * p + kx];
          const float2 xv = make_float2(xs, xs);
#pragma unroll
          for (int o = 0; o < 8; ++o) acc[p][o] = make_float2(fmaf(xv.x, wv[o].x, acc[p][o].x), fmaf(xv.y, wv[o].y, acc[p][o].y));
        }
      }
    }
  const float4* b4 = reinterpret_cast<const float4*>(bias + cg * 16);
  const float4 bb0 = __ldg(&b4[0]), bb1 = __ldg(&b4[1]), bb2 = __ldg(&b4[2]), bb3 = __ldg(&b4[3]);
  const int oy = oy0 + ty;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int ox = ox0 + qx * 4 + p;
    if (oy < Ho && ox < Wo) {
      float4* d = reinterpret_cast<float4*>(out + ((static_cast<size_t>(b) * Ho + oy) * Wo + ox) * 64 + cg * 16);
      d[0] = make_float4(fmaxf(acc[p][0].x + bb0.x, 0.f), fmaxf(acc[p][0].y + bb0.y, 0.f),
                         fmaxf(acc[p][1].x + bb0.z, 0.f), fmaxf(acc[p][1].y + bb0.w, 0.f));
      d[1] = make_float4(fmaxf(acc[p][2].x + bb1.x, 0.f), fmaxf(acc[p][2].y + bb1.y, 0.f),
                         fmaxf(acc[p][3].x + bb1.z, 0.f), fmaxf(acc[p][3].y + bb1.w, 0.f));
      d[2] = make_float4(fmaxf(acc[p][4].x + bb2.x, 0.f), fmaxf(acc[p][4].y + bb2.y, 0.f),
                         fmaxf(acc[p][5].x + bb2.z, 0.f), fmaxf(acc[p][5].y + bb2.w, 0.f));
      d[3] = make_float4(fmaxf(acc[p][6].x + bb3.x, 0.f), fmaxf(acc[p][6].y + bb3.y, 0.f),
                         fmaxf(acc[p][7].x + bb3.z, 0.f), fmaxf(acc[p][7].y + bb3.w, 0.f));
    }
  }
}

// Space-to-depth of the input image for the tensor-core stem: NCHW fp32 [B,3,H,W] -> pieces [B, H/2, W/2 + kS2dPadW, 16],
// channel c16 = (py * 2 + px) * 3 + ch for the 2x2 block's sub-pixel (py, px), channels 12..15 zero; kS2dPadL zero pixels on
// the left and kS2dPadW - kS2dPadL on the right, so that a 4-pixel (64-element) window starting at padded x covers
// s2d pixels x-2 .. x+1 without leaving the row: the 7x7/2 conv becomes a 4x4/1 conv over 12 channels whose 4 horizontal
// taps are ONE contiguous 64-element K block (the A tensor map strides rows by 16 elements: overlapping windows).
constexpr int kS2dPadL = 2;
constexpr int kS2dPadW = 4;      // total horizontal padding (row pitch W/2 + 4)
__global__ void stem_s2d_kernel(const float* __restrict__ img, int B, int H, int W, uint16_t* __restrict__ out,
                                long long out_plane, int planes, int fp16) {
  // grid = (ceil(Wp / 128), Hs, B)
  const int Hs = H / 2, Ws = W / 2, Wp = Ws + kS2dPadW;
  const int xp = blockIdx.x * blockDim.x + threadIdx.x;
  if (xp >= Wp) return;
  const int y = blockIdx.y;
  const long long b = blockIdx.z;
  const long long i = (b * Hs + y) * Wp + xp;
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = 0.f;
  const int x = xp - kS2dPadL;
  if (x >= 0 && x < Ws) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
#pragma unroll
      for (int py = 0; py < 2; ++py) {
        const float2 q = __ldg(reinterpret_cast<const float2*>(
            img + ((b * 3 + ch) * H + (2 * y + py)) * static_cast<long long>(W) + 2 * x));
        v[(py * 2 + 0) * 3 + ch] = q.x;
        v[(py * 2 + 1) * 3 + ch] = q.y;
      }
  }
  const float lo8[8] = {v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]};
  const float hi8[8] = {v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15]};
  act_store8(out, out_plane, planes, fp16, i * 16, lo8);
  act_store8(out, out_plane, planes, fp16, i * 16 + 8, hi8);
}

// MaxPool2d(3, stride 2, pad 1) over NHWC fp32 [B,Hi,Wi,64] -> pieces [B,Hi/2,Wi/2,64].  thread = 8 channels of a pixel.
// `in` is fp32 NHWC (SIMT stem) when in_pieces.base == nullptr, otherwise the piece tensor written by the tensor-core stem.
__global__ void stem_pool_kernel(const float* __restrict__ in, ActView in_pieces, int B, int Hi, int Wi,
                                 uint16_t* __restrict__ out, long long out_plane, int planes, int fp16) {
  // flat index over (image, row, column, channel group); 32-bit div/mod (B * Ho * Wo * 8 < 2^31 is checked by the host)
  const int Ho = Hi / 2, Wo = Wi / 2;
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= static_cast<unsigned>(B) * Ho * Wo * 8u) return;
  const int cg = static_cast<int>(i & 7u);
  const unsigned upix = i >> 3;
  const int ox = static_cast<int>(upix % static_cast<unsigned>(Wo));
  const unsigned t2 = upix / static_cast<unsigned>(Wo);
  const int oy = static_cast<int>(t2 % static_cast<unsigned>(Ho));
  const long long b = t2 / static_cast<unsigned>(Ho);
  const long long pix = upix;
  float m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
  for (int dy = -1; dy <= 1; ++dy) {
    const int iy = oy * 2 + dy;
    if (iy < 0 || iy >= Hi) continue;
    for (int dx = -1; dx <= 1; ++dx) {
      const int ix = ox * 2 + dx;
      if (ix < 0 || ix >= Wi) continue;
      const long long off = ((b * Hi + iy) * Wi + ix) * 64 + cg * 8;
      if (in_pieces.base != nullptr) {
        float v[8];
        act_load8(in_pieces, off, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
        continue;
      }
      const float4* s = reinterpret_cast<const float4*>(in + off);
      const float4 a = __ldg(s), c = __ldg(s + 1);
      m[0] = fmaxf(m[0], a.x); m[1] = fmaxf(m[1], a.y); m[2] = fmaxf(m[2], a.z); m[3] = fmaxf(m[3], a.w);
      m[4] = fmaxf(m[4], c.x); m[5] = fmaxf(m[5], c.y); m[6] = fmaxf(m[6], c.z); m[7] = fmaxf(m[7], c.w);
    }
  }
  act_store8(out, out_plane, planes, fp16, pix * 64 + cg * 8, m);
}

// ------------------------------------------------------------------------------------------------ BiFPN node input
// out[b,y,x,c] = w0*a[b,y,x,c] + w1*b1[nearest] (+ w2*b2[nearest]);  bifpn.py:111-129.  F.interpolate(mode="nearest"):
// src = floor(dst * in / out)  (x2 up-sampling: dst>>1, /2 down-sampling: 2*dst).  thread = 8 channels of a pixel.
struct FuseSrc {
  ActView v;
  int H, W;       // source extents
  float w;
};
// grid = (ceil(W * C/8 / 256), H, B): the row and the image come from the block index, so the only division per thread is a
// 32-bit one (the 64-bit div/mod chain of a flat index was most of this kernel's time)
__global__ void __launch_bounds__(256)
bifpn_fuse_kernel(FuseSrc s0, FuseSrc s1, FuseSrc s2, int nsrc, int B, int H, int W, int C,
                  uint16_t* __restrict__ out, long long out_plane, int planes, int fp16) {
  const unsigned cgs = static_cast<unsigned>(C) >> 3;
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= static_cast<unsigned>(W) * cgs) return;
  const int x = static_cast<int>(t / cgs);
  const int cg = static_cast<int>(t - static_cast<unsigned>(x) * cgs);
  const int y = blockIdx.y;
  const long long b = blockIdx.z;
  const long long pix = (b * H + y) * W + x;
  float acc[8], t0[8], t1[8], t2[8];
  act_load8(s0.v, pix * C + cg * 8, t0);
  {
    const int sy = (y * s1.H) / H, sx = (x * s1.W) / W;
    act_load8(s1.v, ((b * s1.H + sy) * s1.W + sx) * C + cg * 8, t1);
  }
  if (nsrc == 3) {
    const int sy = (y * s2.H) / H, sx = (x * s2.W) / W;
    act_load8(s2.v, ((b * s2.H + sy) * s2.W + sx) * C + cg * 8, t2);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    acc[j] = s0.w * t0[j];
    acc[j] += s1.w * t1[j];
    if (nsrc == 3) acc[j] += s2.w * t2[j];
  }
  act_store8(out, out_plane, planes, fp16, pix * C + cg * 8, acc);
}

// ------------------------------------------------------------------------------------------------ FusionLayer input
// out[b,y,x,:] = [ x[b,y,x,0:Cx] | sigmoid(bilinear_align_corners(heat))[0:Ch_pad] | p5[b,y,x,0:Cp] ]
// (flame_regression.py:33-41).  heat is fp32 NHWC [B,Hh,Wh,ldh]; channels >= n_heat of the middle block are zero.
__global__ void fusion_concat_kernel(ActView x, int Cx, const float* __restrict__ heat, int Hh, int Wh, int ldh,
                                     int n_heat, int Ch_pad, ActView p5, int Cp, int B, int H, int W,
                                     uint16_t* __restrict__ out, long long out_plane, int planes, int fp16) {
  // grid = (pixels of one image, B), block = the Ct/8 channel groups of a pixel (rounded up to a warp multiple)
  const int Ct = Cx + Ch_pad + Cp;
  const int cg = threadIdx.x;
  if (cg >= Ct / 8) return;
  const long long b = blockIdx.y;
  const int pin = blockIdx.x;                      // pixel inside the image
  const long long pix = b * (static_cast<long long>(H) * W) + pin;
  const int c = cg * 8;
  float v[8];
  if (c < Cx) {
    act_load8(x, pix * Cx + c, v);
  } else if (c < Cx + Ch_pad) {
    const int py = pin / W;
    const int px = pin - py * W;
    // align_corners=True: src = dst * (in - 1) / (out - 1)
    const float fy = (H > 1) ? py * (static_cast<float>(Hh - 1) / static_cast<float>(H - 1)) : 0.f;
    const float fx = (W > 1) ? px * (static_cast<float>(Wh - 1) / static_cast<float>(W - 1)) : 0.f;
    const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
    const int y1 = min(y0 + 1, Hh - 1), x1 = min(x0 + 1, Wh - 1);
    const float ly = fy - y0, lx = fx - x0;
    const int ch0 = c - Cx;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = ch0 + j;
      float r = 0.f;
      if (ch < n_heat) {
        const float v00 = __ldg(&heat[((b * Hh + y0) * Wh + x0) * ldh + ch]);
        const float v01 = __ldg(&heat[((b * Hh + y0) * Wh + x1) * ldh + ch]);
        const float v10 = __ldg(&heat[((b * Hh + y1) * Wh + x0) * ldh + ch]);
        const float v11 = __ldg(&heat[((b * Hh + y1) * Wh + x1) * ldh + ch]);
        // same evaluation order as ATen's upsample_bilinear2d: h0l*(w0l*v00 + w1l*v01) + h1l*(w0l*v10 + w1l*v11)
        const float val = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
        r = 1.f / (1.f + expf(-val));
      }
      v[j] = r;
    }
  } else {
    act_load8(p5, pix * Cp + (c - Cx - Ch_pad), v);
  }
  act_store8(out, out_plane, planes, fp16, pix * Ct + c, v);
}

// ------------------------------------------------------------------------------------------------ GAP
// adaptive_avg_pool2d(., 1): [B,HW,C] -> [B,C] pieces.  thread = 8 channels of an image.
// block = one image x 8 channel groups (64 channels); thread = (pixel slice 0..31, channel group): pixels slice, slice+32, ...
// kF32Out also stores the fp32 means [B,C] to means (the frozen-backbone features), the values the pieces are split from.
constexpr int kGapSlices = 32;
template <bool kF32Out>
__global__ void __launch_bounds__(256)
gap_kernel(ActView x, int B, int HW, int C, uint16_t* __restrict__ out, long long out_plane, int planes, int fp16,
           float* __restrict__ means) {
  __shared__ float red[kGapSlices][8][9];
  const int cgs = C / 8;
  const int blocks_per_img = cgs / 8;
  const int b = blockIdx.x / blocks_per_img;
  const int cg = (blockIdx.x % blocks_per_img) * 8 + (threadIdx.x & 7);
  const int slice = threadIdx.x >> 3;
  float acc[8], t[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int p = slice; p < HW; p += kGapSlices) {
    act_load8(x, (static_cast<long long>(b) * HW + p) * C + cg * 8, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += t[j];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[slice][threadIdx.x & 7][j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64) {                           // thread = (channel group, channel): fixed-order sum over the slices
    const int g = threadIdx.x >> 3, j = threadIdx.x & 7;
    float sum = 0.f;
    for (int sl = 0; sl < kGapSlices; ++sl) sum += red[sl][g][j];
    red[0][g][j] = sum / static_cast<float>(HW);
    if (kF32Out) means[static_cast<long long>(b) * C + (blockIdx.x % blocks_per_img) * 64 + threadIdx.x] = red[0][g][j];
  }
  __syncthreads();
  if (threadIdx.x < 8) {
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = red[0][threadIdx.x][j];
    const int cgo = (blockIdx.x % blocks_per_img) * 8 + threadIdx.x;
    act_store8(out, out_plane, planes, fp16, static_cast<long long>(b) * C + cgo * 8, o);
  }
}

// ------------------------------------------------------------------------------------------------ heads
// mlp_out [B, ld] fp32 = [shape 403 | pose 10 | landmarks 136 | pad]  ->  params [B,413] = [tanh(shape)*limit | pose],
// landmarks [B,68,2] = relu(.)   (flame_regression.py:96-106)
__global__ void head_finalize_kernel(const float* __restrict__ mlp_out, int ld, int B, float limit,
                                     float* __restrict__ params, float* __restrict__ landmarks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * 549) return;
  const int b = i / 549, j = i - b * 549;
  const float v = mlp_out[static_cast<size_t>(b) * ld + j];
  if (j < 403) params[static_cast<size_t>(b) * 413 + j] = tanhf(v) * limit;
  else if (j < 413) params[static_cast<size_t>(b) * 413 + j] = v;
  else landmarks[static_cast<size_t>(b) * 136 + (j - 413)] = fmaxf(v, 0.f);
}

// test hook: sum the piece planes back to fp32
__global__ void pieces_to_f32_kernel(ActView a, long long n, float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = act_load(a, i);
}
// test hook: split fp32 values into the piece planes (n8 groups of 8 consecutive elements), the split every kernel stores
__global__ void f32_to_pieces_kernel(const float* __restrict__ in, long long n8, uint16_t* __restrict__ base,
                                     long long plane, int planes, int fp16) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = in[i * 8 + j];
  act_store8(base, plane, planes, fp16, i * 8, v);
}

// heat-map NHWC fp32 [B,HW,ld] -> NCHW fp32 [B,68,HW] (the reference's OUTPUT_LANDMARKS_HEATMAP layout)
__global__ void heatmap_export_kernel(const float* __restrict__ in, int ld, int B, int HW, int C,
                                      float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * C * HW;
  if (i >= total) return;
  const int p = static_cast<int>(i % HW);
  const int c = static_cast<int>((i / HW) % C);
  const long long b = i / (static_cast<long long>(HW) * C);
  out[i] = __ldg(&in[(b * HW + p) * ld + c]);
}

}  // namespace dad3d
