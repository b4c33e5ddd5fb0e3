// FLAME head decoder for sm_90a:  413 params -> 5023x3 vertices (+ weak-perspective projection), and its backward.
// Every pass starts with K1, flame_prep_kernel: per-head small math (betas -> fp16 hi/lo coefficient rows, folded joint
// regression, Rodrigues, kinematic chain, 6-DoF rotation folded into the skinning transforms).  The blend product
// [heads,448] x [15069,448]^T (blend shapes + pose correctives + template) and the skinning then take one of four paths,
// chosen by decode_path:
//   dedicated  (default, layouts with only the jaw posed) flame_decode_kernel (flame_decode.cuh): one fp16 product per MAC,
//              skinning, z offset, rotation and projection in its epilogue
//   lbs        (DAD3D_BLEND_HILO) K2 tile_gemm_kernel<EpiLbs>: fp16 hi/lo operands, 3 products (fp32-class), the same
//              skinning in the epilogue; with DAD3D_DECODE_CLUSTER big passes run as 2x2 clusters with TMA multicast
//   blend      (other layouts, DAD3D_DECODE_UNFUSED) K2 tile_gemm_kernel<EpiBlend> to a v_posed scratch, then K3
//   simt       (DAD3D_BLEND_SIMT) blend_simt_kernel, CUDA-core fp32 product, to the same scratch, then K3
//   K3 lbs_project_kernel   linear-blend skinning + z offset + rotation + projection, shared-memory staged, coalesced
//   K4 gather kernels       landmark subsets
// The backward recomputes the blend product and runs the transposed one on the tile engine (<EpiBlend>, hi/lo operands).
// Reference math: model_training/model/flame.py:182-229, smplx.lbs (0.1.26), model_training/model/utils.py:92-101,
// model_training/head_mesh.py:33-46.  See DESIGN.md for layouts and rooflines.
#include <cuda_fp16.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/dad3d.h"
#include "common.h"
#include "flame_decode.cuh"
#include "tile_gemm.cuh"
#include "tmap.h"

namespace dad3d {

constexpr int kJoints = 5;
constexpr int kMaxShape = 300;        // flame.py:107
constexpr int kMaxExpr = 100;         // flame.py:108
constexpr int kBetas = kMaxShape + kMaxExpr;
constexpr int kPoseFeat = (kJoints - 1) * 9;
constexpr int kKPad = 448;            // 400 betas + 36 pose features + 1 template column, padded to 7 x 64
constexpr int kTmplCol = kBetas + kPoseFeat;   // two columns with coefficient 1.0 carry the (scaled) template exactly,
                                               // so the GEMM itself adds it
constexpr int kXfFloats = 68;         // per-head transform record (see HeadXf layout below)
constexpr int kBlendBlockN = 128;     // unfused path (v_posed scratch)
constexpr int kFusedBlockN = 96;      // fused path: 32 vertices per tile
constexpr int kDecodeChunk = 4096;    // unfused: heads per internal pass (bounds the v_posed scratch to ~250 MB)
constexpr float kMeshOffsetZ = 0.05f; // flame.py:114

struct FlameLayoutDev {
  int n_params;
  int off_shape, n_shape, off_expr, n_expr, off_jaw, n_jaw, off_rot, off_eye, n_eye, off_neck, n_neck, off_trans,
      off_scale;
  int parents[kJoints];
};

// HeadXf record (68 floats): A[j][12] for j<5 (rows of [R | t], already left-multiplied by the 6-DoF rotation),
// then c[3] = R6 * (0,0,0.05), then sc = max(s+1,1e-8), tx, ty, 2 pad.

// ------------------------------------------------------------------------------------------------ K1
__device__ __forceinline__ void rodrigues(const float* r, float* R) {
  // smplx batch_rodrigues: the epsilon is added to the vector inside the norm
  const float ax = r[0] + 1e-8f, ay = r[1] + 1e-8f, az = r[2] + 1e-8f;
  const float angle = sqrtf(ax * ax + ay * ay + az * az);
  const float x = r[0] / angle, y = r[1] / angle, z = r[2] / angle;
  const float s = sinf(angle), c1 = 1.0f - cosf(angle);
  // K = [[0,-z,y],[z,0,-x],[-y,x,0]],  R = I + s K + (1-c) K K
  R[0] = 1.0f + c1 * (-(z * z) - y * y);
  R[1] = s * (-z) + c1 * (x * y);
  R[2] = s * (y) + c1 * (x * z);
  R[3] = s * (z) + c1 * (x * y);
  R[4] = 1.0f + c1 * (-(z * z) - x * x);
  R[5] = s * (-x) + c1 * (y * z);
  R[6] = s * (-y) + c1 * (x * z);
  R[7] = s * (x) + c1 * (y * z);
  R[8] = 1.0f + c1 * (-(y * y) - x * x);
}

__device__ __forceinline__ void mat3_mul(const float* A, const float* B, float* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ void mat3_vec(const float* A, const float* v, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}

__device__ __forceinline__ void split_store(__half* hi, __half* lo, size_t idx, float x) {
  const __half h = __float2half_rn(x);
  hi[idx] = h;
  lo[idx] = __float2half_rn(x - __half2float(h));
}

// One warp per `group` consecutive heads.  Phase 1 (all lanes on one head at a time): betas -> fp16 hi/lo coefficient row, folded
// joint regression J = J_T + J_dirs beta as 15 warp-reduced sums; lane i keeps the joints of head i.  Phase 2 (one LANE per head,
// 32 heads at once): Rodrigues, kinematic chain, 6-DoF frame, skinning transforms -- the scalar tail used to run on lane 0 of a
// warp per head, 31 lanes idle (0.39 ms per 75 776 heads = 16 % of a decode pass; same arithmetic in the same order, so the
// outputs are bit-identical).
__global__ void __launch_bounds__(256)
flame_prep_kernel(const float* __restrict__ params, int B, FlameLayoutDev L, const float* __restrict__ jt,
                  const float* __restrict__ jdirsT, int flags, float inv_scale, __half* __restrict__ a_hi,
                  __half* __restrict__ a_lo, float* __restrict__ xf, int permute, int group) {
  // group = heads per warp: 32 for big batches (throughput), 1 for small ones (latency: every head gets its own warp)
  const int lane = threadIdx.x & 31;
  const int h0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * group;
  if (h0 >= B) return;
  float Jacc[15];
#pragma unroll
  for (int j = 0; j < 15; ++j) Jacc[j] = 0.f;
  const int nh = min(group, B - h0);
  for (int i = 0; i < nh; ++i) {
    const int h = h0 + i;
    const float* p = params + static_cast<size_t>(h) * L.n_params;
    // permute: the dedicated decode kernel wants heads that are equal mod 8 in the same TMEM lane quarter (flame_decode.cuh)
    const size_t arow = static_cast<size_t>(permute ? dec_phys_row(h) : h) * kKPad;
    float acc[15];
#pragma unroll
    for (int j = 0; j < 15; ++j) acc[j] = 0.f;
    for (int l = lane; l < kBetas; l += 32) {
      float b = 0.f;                                   // flame.py:191-200: missing coefficients are registered zeros
      if (l < kMaxShape) {
        if (l < L.n_shape) b = p[L.off_shape + l];
      } else if (l - kMaxShape < L.n_expr) {
        b = p[L.off_expr + l - kMaxShape];
      }
      split_store(a_hi, a_lo, arow + l, b);
#pragma unroll
      for (int j = 0; j < 15; ++j) acc[j] = fmaf(b, __ldg(&jdirsT[j * kBetas + l]), acc[j]);
    }
    for (int l = kTmplCol + lane; l < kKPad; l += 32) {     // template column gets coefficient 1, the rest is padding
      a_hi[arow + l] = __float2half_rn(l < kTmplCol + 2 ? 1.f : 0.f);
      a_lo[arow + l] = __float2half_rn(0.f);
    }
#pragma unroll
    for (int j = 0; j < 15; ++j) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
      if (lane == i) Jacc[j] = acc[j];
    }
  }
  if (lane >= nh) return;
  const int h = h0 + lane;
  const float* p = params + static_cast<size_t>(h) * L.n_params;
  const size_t arow = static_cast<size_t>(permute ? dec_phys_row(h) : h) * kKPad;
  const float* acc = Jacc;

  float J[15];
#pragma unroll
  for (int j = 0; j < 15; ++j) J[j] = __ldg(&jt[j]) + acc[j];       // joints = J_regressor (T + S beta), folded

  // full_pose = [global 0, neck, jaw, eyeballs]   flame.py:201-208
  float pose[15];
#pragma unroll
  for (int j = 0; j < 15; ++j) pose[j] = 0.f;
  if (L.n_neck == 3)
    for (int k = 0; k < 3; ++k) pose[3 + k] = p[L.off_neck + k];
  if (L.n_jaw == 3 && !(flags & DAD3D_ZERO_JAW))
    for (int k = 0; k < 3; ++k) pose[6 + k] = p[L.off_jaw + k];
  if (L.n_eye == 6)
    for (int k = 0; k < 6; ++k) pose[9 + k] = p[L.off_eye + k];

  float R[kJoints][9];
  for (int j = 0; j < kJoints; ++j) rodrigues(&pose[3 * j], R[j]);
  for (int j = 1; j < kJoints; ++j)
    for (int e = 0; e < 9; ++e) {
      const float pf = R[j][e] - ((e == 0 || e == 4 || e == 8) ? 1.0f : 0.0f);
      split_store(a_hi, a_lo, arow + kBetas + (j - 1) * 9 + e, pf);
    }

  // kinematic chain (smplx batch_rigid_transform)
  float GR[kJoints][9], Gt[kJoints][3];
  for (int e = 0; e < 9; ++e) GR[0][e] = R[0][e];
  for (int k = 0; k < 3; ++k) Gt[0][k] = J[k];
  for (int i = 1; i < kJoints; ++i) {
    const int par = L.parents[i];
    float rel[3], tmp[3];
    for (int k = 0; k < 3; ++k) rel[k] = J[3 * i + k] - J[3 * par + k];
    mat3_mul(GR[par], R[i], GR[i]);
    mat3_vec(GR[par], rel, tmp);
    for (int k = 0; k < 3; ++k) Gt[i][k] = tmp[k] + Gt[par][k];
  }

  // 6-DoF rotation (model/utils.py:92-101): columns b1, b2, b3
  float R6[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (!(flags & DAD3D_ZERO_ROT)) {
    const float* r6 = p + L.off_rot;
    const float vx[3] = {r6[0], r6[1], r6[2]}, vy[3] = {r6[3], r6[4], r6[5]};
    const float n1 = fmaxf(sqrtf(vx[0] * vx[0] + vx[1] * vx[1] + vx[2] * vx[2]), 1e-12f);
    const float b1[3] = {vx[0] / n1, vx[1] / n1, vx[2] / n1};
    float c3[3] = {b1[1] * vy[2] - b1[2] * vy[1], b1[2] * vy[0] - b1[0] * vy[2], b1[0] * vy[1] - b1[1] * vy[0]};
    const float n3 = fmaxf(sqrtf(c3[0] * c3[0] + c3[1] * c3[1] + c3[2] * c3[2]), 1e-12f);
    const float b3[3] = {c3[0] / n3, c3[1] / n3, c3[2] / n3};
    const float b2[3] = {-(b1[1] * b3[2] - b1[2] * b3[1]), -(b1[2] * b3[0] - b1[0] * b3[2]),
                         -(b1[0] * b3[1] - b1[1] * b3[0])};
    for (int r = 0; r < 3; ++r) {
      R6[3 * r + 0] = b1[r];
      R6[3 * r + 1] = b2[r];
      R6[3 * r + 2] = b3[r];
    }
  }

  float* o = xf + static_cast<size_t>(h) * kXfFloats;
  for (int i = 0; i < kJoints; ++i) {
    float t[3], rj[3], AR[9], At[3];
    mat3_vec(GR[i], &J[3 * i], rj);                     // rotated rest joint
    for (int k = 0; k < 3; ++k) t[k] = Gt[i][k] - rj[k];
    mat3_mul(R6, GR[i], AR);
    mat3_vec(R6, t, At);
    for (int r = 0; r < 3; ++r) {          // rotation part absorbs 1/basis_scale (exact power of two): it is applied
      o[i * 12 + r * 4 + 0] = AR[3 * r + 0] * inv_scale;   // to the still-scaled GEMM output
      o[i * 12 + r * 4 + 1] = AR[3 * r + 1] * inv_scale;
      o[i * 12 + r * 4 + 2] = AR[3 * r + 2] * inv_scale;
      o[i * 12 + r * 4 + 3] = At[r];
    }
  }
  for (int r = 0; r < 3; ++r) o[60 + r] = R6[3 * r + 2] * kMeshOffsetZ;   // R6 * (0,0,0.05)   flame.py:224
  o[63] = fmaxf(p[L.off_scale] + 1.0f, 1e-8f);                            // head_mesh.py:39
  o[64] = p[L.off_trans + 0];                                             // head_mesh.py:41-42 (z is zeroed)
  o[65] = p[L.off_trans + 1];
  o[66] = 0.f;
  o[67] = 0.f;
}

// ------------------------------------------------------------------------------------------------ K2 epilogue
struct EpiBlend {
  static constexpr int kBf16 = 0;                 // fp16 operands
  static constexpr bool kFragment = false;        // row epilogue over the shared-memory accumulator tile
  struct State {};
  struct Params {
    float* out;          // [rows, ld] fp32 v_posed * basis_scale (x,y,z interleaved, n = 3*vertex + coord)
    int ld;
  };
  static __device__ __forceinline__ void prefetch(const Params&, EpiCtx&, State&) {}
  static __device__ __forceinline__ void run(const Params& ep, EpiCtx& c, State&) {
    int cb, ce;
    epi_chunk_range(*c.g, c.grp, &cb, &ce);
    for (int ch = cb; ch < ce; ++ch) {
      float x[32];
      epi_load32<0>(c, ch * 32, x);
      if (!c.valid) continue;
      float4* dst = reinterpret_cast<float4*>(ep.out + static_cast<size_t>(c.pix) * ep.ld + c.col0 + ch * 32);
#pragma unroll
      for (int j = 0; j < 8; ++j) dst[j] = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
    }
  }
};

// Fused epilogue (layouts without neck / eyeball pose, i.e. the released model): blend-shape accumulator (template
// included, still scaled) -> linear-blend skinning -> z offset / 6-DoF rotation (folded into the per-head transforms) ->
// projection, written straight to the reference's output layouts.  Removes the v_posed round trip (120 KB/head).
// With only the jaw posed, the transforms of the other four joints coincide, so skinning needs two transforms per head
// (rest = joint 0, jaw = joint 2: 30 floats, register-resident) and two weights per vertex (w_rest = sum of the non-jaw
// weights, w_jaw).  Tile = 128 heads x 32 vertices (block_n = 96); warp (wq, grp) owns heads 32*wq.. and vertices
// 16*grp.. of the tile, as two passes of 8 vertices (24 accumulator columns).  Results are staged per warp so that global
// stores are contiguous runs (the reference layout's 60 276-byte row pitch rules out TMA stores).
struct EpiLbs {
  static constexpr int kBf16 = 0;                 // fp16 operands
  static constexpr bool kFragment = false;        // row epilogue over the shared-memory accumulator tile
  struct Params {
    const float* xf;         // [rows][68] per-head transform records (flame_prep_kernel)
    const float* w2;         // [nv][2]  (w_rest, w_jaw)
    int nv;
    float* verts3d;          // [rows][nv][3] or null
    float* proj;             // [rows][nv][pc] or null
    int pc;
    float image_size;
  };
  struct State {             // per-thread, persists across the tiles of a row tile
    float R[12];             // rest transform  [R | t] rows (rotation pre-divided by the basis scale)
    float Jw[12];            // jaw transform
    float cx, cy, cz, sc, tx, ty;
    float wl;                // this lane's entry of the tile's (w_rest, w_jaw) table: lane 2i / 2i+1 <-> vertex i
  };

  // write the warp's staged [32 rows][NCOL floats] (row pitch 25) as contiguous runs of NCOL floats per head row:
  // 4 rows x NCOL floats = NCOL/8 full warp stores; (rr, cc) depend only on (s, lane).
  template <int NCOL>
  static __device__ __forceinline__ void flush(float* __restrict__ dst, size_t row_pitch, const float* stage, int lane,
                                               int head0, int rows, int n_valid_cols) {
    __syncwarp();
    constexpr int kPer = NCOL / 8;
#pragma unroll
    for (int s = 0; s < kPer; ++s) {
      const int e = s * 32 + lane;
      const int rr = e / NCOL, cc = e - rr * NCOL;
      if (cc < n_valid_cols) {
        float* d = dst + static_cast<size_t>(rr) * row_pitch + cc;
        const float* sp = stage + rr * 25 + cc;
#pragma unroll 4
        for (int rg = 0; rg < 8; ++rg) {               // rows rr, rr+4, ... (incremental addressing: few live registers)
          if (head0 + rg * 4 + rr < rows) *d = *sp;
          d += 4 * row_pitch;
          sp += 100;
        }
      }
    }
    __syncwarp();
  }

  // everything that does not depend on the accumulator is fetched while the tile's MMAs still run
  static __device__ __forceinline__ void prefetch(const Params& ep, EpiCtx& c, State& st) {
    const int vb = (c.col0 + c.grp * 48) / 3;                                    // first vertex of this warp
    st.wl = (vb * 2 + c.lane < ep.nv * 2) ? __ldg(&ep.w2[vb * 2 + c.lane]) : 0.f;
    if (c.tc.m_tile != c.prev_m_tile) {            // per-head transforms -> registers, once per row tile
      const int head0 = c.tc.m_tile * kBlockM + c.wq * 32;
      const int h = min(head0 + c.lane, c.g->Wo - 1);
      const float4* src = reinterpret_cast<const float4*>(ep.xf + static_cast<size_t>(h) * kXfFloats);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const float4 a = __ldg(&src[q]);           // joint 0
        const float4 b = __ldg(&src[6 + q]);       // joint 2 (jaw)
        st.R[4 * q] = a.x; st.R[4 * q + 1] = a.y; st.R[4 * q + 2] = a.z; st.R[4 * q + 3] = a.w;
        st.Jw[4 * q] = b.x; st.Jw[4 * q + 1] = b.y; st.Jw[4 * q + 2] = b.z; st.Jw[4 * q + 3] = b.w;
      }
      const float4 u = __ldg(&src[15]);
      const float4 w = __ldg(&src[16]);
      st.cx = u.x; st.cy = u.y; st.cz = u.z; st.sc = u.w; st.tx = w.x; st.ty = w.y;
    }
  }
  static __device__ __forceinline__ void run(const Params& ep, EpiCtx& c, State& st) {
    const int rows = c.g->Wo;
    const int head0 = c.tc.m_tile * kBlockM + c.wq * 32;
    float* stage = reinterpret_cast<float*>(c.stage);

    const int colw = c.grp * 48;
    const int vb = (c.col0 + colw) / 3;                                          // first vertex of this warp
    const float wl = st.wl;

    // ---- the warp's 48 accumulator columns (16 vertices) -> registers in one go
    float xa[48];
    epi_load<0, 48>(c, colw, xa);

#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      float x[24];                                                               // 8 vertices of this pass
#pragma unroll
      for (int j = 0; j < 24; ++j) x[j] = xa[pass * 24 + j];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float px = x[3 * i], py = x[3 * i + 1], pz = x[3 * i + 2];
        const float wr = __shfl_sync(0xffffffffu, wl, 2 * (pass * 8 + i));
        const float wj = __shfl_sync(0xffffffffu, wl, 2 * (pass * 8 + i) + 1);
        const float rx = fmaf(st.R[0], px, fmaf(st.R[1], py, fmaf(st.R[2], pz, st.R[3])));
        const float ry = fmaf(st.R[4], px, fmaf(st.R[5], py, fmaf(st.R[6], pz, st.R[7])));
        const float rz = fmaf(st.R[8], px, fmaf(st.R[9], py, fmaf(st.R[10], pz, st.R[11])));
        const float jx = fmaf(st.Jw[0], px, fmaf(st.Jw[1], py, fmaf(st.Jw[2], pz, st.Jw[3])));
        const float jy = fmaf(st.Jw[4], px, fmaf(st.Jw[5], py, fmaf(st.Jw[6], pz, st.Jw[7])));
        const float jz = fmaf(st.Jw[8], px, fmaf(st.Jw[9], py, fmaf(st.Jw[10], pz, st.Jw[11])));
        x[3 * i] = fmaf(wj, jx, fmaf(wr, rx, st.cx));
        x[3 * i + 1] = fmaf(wj, jy, fmaf(wr, ry, st.cy));
        x[3 * i + 2] = fmaf(wj, jz, fmaf(wr, rz, st.cz));
      }
      const int vfirst = vb + pass * 8;
      const int nvalid = min(8, ep.nv - vfirst);                                 // vertices of this pass inside the mesh
      if (nvalid > 0) {
        if (ep.verts3d) {
#pragma unroll
          for (int j = 0; j < 24; ++j) stage[c.lane * 25 + j] = x[j];
          flush<24>(ep.verts3d + (static_cast<size_t>(head0) * ep.nv + vfirst) * 3, static_cast<size_t>(ep.nv) * 3, stage,
                    c.lane, head0, rows, nvalid * 3);
        }
        if (ep.proj) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float qx = (fmaf(x[3 * i], st.sc, st.tx) + 1.0f) * 0.5f * ep.image_size;       // head_mesh.py:40-43
            const float qy = (fmaf(x[3 * i + 1], st.sc, st.ty) + 1.0f) * 0.5f * ep.image_size;
            if (ep.pc == 2) {
              stage[c.lane * 25 + 2 * i] = qx;
              stage[c.lane * 25 + 2 * i + 1] = qy;
            } else {
              stage[c.lane * 25 + 3 * i] = qx;
              stage[c.lane * 25 + 3 * i + 1] = qy;
              stage[c.lane * 25 + 3 * i + 2] = (fmaf(x[3 * i + 2], st.sc, 0.0f) + 1.0f) * 0.5f * ep.image_size;
            }
          }
          if (ep.pc == 2)
            flush<16>(ep.proj + (static_cast<size_t>(head0) * ep.nv + vfirst) * 2, static_cast<size_t>(ep.nv) * 2, stage,
                      c.lane, head0, rows, nvalid * 2);
          else
            flush<24>(ep.proj + (static_cast<size_t>(head0) * ep.nv + vfirst) * 3, static_cast<size_t>(ep.nv) * 3, stage,
                      c.lane, head0, rows, nvalid * 3);
        }
      }
    }
  }
};

// verification aid (DAD3D_BLEND_SIMT): same product on CUDA cores from the same hi/lo planes
__global__ void blend_simt_kernel(const __half* __restrict__ a_hi, const __half* __restrict__ a_lo,
                                  const __half* __restrict__ b_hi, const __half* __restrict__ b_lo,
                                  int rows, int npad, float* __restrict__ out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int h = blockIdx.y;
  if (n >= npad || h >= rows) return;
  float acc = 0.f;
  for (int k = 0; k < kKPad; ++k) {
    const float a = __half2float(a_hi[static_cast<size_t>(h) * kKPad + k]) + __half2float(a_lo[static_cast<size_t>(h) * kKPad + k]);
    const float b = __half2float(b_hi[static_cast<size_t>(n) * kKPad + k]) + __half2float(b_lo[static_cast<size_t>(n) * kKPad + k]);
    acc = fmaf(a, b, acc);
  }
  out[static_cast<size_t>(h) * npad + n] = acc;            // scaled v_posed (template column included)
}

// ------------------------------------------------------------------------------------------------ K3
constexpr int kLbsThreads = 256;

__global__ void __launch_bounds__(kLbsThreads)
lbs_project_kernel(const float* __restrict__ vposed, int ldv, const float* __restrict__ weights,
                   const float* __restrict__ xf, int B, int nv, float* __restrict__ verts3d,
                   float* __restrict__ proj, int pc, float image_size) {
  __shared__ float s_in[3 * kLbsThreads];
  __shared__ float s_out[3 * kLbsThreads];
  __shared__ float s_proj[3 * kLbsThreads];
  __shared__ float s_xf[kXfFloats];
  const int t = threadIdx.x;
  const int v0 = blockIdx.x * kLbsThreads;
  const int v = v0 + t;
  const int nvalid = min(kLbsThreads, nv - v0);          // vertices in this block
  float w[kJoints];
#pragma unroll
  for (int j = 0; j < kJoints; ++j) w[j] = (v < nv) ? __ldg(&weights[static_cast<size_t>(v) * kJoints + j]) : 0.f;

  for (int h = blockIdx.y; h < B; h += gridDim.y) {
    const float* src = vposed + static_cast<size_t>(h) * ldv + 3 * v0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i = t + k * kLbsThreads;
      if (i < 3 * nvalid) s_in[i] = __ldg(&src[i]);
    }
    if (t < kXfFloats) s_xf[t] = __ldg(&xf[static_cast<size_t>(h) * kXfFloats + t]);
    __syncthreads();
    if (v < nv) {
      const float x = s_in[3 * t], y = s_in[3 * t + 1], z = s_in[3 * t + 2];
      float ox = s_xf[60], oy = s_xf[61], oz = s_xf[62];
#pragma unroll
      for (int j = 0; j < kJoints; ++j) {
        if (w[j] != 0.f) {
          const float* A = &s_xf[12 * j];
          ox = fmaf(w[j], fmaf(A[0], x, fmaf(A[1], y, fmaf(A[2], z, A[3]))), ox);
          oy = fmaf(w[j], fmaf(A[4], x, fmaf(A[5], y, fmaf(A[6], z, A[7]))), oy);
          oz = fmaf(w[j], fmaf(A[8], x, fmaf(A[9], y, fmaf(A[10], z, A[11]))), oz);
        }
      }
      s_out[3 * t] = ox;
      s_out[3 * t + 1] = oy;
      s_out[3 * t + 2] = oz;
      const float sc = s_xf[63];
      const float px = (fmaf(ox, sc, s_xf[64]) + 1.0f) * 0.5f * image_size;     // head_mesh.py:40-43
      const float py = (fmaf(oy, sc, s_xf[65]) + 1.0f) * 0.5f * image_size;
      s_proj[pc * t] = px;
      s_proj[pc * t + 1] = py;
      if (pc == 3) s_proj[3 * t + 2] = (fmaf(oz, sc, 0.0f) + 1.0f) * 0.5f * image_size;
    }
    __syncthreads();
    if (verts3d) {
      float* dst = verts3d + (static_cast<size_t>(h) * nv + v0) * 3;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int i = t + k * kLbsThreads;
        if (i < 3 * nvalid) dst[i] = s_out[i];
      }
    }
    if (proj) {
      float* dst = proj + (static_cast<size_t>(h) * nv + v0) * pc;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int i = t + k * kLbsThreads;
        if (i < pc * nvalid) dst[i] = s_proj[i];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ K4
__global__ void gather_kernel(const float* __restrict__ src, int B, int nv, int nc, const int* __restrict__ idx, int L,
                              float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * L * nc;
  if (i >= total) return;
  const int c = static_cast<int>(i % nc);
  const int l = static_cast<int>((i / nc) % L);
  const long long b = i / (static_cast<long long>(nc) * L);
  out[i] = __ldg(&src[(b * nv + __ldg(&idx[l])) * nc + c]);
}

__global__ void gather_bary_kernel(const float* __restrict__ src, int B, int nv, int nc, const int* __restrict__ tri,
                                   const float* __restrict__ bary, int L, float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * L * nc;
  if (i >= total) return;
  const int c = static_cast<int>(i % nc);
  const int l = static_cast<int>((i / nc) % L);
  const long long b = i / (static_cast<long long>(nc) * L);
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k)
    acc = fmaf(__ldg(&bary[3 * l + k]), __ldg(&src[(b * nv + __ldg(&tri[3 * l + k])) * nc + c]), acc);
  out[i] = acc;
}

}  // namespace dad3d


// =================================================================================================== backward (SURVEY §8f row 3)
// dL/d(params) from dL/d(vertices_3d) and / or dL/d(reprojected vertices): what ``loss.backward()`` needs when the reference's
// losses call HeadMesh (losses/vertices_3d_loss.py:30-47, losses/reprojection_loss.py:22-46, flame_lightning_model.py:329-351).
// Forward model (layouts without neck / eyeball pose, the released one):
//     p_s   = scale * (T + S beta + P phi(jaw))                        blend GEMM (recomputed here into a scratch)
//     out_v = w_r(v) (A0' p_s + t0) + w_j(v) (A2' p_s + t2) + c        [A'|t], c = F(jaw, rot6, J(beta))  (flame_prep_kernel)
//     proj  = ((out * sc + (tx, ty, 0)) + 1) * image/2,  sc = max(s + 1, 1e-8)
// Backward:  g_v = gV + (image/2) sc gP;   dp_s = (w_r A0'^T + w_j A2'^T) g_v;   d coef = Basis_s^T dp_s  -- the dense part,
// a [heads,15104] x [15104,448] wgmma GEMM through the tile engine (fp16 hi/lo operands, 3 products);  the cotangents of
// (A0', t0, A2', t2, c) are per-head sums over the vertices;  the 24-input function F (Rodrigues, kinematic chain, 6-DoF
// Gram-Schmidt) is differentiated in forward mode, one input direction per lane, and contracted with those cotangents.
namespace dad3d {

struct Dual {
  float v, d;
};
__device__ __forceinline__ Dual mk(float v, float d = 0.f) { return Dual{v, d}; }
__device__ __forceinline__ Dual operator+(Dual a, Dual b) { return {a.v + b.v, a.d + b.d}; }
__device__ __forceinline__ Dual operator-(Dual a, Dual b) { return {a.v - b.v, a.d - b.d}; }
__device__ __forceinline__ Dual operator-(Dual a) { return {-a.v, -a.d}; }
__device__ __forceinline__ Dual operator*(Dual a, Dual b) { return {a.v * b.v, fmaf(a.v, b.d, a.d * b.v)}; }
__device__ __forceinline__ Dual operator*(float a, Dual b) { return {a * b.v, a * b.d}; }
__device__ __forceinline__ Dual operator/(Dual a, Dual b) {
  const float q = a.v / b.v;
  return {q, (a.d - q * b.d) / b.v};
}
__device__ __forceinline__ Dual dsqrt(Dual a) {
  const float s = sqrtf(a.v);
  return {s, s > 0.f ? 0.5f * a.d / s : 0.f};
}
__device__ __forceinline__ Dual dsin(Dual a) { return {sinf(a.v), cosf(a.v) * a.d}; }
__device__ __forceinline__ Dual dcos(Dual a) { return {cosf(a.v), -sinf(a.v) * a.d}; }
__device__ __forceinline__ Dual dmaxc(Dual a, float c) { return a.v >= c ? a : mk(c); }      // fmaxf(x, c)

__device__ __forceinline__ void d_rodrigues(const Dual* r, Dual* R) {      // smplx batch_rodrigues, as rodrigues() above
  const Dual ax = r[0] + mk(1e-8f), ay = r[1] + mk(1e-8f), az = r[2] + mk(1e-8f);
  const Dual angle = dsqrt(ax * ax + ay * ay + az * az);
  const Dual x = r[0] / angle, y = r[1] / angle, z = r[2] / angle;
  const Dual s = dsin(angle), c1 = mk(1.0f) - dcos(angle);
  R[0] = mk(1.0f) + c1 * (-(z * z) - y * y);
  R[1] = s * (-z) + c1 * (x * y);
  R[2] = s * y + c1 * (x * z);
  R[3] = s * z + c1 * (x * y);
  R[4] = mk(1.0f) + c1 * (-(z * z) - x * x);
  R[5] = s * (-x) + c1 * (y * z);
  R[6] = s * (-y) + c1 * (x * z);
  R[7] = s * x + c1 * (y * z);
  R[8] = mk(1.0f) + c1 * (-(y * y) - x * x);
}
__device__ __forceinline__ void d_mat3_mul(const Dual* A, const Dual* B, Dual* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ void d_mat3_vec(const Dual* A, const Dual* v, Dual* o) {
  for (int i = 0; i < 3; ++i) o[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}

// F: (jaw[3], rot6[6], J[15]) -> out[36] = A0'[9] (row-major, 1/basis_scale folded in), t0[3], A2'[9], t2[3], c[3], phi_jaw[9];
// the same arithmetic as flame_prep_kernel for layouts whose only posed joint is the jaw (FLAME tree -1,0,1,1,1).
__device__ void head_transforms_dual(const Dual* jaw, const Dual* rot6, const Dual* J, int flags, float inv_scale, Dual* out) {
  Dual zero3[3] = {mk(0.f), mk(0.f), mk(0.f)};
  Dual R0[9], R1[9], R2[9];
  d_rodrigues(zero3, R0);                 // global rotation is not given to lbs (flame.py:205-208); neck pose is zero here
  d_rodrigues(zero3, R1);
  Dual jz[3] = {jaw[0], jaw[1], jaw[2]};
  if (flags & DAD3D_ZERO_JAW) { jz[0] = jz[1] = jz[2] = mk(0.f); }
  d_rodrigues(jz, R2);
  for (int e = 0; e < 9; ++e) out[27 + e] = R2[e] - mk((e == 0 || e == 4 || e == 8) ? 1.0f : 0.0f);
  // kinematic chain: joint 0, 1 (child of 0), 2 (child of 1)
  Dual GR1[9], GR2[9], Gt0[3], Gt1[3], Gt2[3], rel[3], tmp[3];
  for (int k = 0; k < 3; ++k) Gt0[k] = J[k];
  d_mat3_mul(R0, R1, GR1);
  for (int k = 0; k < 3; ++k) rel[k] = J[3 + k] - J[k];
  d_mat3_vec(R0, rel, tmp);
  for (int k = 0; k < 3; ++k) Gt1[k] = tmp[k] + Gt0[k];
  d_mat3_mul(GR1, R2, GR2);
  for (int k = 0; k < 3; ++k) rel[k] = J[6 + k] - J[3 + k];
  d_mat3_vec(GR1, rel, tmp);
  for (int k = 0; k < 3; ++k) Gt2[k] = tmp[k] + Gt1[k];
  // 6-DoF rotation (model/utils.py:92-101)
  Dual R6[9] = {mk(1.f), mk(0.f), mk(0.f), mk(0.f), mk(1.f), mk(0.f), mk(0.f), mk(0.f), mk(1.f)};
  if (!(flags & DAD3D_ZERO_ROT)) {
    const Dual* vx = rot6;
    const Dual* vy = rot6 + 3;
    const Dual n1 = dmaxc(dsqrt(vx[0] * vx[0] + vx[1] * vx[1] + vx[2] * vx[2]), 1e-12f);
    const Dual b1[3] = {vx[0] / n1, vx[1] / n1, vx[2] / n1};
    const Dual c3[3] = {b1[1] * vy[2] - b1[2] * vy[1], b1[2] * vy[0] - b1[0] * vy[2], b1[0] * vy[1] - b1[1] * vy[0]};
    const Dual n3 = dmaxc(dsqrt(c3[0] * c3[0] + c3[1] * c3[1] + c3[2] * c3[2]), 1e-12f);
    const Dual b3[3] = {c3[0] / n3, c3[1] / n3, c3[2] / n3};
    const Dual b2[3] = {-(b1[1] * b3[2] - b1[2] * b3[1]), -(b1[2] * b3[0] - b1[0] * b3[2]), -(b1[0] * b3[1] - b1[1] * b3[0])};
    for (int r = 0; r < 3; ++r) {
      R6[3 * r + 0] = b1[r];
      R6[3 * r + 1] = b2[r];
      R6[3 * r + 2] = b3[r];
    }
  }
  const Dual* GRs[2] = {R0, GR2};
  const Dual* Gts[2] = {Gt0, Gt2};
  const int jidx[2] = {0, 2};
  for (int q = 0; q < 2; ++q) {
    Dual rj[3], t[3], AR[9], At[3];
    d_mat3_vec(GRs[q], &J[3 * jidx[q]], rj);
    for (int k = 0; k < 3; ++k) t[k] = Gts[q][k] - rj[k];
    d_mat3_mul(R6, GRs[q], AR);
    d_mat3_vec(R6, t, At);
    for (int e = 0; e < 9; ++e) out[12 * q + e] = inv_scale * AR[e];
    for (int k = 0; k < 3; ++k) out[12 * q + 9 + k] = At[k];
  }
  for (int r = 0; r < 3; ++r) out[24 + r] = kMeshOffsetZ * R6[3 * r + 2];
}

// per head: max |g_v| over the mesh (g = gV + (image/2) sc gP) -> the power-of-two factor that lifts dp into the fp16 range.
// The exponent is capped at sigma_emax = min(127, 127 - log2(basis_scale)), so that sigma and lift = sigma * basis_scale stay
// finite and unlift = 1 / lift is its exact reciprocal: a head whose gradient is below ~2^(log2(basis_scale) - 118) is lifted
// less than to [512, 1024) (its dp may land among the fp16 subnormals) instead of by an infinite factor (0 * inf = NaN).
// NaN gradient entries do not raise the maximum (fmaxf); an infinite maximum gives sigma = 1.
__global__ void __launch_bounds__(256)
flame_bwd_gmax_kernel(const float* __restrict__ gv, const float* __restrict__ gp, int pc, int nv, const float* __restrict__ xf,
                      float half_img, int sigma_emax, float* __restrict__ sigma) {
  const int h = blockIdx.x;
  const float sc = xf[static_cast<size_t>(h) * kXfFloats + 63] * half_img;
  float m = 0.f;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    float g[3] = {0.f, 0.f, 0.f};
    if (gv) for (int c = 0; c < 3; ++c) g[c] = gv[(static_cast<size_t>(h) * nv + v) * 3 + c];
    if (gp) for (int c = 0; c < pc; ++c) g[c] = fmaf(sc, gp[(static_cast<size_t>(h) * nv + v) * pc + c], g[c]);
    m = fmaxf(m, fmaxf(fabsf(g[0]), fmaxf(fabsf(g[1]), fabsf(g[2]))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float ws[8];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = fmaxf(m, ws[w]);
    int e = 0;
    float s = 1.f;
    if (m > 0.f && isfinite(m)) {
      frexpf(m, &e);                                   // m = f * 2^e, f in [0.5, 1)
      s = ldexpf(1.f, min(10 - e, sigma_emax));        // sigma * m in [512, 1024) unless capped
    }
    sigma[h] = s;
  }
}

constexpr int kBwdPartial = 32;                        // floats per (head, vertex block) partial record
// per (head, vertex): dp -> fp16 hi/lo rows of D; per-block partial sums of the transform cotangents
__global__ void __launch_bounds__(256)
flame_bwd_vertex_kernel(const float* __restrict__ vposed, int ldv, const float* __restrict__ w2, const float* __restrict__ xf,
                        const float* __restrict__ gv, const float* __restrict__ gp, int pc, int nv, float half_img,
                        const float* __restrict__ sigma, float basis_scale, __half* __restrict__ d_hi, __half* __restrict__ d_lo,
                        float* __restrict__ partial) {
  __shared__ float s_xf[kXfFloats];
  __shared__ float s_red[8][kBwdPartial];
  const int h = blockIdx.y;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (threadIdx.x < kXfFloats) s_xf[threadIdx.x] = xf[static_cast<size_t>(h) * kXfFloats + threadIdx.x];
  __syncthreads();
  float acc[30];
#pragma unroll
  for (int i = 0; i < 30; ++i) acc[i] = 0.f;
  if (v < nv) {
    const float sc = s_xf[63];
    float g[3] = {0.f, 0.f, 0.f}, gq[3] = {0.f, 0.f, 0.f};
    if (gv) for (int c = 0; c < 3; ++c) g[c] = gv[(static_cast<size_t>(h) * nv + v) * 3 + c];
    if (gp) for (int c = 0; c < pc; ++c) gq[c] = half_img * gp[(static_cast<size_t>(h) * nv + v) * pc + c];
    const float px = vposed[static_cast<size_t>(h) * ldv + 3 * v], py = vposed[static_cast<size_t>(h) * ldv + 3 * v + 1],
                pz = vposed[static_cast<size_t>(h) * ldv + 3 * v + 2];
    const float wr = w2[2 * v], wj = w2[2 * v + 1];
    const float* A0 = s_xf;            // rows [R | t] of joint 0
    const float* A2 = s_xf + 24;       // joint 2 (jaw)
    // forward value of the vertex (needed for d sc)
    float o[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float a = fmaf(A0[4 * r], px, fmaf(A0[4 * r + 1], py, fmaf(A0[4 * r + 2], pz, A0[4 * r + 3])));
      const float b = fmaf(A2[4 * r], px, fmaf(A2[4 * r + 1], py, fmaf(A2[4 * r + 2], pz, A2[4 * r + 3])));
      o[r] = fmaf(wj, b, fmaf(wr, a, s_xf[60 + r]));
    }
    acc[27] = gq[0] * o[0] + gq[1] * o[1] + gq[2] * o[2];          // d sc
    acc[28] = gq[0];                                               // d tx
    acc[29] = gq[1];                                               // d ty
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = fmaf(sc, gq[c], g[c]);      // total cotangent of out_v
    const float p[3] = {px, py, pz};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        acc[3 * r + c] = wr * g[r] * p[c];                         // G_A0'
        acc[12 + 3 * r + c] = wj * g[r] * p[c];                    // G_A2'
      }
      acc[9 + r] = wr * g[r];                                      // g_t0
      acc[21 + r] = wj * g[r];                                     // g_t2
      acc[24 + r] = g[r];                                          // g_c
    }
    // dp_s = (w_r A0'^T + w_j A2'^T) g, lifted by sigma * basis_scale into the fp16 range
    const float lift = sigma[h] * basis_scale;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float d = wr * (A0[c] * g[0] + A0[4 + c] * g[1] + A0[8 + c] * g[2]) + wj * (A2[c] * g[0] + A2[4 + c] * g[1] + A2[8 + c] * g[2]);
      split_store(d_hi, d_lo, static_cast<size_t>(h) * ldv + 3 * v + c, d * lift);
    }
  }
#pragma unroll
  for (int i = 0; i < 30; ++i) {
    float x = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5][i] = x;
  }
  __syncthreads();
  if (threadIdx.x < 30) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += s_red[w][threadIdx.x];
    partial[(static_cast<size_t>(h) * gridDim.x + blockIdx.x) * kBwdPartial + threadIdx.x] = s;
  }
}

// one warp per head: lanes 0..23 differentiate F along one input each (jaw 0..2, rot6 3..8, J 9..23)
__global__ void __launch_bounds__(128)
flame_bwd_finalize_kernel(const float* __restrict__ params, int B, FlameLayoutDev L, const float* __restrict__ jt,
                          const float* __restrict__ jdirsT, int flags, float inv_scale, const float* __restrict__ dcoef,
                          const float* __restrict__ partial, int n_blocks, const float* __restrict__ sigma, float basis_scale,
                          float* __restrict__ gparams) {
  const int h = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (h >= B) return;
  const float* p = params + static_cast<size_t>(h) * L.n_params;
  // joints J = J_T + J_dirs beta (as flame_prep_kernel)
  float accj[15];
#pragma unroll
  for (int j = 0; j < 15; ++j) accj[j] = 0.f;
  for (int l = lane; l < kBetas; l += 32) {
    float b = 0.f;
    if (l < kMaxShape) { if (l < L.n_shape) b = p[L.off_shape + l]; }
    else if (l - kMaxShape < L.n_expr) b = p[L.off_expr + l - kMaxShape];
#pragma unroll
    for (int j = 0; j < 15; ++j) accj[j] = fmaf(b, __ldg(&jdirsT[j * kBetas + l]), accj[j]);
  }
#pragma unroll
  for (int j = 0; j < 15; ++j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) accj[j] += __shfl_xor_sync(0xffffffffu, accj[j], o);
    accj[j] += __ldg(&jt[j]);
  }
  // cotangents: lane i < 30 sums partial[.][i] over the vertex blocks
  float cot = 0.f;
  if (lane < 30)
    for (int b = 0; b < n_blocks; ++b) cot += partial[(static_cast<size_t>(h) * n_blocks + b) * kBwdPartial + lane];
  const float unlift = 1.0f / (sigma[h] * basis_scale);
  const float* dc = dcoef + static_cast<size_t>(h) * kKPad;
  // directional derivative along input `lane`
  float grad_in = 0.f;
  {
    Dual jaw[3], rot6[6], J[15], out[36];
    for (int k = 0; k < 3; ++k) jaw[k] = mk(L.n_jaw == 3 ? p[L.off_jaw + k] : 0.f, lane == k ? 1.f : 0.f);
    for (int k = 0; k < 6; ++k) rot6[k] = mk(p[L.off_rot + k], lane == 3 + k ? 1.f : 0.f);
    for (int k = 0; k < 15; ++k) J[k] = mk(accj[k], lane == 9 + k ? 1.f : 0.f);
    head_transforms_dual(jaw, rot6, J, flags, inv_scale, out);
    // out order: A0'[9] t0[3] A2'[9] t2[3] c[3] phi[9]; partial order: G_A0'[9] g_t0[3] G_A2'[9] g_t2[3] g_c[3]
    for (int i = 0; i < 27; ++i) grad_in = fmaf(__shfl_sync(0xffffffffu, cot, i), out[i].d, grad_in);
    for (int e = 0; e < 9; ++e) grad_in = fmaf(dc[kBetas + 9 + e] * unlift, out[27 + e].d, grad_in);   // jaw = joint 2: features 9..17
  }
  float* gout = gparams + static_cast<size_t>(h) * L.n_params;
  // betas: dense part + joints part
  float dJ[15];
#pragma unroll
  for (int j = 0; j < 15; ++j) dJ[j] = __shfl_sync(0xffffffffu, grad_in, 9 + j);
  for (int l = lane; l < kBetas; l += 32) {
    float gbeta = dc[l] * unlift;
#pragma unroll
    for (int j = 0; j < 15; ++j) gbeta = fmaf(dJ[j], __ldg(&jdirsT[j * kBetas + l]), gbeta);
    if (l < kMaxShape) { if (l < L.n_shape) gout[L.off_shape + l] = gbeta; }
    else if (l - kMaxShape < L.n_expr) gout[L.off_expr + l - kMaxShape] = gbeta;
  }
  if (lane < 3 && L.n_jaw == 3) gout[L.off_jaw + lane] = (flags & DAD3D_ZERO_JAW) ? 0.f : grad_in;
  if (lane >= 3 && lane < 9) gout[L.off_rot + lane - 3] = (flags & DAD3D_ZERO_ROT) ? 0.f : grad_in;
  const float dsc = __shfl_sync(0xffffffffu, cot, 27), dtx = __shfl_sync(0xffffffffu, cot, 28), dty = __shfl_sync(0xffffffffu, cot, 29);
  if (lane == 0) {
    gout[L.off_scale] = (p[L.off_scale] + 1.0f > 1e-8f) ? dsc : 0.f;      // clamp(s + 1, 1e-8)   head_mesh.py:39
    gout[L.off_trans + 0] = dtx;
    gout[L.off_trans + 1] = dty;
    gout[L.off_trans + 2] = 0.f;                                           // z translation is zeroed in the forward (head_mesh.py:41)
  }
}

}  // namespace dad3d

// =================================================================================================== host side
using namespace dad3d;

struct dad3d_flame {
  int device = 0;
  GemmLaunchCache gemm_lbs, gemm_blend;      // tile-engine launches with <EpiLbs> / <EpiBlend>
  bool decode_configured = false;            // per handle (= per device): max dynamic smem set for flame_decode_kernel
  int nv = 0, n3 = 0, npad = 0;
  int num_sms = 0;
  FlameLayoutDev layout{};
  float basis_scale = 1.f;
  __half* d_basis[2] = {nullptr, nullptr};   // [npad, kKPad] fp16 hi / lo planes of scale * [shapedirs | posedirs^T]
  float* d_w2 = nullptr;                     // [nv, 2] (sum of non-jaw weights, jaw weight) for the fused path
  float* d_w2p = nullptr;                    // decode kernel: per vertex PAIR (w_rest v, w_rest v+1, w_jaw v, w_jaw v+1), whole tiles
  __half* d_basis_dec = nullptr;             // decode kernel: hi plane with the rows of every 64-vertex tile regrouped per vertex
                                             // pair as (x x' y y' z z') -- operands of the packed fp32 FMAs (flame_decode.cuh)
  bool jaw_only = false;                     // layout has no neck / eyeball pose -> fused epilogue is exact
  float* d_weights = nullptr;                // [nv, 5]
  float* d_jt = nullptr;                     // [15]
  float* d_jdirsT = nullptr;                 // [15, 400]
  CUtensorMap map_b[2];                      // box 64 x 128 (unfused path)
  CUtensorMap map_b96[2];                    // box 64 x 96  (fused path)
  CUtensorMap map_b48[2];                    // box 64 x 48  (fused path, 2x2 clusters: each CTA loads half of a B tile)
  __half* d_basisT[2] = {nullptr, nullptr};  // [kKPad, npad] hi / lo planes (transposed basis) for the backward GEMM (lazy)
  CUtensorMap map_bT[2];                     // box 64 x 64 over the transposed planes
  CUtensorMap map_dec;                       // hi plane, box 64 x 192 (decode kernel)
  int fused_chunk = 0;                       // heads per pass of the fused path: 4 row tiles per SM
};

namespace {

// Schedule of one flame_decode_kernel launch over `rows` heads: fills rows, nv, n_tiles, m_units, splits and stages of *p and
// returns the grid size (CTAs).  Shared by the launch and dad3d_flame_describe.
int dec_schedule(const dad3d_flame* h, int rows, DecodeParams* p) {
  p->rows = rows;
  p->nv = h->nv;
  p->n_tiles = ceil_div(h->n3, kDecN);
  p->m_units = dec_rows_padded(rows) / kDecBlockM;                // whole permutation blocks: two row tiles per 256 heads
  const int groups_max = h->num_sms;
  // fewer row tiles than SMs: split every row tile's sweep over the vertex tiles so that all SMs get work
  p->splits = p->m_units >= groups_max ? 1 : ceil_div(groups_max, p->m_units);
  if (p->splits > p->n_tiles) p->splits = p->n_tiles;
  const int units = p->m_units * p->splits;
  p->stages = dec_max_stages();
  return units < groups_max ? units : groups_max;
}

// One launch of flame_decode_kernel over `rows` heads whose fp16 coefficient rows (a_hi) and transform records (xf) the prep
// kernel has written.
int launch_flame_decode(dad3d_flame* h, const __half* a_hi, int rows, const float* xf, float* v3, float* pj, int pc,
                        float image_size, cudaStream_t stream) {
  if (!h->decode_configured) {
    DAD3D_CUDA_OK(cudaFuncSetAttribute(flame_decode_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemLimit));
    DAD3D_CUDA_OK(cudaFuncSetAttribute(flame_decode_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemLimit));
    h->decode_configured = true;
  }
  CUtensorMap map_a;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(kKPad), static_cast<uint64_t>(dec_rows_padded(rows))};
    const uint64_t strides[1] = {static_cast<uint64_t>(kKPad) * 2};
    const uint32_t box[2] = {kDecBlockK, kDecBlockM};
    if (!make_tmap_16bit(&map_a, a_hi, 2, dims, strides, box, nullptr)) return DAD3D_ERR_CUDA;
  }
  DecodeParams p;
  const int groups = dec_schedule(h, rows, &p);
  if (p.stages < 2) { set_error("decode pipeline does not fit shared memory"); return DAD3D_ERR_INVALID; }
  p.xf = xf;
  p.w2 = h->d_w2p;
  p.verts3d = v3;
  p.proj = pj;
  p.pc = pc;
  p.image_size = image_size;
  {
    const char* e = std::getenv("DAD3D_DECODE_DEBUG");
    p.debug = e ? std::atoi(e) : 0;
    const char* e2 = std::getenv("DAD3D_DECODE_POLL");
    p.poll = e2 ? std::atoi(e2) : 0;
  }
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(kDecThreads);
  cfg.gridDim = dim3(groups);
  cfg.dynamicSmemBytes = dec_smem_bytes(p.stages);
  cfg.stream = stream;
  cfg.numAttrs = 0;
  if (pj) DAD3D_CUDA_OK(cudaLaunchKernelEx(&cfg, flame_decode_kernel<true>, map_a, h->map_dec, p));
  else DAD3D_CUDA_OK(cudaLaunchKernelEx(&cfg, flame_decode_kernel<false>, map_a, h->map_dec, p));
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

inline unsigned short f32_to_f16_bits(float x) {
  // round-to-nearest-even fp32 -> fp16 on the host (finite inputs of modest magnitude only)
  __half h = __float2half_rn(x);
  unsigned short b;
  std::memcpy(&b, &h, 2);
  return b;
}
inline float f16_bits_to_f32(unsigned short b) {
  __half h;
  std::memcpy(&h, &b, 2);
  return __half2float(h);
}

}  // namespace

extern "C" {

int dad3d_flame_create(dad3d_flame** out, const float* shapedirs_h, const float* posedirs_h, const float* v_template_h,
                       const float* j_regressor_h, const int32_t* parents_h, const float* lbs_weights_h,
                       int32_t n_vertices, int32_t n_betas, int32_t n_joints, const dad3d_flame_layout* lay,
                       int32_t device) {
  DAD3D_REQUIRE(out && shapedirs_h && posedirs_h && v_template_h && j_regressor_h && parents_h && lbs_weights_h && lay,
                "null pointer");
  DAD3D_REQUIRE(n_joints == kJoints, "n_joints must be 5 (FLAME)");
  DAD3D_REQUIRE(n_betas == kBetas, "n_betas must be 400 (300 shape + 100 expression)");
  DAD3D_REQUIRE(n_vertices > 0, "n_vertices");
  DAD3D_REQUIRE(lay->rotation == 6, "rotation width must be 6 (model/utils.py:93)");
  DAD3D_REQUIRE(lay->translation == 3 && lay->scale == 1, "translation/scale widths must be 3/1");
  DAD3D_REQUIRE(lay->shape >= 0 && lay->shape <= kMaxShape && lay->expression >= 0 && lay->expression <= kMaxExpr,
                "shape/expression widths");
  DAD3D_REQUIRE((lay->jaw == 0 || lay->jaw == 3) && (lay->neck == 0 || lay->neck == 3) &&
                    (lay->eyeballs == 0 || lay->eyeballs == 6),
                "jaw/neck/eyeballs widths must be 0 or 3/3/6");
  DAD3D_REQUIRE(parents_h[0] == -1, "parents[0] must be -1");
  for (int i = 1; i < kJoints; ++i) DAD3D_REQUIRE(parents_h[i] >= 0 && parents_h[i] < i, "parents must be topologically ordered");

  DAD3D_CUDA_OK(cudaSetDevice(device));
  cudaDeviceProp prop;
  DAD3D_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("libdad3d requires an sm_90 (Hopper) device, found sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
    return DAD3D_ERR_UNSUPPORTED;
  }

  dad3d_flame* h = new dad3d_flame();
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  h->nv = n_vertices;
  h->n3 = 3 * n_vertices;
  h->npad = ceil_div(h->n3, kBlendBlockN) * kBlendBlockN;
  FlameLayoutDev& L = h->layout;
  int cur = 0;
  L.off_shape = cur; L.n_shape = lay->shape; cur += lay->shape;
  L.off_expr = cur; L.n_expr = lay->expression; cur += lay->expression;
  L.off_jaw = cur; L.n_jaw = lay->jaw; cur += lay->jaw;
  L.off_rot = cur; cur += lay->rotation;
  L.off_eye = cur; L.n_eye = lay->eyeballs; cur += lay->eyeballs;
  L.off_neck = cur; L.n_neck = lay->neck; cur += lay->neck;
  L.off_trans = cur; cur += lay->translation;
  L.off_scale = cur; cur += lay->scale;
  L.n_params = cur;
  for (int i = 0; i < kJoints; ++i) L.parents[i] = parents_h[i];

  const int n3 = h->n3, npad = h->npad;
  // power-of-two scale that lifts the basis into the well-conditioned part of the fp16 range (hi AND lo normal)
  float amax = 0.f;
  for (size_t i = 0; i < static_cast<size_t>(n3) * kBetas; ++i) amax = fmaxf(amax, fabsf(shapedirs_h[i]));
  for (size_t i = 0; i < static_cast<size_t>(kPoseFeat) * n3; ++i) amax = fmaxf(amax, fabsf(posedirs_h[i]));
  float tmax = 0.f;
  for (int i = 0; i < n3; ++i) tmax = fmaxf(tmax, fabsf(v_template_h[i]));
  int e = 0;
  if (amax > 0.f) {
    std::frexp(amax, &e);          // amax = m * 2^e, m in [0.5,1)
    e = 10 - e;                     // scaled amax in [512, 1024)
    if (e > 24) e = 24;
    if (e < -8) e = -8;
  }
  if (tmax > 0.f) {                 // the template rides in the same fp16 planes: keep scale * |T| below 2^15
    int et = 0;
    std::frexp(tmax, &et);
    if (e > 15 - et) e = 15 - et;
  }
  h->basis_scale = std::ldexp(1.0f, e);

  std::vector<unsigned short> hi(static_cast<size_t>(npad) * kKPad, 0), lo(static_cast<size_t>(npad) * kKPad, 0);
  for (int n = 0; n < n3; ++n) {
    unsigned short* rh = &hi[static_cast<size_t>(n) * kKPad];
    unsigned short* rl = &lo[static_cast<size_t>(n) * kKPad];
    for (int k = 0; k < kBetas + kPoseFeat; ++k) {
      const float x = (k < kBetas ? shapedirs_h[static_cast<size_t>(n) * kBetas + k]
                                  : posedirs_h[static_cast<size_t>(k - kBetas) * n3 + n]) * h->basis_scale;
      const unsigned short hb = f32_to_f16_bits(x);
      rh[k] = hb;
      rl[k] = f32_to_f16_bits(x - f16_bits_to_f32(hb));
    }
    // template: two columns with coefficient 1 (kTmplCol, kTmplCol+1 -- the prep kernel writes 1.0 into both).  The
    // successive fp16 pieces p0..p3 of scale*T go to (col0.hi, col1.hi, col0.lo, col1.lo): the hi planes alone already
    // carry 22 bits (what the one-product FAST mode sees), all four planes are exact in fp32 unless the last piece underflows
    // fp16 (then within 2^-25).
    float r = v_template_h[n] * h->basis_scale;
    unsigned short pc[4];
    for (int k = 0; k < 4; ++k) {
      pc[k] = f32_to_f16_bits(r);
      r -= f16_bits_to_f32(pc[k]);
    }
    rh[kTmplCol] = pc[0];
    rh[kTmplCol + 1] = pc[1];
    rl[kTmplCol] = pc[2];
    rl[kTmplCol + 1] = pc[3];
  }
  // (sum of the non-jaw weights, jaw weight) per vertex for the jaw-only fused epilogue
  std::vector<float> w2(static_cast<size_t>(n_vertices) * 2, 0.f);
  for (int i = 0; i < n_vertices; ++i) {
    float rest = 0.f;
    for (int j = 0; j < kJoints; ++j)
      if (j != 2) rest += lbs_weights_h[static_cast<size_t>(i) * kJoints + j];
    w2[2 * i] = rest;
    w2[2 * i + 1] = lbs_weights_h[static_cast<size_t>(i) * kJoints + 2];
  }
  // the two-transform epilogue is exact only when every non-jaw joint carries joint 0's transform: no neck / eyeball pose in
  // the layout AND the FLAME kinematic tree (jaw = joint 2, child of the neck, with no children of its own)
  h->jaw_only = (lay->neck == 0 && lay->eyeballs == 0 && parents_h[1] == 0 && parents_h[2] == 1 && parents_h[3] == 1 &&
                 parents_h[4] == 1);

  // folded joint regressor: J = Jreg * T + (Jreg * S) beta   (smplx vertices2joints applied to v_shaped)
  std::vector<float> jt(15, 0.f), jdirsT(15 * kBetas, 0.f);
  {
    std::vector<double> jt_d(15, 0.0), jd(15 * kBetas, 0.0);
    for (int j = 0; j < kJoints; ++j)
      for (int i = 0; i < n_vertices; ++i) {
        const double wji = j_regressor_h[static_cast<size_t>(j) * n_vertices + i];
        if (wji == 0.0) continue;
        for (int c = 0; c < 3; ++c) {
          jt_d[3 * j + c] += wji * v_template_h[3 * i + c];
          const float* srow = &shapedirs_h[(static_cast<size_t>(i) * 3 + c) * kBetas];
          double* drow = &jd[static_cast<size_t>(3 * j + c) * kBetas];
          for (int l = 0; l < kBetas; ++l) drow[l] += wji * srow[l];
        }
      }
    for (int i = 0; i < 15; ++i) jt[i] = static_cast<float>(jt_d[i]);
    for (size_t i = 0; i < jd.size(); ++i) jdirsT[i] = static_cast<float>(jd[i]);
  }

  auto fail = [&](int code) { dad3d_flame_destroy(h); return code; };
#define CK(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { set_error(std::string(#expr) + " -> " + cudaGetErrorString(_e)); return fail(DAD3D_ERR_CUDA); } } while (0)
  const size_t plane = static_cast<size_t>(npad) * kKPad * sizeof(__half);
  CK(cudaMalloc(&h->d_basis[0], plane));
  CK(cudaMalloc(&h->d_basis[1], plane));
  // decode-kernel copies: vertex-pair weight table and the pair-regrouped hi plane
  const int dec_tiles = ceil_div(n3, kDecN);
  std::vector<float> w2p(static_cast<size_t>(dec_tiles) * (kDecN / 3) * 2, 0.f);
  std::vector<unsigned short> hi_dec(static_cast<size_t>(dec_tiles) * kDecN * kKPad, 0);
  for (int t = 0; t < dec_tiles; ++t)
    for (int j = 0; j < kDecN / 6; ++j) {                        // vertex pair j of tile t
      const int v0 = t * (kDecN / 3) + 2 * j;
      for (int e = 0; e < 2; ++e) {
        const int v = v0 + e;
        if (v >= n_vertices) continue;
        w2p[(static_cast<size_t>(t) * (kDecN / 6) + j) * 4 + e] = w2[2 * v];
        w2p[(static_cast<size_t>(t) * (kDecN / 6) + j) * 4 + 2 + e] = w2[2 * v + 1];
        for (int c = 0; c < 3; ++c)
          std::memcpy(&hi_dec[(static_cast<size_t>(t) * kDecN + 6 * j + 2 * c + e) * kKPad], &hi[(static_cast<size_t>(v) * 3 + c) * kKPad],
                      kKPad * sizeof(unsigned short));
      }
    }
  CK(cudaMalloc(&h->d_w2p, w2p.size() * sizeof(float)));
  CK(cudaMalloc(&h->d_basis_dec, hi_dec.size() * sizeof(unsigned short)));
  CK(cudaMemcpy(h->d_w2p, w2p.data(), w2p.size() * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_basis_dec, hi_dec.data(), hi_dec.size() * sizeof(unsigned short), cudaMemcpyHostToDevice));
  CK(cudaMalloc(&h->d_w2, w2.size() * sizeof(float)));
  CK(cudaMalloc(&h->d_weights, static_cast<size_t>(n_vertices) * kJoints * sizeof(float)));
  CK(cudaMalloc(&h->d_jt, 15 * sizeof(float)));
  CK(cudaMalloc(&h->d_jdirsT, 15 * kBetas * sizeof(float)));
  CK(cudaMemcpy(h->d_basis[0], hi.data(), plane, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_basis[1], lo.data(), plane, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_w2, w2.data(), w2.size() * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_weights, lbs_weights_h, static_cast<size_t>(n_vertices) * kJoints * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_jt, jt.data(), 15 * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_jdirsT, jdirsT.data(), 15 * kBetas * sizeof(float), cudaMemcpyHostToDevice));
#undef CK
  for (int p = 0; p < 2; ++p) {
    const uint64_t dims[2] = {static_cast<uint64_t>(kKPad), static_cast<uint64_t>(npad)};
    const uint64_t strides[1] = {static_cast<uint64_t>(kKPad) * 2};
    const uint32_t box[2] = {kBlockK, kBlendBlockN};
    if (!make_tmap_16bit(&h->map_b[p], h->d_basis[p], 2, dims, strides, box, nullptr)) return fail(DAD3D_ERR_CUDA);
    const uint32_t box96[2] = {kBlockK, kFusedBlockN};
    if (!make_tmap_16bit(&h->map_b96[p], h->d_basis[p], 2, dims, strides, box96, nullptr)) return fail(DAD3D_ERR_CUDA);
    const uint32_t box48[2] = {kBlockK, kFusedBlockN / 2};
    if (!make_tmap_16bit(&h->map_b48[p], h->d_basis[p], 2, dims, strides, box48, nullptr)) return fail(DAD3D_ERR_CUDA);
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(kKPad), static_cast<uint64_t>(ceil_div(n3, kDecN) * kDecN)};
    const uint64_t strides[1] = {static_cast<uint64_t>(kKPad) * 2};
    const uint32_t box192[2] = {kDecBlockK, kDecN};
    if (!make_tmap_16bit(&h->map_dec, h->d_basis_dec, 2, dims, strides, box192, nullptr)) return fail(DAD3D_ERR_CUDA);
  }
  h->fused_chunk = h->num_sms * kBlockM * 4;
  *out = h;
  return DAD3D_OK;
}

void dad3d_flame_destroy(dad3d_flame* h) {
  if (!h) return;
  cudaFree(h->d_basis[0]);
  cudaFree(h->d_basis[1]);
  cudaFree(h->d_w2);
  cudaFree(h->d_w2p);
  cudaFree(h->d_basis_dec);
  cudaFree(h->d_weights);
  cudaFree(h->d_jt);
  cudaFree(h->d_jdirsT);
  cudaFree(h->d_basisT[0]);
  cudaFree(h->d_basisT[1]);
  delete h;
}

int32_t dad3d_flame_num_params(const dad3d_flame* h) { return h ? h->layout.n_params : 0; }
int32_t dad3d_flame_num_vertices(const dad3d_flame* h) { return h ? h->nv : 0; }

// coefficient rows: padded to whole 256-head permutation blocks (the dedicated decode kernel stores them permuted)
static size_t ws_coef_bytes(int rows) { return align_up(static_cast<size_t>(dec_rows_padded(rows)) * kKPad * sizeof(__half), 1024); }
static size_t ws_xf_bytes(int rows) { return align_up(static_cast<size_t>(rows) * kXfFloats * sizeof(float), 1024); }
static size_t ws_vposed_bytes(const dad3d_flame* h, int rows) { return align_up(static_cast<size_t>(rows) * h->npad * sizeof(float), 1024); }

size_t dad3d_flame_workspace_bytes(const dad3d_flame* h, int32_t B) {
  if (!h || B <= 0) return 0;
  const int rows_u = B < kDecodeChunk ? B : kDecodeChunk;                 // unfused / SIMT passes
  const size_t unfused = 2 * ws_coef_bytes(rows_u) + ws_xf_bytes(rows_u) + ws_vposed_bytes(h, rows_u) + 1024;
  const int rows_f = B < h->fused_chunk ? B : h->fused_chunk;             // fused passes need no v_posed scratch
  const size_t fused = 2 * ws_coef_bytes(rows_f) + ws_xf_bytes(rows_f) + 1024;
  return unfused > fused ? unfused : fused;
}

// The four decode paths.  Default: the dedicated one-product decode kernel (flame_decode.cuh); DAD3D_BLEND_HILO = 3-product hi/lo
// operands through the tile engine with the fused EpiLbs epilogue (fp32-class blend product); general layouts and
// DAD3D_DECODE_UNFUSED: EpiBlend to a v_posed scratch + lbs_project_kernel; DAD3D_BLEND_SIMT: CUDA-core product +
// lbs_project_kernel.  DAD3D_BLEND_FAST is the old name of today's default and is accepted as a no-op.
enum DecodePath { kPathDedicated, kPathLbs, kPathBlend, kPathSimt };
static DecodePath decode_path(const dad3d_flame* h, int flags) {
  const bool fused = h->jaw_only && !(flags & (DAD3D_BLEND_SIMT | DAD3D_DECODE_UNFUSED));
  if (fused) return (flags & DAD3D_BLEND_HILO) ? kPathLbs : kPathDedicated;
  return (flags & DAD3D_BLEND_SIMT) ? kPathSimt : kPathBlend;
}
static bool path_fused(DecodePath path) { return path == kPathDedicated || path == kPathLbs; }
// heads per pass: the fused paths need no v_posed scratch
static int decode_chunk(const dad3d_flame* h, DecodePath path) { return path_fused(path) ? h->fused_chunk : kDecodeChunk; }
// big fused passes (>= one row tile per SM): 2x2 thread-block clusters with TMA multicast of both operands (opt-in)
static bool decode_clustered(const dad3d_flame* h, DecodePath path, int rows, int flags) {
  return path == kPathLbs && ceil_div(rows, kBlockM) >= h->num_sms && (flags & DAD3D_DECODE_CLUSTER);
}

// Tile-engine geometry of a plain row GEMM  D[rows, n_cols] = A[rows, 64 k_blocks] B[n_cols, 64 k_blocks]^T  with
// `pieces`-piece operands: single CTAs, tiles round-robin, the deepest operand ring that fits
static GemmGeom row_gemm_geom(int rows, int k_blocks, int n_cols, int block_n, int pieces) {
  GemmGeom g;
  std::memset(&g, 0, sizeof(g));
  g.tw = kBlockM; g.th = 1; g.tn = 1;
  g.tiles_w = ceil_div(rows, kBlockM); g.tiles_h = 1; g.tiles_n = 1;
  g.Wo = rows; g.Ho = 1; g.Nimg = 1;
  g.stride = 1; g.R = 1; g.S = 1;
  g.cin_blocks = k_blocks;
  g.cl_m = 1; g.cl_n = 1;
  g.n_tiles = ceil_div(n_cols, block_n);
  g.block_n = block_n;
  gemm_products(g, pieces);
  g.stages = gemm_max_stages(g);
  return g;
}

// Tensor maps of a row GEMM: A = the fp16 plane pair hi / lo, each [rows, k] (box 64 x box_rows), and the B planes b[0..1]
static int row_gemm_maps(GemmMaps* maps, const __half* hi, const __half* lo, int rows, int k, int box_rows,
                         const CUtensorMap* b) {
  std::memset(maps, 0, sizeof(*maps));
  const __half* planes[2] = {hi, lo};
  for (int pi = 0; pi < 2; ++pi) {
    const uint64_t dims[4] = {static_cast<uint64_t>(k), static_cast<uint64_t>(rows), 1, 1};
    const uint64_t strides[3] = {static_cast<uint64_t>(k) * 2, static_cast<uint64_t>(k) * 2 * rows,
                                 static_cast<uint64_t>(k) * 2 * rows};
    const uint32_t box[4] = {kBlockK, static_cast<uint32_t>(box_rows), 1, 1};
    if (!make_tmap_16bit(&maps->a[pi], planes[pi], 4, dims, strides, box, nullptr)) return DAD3D_ERR_CUDA;
    maps->b[pi] = b[pi];
  }
  return DAD3D_OK;
}

// Tile-engine geometry of the blend product of one pass (kPathLbs / kPathBlend)
static GemmGeom blend_geom(const dad3d_flame* h, DecodePath path, int rows, int flags) {
  const bool fused = path == kPathLbs;
  const int pieces = (flags & DAD3D_BLEND_FAST) && !(flags & DAD3D_BLEND_HILO) ? 1 : 2;   // unfused A/B path: one product
  GemmGeom g = row_gemm_geom(rows, kKPad / kBlockK, h->n3, fused ? kFusedBlockN : kBlendBlockN, pieces);
  if (decode_clustered(h, path, rows, flags)) { g.cl_m = 2; g.cl_n = 2; }
  g.sched = fused && g.tiles_w >= h->num_sms ? 1 : 0;   // enough row tiles to give every SM its own
  return g;
}

// K1 alone: coefficient rows (permuted for the dedicated kernel) and transform records of `rows` heads
static int flame_prep(dad3d_flame* h, const float* p, int rows, int flags, __half* a_hi, __half* a_lo, float* xf, bool permute,
                      cudaStream_t stream) {
  const int threads = 256;
  const int group = rows >= 32 * 8 * h->num_sms ? 32 : 1;              // heads per warp (see the kernel)
  const int blocks = ceil_div(ceil_div(rows, group) * 32, threads);
  flame_prep_kernel<<<blocks, threads, 0, stream>>>(p, rows, h->layout, h->d_jt, h->d_jdirsT, flags, 1.0f / h->basis_scale, a_hi,
                                                    a_lo, xf, permute ? 1 : 0, group);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

// Everything after K1 for one pass of `rows` <= decode_chunk heads: the product and skinning of the path `flags` selects
static int flame_decode_stage(dad3d_flame* h, const __half* a_hi, const __half* a_lo, const float* xf, int rows, int flags,
                              float* v3, float* pj, int pc, float image_size, float* vposed, cudaStream_t stream) {
  const DecodePath path = decode_path(h, flags);
  if (path == kPathDedicated) return launch_flame_decode(h, a_hi, rows, xf, v3, pj, pc, image_size, stream);
  if (path == kPathSimt) {
    dim3 grid(ceil_div(h->npad, 256), rows);
    blend_simt_kernel<<<grid, 256, 0, stream>>>(a_hi, a_lo, h->d_basis[0], h->d_basis[1], rows, h->npad, vposed);
    count_launch();
    DAD3D_CUDA_OK(cudaGetLastError());
  } else {
    const bool clustered = decode_clustered(h, path, rows, flags);
    GemmMaps maps;
    int rc = row_gemm_maps(&maps, a_hi, a_lo, rows, kKPad, clustered ? kBlockM / 2 : kBlockM,
                           path == kPathLbs ? (clustered ? h->map_b48 : h->map_b96) : h->map_b);
    if (rc != DAD3D_OK) return rc;
    const GemmGeom g = blend_geom(h, path, rows, flags);
    if (path == kPathLbs) {
      EpiLbs::Params ep{xf, h->d_w2, h->nv, v3, pj, pc, image_size};
      return gemm_launch<EpiLbs>(maps, g, ep, h->num_sms, &h->gemm_lbs, false, stream);
    }
    EpiBlend::Params ep{vposed, h->npad};
    rc = gemm_launch<EpiBlend>(maps, g, ep, h->num_sms, &h->gemm_blend, false, stream);
    if (rc != DAD3D_OK) return rc;
  }
  dim3 grid(ceil_div(h->nv, kLbsThreads), rows < 1024 ? rows : 1024);
  lbs_project_kernel<<<grid, kLbsThreads, 0, stream>>>(vposed, h->npad, h->d_weights, xf, rows, h->nv, v3, pj, pc, image_size);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_flame_decode(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, float* vertices3d_d,
                       float* projected_d, float image_size, int32_t to_2d, void* workspace_d, size_t workspace_bytes,
                       dad3d_stream stream_) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && params_d, "params");
  DAD3D_REQUIRE(vertices3d_d || projected_d, "at least one output must be requested");
  DAD3D_REQUIRE(workspace_d && workspace_bytes >= dad3d_flame_workspace_bytes(h, B), "workspace too small");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const DecodePath path = decode_path(h, flags);
  const int chunk = decode_chunk(h, path);
  const int rows_max = B < chunk ? B : chunk;
  uint8_t* ws = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(workspace_d), 1024));
  __half* a_hi = reinterpret_cast<__half*>(ws);
  __half* a_lo = reinterpret_cast<__half*>(ws + ws_coef_bytes(rows_max));
  float* xf = reinterpret_cast<float*>(ws + 2 * ws_coef_bytes(rows_max));
  float* vposed = reinterpret_cast<float*>(ws + 2 * ws_coef_bytes(rows_max) + ws_xf_bytes(rows_max));
  const int pc = to_2d ? 2 : 3;

  for (int b0 = 0; b0 < B; b0 += chunk) {
    const int rows = (B - b0) < chunk ? (B - b0) : chunk;
    const float* p = params_d + static_cast<size_t>(b0) * h->layout.n_params;
    float* v3 = vertices3d_d ? vertices3d_d + static_cast<size_t>(b0) * h->nv * 3 : nullptr;
    float* pj = projected_d ? projected_d + static_cast<size_t>(b0) * h->nv * pc : nullptr;
    int rc = flame_prep(h, p, rows, flags, a_hi, a_lo, xf, path == kPathDedicated, stream);
    if (rc != DAD3D_OK) return rc;
    rc = flame_decode_stage(h, a_hi, a_lo, xf, rows, flags, v3, pj, pc, image_size, vposed, stream);
    if (rc != DAD3D_OK) return rc;
  }
  return DAD3D_OK;
}

int dad3d_flame_prep(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, void* coef_hi_d, void* coef_lo_d,
                     float* xf_d, int32_t permute, dad3d_stream stream) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && params_d && coef_hi_d && coef_lo_d && xf_d, "null pointer");
  return flame_prep(h, params_d, B, flags, static_cast<__half*>(coef_hi_d), static_cast<__half*>(coef_lo_d), xf_d, permute != 0,
                    reinterpret_cast<cudaStream_t>(stream));
}

int dad3d_flame_decode_from(dad3d_flame* h, const void* coef_hi_d, const void* coef_lo_d, const float* xf_d, int32_t B,
                            int32_t flags, float* vertices3d_d, float* projected_d, float image_size, int32_t to_2d,
                            void* workspace_d, size_t workspace_bytes, dad3d_stream stream) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && coef_hi_d && coef_lo_d && xf_d, "null pointer");
  DAD3D_REQUIRE(vertices3d_d || projected_d, "at least one output must be requested");
  const DecodePath path = decode_path(h, flags);
  DAD3D_REQUIRE(B <= decode_chunk(h, path), "B exceeds one pass of the selected decode path");
  float* vposed = nullptr;
  if (!path_fused(path)) {
    DAD3D_REQUIRE(workspace_d && workspace_bytes >= ws_vposed_bytes(h, B) + 1024, "workspace too small");
    vposed = reinterpret_cast<float*>(align_up(reinterpret_cast<uintptr_t>(workspace_d), 1024));
  }
  return flame_decode_stage(h, static_cast<const __half*>(coef_hi_d), static_cast<const __half*>(coef_lo_d), xf_d, B, flags,
                            vertices3d_d, projected_d, to_2d ? 2 : 3, image_size, vposed, reinterpret_cast<cudaStream_t>(stream));
}

int dad3d_flame_describe(dad3d_flame* h, int32_t B, int32_t flags, char* json, size_t cap) {
  DAD3D_REQUIRE(h && json && cap > 0, "null pointer");
  DAD3D_REQUIRE(B >= 0, "B");
  const DecodePath path = decode_path(h, flags);
  const int chunk = decode_chunk(h, path);
  static const char* kNames[4] = {"dedicated", "lbs", "blend", "simt"};
  char scale[32];
  std::snprintf(scale, sizeof(scale), "%.17g", static_cast<double>(h->basis_scale));
  std::string out = "{\"basis_scale\": " + std::string(scale) + ", \"jaw_only\": " + (h->jaw_only ? "true" : "false") +
                    ", \"nv\": " + std::to_string(h->nv) + ", \"npad\": " + std::to_string(h->npad) +
                    ", \"fused_chunk\": " + std::to_string(h->fused_chunk) + ", \"num_sms\": " + std::to_string(h->num_sms) +
                    ", \"passes\": [";
  for (int b0 = 0; b0 < B; b0 += chunk) {
    const int rows = (B - b0) < chunk ? (B - b0) : chunk;
    int m_units = 0, splits = 1, grid = 0, stages = 0;
    bool clustered = false;
    if (path == kPathDedicated) {
      DecodeParams p;
      grid = dec_schedule(h, rows, &p);
      m_units = p.m_units;
      splits = p.splits;
      stages = p.stages;
    } else if (path == kPathSimt) {
      m_units = rows;
      grid = ceil_div(h->npad, 256) * rows;
    } else {
      const GemmGeom g = blend_geom(h, path, rows, flags);
      cudaLaunchConfig_t cfg;
      cudaLaunchAttribute attr[2];
      int rc = path == kPathLbs ? gemm_launch_config<EpiLbs>(g, h->num_sms, &h->gemm_lbs, false, &cfg, attr)
                                : gemm_launch_config<EpiBlend>(g, h->num_sms, &h->gemm_blend, false, &cfg, attr);
      if (rc != DAD3D_OK) return rc;
      m_units = g.tiles_w;
      grid = static_cast<int>(cfg.gridDim.x);
      stages = g.stages;
      clustered = g.cl_m * g.cl_n > 1;
    }
    out += std::string(b0 ? ", " : "") + "{\"path\": \"" + kNames[path] + "\", \"rows\": " + std::to_string(rows) +
           ", \"m_units\": " + std::to_string(m_units) + ", \"splits\": " + std::to_string(splits) +
           ", \"grid\": " + std::to_string(grid) + ", \"stages\": " + std::to_string(stages) +
           ", \"clustered\": " + (clustered ? "true" : "false") + "}";
  }
  out += "]}";
  DAD3D_REQUIRE(out.size() < cap, "json buffer too small");
  std::memcpy(json, out.c_str(), out.size() + 1);
  return DAD3D_OK;
}

// ------------------------------------------------------------------------------------------------ backward host side
static size_t ws_d_bytes(const dad3d_flame* h, int rows) { return align_up(static_cast<size_t>(rows) * h->npad * sizeof(__half), 1024); }
static size_t ws_dcoef_bytes(int rows) { return align_up(static_cast<size_t>(rows) * kKPad * sizeof(float), 1024); }
static size_t ws_partial_bytes(const dad3d_flame* h, int rows) {
  return align_up(static_cast<size_t>(rows) * ceil_div(h->nv, 256) * kBwdPartial * sizeof(float), 1024);
}

size_t dad3d_flame_backward_workspace_bytes(const dad3d_flame* h, int32_t B) {
  if (!h || B <= 0) return 0;
  const int rows = B < kDecodeChunk ? B : kDecodeChunk;
  return 2 * ws_coef_bytes(rows) + ws_xf_bytes(rows) + ws_vposed_bytes(h, rows) + 2 * ws_d_bytes(h, rows) + ws_dcoef_bytes(rows) +
         ws_partial_bytes(h, rows) + align_up(static_cast<size_t>(rows) * sizeof(float), 1024) + 2048;
}

static int ensure_backward_assets(dad3d_flame* h) {
  if (h->d_basisT[0]) return DAD3D_OK;
  const size_t n = static_cast<size_t>(h->npad) * kKPad;
  std::vector<unsigned short> src(n), dst(n);
  for (int pl = 0; pl < 2; ++pl) {
    DAD3D_CUDA_OK(cudaMemcpy(src.data(), h->d_basis[pl], n * 2, cudaMemcpyDeviceToHost));
    for (int r = 0; r < h->npad; ++r)
      for (int k = 0; k < kKPad; ++k) dst[static_cast<size_t>(k) * h->npad + r] = src[static_cast<size_t>(r) * kKPad + k];
    DAD3D_CUDA_OK(cudaMalloc(&h->d_basisT[pl], n * 2));
    DAD3D_CUDA_OK(cudaMemcpy(h->d_basisT[pl], dst.data(), n * 2, cudaMemcpyHostToDevice));
    const uint64_t dims[2] = {static_cast<uint64_t>(h->npad), static_cast<uint64_t>(kKPad)};
    const uint64_t strides[1] = {static_cast<uint64_t>(h->npad) * 2};
    const uint32_t box[2] = {kBlockK, 64};
    if (!make_tmap_16bit(&h->map_bT[pl], h->d_basisT[pl], 2, dims, strides, box, nullptr)) return DAD3D_ERR_CUDA;
  }
  return DAD3D_OK;
}

// The stages of one backward pass of `rows` <= kDecodeChunk heads.  dad3d_flame_backward runs them in this order; the
// dad3d_flame_backward_* test hooks run each one alone on caller buffers.
// Forward blend product (recomputed): v_posed * basis_scale [rows, npad] fp32 from the prep kernel's coefficient rows
static int bwd_blend_stage(dad3d_flame* h, const __half* a_hi, const __half* a_lo, int rows, float* vposed, cudaStream_t stream) {
  GemmMaps maps;
  const int rc = row_gemm_maps(&maps, a_hi, a_lo, rows, kKPad, kBlockM, h->map_b);
  if (rc != DAD3D_OK) return rc;
  const GemmGeom g = row_gemm_geom(rows, kKPad / kBlockK, h->n3, kBlendBlockN, 2);
  EpiBlend::Params ep{vposed, h->npad};
  return gemm_launch<EpiBlend>(maps, g, ep, h->num_sms, &h->gemm_blend, false, stream);
}

// sigma's exponent cap: sigma <= 2^127 and sigma * basis_scale <= 2^127 (flame_bwd_gmax_kernel)
static int sigma_emax(const dad3d_flame* h) {
  int e;
  std::frexp(h->basis_scale, &e);                   // basis_scale = 2^(e - 1)
  return std::min(127, 127 - (e - 1));
}

// Per head sigma; D = dp * sigma * basis_scale as fp16 hi / lo rows [rows, npad] (padding columns zero); per 256-vertex block
// the partial sums of the 30 transform cotangents
static int bwd_vertex_stage(dad3d_flame* h, const float* vposed, const float* xf, const float* gv, const float* gp, int pc, int rows,
                            float half_img, float* sigma, __half* d_hi, __half* d_lo, float* partial, cudaStream_t stream) {
  flame_bwd_gmax_kernel<<<rows, 256, 0, stream>>>(gv, gp, pc, h->nv, xf, half_img, sigma_emax(h), sigma);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  DAD3D_CUDA_OK(cudaMemsetAsync(d_hi, 0, static_cast<size_t>(rows) * h->npad * sizeof(__half), stream));
  DAD3D_CUDA_OK(cudaMemsetAsync(d_lo, 0, static_cast<size_t>(rows) * h->npad * sizeof(__half), stream));
  dim3 grid(ceil_div(h->nv, 256), rows);
  flame_bwd_vertex_kernel<<<grid, 256, 0, stream>>>(vposed, h->npad, h->d_w2, xf, gv, gp, pc, h->nv, half_img, sigma,
                                                    h->basis_scale, d_hi, d_lo, partial);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

// The dense part: d coef [rows, 448] = D [rows, npad] x Basis_s [npad, 448]   (wgmma, fp16 hi/lo, 3 products)
static int bwd_dense_stage(dad3d_flame* h, const __half* d_hi, const __half* d_lo, int rows, float* dcoef, cudaStream_t stream) {
  GemmMaps maps;
  const int rc = row_gemm_maps(&maps, d_hi, d_lo, rows, h->npad, kBlockM, h->map_bT);
  if (rc != DAD3D_OK) return rc;
  const GemmGeom g = row_gemm_geom(rows, h->npad / kBlockK, kKPad, 64, 2);
  EpiBlend::Params ep{dcoef, kKPad};
  return gemm_launch<EpiBlend>(maps, g, ep, h->num_sms, &h->gemm_blend, false, stream);
}

// d coef and the cotangents -> the 413 parameter gradients of `rows` heads
static int bwd_finalize_stage(dad3d_flame* h, const float* p, int rows, int flags, const float* dcoef, const float* partial,
                              const float* sigma, float* gout, cudaStream_t stream) {
  flame_bwd_finalize_kernel<<<ceil_div(rows * 32, 128), 128, 0, stream>>>(p, rows, h->layout, h->d_jt, h->d_jdirsT, flags,
                                                                         1.0f / h->basis_scale, dcoef, partial,
                                                                         ceil_div(h->nv, 256), sigma, h->basis_scale, gout);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_flame_backward_blend(dad3d_flame* h, const void* coef_hi_d, const void* coef_lo_d, int32_t B, float* vposed_d,
                               dad3d_stream stream) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && B <= kDecodeChunk, "B must fit one backward pass (1..4096 heads)");
  DAD3D_REQUIRE(coef_hi_d && coef_lo_d && vposed_d, "null pointer");
  DAD3D_REQUIRE(reinterpret_cast<uintptr_t>(vposed_d) % 16 == 0, "vposed_d must be 16-byte aligned (float4 stores)");
  return bwd_blend_stage(h, static_cast<const __half*>(coef_hi_d), static_cast<const __half*>(coef_lo_d), B, vposed_d,
                         reinterpret_cast<cudaStream_t>(stream));
}

int dad3d_flame_backward_vertex(dad3d_flame* h, const float* vposed_d, const float* xf_d, const float* grad_vertices_d,
                                const float* grad_projected_d, int32_t B, float image_size, int32_t to_2d, float* sigma_d,
                                void* d_hi_d, void* d_lo_d, float* partial_d, dad3d_stream stream) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && B <= kDecodeChunk, "B must fit one backward pass (1..4096 heads)");
  DAD3D_REQUIRE(vposed_d && xf_d && sigma_d && d_hi_d && d_lo_d && partial_d, "null pointer");
  DAD3D_REQUIRE(grad_vertices_d || grad_projected_d, "at least one incoming gradient must be given");
  return bwd_vertex_stage(h, vposed_d, xf_d, grad_vertices_d, grad_projected_d, to_2d ? 2 : 3, B, 0.5f * image_size, sigma_d,
                          static_cast<__half*>(d_hi_d), static_cast<__half*>(d_lo_d), partial_d,
                          reinterpret_cast<cudaStream_t>(stream));
}

int dad3d_flame_backward_dense(dad3d_flame* h, const void* d_hi_d, const void* d_lo_d, int32_t B, float* dcoef_d,
                               dad3d_stream stream) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && B <= kDecodeChunk, "B must fit one backward pass (1..4096 heads)");
  DAD3D_REQUIRE(d_hi_d && d_lo_d && dcoef_d, "null pointer");
  DAD3D_REQUIRE(reinterpret_cast<uintptr_t>(dcoef_d) % 16 == 0, "dcoef_d must be 16-byte aligned (float4 stores)");
  DAD3D_REQUIRE(h->jaw_only, "backward is implemented for layouts without neck / eyeball pose (the released model)");
  const int rc = ensure_backward_assets(h);
  if (rc != DAD3D_OK) return rc;
  return bwd_dense_stage(h, static_cast<const __half*>(d_hi_d), static_cast<const __half*>(d_lo_d), B, dcoef_d,
                         reinterpret_cast<cudaStream_t>(stream));
}

int dad3d_flame_backward_finalize(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, const float* dcoef_d,
                                  const float* partial_d, const float* sigma_d, float* grad_params_d, dad3d_stream stream) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && B <= kDecodeChunk, "B must fit one backward pass (1..4096 heads)");
  DAD3D_REQUIRE(params_d && dcoef_d && partial_d && sigma_d && grad_params_d, "null pointer");
  DAD3D_REQUIRE(h->jaw_only, "backward is implemented for layouts without neck / eyeball pose (the released model)");
  return bwd_finalize_stage(h, params_d, B, flags, dcoef_d, partial_d, sigma_d, grad_params_d,
                            reinterpret_cast<cudaStream_t>(stream));
}

int dad3d_flame_backward(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, const float* grad_vertices_d,
                         const float* grad_projected_d, float image_size, int32_t to_2d, float* grad_params_d,
                         void* workspace_d, size_t workspace_bytes, dad3d_stream stream_) {
  DAD3D_REQUIRE(h, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && params_d && grad_params_d, "params / grad_params");
  DAD3D_REQUIRE(grad_vertices_d || grad_projected_d, "at least one incoming gradient must be given");
  DAD3D_REQUIRE(h->jaw_only, "backward is implemented for layouts without neck / eyeball pose (the released model)");
  DAD3D_REQUIRE(workspace_d && workspace_bytes >= dad3d_flame_backward_workspace_bytes(h, B), "workspace too small");
  int rc = ensure_backward_assets(h);
  if (rc != DAD3D_OK) return rc;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int chunk = kDecodeChunk;
  const int rows_max = B < chunk ? B : chunk;
  uint8_t* ws = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(workspace_d), 1024));
  __half* a_hi = reinterpret_cast<__half*>(ws); ws += ws_coef_bytes(rows_max);
  __half* a_lo = reinterpret_cast<__half*>(ws); ws += ws_coef_bytes(rows_max);
  float* xf = reinterpret_cast<float*>(ws); ws += ws_xf_bytes(rows_max);
  float* vposed = reinterpret_cast<float*>(ws); ws += ws_vposed_bytes(h, rows_max);
  __half* d_hi = reinterpret_cast<__half*>(ws); ws += ws_d_bytes(h, rows_max);
  __half* d_lo = reinterpret_cast<__half*>(ws); ws += ws_d_bytes(h, rows_max);
  float* dcoef = reinterpret_cast<float*>(ws); ws += ws_dcoef_bytes(rows_max);
  float* partial = reinterpret_cast<float*>(ws); ws += ws_partial_bytes(h, rows_max);
  float* sigma = reinterpret_cast<float*>(ws);
  const int pc = to_2d ? 2 : 3;
  const float half_img = 0.5f * image_size;

  for (int b0 = 0; b0 < B; b0 += chunk) {
    const int rows = (B - b0) < chunk ? (B - b0) : chunk;
    const float* p = params_d + static_cast<size_t>(b0) * h->layout.n_params;
    const float* gv = grad_vertices_d ? grad_vertices_d + static_cast<size_t>(b0) * h->nv * 3 : nullptr;
    const float* gp = grad_projected_d ? grad_projected_d + static_cast<size_t>(b0) * h->nv * pc : nullptr;
    float* gout = grad_params_d + static_cast<size_t>(b0) * h->layout.n_params;
    flame_prep_kernel<<<ceil_div(rows * 32, 256), 256, 0, stream>>>(p, rows, h->layout, h->d_jt, h->d_jdirsT, flags,
                                                                     1.0f / h->basis_scale, a_hi, a_lo, xf, 0, 1);
    count_launch();
    DAD3D_CUDA_OK(cudaGetLastError());
    if ((rc = bwd_blend_stage(h, a_hi, a_lo, rows, vposed, stream)) != DAD3D_OK) return rc;
    if ((rc = bwd_vertex_stage(h, vposed, xf, gv, gp, pc, rows, half_img, sigma, d_hi, d_lo, partial, stream)) != DAD3D_OK)
      return rc;
    if ((rc = bwd_dense_stage(h, d_hi, d_lo, rows, dcoef, stream)) != DAD3D_OK) return rc;
    if ((rc = bwd_finalize_stage(h, p, rows, flags, dcoef, partial, sigma, gout, stream)) != DAD3D_OK) return rc;
  }
  return DAD3D_OK;
}

int dad3d_gather_landmarks(const float* src_d, int32_t B, int32_t n_vertices, int32_t ncomp, const int32_t* idx_d,
                           int32_t L, float* out_d, dad3d_stream stream) {
  DAD3D_REQUIRE(src_d && idx_d && out_d, "null pointer");
  DAD3D_REQUIRE(B >= 0 && L >= 0 && n_vertices > 0 && (ncomp == 2 || ncomp == 3), "shape");
  const long long total = static_cast<long long>(B) * L * ncomp;
  if (total == 0) return DAD3D_OK;
  gather_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src_d, B, n_vertices, ncomp, idx_d, L, out_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_gather_landmarks_bary(const float* src_d, int32_t B, int32_t n_vertices, int32_t ncomp,
                                const int32_t* tri_idx_d, const float* bary_d, int32_t L, float* out_d,
                                dad3d_stream stream) {
  DAD3D_REQUIRE(src_d && tri_idx_d && bary_d && out_d, "null pointer");
  DAD3D_REQUIRE(B >= 0 && L >= 0 && n_vertices > 0 && (ncomp == 2 || ncomp == 3), "shape");
  const long long total = static_cast<long long>(B) * L * ncomp;
  if (total == 0) return DAD3D_OK;
  gather_bary_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src_d, B, n_vertices, ncomp, tri_idx_d, bary_d, L, out_d);
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // extern "C"
