// Dedicated FLAME decode kernel for sm_90a (the default path of dad3d_flame_decode):
//
//   vertices[h, v, :] = skin( T + S beta_h + P theta_h )                 flame.py:182-229, smplx.lbs, model/utils.py:92-101
//
// as ONE persistent wgmma kernel: blend shapes + pose correctives + template as a [heads,448] x [15069,448]^T fp16 GEMM
// (fp32 accumulate; the template rides in two K columns and is exact to 22 bits), followed in the epilogue by linear-blend
// skinning, the z offset, the 6-DoF rotation and the weak-perspective projection (head_mesh.py:33-46), written straight into
// the reference's [B,5023,3] / [B,5023,2|3] layouts.
//
// Compared with the generic tile engine (tile_gemm.cuh, still used by the strict hi/lo mode): one tensor-core product per MAC
// (fp16 operands, 11-bit mantissa like TF32; the power-of-two pre-scaled basis keeps every operand normal; relL2 of the
// vertices against the fp64 reference ~1.5e-5, inside the 1e-4 contract), vertex tiles of 192 columns (64 vertices), and an
// epilogue built around whole-sector stores.
// Roles (384 threads): warp 0 TMA producer (one ring slot = one 64-wide k-block of the 128-head coefficient tile and of the
// 192-column basis tile); warpgroups 1 and 2 consume: warpgroup w issues m64n192k16 wgmma for heads rows 64w.. into register
// accumulators, writes them to a shared-memory accumulator tile and runs the epilogue on it.  Epilogue warp (w, i) owns rows
// 32*(2w + i%2).. (= 32 heads) and one half of the tile's columns (96 columns = 32 vertices = 4 passes of 8 vertices); the two
// warps of a row quarter SWAP halves every tile.  Per pass: shared memory -> registers -> skinning -> global stores straight
// from registers.
//
// Stores.  Rows of the reference layout [B,5023,3] are only 4-byte aligned (pitch 60 276 B), and a store that covers part of a
// 32-byte sector costs the L2 a read-modify-write.  Each lane therefore writes ITS OWN row: it keeps the last 8 floats of the
// previous pass (the carry) and writes the window of 24 floats that starts c floats earlier, at the previous sector boundary,
// as whole sectors.  c = (address of the pass's first float, in floats) mod 8 is constant along a row (every pass advances by
// 3 sectors) and depends on the head index only through head mod 8 (8 x pitch = 0 mod 8 floats), so the coefficient rows are
// PERMUTED (dec_phys_row / dec_head_of: physical row tile 2b+t, row quarter wq, lane l <-> head 256 b + 8 l + 4 t + wq) to
// give all 32 lanes of a warp the same c: the window selection is a warp-uniform switch over c with compile-time register
// choices.  Sector boundaries that fall between two warps' column ranges: at a tile boundary the carry stays in the registers
// of the warp that swaps from half 1 to half 0; inside a tile, half 1 recomputes the two vertex pairs in front of its range
// from the same accumulator (+6 % arithmetic).  Partial sectors remain only at the two ends of a unit's column range.
#pragma once
#include "ptx.cuh"

namespace dad3d {

constexpr int kDecBlockM = 128;
constexpr int kDecBlockK = 64;
constexpr int kDecN = 192;                         // columns per vertex tile = 64 vertices
constexpr int kDecKBlocks = 7;                     // 448 / 64
constexpr int kDecABytes = kDecBlockM * kDecBlockK * 2;          // 16 KiB: one k-block of the coefficient tile
constexpr int kDecStageBytes = kDecABytes + kDecN * kDecBlockK * 2;   // + 24 KiB of basis per ring slot
constexpr int kDecAccStride = kDecN + 4;           // floats per accumulator row (= 4 mod 32: conflict-free row-per-lane reads)
constexpr int kDecAccBytes = kDecBlockM * kDecAccStride * 4;
constexpr int kDecThreads = 384;
constexpr int kDecEpiWarps = 8;
constexpr int kDecPassCols = 24;                   // 8 vertices per pass
constexpr int kDecWarpCols = kDecN / 2;             // columns of a tile per epilogue warp (two column groups)
constexpr int kDecPasses = kDecWarpCols / kDecPassCols;   // 4
constexpr int kDecWtabBytes = 20 * 16;             // (w_rest, w_jaw) per vertex pair: the warp's 16 pairs of a tile + the 2 in front
constexpr int kDecXfFloats = 68;
constexpr int kDecSmemLimit = 227 * 1024;
constexpr int kDecRowBlock = 256;                  // heads per permutation block (two row tiles)

// physical coefficient row of head h, and its inverse for (row tile, lane quarter, lane)
__host__ __device__ inline int dec_phys_row(int h) {
  return (h & ~255) + ((h & 7) >> 2) * 128 + (h & 3) * 32 + ((h & 255) >> 3);
}
__host__ __device__ inline int dec_head_of(int m_tile, int wq, int lane) {
  return (m_tile >> 1) * 256 + lane * 8 + (m_tile & 1) * 4 + wq;
}
__host__ __device__ inline int dec_rows_padded(int rows) { return (rows + kDecRowBlock - 1) / kDecRowBlock * kDecRowBlock; }

struct DecodeParams {
  int rows;                 // heads in this launch (coefficient rows are stored permuted: dec_phys_row; rows padded to 256)
  int nv;                   // vertices (5023)
  int n_tiles;              // ceil(3*nv / 192)
  int m_units;              // row tiles (always whole 256-head blocks)
  int splits;               // each m unit is split into `splits` contiguous ranges of vertex tiles
  int stages;               // depth of the operand ring (slots)
  const float* xf;          // [rows][68] per-head transform records (flame_prep_kernel)
  const float* w2;          // [n_tiles * 64][2] (w_rest, w_jaw), zero-padded past nv
  float* verts3d;           // [rows][nv][3] or null
  float* proj;              // [rows][nv][pc] or null
  int pc;
  float image_size;
  int poll;                 // 1: producer / consumer warps poll the ring barriers with test_wait instead of try_wait (A/B)
  int debug;                // diagnostics only (DAD3D_DECODE_DEBUG): 2 = stores predicated off at run time, 3 = no epilogue
                            // (pure main-loop rate)
};

__host__ inline int dec_fixed_smem_bytes() { return kDecAccBytes + kDecEpiWarps * kDecWtabBytes + 1024 + 512; }
__host__ inline int dec_max_stages() {
  const int s = (kDecSmemLimit - dec_fixed_smem_bytes()) / kDecStageBytes;
  return s > 8 ? 8 : s;
}
__host__ inline int dec_smem_bytes(int stages) { return stages * kDecStageBytes + dec_fixed_smem_bytes(); }

// unit u of this CTA: row tile m, vertex tiles [n0, n1)
__device__ __forceinline__ bool dec_unit_at(const DecodeParams& p, int group, int n_groups, int i, int* m, int* n0, int* n1) {
  const int u = group + i * n_groups;
  if (u >= p.m_units * p.splits) return false;
  *m = u / p.splits;
  const int part = u - *m * p.splits;
  *n0 = static_cast<int>(static_cast<long long>(part) * p.n_tiles / p.splits);
  *n1 = static_cast<int>(static_cast<long long>(part + 1) * p.n_tiles / p.splits);
  return true;
}

// ---- window stores.  ext = carry[8] ++ x[RUN] are the floats [g0 - 8, g0 + RUN) of this lane's row (g0 = the pass's first float);
// the window [g0 - C, g0 - C + RUN) = ext[8 - C, 8 - C + RUN) starts on a sector boundary and leaves as RUN/8 whole-sector
// stores.  `head`: no valid carry (first pass of the warp's column range) -- the first sector is partial and its own 8 - C floats
// go out as scalar stores; `tail`: last pass of the range -- the C floats behind the window follow as scalar stores.
template <int RUN, int C>
__device__ __forceinline__ void dec_store_c(float* __restrict__ dst, const float (&carry)[8], const float (&x)[RUN], bool head,
                                            bool tail) {
#define DEC_EXT(e) ((e) < 8 ? carry[(e) < 8 ? (e) : 0] : x[(e) >= 8 ? (e) - 8 : 0])
  float* w = dst - C;
  if (C == 0 || !head) {
    ptx::st_global_8f(w, DEC_EXT(8 - C), DEC_EXT(9 - C), DEC_EXT(10 - C), DEC_EXT(11 - C), DEC_EXT(12 - C), DEC_EXT(13 - C),
                      DEC_EXT(14 - C), DEC_EXT(15 - C));
  } else {
#pragma unroll
    for (int j = 0; j < 8 - C; ++j) dst[j] = x[j];
  }
#pragma unroll
  for (int k = 1; k < RUN / 8; ++k)
    ptx::st_global_8f(w + 8 * k, DEC_EXT(8 - C + 8 * k), DEC_EXT(9 - C + 8 * k), DEC_EXT(10 - C + 8 * k), DEC_EXT(11 - C + 8 * k),
                      DEC_EXT(12 - C + 8 * k), DEC_EXT(13 - C + 8 * k), DEC_EXT(14 - C + 8 * k), DEC_EXT(15 - C + 8 * k));
  if (C > 0 && tail) {
#pragma unroll
    for (int j = 0; j < C; ++j) dst[RUN - C + j] = x[RUN - C + j];
  }
#undef DEC_EXT
}
template <int RUN>
__device__ __forceinline__ void dec_store(float* __restrict__ dst, unsigned c, const float (&carry)[8], const float (&x)[RUN],
                                          bool head, bool tail) {
  switch (c) {                                         // warp-uniform
    case 0: dec_store_c<RUN, 0>(dst, carry, x, head, tail); break;
    case 1: dec_store_c<RUN, 1>(dst, carry, x, head, tail); break;
    case 2: dec_store_c<RUN, 2>(dst, carry, x, head, tail); break;
    case 3: dec_store_c<RUN, 3>(dst, carry, x, head, tail); break;
    case 4: dec_store_c<RUN, 4>(dst, carry, x, head, tail); break;
    case 5: dec_store_c<RUN, 5>(dst, carry, x, head, tail); break;
    case 6: dec_store_c<RUN, 6>(dst, carry, x, head, tail); break;
    default: dec_store_c<RUN, 7>(dst, carry, x, head, tail); break;
  }
}
// Last, partly valid pass of a row (the mesh ends inside it): the carried floats in front of it, then the valid new ones.
template <int RUN>
__device__ __forceinline__ void dec_store_edge(float* __restrict__ dst, unsigned c, const float (&carry)[8], const float (&x)[RUN],
                                            bool head, int nvalid) {
  if (!head) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j >= 8 - static_cast<int>(c)) dst[j - 8] = carry[j];
  }
#pragma unroll
  for (int j = 0; j < RUN; ++j)
    if (j < nvalid) dst[j] = x[j];
}

__device__ __forceinline__ void dec_wait(uint64_t* bar, uint32_t parity, int poll) {
  if (poll) ptx::mbar_wait_poll(bar, parity);
  else ptx::mbar_wait(bar, parity);
}

// kProj: the projected output is requested too (its carry and constants cost registers: own instantiation)
template <bool kProj = true>
__global__ void __launch_bounds__(kDecThreads, 1)
flame_decode_kernel(const __grid_constant__ CUtensorMap map_a,     // coefficients [rows, 448] fp16, box 64 x 128
                    const __grid_constant__ CUtensorMap map_b,     // basis [npad, 448] fp16, box 64 x 192
                    const DecodeParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ring = smem;                                            // [stages][A 16 KiB | B 24 KiB]
  float* acc_smem = reinterpret_cast<float*>(smem + p.stages * kDecStageBytes);   // [128][kDecAccStride]
  uint8_t* wtab_all = smem + p.stages * kDecStageBytes + kDecAccBytes;            // [8][320 B] per-warp (w_rest, w_jaw) table
  uint64_t* bars = reinterpret_cast<uint64_t*>(wtab_all + kDecEpiWarps * kDecWtabBytes);
  uint64_t* full_bar = bars;                  // [8]
  uint64_t* empty_bar = bars + 8;             // [8]

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int group = static_cast<int>(blockIdx.x);
  const int n_groups = static_cast<int>(gridDim.x);

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&map_a);
    ptx::prefetch_tmap(&map_b);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < 8; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);          // one arrive per consumer warpgroup
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();

  if (warp == 0) {
    // ===================================================== TMA producer (whole warp walks the schedule, one lane issues)
    int stage = 0;
    uint32_t phase = 0;
    int m, n0, n1;
    for (int ui = 0; dec_unit_at(p, group, n_groups, ui, &m, &n0, &n1); ++ui) {
      for (int n = n0; n < n1; ++n) {
        for (int kb = 0; kb < kDecKBlocks; ++kb) {
          dec_wait(&empty_bar[stage], phase ^ 1u, p.poll);
          if (ptx::elect_one_sync()) {
            uint8_t* st = ring + stage * kDecStageBytes;
            ptx::mbar_expect_tx(&full_bar[stage], static_cast<uint32_t>(kDecStageBytes));
            ptx::tma_load_2d(st, &map_a, &full_bar[stage], kb * kDecBlockK, m * kDecBlockM);
            ptx::tma_load_2d(st + kDecABytes, &map_b, &full_bar[stage], kb * kDecBlockK, n * kDecN);
          }
          __syncwarp();
          if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================================================== consumer warpgroups: wgmma main loop + skinning epilogue
    const int wg = (warp - 4) >> 2;                // tile rows 64*wg ..
    const int wl = warp & 3;
    const int wq = 2 * wg + (wl & 1);              // row quarter of the epilogue: rows 32*wq + lane
    const int grp = wl >> 1;                       // column half of even tiles (the halves swap every tile)
    const bool signaller = wl == 0 && lane == 0;
    float4* wtab = reinterpret_cast<float4*>(wtab_all + (warp - 4) * kDecWtabBytes);
    const float* arow = acc_smem + (wq * 32 + lane) * kDecAccStride;   // this thread's accumulator row
    float acc[kDecN / 2];
#pragma unroll
    for (int i = 0; i < kDecN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    float R[12], J[12], c0x, c0y, c0z;             // per-head transforms (rest, jaw) and offset
    float sc = 1.f, tx = 0.f, ty = 0.f;
    int m, n0, n1;
    const int nv3 = p.nv * 3;
    const int pc = p.pc;
    const float hs = 0.5f * p.image_size;
    float vcar[8], qcar[8];                        // this row's last 8 floats of the previous pass (the carry), per output
#pragma unroll
    for (int j = 0; j < 8; ++j) vcar[j] = qcar[j] = 0.f;
    for (int ui = 0; dec_unit_at(p, group, n_groups, ui, &m, &n0, &n1); ++ui) {
      const int head = dec_head_of(m, wq, lane);
      const bool row_ok = head < p.rows && p.debug != 2;
      auto load_transforms = [&]() {   // rows past the batch read the last valid record; never stored
        const int h = min(head, p.rows - 1);
        const float4* src = reinterpret_cast<const float4*>(p.xf + static_cast<size_t>(h) * kDecXfFloats);
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const float4 a = __ldg(&src[q]);           // joint 0 (rest)
          const float4 b = __ldg(&src[6 + q]);       // joint 2 (jaw)
          R[4 * q] = a.x; R[4 * q + 1] = a.y; R[4 * q + 2] = a.z; R[4 * q + 3] = a.w;
          J[4 * q] = b.x; J[4 * q + 1] = b.y; J[4 * q + 2] = b.z; J[4 * q + 3] = b.w;
        }
        const float4 u = __ldg(&src[15]);
        const float4 w = __ldg(&src[16]);
        c0x = u.x; c0y = u.y; c0z = u.z;
        sc = u.w; tx = w.x; ty = w.y;
      };
      float* const v_row = p.verts3d ? p.verts3d + static_cast<size_t>(min(head, p.rows - 1)) * nv3 : nullptr;
      float* const q_row = (kProj && p.proj) ? p.proj + static_cast<size_t>(min(head, p.rows - 1)) * p.nv * pc : nullptr;
      // sector phase of the row (floats mod 8): the same for all lanes of the warp (heads = const mod 8), constant along the row
      const unsigned c_v = __shfl_sync(0xffffffffu, static_cast<unsigned>((reinterpret_cast<uintptr_t>(v_row) >> 2) & 7u), 0);
      const unsigned c_q = __shfl_sync(0xffffffffu, static_cast<unsigned>((reinterpret_cast<uintptr_t>(q_row) >> 2) & 7u), 0);
      for (int n = n0; n < n1; ++n) {
        // ---- main loop: this warpgroup's 64 coefficient rows x the 192 basis columns of tile n, K = 448
        int pend = -1;
        for (int kb = 0; kb < kDecKBlocks; ++kb) {
          dec_wait(&full_bar[stage], phase, p.poll);
          const uint32_t sa = ptx::smem_u32(ring + stage * kDecStageBytes) + static_cast<uint32_t>(wg * 64 * kDecBlockK * 2);
          const uint32_t sb = ptx::smem_u32(ring + stage * kDecStageBytes + kDecABytes);
          const uint64_t adesc = ptx::make_kmajor_sw128_desc(sa);
          const uint64_t bdesc = ptx::make_kmajor_sw128_desc(sb);
          ptx::wgmma_fence();
#pragma unroll
          for (int k = 0; k < kDecBlockK / 16; ++k)
            ptx::wgmma_m64k16<kDecN, 0>(acc, adesc + 2u * k, bdesc + 2u * k, (kb > 0 || k > 0) ? 1u : 0u);
          ptx::wgmma_commit();
          ptx::wgmma_wait<1>();                  // the previous k-block's group is complete: its slot may be refilled
          if (pend >= 0 && signaller) ptx::mbar_arrive(&empty_bar[pend]);
          pend = stage;
          if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        }
        ptx::wgmma_wait<0>();
        if (signaller) ptx::mbar_arrive(&empty_bar[pend]);
        ptx::reg_fence(acc);
        // ---- accumulator (this warpgroup's 64 rows) -> shared memory; each epilogue lane then reads its own row
        ptx::bar_sync(1 + wg, 128);              // the previous tile's rows have been read by every warp of the warpgroup
        {
          const int r0 = wg * 64 + wl * 16 + (lane >> 2);
#pragma unroll
          for (int j = 0; j < kDecN / 8; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
            *reinterpret_cast<float2*>(acc_smem + r0 * kDecAccStride + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(acc_smem + (r0 + 8) * kDecAccStride + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
        }
        ptx::bar_sync(1 + wg, 128);
        if (p.debug == 3) continue;
        load_transforms();                       // per tile (L1-resident): not live across the main loop's accumulators
        // Column half of this warp: the two warps of a row quarter SWAP halves every tile, so the warp that ends tile n (half 1)
        // begins tile n+1 (half 0) and the carry across the tile boundary stays in its registers.  Half 1 begins inside the tile:
        // it recomputes the two vertex pairs in front of its range from the same accumulator (12 more columns, +6 % arithmetic)
        // to get its carry.  With that every sector inside a unit's column range is written whole, by one lane.
        const int half = grp ^ (n & 1);
        const float* a_lane = arow + half * kDecWarpCols;
        // (w_rest, w_jaw) per vertex pair -- pairs [14 half, 14 half + 18) of the tile: entries 0, 1 are the two pairs in front of
        // half 1 (unused by half 0), entries 2.. the warp's own 16.
        const float4 wv = __ldg(reinterpret_cast<const float4*>(p.w2) + static_cast<size_t>(n) * (kDecN / 6) +
                                min(max(16 * half - 2 + lane, 0), kDecN / 6 - 1));
        const int col_t = n * kDecN + half * kDecWarpCols;   // first float of the warp's column range within a row
        // Skinning of one vertex pair: the basis rows of a tile are regrouped per vertex pair as (x x' y y' z z'), so the
        // accumulator columns of the two vertices are interleaved.
        auto skin_pair = [&](const float* a6, const float4& w4, float* o6) {
#pragma unroll
          for (int v = 0; v < 2; ++v) {
            const float wr = v ? w4.y : w4.x, wj = v ? w4.w : w4.z;
            const float px = a6[v], py = a6[2 + v], pz = a6[4 + v];
            const float rx = fmaf(R[0], px, fmaf(R[1], py, fmaf(R[2], pz, R[3])));
            const float ry = fmaf(R[4], px, fmaf(R[5], py, fmaf(R[6], pz, R[7])));
            const float rz = fmaf(R[8], px, fmaf(R[9], py, fmaf(R[10], pz, R[11])));
            const float jx = fmaf(J[0], px, fmaf(J[1], py, fmaf(J[2], pz, J[3])));
            const float jy = fmaf(J[4], px, fmaf(J[5], py, fmaf(J[6], pz, J[7])));
            const float jz = fmaf(J[8], px, fmaf(J[9], py, fmaf(J[10], pz, J[11])));
            o6[3 * v] = fmaf(wj, jx, fmaf(wr, rx, c0x));
            o6[3 * v + 1] = fmaf(wj, jy, fmaf(wr, ry, c0y));
            o6[3 * v + 2] = fmaf(wj, jz, fmaf(wr, rz, c0z));
          }
        };
        auto load_cols = [&](const float* src, float* dst, int n4) {
          for (int j = 0; j < n4; ++j) {
            const float4 v = *reinterpret_cast<const float4*>(src + 4 * j);
            dst[4 * j] = v.x; dst[4 * j + 1] = v.y; dst[4 * j + 2] = v.z; dst[4 * j + 3] = v.w;
          }
        };
        __syncwarp();                                // the previous tile's table reads are done
        if (lane < 18) wtab[lane] = wv;
        __syncwarp();
        if (half) {                                  // carry of half 1: the last 8 floats in front of column 96 of the tile
          float xb[16];
          load_cols(a_lane - 16, xb, 4);             // the 12 columns in front of half 1 (4 more ride along)
          float xpre[12];
          skin_pair(xb + 4, wtab[0], xpre);
          skin_pair(xb + 10, wtab[1], xpre + 6);
#pragma unroll
          for (int j = 0; j < 8; ++j) vcar[j] = xpre[4 + j];
          if constexpr (kProj) {
            if (pc == 2) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                qcar[2 * i] = (fmaf(xpre[3 * i], sc, tx) + 1.0f) * hs;
                qcar[2 * i + 1] = (fmaf(xpre[3 * i + 1], sc, ty) + 1.0f) * hs;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const int e = 4 + j;                 // float e of the 12: coordinate e % 3
                qcar[j] = (fmaf(xpre[e], sc, e % 3 == 0 ? tx : e % 3 == 1 ? ty : 0.0f) + 1.0f) * hs;
              }
            }
          }
        }
#pragma unroll 1
        for (int q = 0; q < kDecPasses; ++q) {       // 4 passes of 8 vertices (24 accumulator columns)
          float xa[24];
          load_cols(a_lane + q * kDecPassCols, xa, 6);
          float x[24];
#pragma unroll
          for (int i = 0; i < 4; ++i) skin_pair(xa + 6 * i, wtab[2 + 4 * q + i], x + 6 * i);
          const int col0 = col_t + q * kDecPassCols;
          const int ncols = nv3 - col0;              // valid floats from this pass's first one to the end of the row
          if (ncols > 0) {
            // no carry only at the start of the unit's column range; a tail only at its end or at the end of the row
            const bool first = q == 0 && half == 0 && n == n0;
            const bool last = (q == kDecPasses - 1 && half == 1 && n == n1 - 1) || ncols == kDecPassCols;
            if (v_row) {
              if (row_ok) {
                if (ncols >= kDecPassCols) dec_store<24>(v_row + col0, c_v, vcar, x, first, last);
                else dec_store_edge<24>(v_row + col0, c_v, vcar, x, first, ncols);
              }
#pragma unroll
              for (int j = 0; j < 8; ++j) vcar[j] = x[16 + j];
            }
            if constexpr (kProj) if (q_row) {
              // head_mesh.py:39-43 (z translation is zero)
              const int vfirst = col0 / 3;
              if (pc == 2) {
                float qv[16];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  qv[2 * i] = (fmaf(x[3 * i], sc, tx) + 1.0f) * hs;
                  qv[2 * i + 1] = (fmaf(x[3 * i + 1], sc, ty) + 1.0f) * hs;
                }
                if (row_ok) {
                  if (ncols >= kDecPassCols) dec_store<16>(q_row + vfirst * 2, c_q, qcar, qv, first, last);
                  else dec_store_edge<16>(q_row + vfirst * 2, c_q, qcar, qv, first, (ncols / 3) * 2);
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) qcar[j] = qv[8 + j];
              } else {
                float qv[24];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  qv[3 * i] = (fmaf(x[3 * i], sc, tx) + 1.0f) * hs;
                  qv[3 * i + 1] = (fmaf(x[3 * i + 1], sc, ty) + 1.0f) * hs;
                  qv[3 * i + 2] = (fmaf(x[3 * i + 2], sc, 0.0f) + 1.0f) * hs;
                }
                if (row_ok) {
                  if (ncols >= kDecPassCols) dec_store<24>(q_row + col0, c_q, qcar, qv, first, last);
                  else dec_store_edge<24>(q_row + col0, c_q, qcar, qv, first, ncols);
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) qcar[j] = qv[16 + j];
              }
            }
          }
        }
      }
    }
  }
  __syncthreads();
}

}  // namespace dad3d
