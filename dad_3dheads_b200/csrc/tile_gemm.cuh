// Persistent, warp-specialised wgmma tile engine for sm_90a.
//
//   D[128 x block_n] (fp32)  =  sum over k-blocks, over (a_piece, b_piece) pairs   A_piece[128 x 64] * B_piece[block_n x 64]^T
//
// One kernel serves every dense contraction on the hot path:
//   * the FLAME blend-shape product  (plain GEMM: rows = heads, K = betas | pose features, N = 3*5023 coordinates), and
//   * every convolution of the encoder as an implicit GEMM over NHWC activations (rows = output pixels, the k loop walks
//     filter taps x 64-channel blocks; the A tile for a tap is a TMA box at shifted coordinates, zero-filled outside the
//     image, so padding costs nothing and no im2col buffer exists).
//
// Operands are 16-bit (fp16 or bf16).  fp32-class accuracy comes from splitting each fp32 operand into "pieces"
// (x = p0 + p1 [+ p2], each piece 16-bit) stored as separate planes; the MMA list names which (A piece, B piece) products
// are accumulated (1 product = plain 16-bit GEMM, 3 = hi*hi + hi*lo + lo*hi, 6 = three-way).
//
// Accumulator classes: the tensor core adds into its fp32 accumulator with truncation, so every MMA issued against a
// LARGE accumulator costs up to one ulp of systematic (round-toward-zero) error.  With n_acc = 2 the dominant hi*hi
// products go to accumulator 0 and all the small correction products to accumulator 1; the two are added in fp32 with
// round-to-nearest when the tile is written out.  That cuts the number of truncating steps on the large accumulator by
// n_mma (6x / 3x).
//
// Roles (384 threads = 3 warpgroups): warp 0 = TMA producer (the whole warp walks the schedule, one elect.sync lane issues;
// warps 1..3 only give their registers back: the producer warpgroup drops to kProducerRegs registers per thread and the
// consumer warpgroups grow to kConsumerRegs); warpgroups 1 and 2 = consumers: warpgroup w issues the wgmma for tile rows
// 64w .. 64w+63 (register accumulators) and runs the epilogue.  Two epilogue forms, chosen per launch by GemmGeom::frag_epi:
//   * fragment (frag_epi = 1): each thread works on its own wgmma accumulator registers (warp i of the warpgroup: tile
//     rows 64w + 16i + lane/4 and +8, column pairs 8j + 2(lane%4)), writes 16-bit results into a swizzled staging tile and
//     issues TMA stores of its warp's 16 rows x 32 channels.  No shared-memory accumulator tile exists.
//   * row (frag_epi = 0): the accumulators go to a shared-memory fp32 tile (gemm_acc_bytes) and each thread then owns one
//     accumulator row (warp (w, i): rows 32*(2w + i%2) + lane, column group i/2) -- for epilogues that need whole rows.
// Pipeline: smem ring (full/empty mbarriers) between TMA and the consumers; a consumer releases a slot as soon as the
// wgmma group that read it has completed, so the producer refills it while the next k-block's MMAs run and while the
// epilogue of a tile runs.  Each epilogue warp owns a 4 KiB shared-memory staging area.
// The operand format (fp16 / bf16) is Epi::kBf16, a compile-time constant of the epilogue type.
// Variants selected per launch in GemmGeom: halo (3x3 stride-1 convolutions: one halo patch per channel block feeds all nine
// taps through shifted descriptors; separate weights ring), res_kb / res_kind (residual or second source on the K axis),
// cl_m x cl_n multicast clusters, and ping-pong consumers (GemmGeom::pingpong: each warpgroup owns whole 128 x 64 tiles and the
// two take turns in the main loop, so one warpgroup's epilogue runs under the other's main loop; gemm_consumer_pingpong).
// Host side (end of file): the product list of a piece count, and the launch configuration and launch of the kernel.
#pragma once
#include "../../include/dad3d.h"
#include "common.h"
#include "ptx.cuh"

namespace dad3d {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                       // 64 x 16-bit = 128 B = one swizzle-128B row
constexpr int kTileABytes = kBlockM * kBlockK * 2;   // 16 KiB per A piece per stage
constexpr int kMaxPieces = 3;
constexpr int kMaxMma = 6;
constexpr int kEpiWarps = 8;
constexpr int kFirstEpiWarp = 4;
constexpr int kGemmThreads = (kFirstEpiWarp + kEpiWarps) * 32;   // 384 threads
// per-role register budgets (setmaxnreg): 128 x 40 + 256 x 232 = 64 512 = the 384 x 168 the launch allocates
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
constexpr int kStageOutBytes = 4096;              // per epilogue warp: 32 rows x 128 B
constexpr int kGemmSmemLimit = 227 * 1024;
// halo mode (3x3 stride-1 convolutions): output tiles of 8 x 16 pixels, input halo patch of 10 x 18 pixels per 64-channel
// block and piece = 180 rows of 128 B, padded to a multiple of 1024 B per piece
constexpr int kHaloTW = 8, kHaloTH = 16, kHaloPW = kHaloTW + 2, kHaloPH = kHaloTH + 2;
constexpr int kHaloBytes = kHaloPW * kHaloPH * kBlockK * 2;        // 23040
constexpr int kHaloPieceBytes = 23 * 1024;                         // 23552

struct GemmGeom {
  // output tile = tn images x th rows x tw columns of output pixels (tw*th*tn == 128); plain GEMM: tw=128, th=tn=1
  int tw, th, tn;
  int tiles_w, tiles_h, tiles_n;   // tile counts along W, H, N(images)
  int Wo, Ho, Nimg;                // output extents (store bounds)
  int stride;                      // convolution stride (A tensor map carries matching element strides)
  int R, S, pad_h, pad_w;          // filter taps and padding
  int cin_blocks;                  // padded Cin / 64
  int n_tiles;                     // padded Cout / block_n
  int block_n;                     // wgmma N: 64, 80, 96 or 128
  int nA, nB;                      // operand pieces
  int n_mma;                       // number of (a,b) piece products
  int mma_a[kMaxMma], mma_b[kMaxMma];
  int n_acc;                       // 1 or 2 register accumulators per tile
  int mma_acc[kMaxMma];            // which accumulator each product goes to (see "accumulator classes" above)
  int res_kb;                      // residual-as-K-extension: after the conv's k-blocks, block_n/64 more k-blocks whose A
                                   // tiles come from the residual tensor (maps.r, at the OUTPUT pixel coordinates, the
                                   // tile's own channel range) and whose B tiles are the identity columns appended to the
                                   // packed weights -- the tensor core performs "+ identity(x)" and the residual rides the
                                   // TMA pipeline (deep prefetch, no epilogue loads).  0 = off.
  int res_kind;                    // 0: identity residual as described; 1: SECOND CONV SOURCE -- res_kb k-blocks of a 1x1
                                   // convolution over another tensor (maps.r, element stride res_stride) whose weights
                                   // are K-concatenated behind the main ones: D = [W | W2] [a ; a2] (projection shortcut
                                   // fused into the last conv of a ResUnit).  All B pieces, the full product list.
  int res_stride;
  int n_mma_res;                   // products issued for a residual k-block: (mma_res_a[i], B piece 0) -> mma_res_acc[i]
  int mma_res_a[kMaxPieces], mma_res_acc[kMaxPieces];
  int stages;                      // smem ring depth
  int frag_epi;                    // 1: the epilogue works on the wgmma register fragments (Epi::run_frag) and no fp32
                                   // accumulator tile is allocated; 0: row epilogue over the shared-memory tile (Epi::run)
  int cl_m, cl_n;                  // thread-block cluster of cl_m x cl_n CTAs (1 or 2 each; plain-GEMM geometry and
                                   // sched 1 only): CTA (ci, cj) of a cluster computes row tile cl_m*Ms+ci, column tile
                                   // cl_n*Ns+cj; the cl_n CTAs sharing a row tile each load 1/cl_n of the A tile and
                                   // TMA-multicast it to the others, likewise the cl_m CTAs sharing a column tile for B.
                                   // Operand traffic from L2 per CTA drops to A/cl_n + B/cl_m.
  int halo;                        // 1: 3x3 / stride 1 / pad 1 convolution with HALO REUSE: tiles are 8 x 16 pixels of one image; per
                                   // 64-channel block ONE (10 x 18)-pixel halo patch is loaded (A ring, `stages` deep) and all
                                   // nine taps read it through descriptors that differ only in their start row (r*10 + s)
                                   // with an 8-row-group stride of 10 rows; the weights stream tap by tap through their own
                                   // ring (`stages_b` deep).  k order: channel block outer, tap inner.  A bytes per tile
                                   // drop 9 x 16 KiB -> 22.5 KiB per block and piece.
  int stages_b;                    // halo mode: depth of the B (weights) ring
  int rowmap_n;                    // > 0: only `rowmap_n` groups of th output rows are computed; tile row index ih maps to
  unsigned char rowmap[32];        // first output row rowmap[ih] (tiles_h == rowmap_n).  Used for the heat-map head when only the
                                   // bilinear support of the FusionLayer's 64 -> 16 resampling is needed (flame_regression.py:33-41)
  int sched;                       // 0: tiles round-robin over CTAs with the column tile fastest (default);
                                   // 1: row-tile persistent -- CTA b owns row tiles b, b+grid, ... and walks ALL column
                                   //    tiles of each (per-row-tile epilogue state is loaded once; all CTAs sweep the
                                   //    B operand in step, so it stays hot in L2)
  int pingpong;                    // 1: PING-PONG consumers (fragment epilogue, block_n = 64, no halo, no cluster, stages >= 2):
                                   // warpgroup w owns whole tiles -- positions w, w + 2, ... of the CTA's sequence -- and
                                   // their main loops take turns, so one warpgroup's epilogue runs under the other's main
                                   // loop (gemm_consumer_pingpong).  0: both warpgroups split every tile by rows.
};

struct GemmMaps {
  CUtensorMap a[kMaxPieces];       // rank-4 (C, W, H, N), box (64, tw*stride, th*stride, tn), swizzle 128B
  CUtensorMap b[kMaxPieces];       // rank-2 (Ktot, Cout_pad), box (64, block_n), swizzle 128B
  CUtensorMap c[kMaxPieces];       // output planes, rank-4 (C, Wo, Ho, N), box (32 ch, 32-pixel sub-box), for TMA stores
  CUtensorMap r[kMaxPieces];       // residual planes, rank-4 (C, Wo, Ho, N), box (64, tw, th, tn)  (res_kb > 0)
};

__host__ __device__ inline int gemm_stage_bytes(const GemmGeom& g) {
  return g.nA * kTileABytes + g.nB * g.block_n * kBlockK * 2;
}
__host__ __device__ inline int gemm_halo_a_stage_bytes(const GemmGeom& g) { return g.nA * kHaloPieceBytes; }
__host__ __device__ inline int gemm_b_stage_bytes(const GemmGeom& g) { return g.nB * g.block_n * kBlockK * 2; }
// shared-memory accumulator tile (row epilogues only): 128 rows of gemm_acc_stride floats, 16-byte chunks XOR-swizzled by
// (row & 7)
__host__ __device__ inline int gemm_acc_stride(const GemmGeom& g) { return (g.block_n + 31) / 32 * 32; }
__host__ __device__ inline int gemm_acc_bytes(const GemmGeom& g) {
  return g.frag_epi ? 0 : kBlockM * gemm_acc_stride(g) * 4;
}
__host__ inline int gemm_fixed_smem_bytes(const GemmGeom& g) {
  return kEpiWarps * kStageOutBytes + gemm_acc_bytes(g) + 1024 /*align slack*/ + 512 /*barriers*/;
}
__host__ inline int gemm_max_stages(const GemmGeom& g) {
  int s = (kGemmSmemLimit - gemm_fixed_smem_bytes(g)) / gemm_stage_bytes(g);
  return s > 8 ? 8 : s;
}
// halo mode: A ring fixed at 2 stages, the rest goes to the weights ring (0 if it does not fit)
__host__ inline int gemm_halo_b_stages(const GemmGeom& g, int a_stages = 2) {
  int s = (kGemmSmemLimit - gemm_fixed_smem_bytes(g) - a_stages * gemm_halo_a_stage_bytes(g)) / gemm_b_stage_bytes(g);
  return s > 8 ? 8 : s;
}
__host__ inline int gemm_smem_bytes(const GemmGeom& g) {
  if (g.halo) return g.stages * gemm_halo_a_stage_bytes(g) + g.stages_b * gemm_b_stage_bytes(g) + gemm_fixed_smem_bytes(g);
  return g.stages * gemm_stage_bytes(g) + gemm_fixed_smem_bytes(g);
}

struct TileCoord {
  int m_tile, n_tile;
  int n0, h0, w0;   // first output image / row / column of the tile
};

__device__ __forceinline__ TileCoord decode_tile(const GemmGeom& g, int m_tile, int n_tile) {
  TileCoord c;
  c.n_tile = n_tile;
  c.m_tile = m_tile;
  int iw = c.m_tile % g.tiles_w;
  int ih = (c.m_tile / g.tiles_w) % g.tiles_h;
  int in = c.m_tile / (g.tiles_w * g.tiles_h);
  c.n0 = in * g.tn;
  c.h0 = g.rowmap_n > 0 ? static_cast<int>(g.rowmap[ih]) : ih * g.th;
  c.w0 = iw * g.tw;
  return c;
}

// The schedule: (row tile m, column tile n) of the i-th tile of CTA `cta` of `grid` (`rank`: its rank in a cluster);
// false when the CTA is out of work.  The producer, the consumers and the host's plan description all enumerate tiles
// through this one function.
__host__ __device__ inline bool gemm_tile_index(const GemmGeom& g, int cta, int grid, int rank, int i, int* m, int* n) {
  const int m_tiles = g.tiles_w * g.tiles_h * g.tiles_n;
  if (g.sched == 0) {
    const int t = cta + i * grid;
    if (t >= m_tiles * g.n_tiles) return false;
    *n = t % g.n_tiles;
    *m = t / g.n_tiles;
  } else if (g.cl_m * g.cl_n == 1) {
    *m = cta + (i / g.n_tiles) * grid;
    if (*m >= m_tiles) return false;
    *n = i % g.n_tiles;
  } else {
    // clusters walk (row super tile, column super tile) in lock step; tiles past the edge ("ghosts") are still processed
    // (zero-filled loads, masked stores) so that every CTA of the cluster performs the same number of pipeline steps
    const int csize = g.cl_m * g.cl_n;
    const int n_super = (g.n_tiles + g.cl_n - 1) / g.cl_n;
    const int m_super = (m_tiles + g.cl_m - 1) / g.cl_m;
    const int ms = cta / csize + (i / n_super) * (grid / csize);
    if (ms >= m_super) return false;
    *m = ms * g.cl_m + rank / g.cl_n;
    *n = (i % n_super) * g.cl_n + rank % g.cl_n;
  }
  return true;
}

// number of tiles CTA `cta` of `grid` processes
__host__ inline int gemm_cta_tiles(const GemmGeom& g, int cta, int grid) {
  int i = 0, m, n;
  while (gemm_tile_index(g, cta, grid, cta % (g.cl_m * g.cl_n), i, &m, &n)) ++i;
  return i;
}

// i-th tile of this CTA under the geometry's schedule; false when the CTA is out of work
__device__ __forceinline__ bool tile_at(const GemmGeom& g, int i, TileCoord* tc) {
  const int rank = g.sched != 0 && g.cl_m * g.cl_n > 1 ? static_cast<int>(ptx::cluster_ctarank()) : 0;
  int m, n;
  if (!gemm_tile_index(g, static_cast<int>(blockIdx.x), static_cast<int>(gridDim.x), rank, i, &m, &n)) return false;
  *tc = decode_tile(g, m, n);
  return true;
}

// Everything a row-epilogue thread needs for one tile.
struct EpiCtx {
  const GemmGeom* g;
  const GemmMaps* maps;
  TileCoord tc;
  int wq;            // row quarter of this warp (0..3): accumulator rows 32*wq .. 32*wq+31
  int grp;           // column group (0/1)
  int lane;
  const float* acc;  // this thread's row of the shared-memory accumulator tile (both accumulator classes summed)
  int swz;           // its 16-byte chunk swizzle (row & 7)
  uint8_t* stage;    // warp-private 4 KiB staging tile (1024-byte aligned)
  int prev_m_tile;   // row tile of the previous tile this CTA processed (-1 for the first)
  mutable int store_seq;   // number of TMA stores this warp has issued (epilogues alternating between two staging tiles)
  // this thread's accumulator row
  int n, h, w;
  bool valid;
  long long pix;     // (n*Ho + h)*Wo + w
  int col0;          // first output column of the tile
  // the warp's 32-row sub-box origin inside the output tensor
  int bw0, bh0, bn0;
};

// N columns [c0, c0+N) of this thread's accumulator row into x[OFF..OFF+N)  (c0 a multiple of 4)
template <int OFF, int N, int M>
__device__ __forceinline__ void epi_load(const EpiCtx& c, int c0, float (&x)[M]) {
  static_assert(OFF + N <= M && N % 4 == 0, "slice out of range");
#pragma unroll
  for (int j = 0; j < N / 4; ++j) {
    const float4 v = *reinterpret_cast<const float4*>(c.acc + ((((c0 >> 2) + j) ^ c.swz) << 2));
    x[OFF + 4 * j] = v.x; x[OFF + 4 * j + 1] = v.y; x[OFF + 4 * j + 2] = v.z; x[OFF + 4 * j + 3] = v.w;
  }
}
// columns [c0, c0+32) of this thread's row
template <int OFF, int N>
__device__ __forceinline__ void epi_load32(const EpiCtx& c, int c0, float (&x)[N]) { epi_load<OFF, 32>(c, c0, x); }
// 16 columns [c0, c0+16) into x[OFF..OFF+15]
template <int OFF, int N>
__device__ __forceinline__ void epi_load16(const EpiCtx& c, int c0, float (&x)[N]) { epi_load<OFF, 16>(c, c0, x); }
// Everything a fragment-epilogue thread needs for one tile: its two accumulator rows r0 = 16*wl + lane/4 (within the
// warpgroup's 64) and r0 + 8, and its warp's 16-row store box.
struct FragCtx {
  const GemmGeom* g;
  const GemmMaps* maps;
  int lane;
  uint8_t* stage;        // warp-private 4 KiB staging area: four 1 KiB store tiles used in turn
  int store_seq;         // number of TMA stores this warp has issued
  long long pix[2];      // (n*Ho + h)*Wo + w of rows r0, r0 + 8
  bool valid[2];
  int col0;              // first output column of the tile
  int bw0, bh0, bn0;     // the warp's 16-row sub-box origin inside the output tensor
};

// 32-column chunks [cb, ce) of the tile that column group grp handles
__device__ __forceinline__ void epi_chunk_range(const GemmGeom& g, int grp, int* cb, int* ce) {
  const int nch = (g.block_n + 31) / 32;          // the last chunk may be 16 columns wide (block_n = 80)
  const int per = (nch + 1) / 2;
  *cb = grp * per;
  *ce = min(nch, *cb + per);
}

// k-steps of one (A piece, B piece) product over a 64-wide k-block into accumulator d (BF16: operand format)
template <int BN, int BF16>
__device__ __forceinline__ void gemm_mma_kblock(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t first) {
#pragma unroll
  for (int k = 0; k < kBlockK / 16; ++k)   // 16 elements (32 B) along K inside the 128 B swizzle row = +2 in (addr >> 4)
    ptx::wgmma_m64k16<BN, BF16>(d, adesc + 2u * k, bdesc + 2u * k, k > 0 ? 1u : first);
}

// One consumer warpgroup (rows 64*wg ..) over all tiles of this CTA: main loop into registers, then the fragment epilogue,
// or the accumulator tile to shared memory and the row epilogue.
template <class Epi, int BN>
__device__ __forceinline__ void gemm_consumer(const GemmMaps& maps, const GemmGeom& g, const typename Epi::Params& ep,
                                              uint8_t* smem, uint8_t* smem_b, float* acc_smem, uint64_t* full_bar,
                                              uint64_t* empty_bar, uint64_t* bfull_bar, uint64_t* bempty_bar, EpiCtx& c,
                                              int wg, int wl, uint16_t mask_peers, uint16_t mask_b, int csize) {
  const int lane = c.lane;
  const int stage_bytes = g.halo ? gemm_halo_a_stage_bytes(g) : gemm_stage_bytes(g);
  const int b_stage_bytes = gemm_b_stage_bytes(g);
  const int num_kb = g.R * g.S * g.cin_blocks;
  const int astride = gemm_acc_stride(g);
  const bool signaller = wl == 0 && lane == 0;     // one arrive per consumer warpgroup on every barrier it releases
  // slot release: every CTA that writes into the slot (multicast peers) waits for both consumer warpgroups of each reader
  auto release = [&](uint64_t* bar, uint16_t mask) {
    if (!signaller) return;
    if (csize == 1) {
      ptx::mbar_arrive(bar);
    } else {
      for (int r = 0; r < csize; ++r)
        if (mask & (1u << r)) ptx::mbar_arrive_cluster(ptx::mapa_u32(bar, static_cast<uint32_t>(r)));
    }
  };
  float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
  FragCtx f;
  f.g = &g;
  f.maps = &maps;
  f.lane = lane;
  f.stage = c.stage;
  f.store_seq = 0;
  typename Epi::State user_state;                // per-thread state that persists across this CTA's tiles
  const int row = c.wq * 32 + lane;
  const int iw = row % g.tw;
  const int ih = (row / g.tw) % g.th;
  const int in = row / (g.tw * g.th);
  const int row0 = c.wq * 32;
  const int biw = row0 % g.tw, bih = (row0 / g.tw) % g.th, bin = row0 / (g.tw * g.th);
  int stage = 0, sbi = 0;
  uint32_t phase = 0, phb = 0;
  const uint32_t a_rows = static_cast<uint32_t>(wg * 64 * kBlockK * 2);     // this warpgroup's rows of an A tile
  for (int ti = 0; tile_at(g, ti, &c.tc); ++ti) {
    uint32_t started = 0;                        // bit a set once accumulator a has received its first MMA
    if (g.halo) {
      // ---- halo mode: per channel block one halo patch, nine taps = nine start rows into it (8-row groups = output rows)
      int pend_b = -1, pend_a = -1;              // slots read by the wgmma group in flight
      for (int cb = 0; cb < g.cin_blocks; ++cb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = ptx::smem_u32(smem + stage * stage_bytes) +
                            static_cast<uint32_t>(wg * 8 * kHaloPW * kBlockK * 2);
        for (int tap = 0; tap < 9; ++tap) {
          ptx::mbar_wait(&bfull_bar[sbi], phb);
          const uint32_t sb = ptx::smem_u32(smem_b + sbi * b_stage_bytes);
          const uint32_t a_off = static_cast<uint32_t>(((tap / 3) * kHaloPW + (tap % 3)) * kBlockK * 2);
          ptx::wgmma_fence();
          for (int i = 0; i < g.n_mma; ++i) {
            const uint64_t adesc = ptx::make_kmajor_sw128_desc_sbo(sa + g.mma_a[i] * kHaloPieceBytes + a_off,
                                                                   kHaloPW * kBlockK * 2);
            const uint64_t bdesc = ptx::make_kmajor_sw128_desc(sb + g.mma_b[i] * g.block_n * kBlockK * 2);
            const uint32_t a_id = static_cast<uint32_t>(g.mma_acc[i]);
            const uint32_t first = (started >> a_id) & 1u;
            started |= 1u << a_id;
            if (a_id) gemm_mma_kblock<BN, Epi::kBf16>(acc1, adesc, bdesc, first);
            else gemm_mma_kblock<BN, Epi::kBf16>(acc0, adesc, bdesc, first);
          }
          ptx::wgmma_commit();
          ptx::wgmma_wait<1>();                  // the previous group has finished reading its slots
          if (pend_b >= 0) release(&bempty_bar[pend_b], mask_b);
          if (pend_a >= 0) release(&empty_bar[pend_a], 1u << (csize > 1 ? ptx::cluster_ctarank() : 0u));
          pend_b = sbi;
          pend_a = tap == 8 ? stage : -1;        // the halo patch may be overwritten once the last tap has read it
          if (++sbi == g.stages_b) { sbi = 0; phb ^= 1u; }
        }
        if (++stage == g.stages) { stage = 0; phase ^= 1u; }
      }
      ptx::wgmma_wait<0>();
      release(&bempty_bar[pend_b], mask_b);
      if (pend_a >= 0) release(&empty_bar[pend_a], 1u << (csize > 1 ? ptx::cluster_ctarank() : 0u));
    } else {
      int pend = -1;
      for (int kb = 0; kb < num_kb + g.res_kb; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = ptx::smem_u32(smem + stage * stage_bytes);
        const uint32_t sb = sa + g.nA * kTileABytes;
        const bool res_block = kb >= num_kb && g.res_kind == 0;    // a second conv source uses the normal product list
        const int n_prod = res_block ? g.n_mma_res : g.n_mma;
        ptx::wgmma_fence();
        for (int i = 0; i < n_prod; ++i) {
          const int pa = res_block ? g.mma_res_a[i] : g.mma_a[i];
          const int pb = res_block ? 0 : g.mma_b[i];
          const uint64_t adesc = ptx::make_kmajor_sw128_desc(sa + pa * kTileABytes + a_rows);
          const uint64_t bdesc = ptx::make_kmajor_sw128_desc(sb + pb * g.block_n * kBlockK * 2);
          const uint32_t a_id = static_cast<uint32_t>(res_block ? g.mma_res_acc[i] : g.mma_acc[i]);
          const uint32_t first = (started >> a_id) & 1u;     // 0: this accumulator's first MMA of the tile overwrites
          started |= 1u << a_id;
          if (a_id) gemm_mma_kblock<BN, Epi::kBf16>(acc1, adesc, bdesc, first);
          else gemm_mma_kblock<BN, Epi::kBf16>(acc0, adesc, bdesc, first);
        }
        ptx::wgmma_commit();
        if (g.stages == 1) {                     // a one-deep ring: the slot is needed back before the next k-block
          ptx::wgmma_wait<0>();
          release(&empty_bar[stage], mask_peers);
        } else {
          ptx::wgmma_wait<1>();                  // the previous k-block's group is complete: its slot may be refilled
          if (pend >= 0) release(&empty_bar[pend], mask_peers);
          pend = stage;
        }
        if (++stage == g.stages) { stage = 0; phase ^= 1u; }
      }
      ptx::wgmma_wait<0>();
      if (pend >= 0) release(&empty_bar[pend], mask_peers);
    }
    ptx::reg_fence(acc0);
    ptx::reg_fence(acc1);
    if constexpr (Epi::kFragment) {
      if (g.frag_epi) {
        const int row0 = wg * 64 + wl * 16;                   // this warp's 16 tile rows
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = row0 + (lane >> 2) + 8 * hr;
          const int n = c.tc.n0 + r / (g.tw * g.th), h = c.tc.h0 + (r / g.tw) % g.th, w = c.tc.w0 + r % g.tw;
          f.valid[hr] = n < g.Nimg && h < g.Ho && w < g.Wo;
          f.pix[hr] = (static_cast<long long>(n) * g.Ho + h) * g.Wo + w;
        }
        f.col0 = c.tc.n_tile * g.block_n;
        f.bw0 = c.tc.w0 + row0 % g.tw;
        f.bh0 = c.tc.h0 + (row0 / g.tw) % g.th;
        f.bn0 = c.tc.n0 + row0 / (g.tw * g.th);
        Epi::template run_frag<BN>(ep, f, acc0, acc1, g.n_acc == 2);
        continue;
      }
    }
    // ---- accumulator tile (this warpgroup's 64 rows) -> shared memory, then the epilogue reads it row by row
    ptx::bar_sync(1 + wg, 128);                  // every thread of the warpgroup is done with the previous tile's rows
    {
      const int r0 = wg * 64 + wl * 16 + (lane >> 2);
      const bool two = g.n_acc == 2;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = r0 + 8 * hr;
          float2 v = make_float2(acc0[4 * j + 2 * hr], acc0[4 * j + 2 * hr + 1]);
          if (two) { v.x += acc1[4 * j + 2 * hr]; v.y += acc1[4 * j + 2 * hr + 1]; }
          *reinterpret_cast<float2*>(acc_smem + r * astride + ((((col >> 2) ^ (r & 7))) << 2) + (col & 3)) = v;
        }
      }
    }
    ptx::bar_sync(1 + wg, 128);
    c.n = c.tc.n0 + in;
    c.h = c.tc.h0 + ih;
    c.w = c.tc.w0 + iw;
    c.valid = (c.n < g.Nimg) && (c.h < g.Ho) && (c.w < g.Wo);
    c.pix = (static_cast<long long>(c.n) * g.Ho + c.h) * g.Wo + c.w;
    c.col0 = c.tc.n_tile * g.block_n;
    c.bw0 = c.tc.w0 + biw;
    c.bh0 = c.tc.h0 + bih;
    c.bn0 = c.tc.n0 + bin;
    Epi::prefetch(ep, c, user_state);
    Epi::run(ep, c, user_state);
    c.prev_m_tile = c.tc.m_tile;
  }
  if (lane == 0) ptx::bulk_wait_read0();         // staging tile must outlive the last TMA store's read
}

// Ping-pong consumer warpgroup wg (GemmGeom::pingpong): tiles wg, wg + 2, ... of this CTA's sequence, each 128 rows x 64
// columns -- per k16 step and product one m64n64k16 per row half (acc*[0]: tile rows 0..63, acc*[1]: 64..127), so every
// output element sees the products, accumulator classes and k order of the cooperative path.  A ring slot holds one
// k-block of one tile and has this one reader (empty_bar counts 1 arrival).  Order barrier: turn_bar[w] completes one
// phase per hand-over to warpgroup w.  A warpgroup waits for its turn before the first wgmma of a tile (tile 0 needs
// none) and hands over right after committing the tile's last k-block, so slots are read in the producer's order and an
// mbarrier wait never meets a phase two laps old; it then drains its groups, releases its last slot and runs the
// epilogue while the other warpgroup's main loop runs.  A warpgroup without a tile never waits, and the last hand-over
// of a CTA is never waited for.
template <class Epi>
__device__ __forceinline__ void gemm_consumer_pingpong(const GemmMaps& maps, const GemmGeom& g, const typename Epi::Params& ep,
                                                       uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                                       uint64_t* turn_bar, uint8_t* stage_out, int wg, int wl, int lane) {
  constexpr int BN = 64;
  const int stage_bytes = gemm_stage_bytes(g);
  const int nkb = g.R * g.S * g.cin_blocks + g.res_kb;
  const int num_kb = g.R * g.S * g.cin_blocks;
  const bool signaller = wl == 0 && lane == 0;
  float acc0[2][BN / 2], acc1[2][BN / 2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc0[h][i] = acc1[h][i] = 0.f;
  FragCtx f;
  f.g = &g;
  f.maps = &maps;
  f.lane = lane;
  f.stage = stage_out;
  f.store_seq = 0;
  TileCoord tc;
  for (int ti = wg; tile_at(g, ti, &tc); ti += 2) {
    const int pos = ti * nkb;                    // ring position of the tile's first k-block (every tile has nkb)
    int stage = pos % g.stages;
    uint32_t phase = static_cast<uint32_t>(pos / g.stages) & 1u;
    if (ti > 0) ptx::mbar_wait(&turn_bar[wg], static_cast<uint32_t>((ti - 1) >> 1) & 1u);
    uint32_t started = 0;
    int pend = -1;
    for (int kb = 0; kb < nkb; ++kb) {
      ptx::mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = ptx::smem_u32(smem + stage * stage_bytes);
      const uint32_t sb = sa + g.nA * kTileABytes;
      const bool res_block = kb >= num_kb && g.res_kind == 0;
      const int n_prod = res_block ? g.n_mma_res : g.n_mma;
      ptx::wgmma_fence();
      for (int i = 0; i < n_prod; ++i) {
        const int pa = res_block ? g.mma_res_a[i] : g.mma_a[i];
        const int pb = res_block ? 0 : g.mma_b[i];
        const uint64_t bdesc = ptx::make_kmajor_sw128_desc(sb + pb * BN * kBlockK * 2);
        const uint32_t a_id = static_cast<uint32_t>(res_block ? g.mma_res_acc[i] : g.mma_acc[i]);
        const uint32_t first = (started >> a_id) & 1u;
        started |= 1u << a_id;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t adesc = ptx::make_kmajor_sw128_desc(sa + pa * kTileABytes + h * 64 * kBlockK * 2);
          if (a_id) gemm_mma_kblock<BN, Epi::kBf16>(acc1[h], adesc, bdesc, first);
          else gemm_mma_kblock<BN, Epi::kBf16>(acc0[h], adesc, bdesc, first);
        }
      }
      ptx::wgmma_commit();
      if (kb == nkb - 1 && signaller) ptx::mbar_arrive(&turn_bar[wg ^ 1]);   // hand over: every k-block is issued
      ptx::wgmma_wait<1>();                      // the previous k-block's group is complete: its slot may be refilled
      if (pend >= 0 && signaller) ptx::mbar_arrive(&empty_bar[pend]);
      pend = stage;
      if (++stage == g.stages) { stage = 0; phase ^= 1u; }
    }
    ptx::wgmma_wait<0>();
    if (signaller) ptx::mbar_arrive(&empty_bar[pend]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      ptx::reg_fence(acc0[h]);
      ptx::reg_fence(acc1[h]);
    }
    f.col0 = tc.n_tile * BN;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row0 = h * 64 + wl * 16;                      // this warp's 16 tile rows of row half h
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = row0 + (lane >> 2) + 8 * hr;
        const int n = tc.n0 + r / (g.tw * g.th), hh = tc.h0 + (r / g.tw) % g.th, w = tc.w0 + r % g.tw;
        f.valid[hr] = n < g.Nimg && hh < g.Ho && w < g.Wo;
        f.pix[hr] = (static_cast<long long>(n) * g.Ho + hh) * g.Wo + w;
      }
      f.bw0 = tc.w0 + row0 % g.tw;
      f.bh0 = tc.h0 + (row0 / g.tw) % g.th;
      f.bn0 = tc.n0 + row0 / (g.tw * g.th);
      Epi::template run_frag<BN>(ep, f, acc0[h], acc1[h], g.n_acc == 2);
    }
  }
  if (lane == 0) ptx::bulk_wait_read0();         // staging tile must outlive the last TMA store's read
}

template <class Epi>
// 12 warps = 3 warpgroups -> 168 registers per thread at launch, redistributed by role (kProducerRegs / kConsumerRegs)
__global__ void __launch_bounds__(kGemmThreads, 1)
tile_gemm_kernel(const __grid_constant__ GemmMaps maps, const GemmGeom g, const typename Epi::Params ep) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atoms (TMA writes and wgmma reads must agree on the pattern).
  // (pointer arithmetic on smem_raw -- not an integer round-trip -- so the compiler keeps the shared address space and
  //  emits LDS/STS instead of generic LD/ST for everything derived from it)
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int stage_bytes = g.halo ? gemm_halo_a_stage_bytes(g) : gemm_stage_bytes(g);
  const int b_stage_bytes = gemm_b_stage_bytes(g);                               // halo mode: the weights ring
  uint8_t* smem_b = smem + g.stages * stage_bytes;                              // [stages_b][nB][block_n x 128 B] (halo mode)
  uint8_t* out_stage = smem_b + (g.halo ? g.stages_b * b_stage_bytes : 0);     // [kEpiWarps][4 KiB]
  float* acc_smem = reinterpret_cast<float*>(out_stage + kEpiWarps * kStageOutBytes);   // [128][gemm_acc_stride]
  uint64_t* bars = reinterpret_cast<uint64_t*>(out_stage + kEpiWarps * kStageOutBytes + gemm_acc_bytes(g));
  uint64_t* full_bar = bars;                     // [stages]
  uint64_t* empty_bar = bars + g.stages;         // [stages]
  uint64_t* bfull_bar = bars + 2 * g.stages;     // [stages_b]   (halo mode)
  uint64_t* bempty_bar = bfull_bar + 8;          // [stages_b]
  uint64_t* turn_bar = bempty_bar + 8;           // [2]          (ping-pong order barrier)

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // provably warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const int num_kb = g.R * g.S * g.cin_blocks;
  const int csize = g.cl_m * g.cl_n;

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < g.nA; ++i) ptx::prefetch_tmap(&maps.a[i]);
    for (int i = 0; i < g.nB; ++i) ptx::prefetch_tmap(&maps.b[i]);
  }
  if (warp == 1 && lane == 0) {
    const int n_peers = g.cl_m + g.cl_n - 1;       // CTAs that read what I multicast == CTAs that multicast to me
    for (int s = 0; s < g.stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], g.pingpong ? 1 : 2 * (g.halo ? 1 : n_peers));   // ping-pong: the tile's warpgroup;
                                      // else both consumer warpgroups of every CTA that reads my slices (halo patches are
                                      // never shared)
    }
    ptx::mbar_init(&turn_bar[0], 1);
    ptx::mbar_init(&turn_bar[1], 1);
    if (g.halo)
      for (int s = 0; s < g.stages_b; ++s) {
        ptx::mbar_init(&bfull_bar[s], 1);
        ptx::mbar_init(&bempty_bar[s], 2 * g.cl_m); // cluster: every CTA that I multicast weight slices to must release the slot
      }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  // ---- cluster bookkeeping (csize == 1: everything below degenerates to the single-CTA protocol)
  const int crank = csize > 1 ? static_cast<int>(ptx::cluster_ctarank()) : 0;
  const int ci = crank / g.cl_n, cj = crank % g.cl_n;
  uint16_t mask_a = 0, mask_b = 0;                 // CTAs sharing my row tile (A) / my column tile (B)
  for (int j = 0; j < g.cl_n; ++j) mask_a |= static_cast<uint16_t>(1u << (ci * g.cl_n + j));
  for (int i = 0; i < g.cl_m; ++i) mask_b |= static_cast<uint16_t>(1u << (i * g.cl_n + cj));
  const uint16_t mask_peers = mask_a | mask_b;     // everyone I exchange operand slices with (including myself)
  if (csize > 1) ptx::cluster_sync_all();          // peers' barriers are initialised before anyone signals them
  // PDL: everything above (barrier init, descriptor prefetch) may overlap the previous kernel's tail; nothing below may
  // touch global memory before the previous grid has fully completed.
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();

  // The register budget changes in the same branch as the role code, so that ptxas allocates each role's code under its
  // own budget.
  if (warp < kFirstEpiWarp) {
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      // ===================================================== TMA producer
      // The WHOLE warp walks the schedule (all control flow and operands stay warp-uniform -> uniform registers); one elected
      // lane issues the TMA instructions.
      if (g.halo) {
        // ---- halo mode: units (tile, channel block) in sequence; the halo patch of unit u+1 is requested while the taps of
        // unit u are still streaming (after its second tap), the nine weight tiles of a unit follow one another
        int sa = 0, sbi = 0;
        uint32_t pha = 0, phb = 0;
        auto issue_a = [&](const TileCoord& t, int cb) {
          ptx::mbar_wait(&empty_bar[sa], pha ^ 1u);
          if (ptx::elect_one_sync()) {
            ptx::mbar_expect_tx(&full_bar[sa], static_cast<uint32_t>(g.nA * kHaloBytes));
            for (int i = 0; i < g.nA; ++i)
              ptx::tma_load_4d(smem + sa * stage_bytes + i * kHaloPieceBytes, &maps.a[i], &full_bar[sa], cb * kBlockK, t.w0 - 1,
                               t.h0 - 1, t.n0);
          }
          __syncwarp();
          if (++sa == g.stages) { sa = 0; pha ^= 1u; }
        };
        int ti = 0, cb = 0;
        TileCoord tc;
        bool valid = tile_at(g, 0, &tc);
        if (valid) issue_a(tc, 0);
        while (valid) {
          int nti = ti, ncb = cb + 1;
          TileCoord ntc = tc;
          bool nvalid = true;
          if (ncb == g.cin_blocks) { ncb = 0; ++nti; nvalid = tile_at(g, nti, &ntc); }
          for (int tap = 0; tap < 9; ++tap) {
            if (tap == 2 && nvalid) issue_a(ntc, ncb);
            ptx::mbar_wait(&bempty_bar[sbi], phb ^ 1u);
            if (ptx::elect_one_sync()) {
              ptx::mbar_expect_tx(&bfull_bar[sbi], static_cast<uint32_t>(b_stage_bytes));
              if (csize == 1) {
                for (int i = 0; i < g.nB; ++i)
                  ptx::tma_load_2d(smem_b + sbi * b_stage_bytes + i * g.block_n * kBlockK * 2, &maps.b[i], &bfull_bar[sbi],
                                   (tap * g.cin_blocks + cb) * kBlockK, tc.n_tile * g.block_n);
              } else {
                // cluster of cl_m row tiles sharing the column tile: I fetch 1/cl_m of the weight rows and multicast them
                const int b_rows = g.block_n / g.cl_m;
                for (int i = 0; i < g.nB; ++i)
                  ptx::tma_load_2d_mc(smem_b + sbi * b_stage_bytes + i * g.block_n * kBlockK * 2 + ci * b_rows * kBlockK * 2,
                                      &maps.b[i], &bfull_bar[sbi], (tap * g.cin_blocks + cb) * kBlockK,
                                      tc.n_tile * g.block_n + ci * b_rows, mask_b);
              }
            }
            __syncwarp();
            if (++sbi == g.stages_b) { sbi = 0; phb ^= 1u; }
          }
          ti = nti; cb = ncb; tc = ntc; valid = nvalid;
        }
      } else {
        int stage = 0;
        uint32_t phase = 0;
        const uint32_t tx_bytes = static_cast<uint32_t>(stage_bytes);
        TileCoord tc;
        for (int ti = 0; tile_at(g, ti, &tc); ++ti) {
          for (int kb = 0; kb < num_kb + g.res_kb; ++kb) {
            if (kb >= num_kb) {                      // extra k-blocks fed from the second tensor (maps.r)
              ptx::mbar_wait(&empty_bar[stage], phase ^ 1u);
              uint8_t* st = smem + stage * stage_bytes;
              const int r = kb - num_kb;
              if (ptx::elect_one_sync()) {
                if (g.res_kind == 0) {
                  // identity residual: A = residual tile (the tile's own channels), B = identity columns (piece 0 only: the
                  // other planes are zero there and are never multiplied)
                  ptx::mbar_expect_tx(&full_bar[stage], static_cast<uint32_t>(g.nA * kTileABytes + g.block_n * kBlockK * 2));
                  const int rc = tc.n_tile * g.block_n + r * kBlockK;
                  for (int i = 0; i < g.nA; ++i)
                    ptx::tma_load_4d(st + i * kTileABytes, &maps.r[i], &full_bar[stage], rc, tc.w0, tc.h0, tc.n0);
                  ptx::tma_load_2d(st + g.nA * kTileABytes, &maps.b[0], &full_bar[stage], num_kb * kBlockK + rc,
                                   tc.n_tile * g.block_n);
                } else {
                  // second 1x1 source: A = 64 channels of the other tensor at (strided) pixel coordinates, B = its weights
                  ptx::mbar_expect_tx(&full_bar[stage], tx_bytes);
                  for (int i = 0; i < g.nA; ++i)
                    ptx::tma_load_4d(st + i * kTileABytes, &maps.r[i], &full_bar[stage], r * kBlockK, tc.w0 * g.res_stride,
                                     tc.h0 * g.res_stride, tc.n0);
                  uint8_t* sb2 = st + g.nA * kTileABytes;
                  for (int i = 0; i < g.nB; ++i)
                    ptx::tma_load_2d(sb2 + i * g.block_n * kBlockK * 2, &maps.b[i], &full_bar[stage], (num_kb + r) * kBlockK,
                                     tc.n_tile * g.block_n);
                }
              }
              __syncwarp();
              if (++stage == g.stages) { stage = 0; phase ^= 1u; }
              continue;
            }
            const int tap = kb / g.cin_blocks;
            const int cb = kb - tap * g.cin_blocks;
            const int r = tap / g.S;
            const int s = tap - r * g.S;
            ptx::mbar_wait(&empty_bar[stage], phase ^ 1u);
            uint8_t* st = smem + stage * stage_bytes;
            const int cw = tc.w0 * g.stride + s - g.pad_w;
            const int ch = tc.h0 * g.stride + r - g.pad_h;
            uint8_t* sb = st + g.nA * kTileABytes;
            const int kcol = kb * kBlockK;
            if (ptx::elect_one_sync()) {
              ptx::mbar_expect_tx(&full_bar[stage], tx_bytes);
              if (csize == 1) {
                for (int i = 0; i < g.nA; ++i)
                  ptx::tma_load_4d(st + i * kTileABytes, &maps.a[i], &full_bar[stage], cb * kBlockK, cw, ch, tc.n0);
                for (int i = 0; i < g.nB; ++i)
                  ptx::tma_load_2d(sb + i * g.block_n * kBlockK * 2, &maps.b[i], &full_bar[stage], kcol,
                                   tc.n_tile * g.block_n);
              } else {
                // my 1/cl_n slice of the A rows and 1/cl_m slice of the B rows, multicast to the CTAs that share them
                const int a_rows = kBlockM / g.cl_n, b_rows = g.block_n / g.cl_m;
                for (int i = 0; i < g.nA; ++i)
                  ptx::tma_load_4d_mc(st + i * kTileABytes + cj * a_rows * kBlockK * 2, &maps.a[i], &full_bar[stage],
                                      cb * kBlockK, cw + cj * a_rows, ch, tc.n0, mask_a);
                for (int i = 0; i < g.nB; ++i)
                  ptx::tma_load_2d_mc(sb + i * g.block_n * kBlockK * 2 + ci * b_rows * kBlockK * 2, &maps.b[i],
                                      &full_bar[stage], kcol, tc.n_tile * g.block_n + ci * b_rows, mask_b);
              }
            }
            __syncwarp();
            if (++stage == g.stages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<kConsumerRegs>();
    // ===================================================== consumer warpgroups: wgmma main loop + epilogue
    const int wg = (warp - kFirstEpiWarp) >> 2;
    const int wl = warp & 3;
    EpiCtx c;
    c.g = &g;
    c.maps = &maps;
    c.wq = 2 * wg + (wl & 1);
    c.grp = wl >> 1;
    c.lane = lane;
    const int row = c.wq * 32 + lane;
    c.acc = acc_smem + row * gemm_acc_stride(g);
    c.swz = row & 7;
    c.stage = out_stage + (warp - kFirstEpiWarp) * kStageOutBytes;
    c.prev_m_tile = -1;
    c.store_seq = 0;
    bool done = false;
    if constexpr (Epi::kFragment) {
      if (g.pingpong) {
        gemm_consumer_pingpong<Epi>(maps, g, ep, smem, full_bar, empty_bar, turn_bar, c.stage, wg, wl, lane);
        done = true;
      }
    }
    if (!done) switch (g.block_n) {
      case 64:
        gemm_consumer<Epi, 64>(maps, g, ep, smem, smem_b, acc_smem, full_bar, empty_bar, bfull_bar, bempty_bar, c, wg, wl,
                               mask_peers, mask_b, csize);
        break;
      case 80:
        gemm_consumer<Epi, 80>(maps, g, ep, smem, smem_b, acc_smem, full_bar, empty_bar, bfull_bar, bempty_bar, c, wg, wl,
                               mask_peers, mask_b, csize);
        break;
      case 96:
        gemm_consumer<Epi, 96>(maps, g, ep, smem, smem_b, acc_smem, full_bar, empty_bar, bfull_bar, bempty_bar, c, wg, wl,
                               mask_peers, mask_b, csize);
        break;
      default:
        gemm_consumer<Epi, 128>(maps, g, ep, smem, smem_b, acc_smem, full_bar, empty_bar, bfull_bar, bempty_bar, c, wg, wl,
                                mask_peers, mask_b, csize);
        break;
    }
  }

  __syncthreads();
  if (csize > 1) ptx::cluster_sync_all();          // nobody leaves while a peer may still write my smem / barriers
}

// =================================================================================================== host side
// Operand pieces and product list of `pieces`-piece operands (1, 2 or 3), smallest terms first so that they are not
// swamped in the fp32 accumulator; with more than one piece every product but p0*p0 goes to accumulator class 1.
__host__ inline void gemm_products(GemmGeom& g, int pieces) {
  static const int pa[3][kMaxMma] = {{0}, {1, 0, 0}, {2, 0, 1, 1, 0, 0}};
  static const int pb[3][kMaxMma] = {{0}, {0, 1, 0}, {0, 2, 1, 0, 1, 0}};
  static const int pc[3][kMaxMma] = {{0}, {1, 1, 0}, {1, 1, 1, 1, 1, 0}};
  g.nA = pieces;
  g.nB = pieces;
  g.n_mma = pieces == 1 ? 1 : pieces == 2 ? 3 : 6;
  g.n_acc = pieces == 1 ? 1 : 2;
  for (int i = 0; i < g.n_mma; ++i) {
    g.mma_a[i] = pa[pieces - 1][i];
    g.mma_b[i] = pb[pieces - 1][i];
    g.mma_acc[i] = pc[pieces - 1][i];
  }
}

// What launches of one tile_gemm_kernel<Epi> remember.  Function attributes and occupancy are per device, so this lives
// in the handle that owns the launches, not in a process-wide static.
struct GemmLaunchCache {
  bool smem_set = false;     // max dynamic shared memory set on the kernel
  int max_clusters[5] = {};  // co-resident clusters, by cluster size cl_m * cl_n (0: not queried yet)
};

// Launch configuration of one launch, without the stream: grid, dynamic shared memory, the cluster attribute and, with
// `pdl`, programmatic dependent launch (`attr` holds two).  At most one CTA per SM: a plain launch runs
// min(work units, #SM) CTAs, where a work unit is a row tile under sched 1 and a tile otherwise; a clustered launch runs
// as many whole clusters as are co-resident, at most one per row super tile.
template <class Epi>
__host__ int gemm_launch_config(const GemmGeom& g, int num_sms, GemmLaunchCache* cache, bool pdl, cudaLaunchConfig_t* cfg,
                                cudaLaunchAttribute* attr) {
  if (!cache->smem_set) {
    DAD3D_CUDA_OK(cudaFuncSetAttribute(tile_gemm_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemmSmemLimit));
    cache->smem_set = true;
  }
  const int m_tiles = g.tiles_w * g.tiles_h * g.tiles_n;
  const int csize = g.cl_m * g.cl_n;
  *cfg = cudaLaunchConfig_t{};
  cfg->blockDim = dim3(kGemmThreads);
  cfg->dynamicSmemBytes = gemm_smem_bytes(g);
  cfg->attrs = attr;
  cfg->numAttrs = 0;
  if (csize > 1) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = csize;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg->numAttrs = 1;
    int& max_clusters = cache->max_clusters[csize];   // GPC packing: can be fewer than #SM / csize
    if (max_clusters == 0) {
      cfg->gridDim = dim3(num_sms / csize * csize);
      DAD3D_CUDA_OK(cudaOccupancyMaxActiveClusters(&max_clusters, tile_gemm_kernel<Epi>, cfg));
      if (max_clusters < 1) { set_error("no co-resident cluster fits"); return DAD3D_ERR_CUDA; }
    }
    const int m_super = ceil_div(m_tiles, g.cl_m);
    cfg->gridDim = dim3((m_super < max_clusters ? m_super : max_clusters) * csize);
  } else {
    const int units = g.sched == 1 ? m_tiles : m_tiles * g.n_tiles;
    cfg->gridDim = dim3(units < num_sms ? units : num_sms);
  }
  if (pdl) {
    attr[cfg->numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[cfg->numAttrs].val.programmaticStreamSerializationAllowed = 1;
    ++cfg->numAttrs;
  }
  return DAD3D_OK;
}

// One launch of tile_gemm_kernel<Epi> on `stream`.
template <class Epi>
__host__ int gemm_launch(const GemmMaps& maps, const GemmGeom& g, const typename Epi::Params& ep, int num_sms,
                         GemmLaunchCache* cache, bool pdl, cudaStream_t stream) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  const int rc = gemm_launch_config<Epi>(g, num_sms, cache, pdl, &cfg, attr);
  if (rc != DAD3D_OK) return rc;
  cfg.stream = stream;
  DAD3D_CUDA_OK(cudaLaunchKernelEx(&cfg, tile_gemm_kernel<Epi>, maps, g, ep));
  count_launch();
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

}  // namespace dad3d
