// DAD-3DNet encoder (FlameRegression.forward, model_training/model/flame_regression.py:87-106) for sm_90a.
// Host side: folded weights -> bf16 piece planes + TMA maps (create), a per-batch-size execution plan with a
// liveness-based workspace layout (plan), and the launch loop (forward).  Device side: tile_gemm.cuh (every conv /
// linear layer as an implicit GEMM on wgmma) + encoder_kernels.cuh (stem, pooling, BiFPN sums, fusion concat, heads).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/dad3d.h"
#include "common.h"
#include "encoder_kernels.cuh"
#include "tmap.h"

using namespace dad3d;

namespace {

constexpr int kImg = 256;
constexpr int kStageUnits[4] = {3, 4, 6, 3};
constexpr int kNumFilters = 256;
constexpr int kHeat = 68;
constexpr int kHeatCat = 128;      // heat-map slot inside the FusionLayer concat (64-channel granularity)
constexpr int kMlpOut = 549;       // 403 + 10 + 136
constexpr float kLimitValue = 3.0f;

struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
template <class T>
using DevPtr = std::unique_ptr<T, CudaFree>;   // device memory, freed with its owner

template <class T>
bool upload(DevPtr<T>* d, const T* h, size_t n) {
  void* p = nullptr;
  if (cudaMalloc(&p, n * sizeof(T)) != cudaSuccess) return false;
  d->reset(static_cast<T*>(p));
  return cudaMemcpy(p, h, n * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess;
}

struct ConvW {
  std::string name;
  int cout = 0, cin = 0, R = 1, S = 1;
  int cout_pad = 0, cin_pad = 0, block_n = 0;
  DevPtr<uint16_t> d_w;         // [P][cout_pad][R*S*cin_pad] bf16 pieces
  DevPtr<float> d_bias;         // [cout_pad]
  DevPtr<float> d_scale;        // [cout_pad] 2^-s per output channel (fp16 pieces: weights are stored as w * 2^s)
  CUtensorMap map_b[kMaxPieces];      // box 64 x block_n
  CUtensorMap map_b64[kMaxPieces];    // box 64 x 64 (small problems: more, narrower tiles to fill the SMs)
  bool has_b64 = false;
  bool has_identity = false;          // identity columns appended after the conv's K columns (residual-as-K-extension)
};

int pick_block_n(int cout) {
  if (cout % 128 == 0) return 128;
  if (cout % 64 == 0) return 64;
  if (cout <= 80) return 80;                  // heat-map head: 68 -> one 80-wide tile (wgmma N % 8 == 0)
  return 96;                                  // 549 -> 6 x 96
}

inline uint16_t host_bf16(float x) {          // round-to-nearest-even fp32 -> bf16
  uint32_t u;
  std::memcpy(&u, &x, 4);
  if ((u & 0x7f800000u) == 0x7f800000u) return static_cast<uint16_t>(u >> 16);
  u += 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(u >> 16);
}
inline uint16_t host_f16(float x) { return __half_as_ushort(__float2half_rn(x)); }   // RN, subnormals kept
inline float host_f16_to_f32(uint16_t b) { return __half2float(__ushort_as_half(b)); }
inline float host_bf16_to_f32(uint16_t b) {
  uint32_t u = static_cast<uint32_t>(b) << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

// ---------------------------------------------------------------------------------------------- plan structures
struct TensorInfo {
  int N = 0, H = 0, W = 0, C = 0;
  bool f32 = false;
  int planes = 1;
  size_t bytes = 0;
  int first = 1 << 30, last = -1;
  size_t off = 0;
  uint8_t* ptr = nullptr;
  std::string name;                 // debug tag (layer that produced it)
  long long plane_elems() const { return static_cast<long long>(N) * H * W * C; }
  // piece plane p lives at ptr + p * plane_elems(), NHWC
  uint16_t* plane(int p) const { return reinterpret_cast<uint16_t*>(ptr) + static_cast<size_t>(p) * plane_elems(); }
  ActView view(int fp16) const { return ActView{plane(0), plane_elems(), planes, C, fp16}; }
  // 4-D (C, W, H, N) tensor map of plane p; box and element strides (nullptr: 1) as make_tmap_16bit takes them.  c_ext /
  // w_ext (when non-zero) replace the two innermost extents while the strides stay those of the tensor: the stem reads
  // overlapping 64-element windows that start at every 16-channel pixel.
  bool nhwc_map(CUtensorMap* m, int p, const uint32_t* box, const uint32_t* es, int swizzle_bytes, uint64_t c_ext = 0,
                uint64_t w_ext = 0) const {
    const uint64_t dims[4] = {c_ext ? c_ext : static_cast<uint64_t>(C), w_ext ? w_ext : static_cast<uint64_t>(W),
                              static_cast<uint64_t>(H), static_cast<uint64_t>(N)};
    const uint64_t strides[3] = {static_cast<uint64_t>(C) * 2, static_cast<uint64_t>(W) * C * 2,
                                 static_cast<uint64_t>(H) * W * C * 2};
    return make_tmap_16bit(m, plane(p), 4, dims, strides, box, es, swizzle_bytes);
  }
};

enum StepKind { kStemConv, kStemS2d, kStemPool, kConv, kFuse, kConcat, kGap, kFinalize, kHeatExport };

// Step::res_mode, how Step::res enters a conv: residual add (on the K axis when the weights have identity columns), gate
// multiply in the epilogue (FusionLayer), second 1x1 source (stride res_stride) whose weights are K-concatenated behind
enum ResMode { kResNone = 0, kResAdd = 1, kResGate = 2, kResSource2 = 4 };
// Step::variant: the step runs always, only when the caller asks for the heat-map, or only when it does not
enum Variant { kAlways = 0, kWithHeatmap = 1, kWithoutHeatmap = 2 };

struct Step {
  StepKind kind;
  // generic tensor slots
  int in = -1, out = -1, res = -1, out_f32 = -1, in2 = -1, in3 = -1;
  // conv
  const ConvW* w = nullptr;
  int stride = 1, pad = 0, relu = 0, res_mode = kResNone, res_stride = 1;
  int up2 = 0;                  // output stored 2x nearest-up-sampled ([N, 2Ho, 2Wo, C])
  int parity = 0;               // 1 + 2a + b: 1x1 conv over the input pixels (2i + a, 2j + b) only, output stored to the same
                                // pixels of the full-resolution tensor; the residual (res) lives on the half-resolution grid
  int variant = kAlways;
  int sparse_rows = 0;          // heat-map head restricted to the output rows the FusionLayer's bilinear resampling reads
  int stem = 0;                 // the stem as a GEMM: input = space-to-depth image, A map = overlapping 4-pixel windows
  GemmMaps maps{};
  GemmGeom geom{};
  EpiConv::Params epi{};
  // fuse
  float fw[3] = {0, 0, 0};
  int nsrc = 0;
};

struct Plan {
  int B = 0;
  void* ws = nullptr;
  size_t ws_bytes = 0;
  std::vector<TensorInfo> tensors;
  std::vector<Step> steps;
  int t_mlp_out = -1, t_heat = -1, t_c4 = -1;
};

// the DAD3D_* switches, read once at dad3d_encoder_create (DESIGN.md 4.4)
struct Switches {
  bool stem_simt = false;          // DAD3D_STEM_SIMT=1: run the stem on the fp32 CUDA-core kernel instead of the tile engine
  bool halo = true;                // halo-reuse tiles for the 3x3 stride-1 layers (DAD3D_HALO=0 selects the per-tap path)
  int halo_cluster = 1;            // DAD3D_HALO_CLUSTER=2: halo layers run as clusters of 2 row tiles that multicast the weights
  bool td_parity = false;          // DAD3D_TD_PARITY=1: large top-down nodes as four parity launches
  bool heat_sparse = true;         // DAD3D_HEAT_SPARSE=0: always compute the full heat-map
  bool pdl = false;                // programmatic dependent launch for the tile-engine kernels (DAD3D_PDL=1 enables)
};

Switches read_switches() {
  auto first = [](const char* name) { const char* e = std::getenv(name); return e ? e[0] : '\0'; };
  Switches sw;
  sw.pdl = first("DAD3D_PDL") == '1';
  sw.halo = first("DAD3D_HALO") != '0';
  sw.halo_cluster = first("DAD3D_HALO_CLUSTER") == '2' ? 2 : 1;
  sw.td_parity = first("DAD3D_TD_PARITY") == '1';
  const char* heat = std::getenv("DAD3D_HEAT_SPARSE");
  sw.heat_sparse = !(heat && std::atoi(heat) == 0);
  sw.stem_simt = first("DAD3D_STEM_SIMT") == '1';
  return sw;
}

}  // namespace

struct dad3d_encoder {
  int device = 0;
  int num_sms = 0;
  int P = 3;                       // pieces per operand
  int fp16 = 0;                    // piece format: 0 = bf16 (1-3 pieces), 1 = fp16 hi/lo (per-channel scaled weights)
  std::map<std::string, ConvW> convs;
  DevPtr<float> d_stem_w;          // [147][64]
  DevPtr<float> d_stem_b;          // [64]
  float bifpn_w[2][20];            // per block: w1 normalised [2][4] then w2 normalised [3][4]
  std::unique_ptr<Plan> plan;
  size_t ws_cache_B = 0, ws_cache_bytes = 0;
  Switches sw;
  GemmLaunchCache gemm_cache;      // the tile engine of this handle's operand format (the only one it launches)
  bool stem_configured = false;    // cudaFuncSetAttribute done on this handle's device
  bool debug_keep_all = false;     // disable buffer reuse so every activation can be read back after a forward
  // live profiling of the dominant kernel (bench.py roofline): CUDA events around every tile_gemm launch
  bool profile = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
  size_t prof_used = 0;
  std::vector<const void*> prof_steps;   // the Step each recorded launch ran (valid while the plan lives)
  double prof_flops = 0.0;         // algorithmic (useful, unpadded, one-product) FLOPs of the recorded launches
  double prof_bytes = 0.0;         // algorithmic HBM bytes of the recorded launches (inputs + weights + outputs once)
};

namespace {

// ---------------------------------------------------------------------------------------------- plan building
// what a conv / linear layer step does besides reading its input; call sites name the fields they set
struct ConvArgs {
  int stride = 1, pad = 0;
  bool relu = false;
  int res = -1;                  // second tensor, entering as res_mode says
  int res_mode = kResNone;
  int res_stride = 1;            // kResSource2: stride of the second source
  bool up2 = false;              // the output is written nearest-up-sampled by 2
  bool f32_out = false;          // an fp32 output ...
  bool pieces_out = true;        // ... and / or the piece planes
  int* f32_id = nullptr;         // receives the fp32 output's tensor id
  int reuse_f32 = -1;            // write the fp32 output into this tensor instead of a new one
  int variant = kAlways;
  bool sparse_rows = false;
};

struct Builder {
  dad3d_encoder* enc;
  Plan* plan;
  int B;

  int tensor(const std::string& name, int N, int H, int W, int C, bool f32 = false) {
    TensorInfo t;
    t.name = name;
    t.N = N; t.H = H; t.W = W; t.C = C; t.f32 = f32;
    t.planes = f32 ? 1 : enc->P;
    t.bytes = align_up(static_cast<size_t>(t.plane_elems()) * (f32 ? 4 : 2) * t.planes, 1024);
    plan->tensors.push_back(t);
    return static_cast<int>(plan->tensors.size()) - 1;
  }
  void touch(int t, int step) {
    if (t < 0) return;
    TensorInfo& ti = plan->tensors[t];
    ti.first = std::min(ti.first, step);
    ti.last = std::max(ti.last, step);
  }
  int push(Step s) {
    const int idx = static_cast<int>(plan->steps.size());
    for (int t : {s.in, s.out, s.res, s.out_f32, s.in2, s.in3}) touch(t, idx);
    plan->steps.push_back(s);
    return idx;
  }
  const ConvW* W(const std::string& name) {
    auto it = enc->convs.find(name);
    return it == enc->convs.end() ? nullptr : &it->second;
  }
  // conv / linear layer; returns the output tensor id (pieces), -1 without piece output
  int conv(const std::string& name, int in, const ConvArgs& a) {
    const ConvW* w = W(name);
    const TensorInfo ti = plan->tensors[in];
    const int Ho = (ti.H + 2 * a.pad - w->R) / a.stride + 1;
    const int Wo = (ti.W + 2 * a.pad - w->S) / a.stride + 1;
    Step s{.kind = kConv, .in = in, .res = a.res, .w = w, .stride = a.stride, .pad = a.pad, .relu = a.relu,
           .res_mode = a.res_mode, .res_stride = a.res_stride, .up2 = a.up2, .variant = a.variant,
           .sparse_rows = a.sparse_rows};
    s.out = a.pieces_out ? tensor(name, ti.N, a.up2 ? 2 * Ho : Ho, a.up2 ? 2 * Wo : Wo, w->cout_pad) : -1;
    if (a.f32_out)
      s.out_f32 = a.reuse_f32 >= 0 ? a.reuse_f32 : tensor(name + (a.pieces_out ? ".f32" : ""), ti.N, Ho, Wo, w->cout_pad, true);
    if (a.f32_id) *a.f32_id = s.out_f32;
    push(s);
    return s.out;
  }
};

void pick_tile(int Wo, int Ho, int* tw, int* th, int* tn) {
  int w = 1;
  while (w < Wo && w < kBlockM) w <<= 1;
  *tw = w;
  int h = 1;
  while (h < Ho && w * h < kBlockM) h <<= 1;
  *th = h;
  *tn = kBlockM / (w * h);
}

// ResNet-50 stage si over x (pytorchcv resnet50: stride on the first 1x1 of the first unit of stages 2..4)
int res_stage(Builder& b, int si, int x) {
  int cur = x;
  for (int ui = 0; ui < kStageUnits[si]; ++ui) {
    const std::string p = "s" + std::to_string(si + 1) + "u" + std::to_string(ui + 1);
    const int stride = (ui == 0 && si != 0) ? 2 : 1;
    int y = b.conv(p + "c1", cur, {.stride = stride, .relu = true});
    y = b.conv(p + "c2", y, {.pad = 1, .relu = true});
    if (ui == 0) {
      // first unit of a stage: the projection shortcut (1x1, stride s, BN) is K-concatenated behind the last 1x1 --
      // out = relu([W3 | Wid] [y ; x_strided] + b3 + bid): one GEMM, the shortcut tensor is never materialised
      cur = b.conv(p + "c3", y, {.relu = true, .res = cur, .res_mode = kResSource2, .res_stride = stride});
    } else {
      cur = b.conv(p + "c3", y, {.relu = true, .res = cur, .res_mode = kResAdd});
    }
  }
  return cur;
}

// one BiFPNBlock (bifpn.py:101-131) over the five levels feat[], which it replaces by its outputs
void bifpn_block(Builder& b, int li, int feat[5]) {
  Plan* plan = b.plan;
  auto fuse = [&](int a, float wa, int s1, float w1, int s2, float w2) {
    const TensorInfo ta = plan->tensors[a];
    const int out = b.tensor("fuse" + std::to_string(plan->steps.size()), ta.N, ta.H, ta.W, ta.C);
    b.push({.kind = kFuse, .in = a, .out = out, .in2 = s1, .in3 = s2, .fw = {wa, w1, w2}, .nsrc = s2 >= 0 ? 3 : 2});
    return out;
  };
  // (w1 [2][4], the top-down fusion scalars, is folded into the weights on the host)
  const float* w2 = &b.enc->bifpn_w[li][8];     // [3][4]
  const std::string p = "b" + std::to_string(li) + "_";
  const int p3x = feat[0], p4x = feat[1], p5x = feat[2], p6x = feat[3], p7x = feat[4];
  const int p7td = p7x;
  // top-down nodes (bifpn.py:111-114): node(w0*a + w1*up(b)) = relu(W0 a + up(W1 b) + shift); the fusion scalars are
  // folded into the two weight sets on the host.  The low-resolution product is stored nearest-up-sampled (every pixel
  // to its 2x2 block) and enters the node's GEMM through identity columns on the K axis, like a ResUnit residual.
  // DAD3D_TD_PARITY=1, maps of >= 32 rows: the up-sampled branch is never materialised -- the node runs as four launches,
  // one per pixel parity (a, b): a stride-2 view of the input starting at (a, b), the half-resolution product as the
  // K-axis residual, and a store to the pixels (2i + a, 2j + b).  Measured slower than the default (one launch over the
  // full map with the 4x-stored branch as residual: P3 node 222 -> 231 us, P4 73 -> 103 us), so it is opt-in.
  auto td_node = [&](const std::string& name, int a, int lower) {
    const TensorInfo ta = plan->tensors[a];
    if (!b.enc->sw.td_parity || ta.H < 32) {
      const int u = b.conv(name + "_u", lower, {.up2 = true});
      return b.conv(name, a, {.relu = true, .res = u, .res_mode = kResAdd});
    }
    const int u = b.conv(name + "_u", lower, {});
    const ConvW* w = b.W(name);
    const int out = b.tensor(name, ta.N, ta.H, ta.W, w->cout_pad);
    for (int ab = 0; ab < 4; ++ab)
      b.push({.kind = kConv, .in = a, .out = out, .res = u, .w = w, .stride = 2, .relu = 1, .res_mode = kResAdd,
              .parity = 1 + ab});
    return out;
  };
  const int p6td = td_node(p + "p6td", p6x, p7td);
  const int p5td = td_node(p + "p5td", p5x, p6td);
  const int p4td = td_node(p + "p4td", p4x, p5td);
  const int p3td = td_node(p + "p3td", p3x, p4td);
  const int p3out = p3td;
  const int p4out = b.conv(p + "p4out", fuse(p4x, w2[0], p4td, w2[4 + 0], p3out, w2[8 + 0]), {.relu = true});
  const int p5out = b.conv(p + "p5out", fuse(p5x, w2[1], p5td, w2[4 + 1], p4out, w2[8 + 1]), {.relu = true});
  const int p6out = b.conv(p + "p6out", fuse(p6x, w2[2], p6td, w2[4 + 2], p5out, w2[8 + 2]), {.relu = true});
  const int p7out = b.conv(p + "p7out", fuse(p7x, w2[3], p7td, w2[4 + 3], p6out, w2[8 + 3]), {.relu = true});
  feat[0] = p3out; feat[1] = p4out; feat[2] = p5out; feat[3] = p6out; feat[4] = p7out;
}

int build_graph(Builder& b) {
  const int B = b.B;
  Plan* plan = b.plan;
  // ---- stem: conv7x7/2 + BN + ReLU (fp32 SIMT) -> maxpool 3x3/2 -> pieces [B,64,64,64]
  const int t_stem = b.tensor("stem_conv", B, kImg / 2, kImg / 2, 64, /*f32=*/b.enc->sw.stem_simt);   // tensor-core stem: piece planes
  if (b.enc->sw.stem_simt) {
    b.push({.kind = kStemConv, .out_f32 = t_stem});
  } else {
    // tensor-core stem: 2x2 space-to-depth (+ piece split) of the image, then a 4x4/1 conv over 12 channels whose four
    // horizontal taps form one 64-element K block (4 k-blocks, K = 256 of which 147 are non-zero)
    const int t_s2d = b.tensor("s2d", B, kImg / 2, kImg / 2 + kS2dPadW, 16);
    b.push({.kind = kStemS2d, .out = t_s2d});
    b.push({.kind = kConv, .in = t_s2d, .out = t_stem, .w = b.W("stem"), .relu = 1, .stem = 1});
  }
  int x = b.tensor("stem", B, kImg / 4, kImg / 4, 64);
  b.push({.kind = kStemPool, .in = t_stem, .out = x});
  // ---- ResNet-50 stages 1..3
  int c_out[4] = {-1, -1, -1, -1};
  for (int si = 0; si < 3; ++si) {
    x = res_stage(b, si, x);
    c_out[si] = x;
  }
  const int c2 = c_out[0], c3 = c_out[1], c4 = c_out[2];
  // ---- BiFPN laterals (bifpn.py:137-145, 152-161)
  int feat[5];
  // P3's lateral conv is normally composed into b0_p3td on the host (its only consumer); a "lat3" record keeps it separate
  feat[0] = b.W("lat3") ? b.conv("lat3", c2, {}) : c2;
  feat[1] = b.conv("lat4", c3, {});
  feat[2] = b.conv("lat5", c4, {});
  feat[3] = b.conv("lat6", c4, {.stride = 2, .pad = 1});
  feat[4] = b.conv("lat7", feat[3], {.stride = 2, .pad = 1, .relu = true});
  for (int li = 0; li < 2; ++li) bifpn_block(b, li, feat);
  // ---- heat-map head (flame_regression.py:22-25): 3x3 conv 256 -> 68 (+bias), kept in fp32
  int t_heat = -1;
  // Two variants of the same layer: the full 64 x 64 map when the caller asks for the heat-map, otherwise only the output
  // rows that FusionLayer's align_corners bilinear 64 -> 16 resampling reads (31 of 64: the rows floor(i * 63 / 15) and the
  // next one) -- env DAD3D_HEAT_SPARSE=0 keeps the full map always.
  const bool heat_sparse = b.enc->sw.heat_sparse;
  b.conv("heat", feat[0], {.pad = 1, .f32_out = true, .pieces_out = false, .f32_id = &t_heat,
                           .variant = heat_sparse ? kWithHeatmap : kAlways});
  if (heat_sparse)
    b.conv("heat", feat[0], {.pad = 1, .f32_out = true, .pieces_out = false, .reuse_f32 = t_heat,
                             .variant = kWithoutHeatmap, .sparse_rows = true});
  plan->t_heat = t_heat;
  // ---- FusionLayer (flame_regression.py:33-42)
  plan->t_c4 = c4;
  const TensorInfo tc4 = plan->tensors[c4];
  const int t_cat = b.tensor("cat", B, tc4.H, tc4.W, 1024 + kHeatCat + kNumFilters);
  b.push({.kind = kConcat, .in = c4, .out = t_cat, .in2 = t_heat, .in3 = feat[2]});
  x = b.conv("fusion", t_cat, {.res = c4, .res_mode = kResGate});
  // ---- stage 4
  x = res_stage(b, 3, x);
  // ---- heads (flame_regression.py:45-59, 96-106): GAP -> [3 x Linear 2048->512 + ReLU] -> block-diagonal second layers
  const TensorInfo tx = plan->tensors[x];
  const int t_gap = b.tensor("gap", 1, 1, B, tx.C);
  b.push({.kind = kGap, .in = x, .out = t_gap});
  const int t_h = b.conv("mlp1", t_gap, {.relu = true});
  int t_out = -1;
  b.conv("mlp2", t_h, {.f32_out = true, .pieces_out = false, .f32_id = &t_out});
  plan->t_mlp_out = t_out;
  b.push({.kind = kFinalize, .in = t_out});
  b.push({.kind = kHeatExport, .in = t_heat});
  return DAD3D_OK;
}

// first-fit offset assignment over live ranges [first, last]
size_t assign_offsets(std::vector<TensorInfo>& ts) {
  std::vector<int> order(ts.size());
  for (size_t i = 0; i < ts.size(); ++i) order[i] = static_cast<int>(i);
  std::sort(order.begin(), order.end(), [&](int a, int b) {
    if (ts[a].first != ts[b].first) return ts[a].first < ts[b].first;
    return ts[a].bytes > ts[b].bytes;
  });
  std::vector<int> placed;
  size_t total = 0;
  for (int id : order) {
    TensorInfo& t = ts[id];
    if (t.last < 0) { t.off = 0; continue; }
    std::vector<std::pair<size_t, size_t>> busy;       // [off, off+bytes) of overlapping-lifetime tensors
    for (int pid : placed) {
      const TensorInfo& p = ts[pid];
      if (p.last < t.first || p.first > t.last) continue;
      busy.emplace_back(p.off, p.off + p.bytes);
    }
    std::sort(busy.begin(), busy.end());
    size_t off = 0;
    for (auto& iv : busy) {
      if (off + t.bytes <= iv.first) break;
      off = std::max(off, iv.second);
    }
    t.off = off;
    total = std::max(total, off + t.bytes);
    placed.push_back(id);
  }
  return total;
}

// the residual rides the K axis: through the weights' identity columns, or as a second 1x1 source
bool res_identity(const Step& s) { return s.res >= 0 && s.res_mode == kResAdd && s.w->has_identity; }
bool res_source2(const Step& s) { return s.res >= 0 && s.res_mode == kResSource2; }

// the operand ring of this handle's pieces at width block_n, before a tile is chosen: asks what shared memory fits
GemmGeom ring_probe(int P, int block_n, int frag_epi) {
  GemmGeom g{};
  g.nA = P; g.nB = P; g.block_n = block_n; g.frag_epi = frag_epi;
  return g;
}

// Every launch decision of one conv step, from shapes and the handle's switches (no pointers), and the checks on them.
// Written in the order of tests/pingpong_model.py::geometry, which restates it for the CPU tests: change both together.
int conv_geometry(const dad3d_encoder* enc, const Plan& plan, const Step& s, GemmGeom* out) {
  const TensorInfo& ti = plan.tensors[s.in];
  const ConvW* w = s.w;
  const int P = enc->P;
  const bool res_in_k = res_identity(s), src2 = res_source2(s);
  const int cin2 = src2 ? plan.tensors[s.res].C : 0;
  if (!s.stem && ti.C + cin2 != w->cin_pad) {
    set_error("layer " + w->name + ": input has " + std::to_string(ti.C) + "+" + std::to_string(cin2) +
              " channels, weights expect " + std::to_string(w->cin_pad));
    return DAD3D_ERR_INVALID;
  }
  GemmGeom g{};
  const int Ho = s.stem ? ti.H : s.parity ? ti.H / 2 : (ti.H + 2 * s.pad - w->R) / s.stride + 1;
  const int Wo = s.stem ? ti.W - kS2dPadW : s.parity ? ti.W / 2 : (ti.W + 2 * s.pad - w->S) / s.stride + 1;
  g.Wo = Wo; g.Ho = Ho; g.Nimg = ti.N;
  g.stride = s.stride;
  g.R = w->R; g.S = w->S; g.pad_h = s.pad; g.pad_w = s.pad;
  if (s.stem) { g.pad_h = 2; g.pad_w = 0; }                                             // 4 vertical taps
  if (s.parity) { g.pad_h = -((s.parity - 1) >> 1); g.pad_w = -((s.parity - 1) & 1); }   // input pixel (2i + a, 2j + b)
  g.cl_m = 1; g.cl_n = 1;
  g.frag_epi = s.out >= 0 ? 1 : 0;                  // piece outputs: fragment epilogue, no shared-memory accumulator tile
  pick_tile(Wo, Ho, &g.tw, &g.th, &g.tn);
  // 3x3 / stride 1 / pad 1 layers: 8 x 16-pixel tiles whose nine taps share one halo patch in shared memory (tile_gemm.cuh
  // "halo mode"); needs a map of at least 8 x 16 pixels and room for two halo patches + a two-deep weights ring (bf16x3
  // at N = 128 has none).  The sparse heat rows use row-pair tiles (2 rows x 64 columns) through the per-tap path.
  const bool halo = enc->sw.halo && !s.stem && w->R == 3 && w->S == 3 && s.stride == 1 && s.pad == 1 &&
                    Wo >= kHaloTW && Ho >= kHaloTH && gemm_halo_b_stages(ring_probe(P, w->block_n, g.frag_epi)) >= 2 &&
                    !s.sparse_rows;
  if (halo) { g.tw = kHaloTW; g.th = kHaloTH; g.tn = 1; }
  g.tiles_w = ceil_div(Wo, g.tw);
  g.tiles_h = ceil_div(Ho, g.th);
  if (s.sparse_rows) {
    // FusionLayer: F.interpolate(heatmap, size=(16, 16), mode="bilinear", align_corners=True) reads source rows
    // y0 = floor(i * (Ho - 1) / 15) and min(y0 + 1, Ho - 1), i = 0..15 (flame_regression.py:33-41)
    g.tw = Wo; g.th = 2; g.tn = 1;
    if (g.tw * g.th != kBlockM) { set_error("sparse heat rows need a 64-pixel-wide map"); return DAD3D_ERR_INVALID; }
    g.tiles_w = 1;
    const int Hd = plan.tensors[plan.t_c4].H;        // the FusionLayer's target height (16)
    g.rowmap_n = 0;
    for (int i = 0; i < Hd && g.rowmap_n < 32; ++i) {
      const float fy = (Hd > 1) ? i * (static_cast<float>(Ho - 1) / static_cast<float>(Hd - 1)) : 0.f;   // as fusion_concat_kernel
      const int y0 = static_cast<int>(fy);
      if (g.rowmap_n == 0 || g.rowmap[g.rowmap_n - 1] != y0) g.rowmap[g.rowmap_n++] = static_cast<unsigned char>(y0);
    }
    g.tiles_h = g.rowmap_n;
  }
  g.tiles_n = ceil_div(ti.N, g.tn);
  // few row tiles (small maps / small batch): halve the tile width so that twice as many CTAs share the work; the
  // full-width tile also needs a two-deep operand ring in shared memory
  const int m_tiles = g.tiles_w * g.tiles_h * g.tiles_n;
  const bool narrow = w->has_b64 && (m_tiles * (w->cout_pad / w->block_n) * 2 <= enc->num_sms ||
                                     gemm_max_stages(ring_probe(P, w->block_n, g.frag_epi)) < 2);
  g.cin_blocks = s.stem ? 1 : ti.C / kBlockK;       // main source (the stem: one 64-element window); a second source adds
  gemm_products(g, P);                              // res_kb blocks below
  // ping-pong consumers (tile_gemm.cuh) on 128 x 64 tiles: fragment-epilogue launches outside halo mode (and so outside
  // clusters) whose 64-wide ring is at least two deep, with more than one product per k-block and at most
  // kPingPongMaxKb k-blocks per tile.  Measured on H100 (profiles/README.md): in fp16x2 at batch 64 every such launch of
  // up to 32 k-blocks ran faster or level, the 3x3 layers of 36 and 72 k-blocks slower; with one product per k-block
  // (bf16, batch 512) ping-pong everywhere was slower, its main loop being bound by the operand bytes that 64-wide
  // tiles raise.
  constexpr int kPingPongMaxKb = 32;
  const int kb64 = w->R * w->S * g.cin_blocks + (res_in_k ? 1 : src2 ? cin2 / kBlockK : 0);   // k-blocks at block_n 64
  g.pingpong = g.frag_epi && !halo && (w->block_n == 64 || w->has_b64) &&
               gemm_max_stages(ring_probe(P, 64, g.frag_epi)) >= 2 && g.n_mma > 1 && kb64 <= kPingPongMaxKb ? 1 : 0;
  g.block_n = narrow || g.pingpong ? 64 : w->block_n;
  g.n_tiles = w->cout_pad / g.block_n;
  if (res_in_k) {                                   // "+ identity(x)" performed by the tensor core
    g.res_kb = g.block_n / kBlockK;
    g.n_mma_res = P;
    for (int i = 0; i < P; ++i) {
      g.mma_res_a[i] = P - 1 - i;                   // smallest piece first
      g.mma_res_acc[i] = (g.n_acc == 2 && g.mma_res_a[i] != 0) ? 1 : 0;
    }
  }
  if (src2) {                                       // projection shortcut as a second K segment
    g.res_kb = cin2 / kBlockK;
    g.res_kind = 1;
    g.res_stride = s.res_stride;
  }
  g.stages = gemm_max_stages(g);
  if (halo) {
    g.halo = 1;
    if (enc->sw.halo_cluster == 2 && g.block_n == 128 && w->has_b64 && m_tiles >= 2 * enc->num_sms) {
      g.cl_m = 2;                                   // two row tiles share every weight tile (each loads half, multicast)
      g.sched = 1;
    }
    g.stages = 2;
    g.stages_b = gemm_halo_b_stages(g);
    if (g.stages_b < 2) { set_error("layer " + w->name + ": halo pipeline does not fit shared memory"); return DAD3D_ERR_INVALID; }
  }
  // (the 80 / 96-wide heads at three pieces fit one operand stage only: the producer then refills behind each k-block)
  if (g.stages < 1) { set_error("layer " + w->name + ": pipeline does not fit shared memory"); return DAD3D_ERR_INVALID; }
  if (s.res >= 0 && !src2 && plan.tensors[s.res].C != w->cout_pad) {
    set_error("layer " + w->name + ": residual channel mismatch");
    return DAD3D_ERR_INVALID;
  }
  if (s.out >= 0 && g.block_n != 64 && g.block_n != 128) {
    set_error("layer " + w->name + ": piece outputs need block_n 64 or 128");
    return DAD3D_ERR_INVALID;
  }
  *out = g;
  return DAD3D_OK;
}

// the tensor maps of one conv step (after conv_geometry): input pieces, weight pieces, residual / second source, outputs
int conv_maps(const dad3d_encoder* enc, const Plan& plan, Step& s) {
  const GemmGeom& g = s.geom;
  const TensorInfo& ti = plan.tensors[s.in];
  const ConvW* w = s.w;
  {
    // stem: row x of the A operand is the 64-element window that starts at padded s2d pixel x (dim 1 advances by one
    // 16-channel pixel = 32 bytes while the window is 128 bytes long: consecutive rows overlap)
    const uint32_t box[4] = {kBlockK, static_cast<uint32_t>(g.halo ? kHaloPW : g.tw * s.stride),
                             static_cast<uint32_t>(g.halo ? kHaloPH : g.th * s.stride), static_cast<uint32_t>(g.tn)};
    const uint32_t es[4] = {1, static_cast<uint32_t>(s.stride), static_cast<uint32_t>(s.stride), 1};
    for (int p = 0; p < enc->P; ++p) {
      if (!ti.nhwc_map(&s.maps.a[p], p, box, es, 128, s.stem ? kBlockK : 0, s.stem ? g.Wo : 0)) return DAD3D_ERR_CUDA;
      s.maps.b[p] = (g.block_n != w->block_n || g.cl_m == 2) ? w->map_b64[p] : w->map_b[p];
    }
  }
  if (res_identity(s) || res_source2(s)) {
    const TensorInfo& tr = plan.tensors[s.res];
    const int rs = res_source2(s) ? s.res_stride : 1;
    const uint32_t box[4] = {kBlockK, static_cast<uint32_t>(g.tw * rs), static_cast<uint32_t>(g.th * rs),
                             static_cast<uint32_t>(g.tn)};
    const uint32_t es[4] = {1, static_cast<uint32_t>(rs), static_cast<uint32_t>(rs), 1};
    for (int p = 0; p < enc->P; ++p)
      if (!tr.nhwc_map(&s.maps.r[p], p, box, es, 128)) return DAD3D_ERR_CUDA;
  }
  if (s.out < 0) return DAD3D_OK;
  const TensorInfo& to = plan.tensors[s.out];
  // per-warp store box: 16 consecutive tile rows = (bw x bh x bn) output pixels x 32 channels (SWIZZLE_64B rows)
  const int nc = 32;
  const int bw = std::min(g.tw, 16);
  const int bh = std::min(g.th, 16 / bw);
  const int bn = 16 / (bw * bh);
  if (s.up2 || s.parity) {
    // [N, 2Ho, 2Wo, C] seen as (C, b, j, a, n*Ho + i): pixel (2i + a, 2j + b); a box with b = a = 1 addresses the
    // sub-grid of one parity, so the same staging tile is stored four times
    const uint64_t C2 = static_cast<uint64_t>(to.C) * 2;
    const uint64_t dims[5] = {static_cast<uint64_t>(to.C), 2, static_cast<uint64_t>(g.Wo), 2,
                              static_cast<uint64_t>(to.N) * g.Ho};
    const uint64_t strides[4] = {C2, 2 * C2, static_cast<uint64_t>(to.W) * C2, 2 * static_cast<uint64_t>(to.W) * C2};
    const uint32_t box[5] = {static_cast<uint32_t>(nc), 1, static_cast<uint32_t>(bw), 1, static_cast<uint32_t>(bh * bn)};
    for (int p = 0; p < to.planes; ++p)
      if (!make_tmap_16bit(&s.maps.c[p], to.plane(p), 5, dims, strides, box, nullptr, nc * 2)) return DAD3D_ERR_CUDA;
    return DAD3D_OK;
  }
  const uint32_t box[4] = {static_cast<uint32_t>(nc), static_cast<uint32_t>(bw), static_cast<uint32_t>(bh),
                           static_cast<uint32_t>(bn)};
  for (int p = 0; p < to.planes; ++p)
    if (!to.nhwc_map(&s.maps.c[p], p, box, nullptr, nc * 2)) return DAD3D_ERR_CUDA;
  return DAD3D_OK;
}

// the epilogue parameters of one conv step
void conv_epilogue(const dad3d_encoder* enc, const Plan& plan, Step& s) {
  EpiConv::Params& ep = s.epi;
  ep.bias = s.w->d_bias.get();
  ep.scale = s.w->d_scale.get();
  ep.relu = s.relu;
  ep.res_mode = (res_identity(s) || res_source2(s)) ? kResNone : s.res_mode;   // a K-axis residual is in the product
  ep.res = s.res >= 0 ? plan.tensors[s.res].view(enc->fp16) : ActView{nullptr, 0, 0, 0, enc->fp16};
  ep.up2 = s.up2;
  ep.parity = s.parity;
  if (s.out >= 0) {
    const TensorInfo& to = plan.tensors[s.out];
    ep.out = to.plane(0);
    ep.out_plane = to.plane_elems();
    ep.out_planes = to.planes;
    ep.ld_out = to.C;
  }
  if (s.out_f32 >= 0) {
    const TensorInfo& to = plan.tensors[s.out_f32];
    ep.out_f32 = reinterpret_cast<float*>(to.ptr);
    ep.ld_f32 = to.C;
  }
}

// the plan of one batch size: the step graph, tensor lifetimes and workspace offsets, then every conv step's launch
int make_plan(dad3d_encoder* enc, int B, void* ws, size_t ws_bytes, bool layout_only, size_t* need) {
  std::unique_ptr<Plan> plan(new Plan());
  plan->B = B;
  Builder b{enc, plan.get(), B};
  int rc = build_graph(b);
  if (rc != DAD3D_OK) return rc;
  if (enc->debug_keep_all)
    for (auto& t : plan->tensors) { t.first = 0; t.last = 1 << 29; }
  const size_t total = assign_offsets(plan->tensors) + 1024;
  if (need) *need = total;
  if (layout_only) return DAD3D_OK;
  if (ws_bytes < total) {
    set_error("encoder workspace too small: need " + std::to_string(total) + " bytes");
    return DAD3D_ERR_INVALID;
  }
  uint8_t* base = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(ws), 1024));
  for (auto& t : plan->tensors) t.ptr = base + t.off;
  plan->ws = ws;
  plan->ws_bytes = ws_bytes;
  for (Step& s : plan->steps) {
    if (s.kind != kConv) continue;
    if ((rc = conv_geometry(enc, *plan, s, &s.geom)) != DAD3D_OK) return rc;
    if ((rc = conv_maps(enc, *plan, s)) != DAD3D_OK) return rc;
    conv_epilogue(enc, *plan, s);
  }
  enc->plan = std::move(plan);
  return DAD3D_OK;
}

double conv_useful_flops(const Step& s) {
  const ConvW* w = s.w;
  const GemmGeom& g = s.geom;
  double cin = w->cin, cout = w->cout;
  if (w->name == "fusion") cin -= 60;                       // zero columns that pad the heat-map slot
  if (w->name == "mlp2") cin /= 3.0;                        // block-diagonal: each output sees one 512-wide block
  if (w->name == "stem") return 2.0 * g.Nimg * g.Ho * g.Wo * cout * 147.0;   // the 7x7x3 taps (the rest of K = 256 is zero)
  double rows = g.Ho;
  if (g.rowmap_n > 0) {                                     // only the rows actually computed count as work done
    rows = 0;
    for (int i = 0; i < g.rowmap_n; ++i)
      for (int r = 0; r < g.th; ++r) rows += (g.rowmap[i] + r < g.Ho) ? 1 : 0;
  }
  return 2.0 * g.Nimg * rows * g.Wo * cout * cin * w->R * w->S;
}

int launch_conv(dad3d_encoder* enc, const Step& s, cudaStream_t stream) {
  std::pair<cudaEvent_t, cudaEvent_t>* ev = nullptr;
  if (enc->profile) {
    if (enc->prof_used == enc->prof_events.size()) {
      cudaEvent_t a, b;
      DAD3D_CUDA_OK(cudaEventCreate(&a));
      DAD3D_CUDA_OK(cudaEventCreate(&b));
      enc->prof_events.emplace_back(a, b);
    }
    if (enc->prof_steps.size() <= enc->prof_used) enc->prof_steps.resize(enc->prof_used + 1);
    enc->prof_steps[enc->prof_used] = &s;
    ev = &enc->prof_events[enc->prof_used++];
    enc->prof_flops += conv_useful_flops(s);
    DAD3D_CUDA_OK(cudaEventRecord(ev->first, stream));
  }
  const int rc = enc->fp16
                     ? gemm_launch<EpiConvH>(s.maps, s.geom, s.epi, enc->num_sms, &enc->gemm_cache, enc->sw.pdl, stream)
                     : gemm_launch<EpiConv>(s.maps, s.geom, s.epi, enc->num_sms, &enc->gemm_cache, enc->sw.pdl, stream);
  if (rc != DAD3D_OK) return rc;
  if (ev) DAD3D_CUDA_OK(cudaEventRecord(ev->second, stream));
  return DAD3D_OK;
}

// one step of the plan, as dad3d_encoder_forward runs it (the single-step test hook runs the same code)
int run_step(dad3d_encoder* enc, const Step& s, const float* images_d, float* params_d, float* landmarks_d, float* heatmap_d,
             cudaStream_t stream) {
  const Plan& plan = *enc->plan;
  const int B = plan.B;
  auto T = [&](int id) -> const TensorInfo& { return plan.tensors[id]; };
  auto view = [&](int id) { return T(id).view(enc->fp16); };
  switch (s.kind) {
    case kStemConv: {
      const TensorInfo& to = T(s.out_f32);
      dim3 grid(ceil_div(to.W, kStemTile), ceil_div(to.H, kStemTile), B);
      if (!enc->stem_configured) {
        DAD3D_CUDA_OK(cudaFuncSetAttribute(stem_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kStemSmemBytes));
        enc->stem_configured = true;
      }
      stem_conv_kernel<<<grid, 256, kStemSmemBytes, stream>>>(images_d, enc->d_stem_w.get(), enc->d_stem_b.get(), kImg, kImg,
                                                 reinterpret_cast<float*>(to.ptr));
      count_launch();
      break;
    }
    case kStemS2d: {
      const TensorInfo& to = T(s.out);
      stem_s2d_kernel<<<dim3(static_cast<unsigned>(ceil_div(to.W, 128)), static_cast<unsigned>(to.H), static_cast<unsigned>(B)),
                        128, 0, stream>>>(
          images_d, B, kImg, kImg, reinterpret_cast<uint16_t*>(to.ptr), to.plane_elems(), to.planes, enc->fp16);
      count_launch();
      break;
    }
    case kStemPool: {
      const TensorInfo& ti = T(s.in);
      const TensorInfo& to = T(s.out);
      ActView pieces{nullptr, 0, 0, 0, enc->fp16};
      if (!ti.f32) pieces = view(s.in);
      const long long total = static_cast<long long>(B) * to.H * to.W * 8;
      DAD3D_REQUIRE(total < (1ll << 31), "pool: batch too large for 32-bit indexing");
      stem_pool_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
          reinterpret_cast<const float*>(ti.ptr), pieces, B, ti.H, ti.W, reinterpret_cast<uint16_t*>(to.ptr),
          to.plane_elems(), to.planes, enc->fp16);
      count_launch();
      break;
    }
    case kConv: {
      if ((s.variant == 1 && !heatmap_d) || (s.variant == 2 && heatmap_d)) break;     // heat-map head: full map / support rows
      int rc = launch_conv(enc, s, stream);
      if (rc != DAD3D_OK) return rc;
      break;
    }
    case kFuse: {
      const TensorInfo& to = T(s.out);
      FuseSrc f0{view(s.in), T(s.in).H, T(s.in).W, s.fw[0]};
      FuseSrc f1{view(s.in2), T(s.in2).H, T(s.in2).W, s.fw[1]};
      FuseSrc f2 = f1;
      if (s.nsrc == 3) f2 = FuseSrc{view(s.in3), T(s.in3).H, T(s.in3).W, s.fw[2]};
      const dim3 fgrid(static_cast<unsigned>(ceil_div(to.W * (to.C / 8), 256)), static_cast<unsigned>(to.H),
                       static_cast<unsigned>(to.N));
      bifpn_fuse_kernel<<<fgrid, 256, 0, stream>>>(
          f0, f1, f2, s.nsrc, to.N, to.H, to.W, to.C, reinterpret_cast<uint16_t*>(to.ptr), to.plane_elems(), to.planes,
          enc->fp16);
      count_launch();
      break;
    }
    case kConcat: {
      const TensorInfo& to = T(s.out);
      const TensorInfo& th = T(s.in2);
      const int cthreads = ceil_div(to.C / 8, 32) * 32;
      DAD3D_REQUIRE(cthreads <= 1024, "concat: too many channels");
      fusion_concat_kernel<<<dim3(static_cast<unsigned>(to.H * to.W), static_cast<unsigned>(to.N)), cthreads, 0, stream>>>(
          view(s.in), T(s.in).C, reinterpret_cast<const float*>(th.ptr), th.H, th.W, th.C, kHeat, kHeatCat, view(s.in3),
          T(s.in3).C, to.N, to.H, to.W, reinterpret_cast<uint16_t*>(to.ptr), to.plane_elems(), to.planes, enc->fp16);
      count_launch();
      break;
    }
    case kGap: {
      const TensorInfo& ti = T(s.in);
      const TensorInfo& to = T(s.out);
      gap_kernel<<<B * (ti.C / 64), 256, 0, stream>>>(view(s.in), B, ti.H * ti.W, ti.C,
                                                           reinterpret_cast<uint16_t*>(to.ptr), to.plane_elems(), to.planes,
                                                           enc->fp16);
      count_launch();
      break;
    }
    case kFinalize: {
      const TensorInfo& ti = T(s.in);
      head_finalize_kernel<<<ceil_div(B * kMlpOut, 256), 256, 0, stream>>>(reinterpret_cast<const float*>(ti.ptr), ti.C, B,
                                                                          kLimitValue, params_d, landmarks_d);
      count_launch();
      break;
    }
    case kHeatExport: {
      if (!heatmap_d) break;
      const TensorInfo& ti = T(s.in);
      const long long total = static_cast<long long>(B) * kHeat * ti.H * ti.W;
      heatmap_export_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
          reinterpret_cast<const float*>(ti.ptr), ti.C, B, ti.H * ti.W, kHeat, heatmap_d);
      count_launch();
      break;
    }
  }
  return DAD3D_OK;
}

// ---------------------------------------------------------------------------------------------- weights
// the SIMT stem's filter on the device: [(c * 7 + r) * 7 + s][64] from [64][7][7][3], and its bias
int upload_stem(dad3d_encoder* enc, const dad3d_conv_weights& L) {
  std::vector<float> w(147 * 64);
  for (int o = 0; o < 64; ++o)
    for (int r = 0; r < 7; ++r)
      for (int s = 0; s < 7; ++s)
        for (int c = 0; c < 3; ++c)
          w[((c * 7 + r) * 7 + s) * 64 + o] = L.weight_h[((static_cast<size_t>(o) * 7 + r) * 7 + s) * 3 + c];
  if (!upload(&enc->d_stem_w, w.data(), w.size()) || !upload(&enc->d_stem_b, L.bias_h, 64)) {
    set_error("stem upload failed");
    return DAD3D_ERR_CUDA;
  }
  return DAD3D_OK;
}

// the stem's 7x7/2 filter [64][7][7][3] re-expressed as 4x4/1 over the 2x2 space-to-depth image, [64][4][64]: K index =
// r * 64 + dx * 16 + (py * 2 + px) * 3 + ch for block row / column offsets r, dx in 0..3 (s2d block oy - 2 + r,
// ox - 2 + dx); the original tap is ky = 2 r + py - 1, kx = 2 dx + px - 1 (zero outside 0..6)
std::vector<float> stem_as_s2d(const float* w7) {
  std::vector<float> w4(static_cast<size_t>(64) * 4 * 64, 0.f);
  for (int o = 0; o < 64; ++o)
    for (int r = 0; r < 4; ++r)
      for (int dx = 0; dx < 4; ++dx)
        for (int py = 0; py < 2; ++py)
          for (int px = 0; px < 2; ++px) {
            const int ky = 2 * r + py - 1, kx = 2 * dx + px - 1;
            if (ky < 0 || ky > 6 || kx < 0 || kx > 6) continue;
            for (int c = 0; c < 3; ++c)
              w4[(static_cast<size_t>(o) * 4 + r) * 64 + dx * 16 + (py * 2 + px) * 3 + c] =
                  w7[((static_cast<size_t>(o) * 7 + ky) * 7 + kx) * 3 + c];
          }
  return w4;
}

// one layer as a tile-engine operand: its shape and padding, the weights as P bf16 / fp16 piece planes
// [P][cout_pad][ktot] (identity columns included) with bias and scales on the device, and its B-operand tensor maps
int pack_conv(const std::string& name, const dad3d_conv_weights& L, int pieces, int fp16, ConvW* cw) {
  cw->name = name;
  cw->cout = L.cout; cw->cin = L.cin; cw->R = L.R; cw->S = L.S;
  cw->block_n = pick_block_n(L.cout);
  cw->cout_pad = ceil_div(L.cout, cw->block_n) * cw->block_n;
  cw->cin_pad = ceil_div(L.cin, kBlockK) * kBlockK;
  // the last 1x1 of a ResUnit ("...c3") gets identity columns appended to its K axis: [W | I] * [a ; residual]
  // (the first unit's c3 carries the projection-shortcut weights in its K axis instead and needs no identity)
  cw->has_identity = name.size() > 4 && L.R == 1 && L.S == 1 &&
                     ((name.compare(name.size() - 2, 2, "c3") == 0 && name.compare(name.size() - 4, 4, "u1c3") != 0) ||
                      name.compare(name.size() - 2, 2, "td") == 0);      // BiFPN top-down nodes add the up-sampled branch
  const size_t ktot_main = static_cast<size_t>(L.R) * L.S * cw->cin_pad;
  const size_t ktot = ktot_main + (cw->has_identity ? cw->cout_pad : 0);
  const size_t plane = static_cast<size_t>(cw->cout_pad) * ktot;
  std::vector<uint16_t> packed(plane * pieces, 0);
  // fp16 pieces: row o is stored as w * 2^s_o with max |w * 2^s_o| <= 2^15 (s_o <= 15 so that the identity entry 2^s_o
  // stays representable); the epilogue multiplies the accumulator by 2^-s_o (exact).  bf16 pieces: s_o = 0.
  std::vector<float> scale(cw->cout_pad, 1.f), up(cw->cout_pad, 1.f);
  if (fp16)
    for (int o = 0; o < L.cout; ++o) {
      float amax = 0.f;
      const float* row = L.weight_h + static_cast<size_t>(o) * L.R * L.S * L.cin;
      for (size_t i = 0; i < static_cast<size_t>(L.R) * L.S * L.cin; ++i) amax = std::max(amax, std::fabs(row[i]));
      int e = 0;
      if (amax > 0.f && std::isfinite(amax)) {
        std::frexp(amax, &e);                       // amax = m * 2^e, m in [0.5, 1)  ->  amax * 2^(15 - e) in [2^14, 2^15)
        e = std::min(15, 15 - e);
        e = std::max(e, -100);
      }
      up[o] = std::ldexp(1.f, e);
      scale[o] = std::ldexp(1.f, -e);
    }
  if (cw->has_identity)
    for (int o = 0; o < cw->cout_pad; ++o)
      packed[static_cast<size_t>(o) * ktot + ktot_main + o] = fp16 ? host_f16(up[o]) : static_cast<uint16_t>(0x3F80);   // piece 0
  for (int o = 0; o < L.cout; ++o)
    for (int t = 0; t < L.R * L.S; ++t)
      for (int c = 0; c < L.cin; ++c) {
        float r = L.weight_h[(static_cast<size_t>(o) * L.R * L.S + t) * L.cin + c] * up[o];
        const size_t idx = static_cast<size_t>(o) * ktot + static_cast<size_t>(t) * cw->cin_pad + c;
        for (int p = 0; p < pieces; ++p) {
          const uint16_t h = fp16 ? host_f16(r) : host_bf16(r);
          packed[p * plane + idx] = h;
          r -= fp16 ? host_f16_to_f32(h) : host_bf16_to_f32(h);
        }
      }
  std::vector<float> bias(cw->cout_pad, 0.f);
  for (int o = 0; o < L.cout; ++o) bias[o] = L.bias_h[o];
  if (!upload(&cw->d_w, packed.data(), packed.size()) || !upload(&cw->d_bias, bias.data(), bias.size()) ||
      !upload(&cw->d_scale, scale.data(), scale.size())) {
    set_error("weight upload failed for " + name);
    return DAD3D_ERR_CUDA;
  }
  // B maps: box 64 x block_n, and 64 x 64 for the 128-wide layers
  const uint64_t dims[2] = {static_cast<uint64_t>(ktot), static_cast<uint64_t>(cw->cout_pad)};
  const uint64_t strides[1] = {static_cast<uint64_t>(ktot) * 2};
  const uint32_t box[2] = {kBlockK, static_cast<uint32_t>(cw->block_n)};
  const uint32_t box64[2] = {kBlockK, 64};
  cw->has_b64 = cw->block_n == 128;
  for (int p = 0; p < pieces; ++p) {
    if (!make_tmap_16bit(&cw->map_b[p], cw->d_w.get() + p * plane, 2, dims, strides, box, nullptr)) return DAD3D_ERR_CUDA;
    if (cw->has_b64 && !make_tmap_16bit(&cw->map_b64[p], cw->d_w.get() + p * plane, 2, dims, strides, box64, nullptr))
      return DAD3D_ERR_CUDA;
  }
  return DAD3D_OK;
}

}  // namespace

// =================================================================================================== C ABI
extern "C" {

int dad3d_encoder_create(dad3d_encoder** out, const dad3d_conv_weights* layers, int32_t n_layers,
                         const float* bifpn_fusion_w_h, int32_t pieces, int32_t operand_format, int32_t device) {
  DAD3D_REQUIRE(out && layers && bifpn_fusion_w_h, "null pointer");
  DAD3D_REQUIRE(pieces >= 1 && pieces <= 3, "pieces must be 1 (one product), 2 (hi/lo, 3 products) or 3 (bf16x3, 6 products)");
  DAD3D_REQUIRE(operand_format == DAD3D_OPERAND_BF16 || (operand_format == DAD3D_OPERAND_FP16 && pieces <= 2),
                "operand_format must be DAD3D_OPERAND_BF16, or DAD3D_OPERAND_FP16 with 1 or 2 pieces");
  DAD3D_CUDA_OK(cudaSetDevice(device));
  cudaDeviceProp prop;
  DAD3D_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("libdad3d requires an sm_90 (Hopper) device");
    return DAD3D_ERR_UNSUPPORTED;
  }
  std::unique_ptr<dad3d_encoder> enc(new dad3d_encoder());
  enc->device = device;
  enc->num_sms = prop.multiProcessorCount;
  enc->P = pieces;
  enc->fp16 = operand_format == DAD3D_OPERAND_FP16 ? 1 : 0;
  std::memcpy(enc->bifpn_w, bifpn_fusion_w_h, sizeof(enc->bifpn_w));
  enc->sw = read_switches();

  std::vector<float> stem_w4;
  for (int li = 0; li < n_layers; ++li) {
    dad3d_conv_weights L = layers[li];
    if (!L.name || !L.weight_h || !L.bias_h || L.cout <= 0 || L.cin <= 0 || L.R <= 0 || L.S <= 0) {
      set_error("invalid layer record " + std::to_string(li));
      return DAD3D_ERR_INVALID;
    }
    const std::string name(L.name);
    if (name == "stem") {
      if (L.cout != 64 || L.cin != 3 || L.R != 7 || L.S != 7) { set_error("stem must be 7x7 3->64"); return DAD3D_ERR_INVALID; }
      const int rc = upload_stem(enc.get(), L);
      if (rc != DAD3D_OK) return rc;
      stem_w4 = stem_as_s2d(L.weight_h);            // the tensor-core stem is packed as a 4x4 conv over 64 channels
      L.weight_h = stem_w4.data();
      L.cin = 64; L.R = 4; L.S = 1;
    }
    ConvW cw;
    const int rc = pack_conv(name, L, pieces, enc->fp16, &cw);
    if (rc != DAD3D_OK) return rc;
    enc->convs[name] = std::move(cw);
  }
  // every layer the graph needs must be present
  std::vector<std::string> need = {"lat4", "lat5", "lat6", "lat7", "heat", "fusion", "mlp1", "mlp2"};
  for (int si = 0; si < 4; ++si)
    for (int ui = 0; ui < kStageUnits[si]; ++ui) {
      const std::string p = "s" + std::to_string(si + 1) + "u" + std::to_string(ui + 1);
      need.push_back(p + "c1"); need.push_back(p + "c2"); need.push_back(p + "c3");
    }
  for (int li = 0; li < 2; ++li)
    for (const char* n : {"p6td", "p5td", "p4td", "p3td", "p6td_u", "p5td_u", "p4td_u", "p3td_u", "p4out", "p5out",
                          "p6out", "p7out"})
      need.push_back("b" + std::to_string(li) + "_" + n);
  for (auto& n : need)
    if (!enc->convs.count(n)) { set_error("missing layer weights: " + n); return DAD3D_ERR_INVALID; }
  if (!enc->d_stem_w) { set_error("missing layer weights: stem"); return DAD3D_ERR_INVALID; }
  *out = enc.release();
  return DAD3D_OK;
}

void dad3d_encoder_destroy(dad3d_encoder* enc) {
  if (!enc) return;
  for (auto& ev : enc->prof_events) {
    cudaEventDestroy(ev.first);
    cudaEventDestroy(ev.second);
  }
  delete enc;
}

size_t dad3d_encoder_workspace_bytes(dad3d_encoder* enc, int32_t B) {
  if (!enc || B <= 0) return 0;
  if (enc->ws_cache_B == static_cast<size_t>(B)) return enc->ws_cache_bytes;
  size_t need = 0;
  if (make_plan(enc, B, nullptr, 0, true, &need) != DAD3D_OK) return 0;
  enc->ws_cache_B = B;
  enc->ws_cache_bytes = need;
  return need;
}

int dad3d_encoder_forward(dad3d_encoder* enc, const float* images_d, int32_t B, float* params_d, float* landmarks_d,
                          float* heatmap_d, void* workspace_d, size_t workspace_bytes, dad3d_stream stream_) {
  DAD3D_REQUIRE(enc, "null handle");
  if (B == 0) return DAD3D_OK;
  DAD3D_REQUIRE(B > 0 && images_d && params_d && landmarks_d && workspace_d, "null pointer / batch");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!enc->plan || enc->plan->B != B || enc->plan->ws != workspace_d || enc->plan->ws_bytes != workspace_bytes) {
    int rc = make_plan(enc, B, workspace_d, workspace_bytes, false, nullptr);
    if (rc != DAD3D_OK) return rc;
  }
  for (const Step& s : enc->plan->steps) {
    int rc = run_step(enc, s, images_d, params_d, landmarks_d, heatmap_d, stream);
    if (rc != DAD3D_OK) return rc;
  }
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

// ---- live kernel timing for bench.py's roofline: events around every tile_gemm_kernel<EpiConv> launch
int dad3d_encoder_set_profile(dad3d_encoder* enc, int32_t on) {
  DAD3D_REQUIRE(enc, "null handle");
  enc->profile = on != 0;
  enc->prof_used = 0;
  enc->prof_flops = 0.0;
  return DAD3D_OK;
}

int dad3d_encoder_profile_read(dad3d_encoder* enc, double* gemm_ms, long long* gemm_launches, double* useful_flops) {
  DAD3D_REQUIRE(enc && gemm_ms && gemm_launches && useful_flops, "null pointer");
  double ms = 0.0;
  for (size_t i = 0; i < enc->prof_used; ++i) {
    DAD3D_CUDA_OK(cudaEventSynchronize(enc->prof_events[i].second));
    float t = 0.f;
    DAD3D_CUDA_OK(cudaEventElapsedTime(&t, enc->prof_events[i].first, enc->prof_events[i].second));
    ms += t;
  }
  *gemm_ms = ms;
  *gemm_launches = static_cast<long long>(enc->prof_used);
  *useful_flops = enc->prof_flops;
  enc->prof_used = 0;
  enc->prof_flops = 0.0;
  return DAD3D_OK;
}

int dad3d_encoder_profile_layer(dad3d_encoder* enc, int32_t index, char* name, int32_t name_cap, double* ms,
                                double* useful_flops, double* algo_bytes, int32_t* info8) {
  DAD3D_REQUIRE(enc && name && name_cap > 0 && ms && useful_flops && algo_bytes && info8, "null pointer");
  DAD3D_REQUIRE(enc->plan, "no forward has run yet");
  if (index < 0 || static_cast<size_t>(index) >= enc->prof_used) return DAD3D_ERR_INVALID;   // end of list (no message)
  const Step& s = *static_cast<const Step*>(enc->prof_steps[index]);
  const GemmGeom& g = s.geom;
  DAD3D_CUDA_OK(cudaEventSynchronize(enc->prof_events[index].second));
  float t = 0.f;
  DAD3D_CUDA_OK(cudaEventElapsedTime(&t, enc->prof_events[index].first, enc->prof_events[index].second));
  *ms = t;
  *useful_flops = conv_useful_flops(s);
  std::snprintf(name, static_cast<size_t>(name_cap), "%s", s.w->name.c_str());
  const Plan& plan = *enc->plan;
  auto bytes_of = [&](int id) -> double {
    if (id < 0) return 0.0;
    const TensorInfo& t = plan.tensors[id];
    const double elems = static_cast<double>(t.N) * t.H * t.W * t.C;
    return t.f32 ? elems * 4.0 : elems * 2.0 * t.planes;
  };
  // every operand once: input map (strided convs read 1/stride^2 of it only for 1x1), residual / second source, weight
  // pieces, outputs
  double in_b = bytes_of(s.in);
  if (s.w->R == 1 && g.stride > 1) in_b /= static_cast<double>(g.stride) * g.stride;
  double res_b = bytes_of(s.res);
  if (g.res_kind == 1 && g.res_stride > 1) res_b /= static_cast<double>(g.res_stride) * g.res_stride;
  const double w_b = static_cast<double>(s.w->cout_pad) * s.w->R * s.w->S * s.w->cin_pad * 2.0 * enc->P;
  *algo_bytes = in_b + res_b + w_b + bytes_of(s.out) + bytes_of(s.out_f32);
  info8[0] = g.Nimg * g.Ho * g.Wo;                       // M: output pixels
  info8[1] = s.w->cin * s.w->R * s.w->S;                 // K (as given, before padding)
  info8[2] = s.w->cout;                                  // N
  info8[3] = g.n_mma;                                    // tensor-core products per MAC
  info8[4] = g.tiles_w * g.tiles_h * g.tiles_n * g.n_tiles;
  info8[5] = g.block_n;
  info8[6] = g.stages;
  info8[7] = g.cin_blocks * g.R * g.S + g.res_kb;        // k-blocks per tile
  return DAD3D_OK;
}

// ---- test hooks: keep every activation alive, read one back as fp32 NHWC (channels padded as stored)
int dad3d_encoder_set_debug(dad3d_encoder* enc, int32_t keep_all) {
  DAD3D_REQUIRE(enc, "null handle");
  enc->debug_keep_all = keep_all != 0;
  enc->plan.reset();
  enc->ws_cache_B = 0;
  return DAD3D_OK;
}

int dad3d_encoder_read_activation(dad3d_encoder* enc, const char* name, float* out_d, size_t capacity_floats,
                                  int32_t* dims4, dad3d_stream stream_) {
  DAD3D_REQUIRE(enc && name && dims4, "null pointer");
  DAD3D_REQUIRE(enc->plan, "no forward has run yet");
  for (const TensorInfo& t : enc->plan->tensors) {
    if (t.name != name) continue;
    dims4[0] = t.N; dims4[1] = t.H; dims4[2] = t.W; dims4[3] = t.C;
    const size_t n = static_cast<size_t>(t.plane_elems());
    if (!out_d) return DAD3D_OK;
    DAD3D_REQUIRE(capacity_floats >= n, "output buffer too small");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (t.f32) {
      DAD3D_CUDA_OK(cudaMemcpyAsync(out_d, t.ptr, n * 4, cudaMemcpyDeviceToDevice, stream));
    } else {
      pieces_to_f32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(t.view(enc->fp16),
                                                                                      static_cast<long long>(n), out_d);
      count_launch();
      DAD3D_CUDA_OK(cudaGetLastError());
    }
    return DAD3D_OK;
  }
  set_error(std::string("no activation named ") + name);
  return DAD3D_ERR_INVALID;
}

int dad3d_encoder_describe_plan(dad3d_encoder* enc, char* buf, size_t cap) {
  DAD3D_REQUIRE(enc && buf, "null pointer");
  DAD3D_REQUIRE(enc->plan, "no forward has run yet");
  static const char* kKinds[] = {"stem_conv", "stem_s2d", "stem_pool", "conv", "fuse", "concat", "gap", "finalize",
                                 "heat_export"};
  const Plan& plan = *enc->plan;
  std::string j = "{\"B\":" + std::to_string(plan.B) + ",\"pieces\":" + std::to_string(enc->P) +
                  ",\"fp16\":" + std::to_string(enc->fp16) + ",\"num_sms\":" + std::to_string(enc->num_sms) + ",\"steps\":[";
  auto num = [&](const char* k, long long v) { j += "\""; j += k; j += "\":" + std::to_string(v) + ","; };
  auto tensor = [&](const char* k, int id) {
    if (id < 0) return;
    const TensorInfo& t = plan.tensors[id];
    j += "\""; j += k;
    j += "\":{\"name\":\"" + t.name + "\",\"N\":" + std::to_string(t.N) + ",\"H\":" + std::to_string(t.H) +
         ",\"W\":" + std::to_string(t.W) + ",\"C\":" + std::to_string(t.C) + ",\"planes\":" + std::to_string(t.planes) +
         ",\"f32\":" + (t.f32 ? "true" : "false") + "},";
  };
  for (size_t i = 0; i < plan.steps.size(); ++i) {
    const Step& s = plan.steps[i];
    j += i ? ",{" : "{";
    j += "\"kind\":\"" + std::string(kKinds[s.kind]) + "\",\"layer\":\"" + (s.w ? s.w->name : std::string()) + "\",";
    num("variant", s.variant);
    tensor("in", s.in); tensor("in2", s.in2); tensor("in3", s.in3); tensor("res", s.res); tensor("out", s.out);
    tensor("out_f32", s.out_f32);
    if (s.kind == kFuse) j += "\"fw\":[" + std::to_string(s.fw[0]) + "," + std::to_string(s.fw[1]) + "," +
                              std::to_string(s.fw[2]) + "],";
    if (s.kind == kConv) {
      const GemmGeom& g = s.geom;
      num("stride", s.stride); num("pad", s.pad); num("relu", s.relu); num("res_mode", s.res_mode); num("stem", s.stem);
      num("R", g.R); num("S", g.S);
      num("tw", g.tw); num("th", g.th); num("tn", g.tn); num("tiles_w", g.tiles_w); num("tiles_h", g.tiles_h);
      num("tiles_n", g.tiles_n); num("block_n", g.block_n); num("n_tiles", g.n_tiles); num("stages", g.stages);
      num("stages_b", g.stages_b); num("halo", g.halo); num("cl_m", g.cl_m); num("cl_n", g.cl_n); num("sched", g.sched);
      num("frag_epi", g.frag_epi); num("res_kb", g.res_kb); num("res_kind", g.res_kind); num("res_stride", g.res_stride);
      num("up2", s.up2); num("parity", s.parity); num("rowmap_n", g.rowmap_n); num("n_mma", g.n_mma); num("n_acc", g.n_acc);
      num("cout", s.w->cout); num("cin", s.w->cin); num("has_identity", s.w->has_identity ? 1 : 0);
      cudaLaunchConfig_t cfg;
      cudaLaunchAttribute attr[2];
      const int rc = enc->fp16 ? gemm_launch_config<EpiConvH>(g, enc->num_sms, &enc->gemm_cache, enc->sw.pdl, &cfg, attr)
                               : gemm_launch_config<EpiConv>(g, enc->num_sms, &enc->gemm_cache, enc->sw.pdl, &cfg, attr);
      if (rc != DAD3D_OK) return rc;
      const int grid = static_cast<int>(cfg.gridDim.x);
      int tmin = 1 << 30, tmax = 0;
      for (int b = 0; b < grid; ++b) {
        const int t = gemm_cta_tiles(g, b, grid);
        tmin = std::min(tmin, t);
        tmax = std::max(tmax, t);
      }
      num("pingpong", g.pingpong); num("grid", grid); num("cta_tiles_min", tmin); num("cta_tiles_max", tmax);
      j += "\"rowmap\":[";
      for (int r = 0; r < g.rowmap_n; ++r) j += (r ? "," : "") + std::to_string(g.rowmap[r]);
      j += "],";
    }
    j.back() = '}';
  }
  j += "]}";
  if (j.size() + 1 > cap) {
    set_error("plan description needs " + std::to_string(j.size() + 1) + " bytes");
    return DAD3D_ERR_INVALID;
  }
  std::memcpy(buf, j.c_str(), j.size() + 1);
  return DAD3D_OK;
}

int dad3d_encoder_write_activation(dad3d_encoder* enc, const char* name, const float* src_d, size_t n, dad3d_stream stream_) {
  DAD3D_REQUIRE(enc && name && src_d, "null pointer");
  DAD3D_REQUIRE(enc->plan && enc->plan->ws, "no forward has run yet");
  // without keep_all, tensors whose lifetimes do not overlap share workspace: a write would clobber live activations
  DAD3D_REQUIRE(enc->debug_keep_all, "write_activation needs dad3d_encoder_set_debug(enc, 1)");
  for (const TensorInfo& t : enc->plan->tensors) {
    if (t.name != name) continue;
    const size_t elems = static_cast<size_t>(t.plane_elems());
    DAD3D_REQUIRE(n == elems, "write_activation: element count does not match the tensor");
    DAD3D_REQUIRE(t.ptr, "write_activation: tensor has no storage");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (t.f32) {
      DAD3D_CUDA_OK(cudaMemcpyAsync(t.ptr, src_d, n * 4, cudaMemcpyDeviceToDevice, stream));
    } else {
      DAD3D_REQUIRE(t.C % 8 == 0, "write_activation: channel count not a multiple of 8");
      const long long n8 = static_cast<long long>(n / 8);
      f32_to_pieces_kernel<<<static_cast<unsigned>((n8 + 255) / 256), 256, 0, stream>>>(
          src_d, n8, reinterpret_cast<uint16_t*>(t.ptr), t.plane_elems(), t.planes, enc->fp16);
      count_launch();
      DAD3D_CUDA_OK(cudaGetLastError());
    }
    return DAD3D_OK;
  }
  set_error(std::string("no activation named ") + name);
  return DAD3D_ERR_INVALID;
}

int dad3d_encoder_run_steps(dad3d_encoder* enc, int32_t first, int32_t count, const float* images_d, float* params_d,
                            float* landmarks_d, float* heatmap_d, dad3d_stream stream_) {
  DAD3D_REQUIRE(enc, "null handle");
  DAD3D_REQUIRE(enc->plan && enc->plan->ws, "no plan: run a forward at this batch size and workspace first");
  const int n = static_cast<int>(enc->plan->steps.size());
  DAD3D_REQUIRE(first >= 0 && count >= 0 && first + count <= n, "step range outside the plan");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  for (int i = first; i < first + count; ++i) {
    const Step& s = enc->plan->steps[i];
    DAD3D_REQUIRE(images_d || (s.kind != kStemConv && s.kind != kStemS2d), "this step reads the images");
    DAD3D_REQUIRE((params_d && landmarks_d) || s.kind != kFinalize, "this step writes params and landmarks");
    int rc = run_step(enc, s, images_d, params_d, landmarks_d, heatmap_d, stream);
    if (rc != DAD3D_OK) return rc;
  }
  DAD3D_CUDA_OK(cudaGetLastError());
  return DAD3D_OK;
}

int dad3d_encoder_num_layers(const dad3d_encoder* enc) { return enc ? static_cast<int>(enc->convs.size()) : 0; }   // "stem" is in convs too

}  // extern "C"
