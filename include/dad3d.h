/* libdad3d.so -- C ABI of the H100-native DAD-3DNet image->3D-head hot path.
 *
 * The reference (PinataFarms/DAD-3DHeads) has no FFI seam: its "operator interface" for this path is three Python
 * objects (SURVEY.md §8b).  Each entry point below names the reference call it replaces (file:line under
 * /root/reference); INTEGRATION.md shows the ctypes stub a reference maintainer would add.
 *
 * Conventions: plain C, no torch types.  Pointers suffixed _h are HOST pointers (read during the call only), _d are
 * DEVICE pointers owned by the caller.  Every compute call is asynchronous on the given CUDA stream.  Return value
 * 0 = OK, negative = error (text via dad3d_last_error(), thread-local).  Handles are opaque, created/destroyed
 * explicitly; one handle may be used by one host thread at a time.  Nothing here ever falls back to the CPU.
 */
#ifndef DAD3D_H_
#define DAD3D_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define DAD3D_API __attribute__((visibility("default")))
#else
#define DAD3D_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* dad3d_stream;      /* == cudaStream_t / CUstream */
typedef struct dad3d_flame dad3d_flame;
typedef struct dad3d_encoder dad3d_encoder;

#define DAD3D_OK 0
#define DAD3D_ERR_INVALID (-1)
#define DAD3D_ERR_CUDA (-2)
#define DAD3D_ERR_UNSUPPORTED (-3)

#define DAD3D_DECODE_CLUSTER 32 /* A/B aid: fused decode as 2x2 thread-block clusters with TMA multicast of both operands
                                  (off by default) */

/* Widths of the fields of the 3DMM parameter vector, sliced in the reference's hard-coded order
 * shape, expression, jaw, rotation, eyeballs, neck, translation, scale
 * (model_training/model/flame.py:41-84 FlameParams.from_3dmm; dad_3dnet.yaml:5-12 gives 300/100/3/6/0/0/3/1 = 413). */
typedef struct dad3d_flame_layout {
  int32_t shape, expression, jaw, rotation, eyeballs, neck, translation, scale;
} dad3d_flame_layout;

/* decode flags */
#define DAD3D_ZERO_ROT 1        /* FLAMELayer.forward(zero_rot=True)   flame.py:225 */
#define DAD3D_ZERO_JAW 2        /* FLAMELayer.forward(zero_jaw=True)   flame.py:206 */
#define DAD3D_BLEND_FAST 4      /* (old name of today's default; accepted, no effect) */
#define DAD3D_BLEND_HILO 64     /* blend-shape product with fp16 hi/lo split operands (3 tensor-core products, 22-bit, vertices
                                   relL2 2e-7 vs fp64) through the generic tile engine.  DEFAULT (flag absent): ONE fp16 product
                                   (11-bit operand mantissa like TF32, template exact to 22 bits; vertices relL2 1.5e-5, inside
                                   the 1e-4 contract) in the dedicated decode kernel (csrc/flame_decode.cuh) */
#define DAD3D_DECODE_PAIR 128   /* accepted, no effect: CTA pairs need a two-CTA MMA, which sm_90 lacks */
#define DAD3D_BLEND_SIMT 8      /* verification aid: blend-shape product on CUDA cores in fp32 (slow) */
#define DAD3D_DECODE_UNFUSED 16 /* A/B aid: tensor-core blend product to a v_posed scratch + separate skinning kernel
                                   (default: skinning / rotation / projection fused into the GEMM epilogue) */

DAD3D_API const char* dad3d_last_error(void);
DAD3D_API int dad3d_version(void);

/* ---- FLAME head decoder -------------------------------------------------------------------------------------------
 * dad3d_flame_create  replaces FLAMELayer.__init__ (model_training/model/flame.py:124-180): takes the fp32 constants
 *   the reference registers as buffers and packs them for the GPU (fp16 hi/lo basis planes, folded joint regressor).
 *   shapedirs_h [n_vertices*3, n_betas] (i.e. [V,3,400] row-major), posedirs_h [(n_joints-1)*9, n_vertices*3],
 *   v_template_h [n_vertices*3], j_regressor_h [n_joints, n_vertices], parents_h [n_joints] (parents[0] = -1),
 *   lbs_weights_h [n_vertices, n_joints].  n_joints must be 5 (FLAME: global, neck, jaw, eye, eye), n_betas 400. */
DAD3D_API int dad3d_flame_create(dad3d_flame** out, const float* shapedirs_h, const float* posedirs_h, const float* v_template_h,
                       const float* j_regressor_h, const int32_t* parents_h, const float* lbs_weights_h,
                       int32_t n_vertices, int32_t n_betas, int32_t n_joints, const dad3d_flame_layout* layout,
                       int32_t device);
DAD3D_API void dad3d_flame_destroy(dad3d_flame* h);
DAD3D_API int32_t dad3d_flame_num_params(const dad3d_flame* h);      /* 413 for the released layout */
DAD3D_API int32_t dad3d_flame_num_vertices(const dad3d_flame* h);
/* scratch the decode needs for a batch of B heads (decode streams internally in chunks, so this saturates) */
DAD3D_API size_t dad3d_flame_workspace_bytes(const dad3d_flame* h, int32_t B);

/* dad3d_flame_decode  replaces HeadMesh.vertices_3d + HeadMesh.reprojected_vertices
 *   (model_training/head_mesh.py:28-46 -> FLAMELayer.forward flame.py:182-229 -> smplx.lbs.lbs) in ONE pass:
 *   params_d   [B, num_params] fp32 row-major (not modified -- the reference's in-place zeroing of translation z,
 *              head_mesh.py:41, is reproduced by the Python wrapper, not here)
 *   vertices3d_d  [B, V, 3] fp32 or NULL : rotated model-space mesh (vertices_3d, zero_rot per flags)
 *   projected_d   [B, V, 2] (to_2d != 0) or [B, V, 3] fp32 or NULL : ((v*max(s+1,1e-8) + [tx,ty,0]) + 1)/2*image_size
 *                 (always uses the 6-DoF rotation, as reprojected_vertices does, unless DAD3D_ZERO_ROT is set) */
DAD3D_API int dad3d_flame_decode(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, float* vertices3d_d,
                       float* projected_d, float image_size, int32_t to_2d, void* workspace_d, size_t workspace_bytes,
                       dad3d_stream stream);

/* test hooks: the two stages of every decode pass, run alone on caller buffers (dad3d_flame_decode runs each pass as
 * dad3d_flame_prep followed by dad3d_flame_decode_from, 2 kernel launches on the fused paths and 3 on the others)
 *   dad3d_flame_prep   flame_prep_kernel alone: coef_hi_d / coef_lo_d [dec_rows_padded(B) = B rounded up to 256, 448] fp16
 *                      hi/lo coefficient rows (row order permuted for the dedicated kernel when permute != 0; padding rows
 *                      are not written), xf_d [B, 68] fp32 per-head transform records
 *   dad3d_flame_decode_from  the product + skinning + projection stage `flags` selects, on caller-written rows and records:
 *                      the dedicated kernel expects permuted rows (and reads all dec_rows_padded(B) of them), the other paths
 *                      unpermuted rows.  B must fit one pass of the path (fused_chunk or 4096 heads, see describe), else
 *                      DAD3D_ERR_INVALID.  The unfused and SIMT paths need dad3d_flame_workspace_bytes(h, B) of workspace
 *                      (v_posed scratch); the fused paths ignore it
 *   dad3d_flame_describe  NUL-terminated JSON: basis_scale, jaw_only, nv, npad, fused_chunk, num_sms and, for every pass of a
 *                      decode of B heads with `flags`, the path ("dedicated", "lbs", "blend", "simt"), rows, m_units (row
 *                      tiles), splits (vertex-tile ranges per row tile), grid (CTAs of the product kernel), stages and
 *                      clustered -- computed by the code the launches use */
DAD3D_API int dad3d_flame_prep(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, void* coef_hi_d, void* coef_lo_d,
                               float* xf_d, int32_t permute, dad3d_stream stream);
DAD3D_API int dad3d_flame_decode_from(dad3d_flame* h, const void* coef_hi_d, const void* coef_lo_d, const float* xf_d, int32_t B,
                                      int32_t flags, float* vertices3d_d, float* projected_d, float image_size, int32_t to_2d,
                                      void* workspace_d, size_t workspace_bytes, dad3d_stream stream);
DAD3D_API int dad3d_flame_describe(dad3d_flame* h, int32_t B, int32_t flags, char* json, size_t cap);

/* dad3d_gather_landmarks  replaces np.take(projected_vertices, indices, axis=0) (demo_utils.py:37-47) and
 *   FLAMELayer.indices_2d style subset selection: out[b,l,:] = src[b, idx[l], :].  ncomp = 2 or 3. */
/* Backward of dad3d_flame_decode (SURVEY §8f row 3): grad_params_d [B, num_params] = d L / d params given
 * grad_vertices_d [B,V,3] = dL/d(vertices3d) and / or grad_projected_d [B,V,2|3] = dL/d(projected) (either may be NULL).
 * What autograd gives the reference when its losses call HeadMesh.vertices_3d / reprojected_vertices
 * (losses/vertices_3d_loss.py:30-47, losses/reprojection_loss.py:22-46, train/flame_lightning_model.py:329-351).  The dense
 * part (d beta, d pose features) is a wgmma GEMM over the transposed basis; layouts without neck / eyeball pose only. */
DAD3D_API size_t dad3d_flame_backward_workspace_bytes(const dad3d_flame* h, int32_t B);
DAD3D_API int dad3d_flame_backward(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, const float* grad_vertices_d,
                                   const float* grad_projected_d, float image_size, int32_t to_2d, float* grad_params_d,
                                   void* workspace_d, size_t workspace_bytes, dad3d_stream stream);

/* test hooks: the stages of every backward pass, run alone on caller buffers.  dad3d_flame_backward runs each pass of up to
 * 4096 heads as flame_prep_kernel (dad3d_flame_prep, permute = 0), then blend, vertex, dense and finalize below; each hook
 * takes 1 <= B <= 4096 heads (else DAD3D_ERR_INVALID).  npad = dad3d_flame_describe's npad (3 V rounded up to 128).
 *   dad3d_flame_backward_blend     the recomputed forward blend product: coef_hi_d / coef_lo_d [B rounded up to 256, 448] fp16
 *                      unpermuted prep rows -> vposed_d [B, npad] fp32 = v_posed * basis_scale, x,y,z interleaved (columns
 *                      3 V .. npad - 1 are written with the product of the zero basis rows); vposed_d 16-byte aligned
 *   dad3d_flame_backward_vertex    vposed_d [B, npad] fp32, xf_d [B, 68] fp32 transform records (dad3d_flame_prep), the
 *                      incoming gradients as in dad3d_flame_backward (either may be NULL, not both) ->
 *                      sigma_d [B] fp32: the power of two that lifts the head's max |gV + (image/2) sc gP| into [512, 1024),
 *                        its exponent capped so that sigma * basis_scale <= 2^127; 1 for an all-zero or non-finite maximum;
 *                      d_hi_d / d_lo_d [B, npad] fp16: fp16 RN hi / lo split of dp * sigma * basis_scale, where
 *                        dp = (w_rest A0'^T + w_jaw A2'^T) g per vertex coordinate; columns 3 V .. npad - 1 are zero;
 *                      partial_d [B, ceil(V / 256), 32] fp32: per 256-vertex block, the block's sums of the cotangents
 *                        G_A0'[9] g_t0[3] G_A2'[9] g_t2[3] g_c[3] d_sc d_tx d_ty (floats 30, 31 are not written)
 *   dad3d_flame_backward_dense     d_hi_d / d_lo_d [B, npad] fp16 -> dcoef_d [B, 448] fp32 = (hi hi + (lo hi + hi lo)) over
 *                      the transposed hi / lo basis planes (columns 0..399 betas, 400..435 pose features, the rest unused);
 *                      dcoef_d 16-byte aligned (the epilogue stores float4)
 *   dad3d_flame_backward_finalize  params_d [B, num_params], flags (DAD3D_ZERO_ROT / DAD3D_ZERO_JAW), dcoef_d, partial_d,
 *                      sigma_d as above -> grad_params_d [B, num_params]: every entry of the released layout is written
 *                      (translation z and the flagged entries as 0).  Non-finite incoming gradients may propagate to their
 *                      own head's gradients; other heads are not affected. */
DAD3D_API int dad3d_flame_backward_blend(dad3d_flame* h, const void* coef_hi_d, const void* coef_lo_d, int32_t B, float* vposed_d,
                                         dad3d_stream stream);
DAD3D_API int dad3d_flame_backward_vertex(dad3d_flame* h, const float* vposed_d, const float* xf_d, const float* grad_vertices_d,
                                          const float* grad_projected_d, int32_t B, float image_size, int32_t to_2d,
                                          float* sigma_d, void* d_hi_d, void* d_lo_d, float* partial_d, dad3d_stream stream);
DAD3D_API int dad3d_flame_backward_dense(dad3d_flame* h, const void* d_hi_d, const void* d_lo_d, int32_t B, float* dcoef_d,
                                         dad3d_stream stream);
DAD3D_API int dad3d_flame_backward_finalize(dad3d_flame* h, const float* params_d, int32_t B, int32_t flags, const float* dcoef_d,
                                            const float* partial_d, const float* sigma_d, float* grad_params_d,
                                            dad3d_stream stream);

DAD3D_API int dad3d_gather_landmarks(const float* src_d, int32_t B, int32_t n_vertices, int32_t ncomp, const int32_t* idx_d,
                           int32_t L, float* out_d, dad3d_stream stream);
/* barycentric variant (model_training/data/utils.py:120-206 get_68_landmarks): out[b,l,:] = sum_k bary[l,k]*src[b,tri[l,k],:] */
DAD3D_API int dad3d_gather_landmarks_bary(const float* src_d, int32_t B, int32_t n_vertices, int32_t ncomp,
                                const int32_t* tri_idx_d, const float* bary_d, int32_t L, float* out_d,
                                dad3d_stream stream);

/* ---- DAD-3DNet encoder ---------------------------------------------------------------------------------------------
 * Replaces the TorchScript module the reference's predictor runs (predictor.py:72,97-100), i.e.
 * FlameRegression.forward (model_training/model/flame_regression.py:87-106): pytorchcv ResNet-50 stages -> BiFPN(256) ->
 * heat-map head -> FusionLayer -> stage 4 -> three MLP heads.
 *
 * Weights arrive BN-folded, one record per GEMM-able layer, fp32, laid out [cout][R][S][cin] (channels-last taps).
 * Layer names (the folding itself is host-side Python, dad_3dheads_b200/encoder.py, from the reference's state_dict):
 *   "stem" (7x7 3->64)                       encoder.model.init_block.conv
 *   "s{1..4}u{k}c{1,2,3}"                    encoder.model.stage{i}.unit{k}.body.conv{1,2,3}; the first unit's c3 carries
 *                                            the projection shortcut K-concatenated: [W3 | W_identity_conv], bias b3 + bid
 *   "lat4".."lat7" (+ optional "lat3")      bifpn.p4 .. bifpn.p7; bifpn.p3 is normally composed into "b0_p3td" (its only
 *                                            consumer: (W_node W_p3) c2 + W_node b_p3), a "lat3" record keeps it separate
 *   "b{0,1}_{p4out,p5out,p6out,p7out}"       bifpn.bifpn.{0,1}.<node> (depthwise scale, pointwise, BN folded)
 *   "b{0,1}_{p6td,p5td,p4td,p3td}" and "..._u"   top-down nodes split in two: W*(w0 a) at the node's resolution and
 *                                            W*(w1 b) at the lower one (fusion scalars folded in; the second has no bias)
 *   "heat"                                   head.heatmap (3x3 256->68 + bias)
 *   "fusion"                                 fusion_layer.conv1x1 with K laid out [x 1024 | heat 68 + 60 zero | p5 256]
 *   "mlp1" (2048 -> 3x512)  "mlp2" (block-diagonal 1536 -> 403|10|136)   {shape,pose,landmarks}.logit_image.{0,3}
 * bifpn_fusion_w_h: [2][20] = per BiFPN block the normalised fusion weights relu(w)/sum + 1e-4, w1 [2][4] then w2 [3][4]
 *   (bifpn.py:105-108).
 * pieces / operand_format select the arithmetic (accumulation is always fp32):
 *   DAD3D_OPERAND_BF16: 1 = plain bf16 operands (1 tensor-core product, throughput mode), 2 = bf16 hi/lo (3 products,
 *     16-bit operand mantissa), 3 = bf16 three-way split (6 products, 24-bit operand mantissa: strict fp32 operands);
 *   DAD3D_OPERAND_FP16: 2 = fp16 hi/lo (3 products, 22-bit operand mantissa; weights scaled per output channel by a power
 *     of two that the epilogue undoes; activations saturate at +-65504 and carry an absolute representation error
 *     <= 2^-25 below |x| = 2^-3), 1 = plain fp16 (11-bit, TF32-class). */
#define DAD3D_OPERAND_BF16 0
#define DAD3D_OPERAND_FP16 1
typedef struct dad3d_conv_weights {
  const char* name;
  const float* weight_h;     /* [cout][R][S][cin] */
  const float* bias_h;       /* [cout] */
  int32_t cout, cin, R, S;
} dad3d_conv_weights;

DAD3D_API int dad3d_encoder_create(dad3d_encoder** out, const dad3d_conv_weights* layers, int32_t n_layers,
                                   const float* bifpn_fusion_w_h, int32_t pieces, int32_t operand_format, int32_t device);
DAD3D_API void dad3d_encoder_destroy(dad3d_encoder* enc);
DAD3D_API int dad3d_encoder_num_layers(const dad3d_encoder* enc);
DAD3D_API size_t dad3d_encoder_workspace_bytes(dad3d_encoder* enc, int32_t B);
/* images_d [B,3,256,256] NCHW fp32 (already normalised, predictor.py:195-203) ->
 *   params_d [B,413] (OUTPUT_3DMM_PARAMS), landmarks_d [B,68,2] (OUTPUT_2D_LANDMARKS, in [0,1] image units),
 *   heatmap_d [B,68,64,64] NCHW fp32 or NULL (OUTPUT_LANDMARKS_HEATMAP). */
DAD3D_API int dad3d_encoder_forward(dad3d_encoder* enc, const float* images_d, int32_t B, float* params_d,
                                    float* landmarks_d, float* heatmap_d, void* workspace_d, size_t workspace_bytes,
                                    dad3d_stream stream);

/* ---- device-side pre-processing (SURVEY §8f "next" row 2) --------------------------------------------------------------
 * dad3d_preprocess replaces FaceMeshPredictor._transform + _array_to_batch (predictor.py:85-89,195-203: albumentations
 *   LongestMaxSize -> PadIfNeeded -> Normalize -> HWC->CHW) for one image: image_d [H,W,3] uint8 RGB (device) ->
 *   out_d [3,img_size,img_size] fp32.  new_h/new_w are the letter-boxed sizes (py3round(dim * img_size / max(H,W)),
 *   computed by the caller exactly as predictor.py:117-123 does); the 8-bit bilinear resize is bit-exact with
 *   cv2.resize(INTER_LINEAR).  mean255_h / inv_std255_h: the three fp32 constants mean*255 and 1/(std*255). */
DAD3D_API int dad3d_preprocess(const uint8_t* image_d, int32_t H, int32_t W, int32_t new_h, int32_t new_w,
                               int32_t img_size, const float* mean255_h, const float* inv_std255_h, float* out_d,
                               dad3d_stream stream);
/* the same for B images of one size: images_d [B,H,W,3] uint8 -> out_d [B,3,img_size,img_size] fp32, one launch */
DAD3D_API int dad3d_preprocess_batch(const uint8_t* images_d, int32_t B, int32_t H, int32_t W, int32_t new_h, int32_t new_w,
                                     int32_t img_size, const float* mean255_h, const float* inv_std255_h, float* out_d,
                                     dad3d_stream stream);

/* ---- heads from boxes in whole frames ----------------------------------------------------------------------------------
 * What a caller of the reference does per head box: crop (model_training/data/flame_dataset.py:96-99), run
 * FaceMeshPredictor.__call__ on the crop (predictor.py:117-176) and move the result into frame pixels -- for R boxes at once,
 * with every geometric value computed on the device, so the boxes may change between replays of a captured graph.
 *   dad3d_roi_setup  boxes_d [R,4] int32 [x, y, w, h] in frame pixels, frame_index_d [R] int32 (NULL: every box is on frame 0)
 *     -> rois_d [R] records.  crop = ensure_bbox_boundaries(extend_bbox(box, extend), (H, W)) (model_training/data/
 *     utils.py:73-115, float64 then truncation to int32; x2 is computed from the already clipped x1, so a box left of the frame
 *     is shifted, not cut); extend_h = (left, right, top, bottom) fractions as extend_bbox takes them.  A record is invalid
 *     (valid = 0: scale 1, new_h = new_w = 0, zero paddings, an all-padding input image) when its frame index is outside
 *     [0, F), its crop is empty, or a letter-boxed side rounds to 0 pixels (cv2.resize refuses that size, so the reference
 *     cannot process the crop either).
 *   dad3d_preprocess_rois  frames_d [F,H,W,3] uint8 RGB -> out_d [R,3,img_size,img_size] fp32: the letter-box of
 *     dad3d_preprocess on each record's crop, read in place with the frame's row pitch (bilinear taps clamp at the crop's
 *     border), bit-exact with cv2 on frame[y:y+h, x:x+w].  R <= 65535.
 *   dad3d_readjust_rois  FaceMeshPredictor._get_predictions' read-back (predictor.py:117-123,141-176) plus the move into frame
 *     pixels, per head, from the encoder's params_d [R,num_params] and landmarks_d [R,num_landmarks,2] (in [0,1] units):
 *     params_out_d [R,num_params] = readjust_3dmm_to_the_input_image in fp32 (scale at scale_index, translation at
 *     translation_index .. +2), then translation xy += [x, y] * 2 / img_size (the arithmetic of HeadMesh.adjust_3dmm_to_paddings,
 *     head_mesh.py:48-60) and translation z = 0 (the in-place side effect of reprojected_vertices, head_mesh.py:41);
 *     points_d [R,num_landmarks,2] int64 = readjust_landmarks_to_the_input_image(clip(lm * 256, 0, 256)) + [x, y], with the
 *     reference's dtypes (fp32 multiply and clip, float64 subtract and divide, truncation).  params_out_d may be params_d. */
typedef struct dad3d_roi {
  int32_t x, y, w, h;             /* the crop, in frame pixels */
  int32_t frame, valid;
  int32_t new_h, new_w;           /* py3round(side * scale): the letter-boxed size */
  int32_t pre_top, pre_left;      /* PadIfNeeded offsets of the letter-box (pre-processing) */
  int32_t post_top, post_left;    /* calculate_paddings(new_h, new_w)[0], [2] (post-processing, predictor.py:117-123) */
  double scale;                   /* img_size / double(max(h, w)) */
  double inv_scale_x, inv_scale_y;  /* cv::resize's 1 / (new_w / w), 1 / (new_h / h) */
} dad3d_roi;
DAD3D_API int dad3d_roi_setup(const int32_t* boxes_d, const int32_t* frame_index_d, int32_t R, int32_t F, int32_t H, int32_t W,
                              int32_t img_size, const double* extend_h, dad3d_roi* rois_d, dad3d_stream stream);
DAD3D_API int dad3d_preprocess_rois(const uint8_t* frames_d, int32_t H, int32_t W, const dad3d_roi* rois_d, int32_t R,
                                    int32_t img_size, const float* mean255_h, const float* inv_std255_h, float* out_d,
                                    dad3d_stream stream);
DAD3D_API int dad3d_readjust_rois(const float* params_d, const float* landmarks_d, const dad3d_roi* rois_d, int32_t R,
                                  int32_t num_params, int32_t num_landmarks, int32_t scale_index, int32_t translation_index,
                                  int32_t img_size, float* params_out_d, int64_t* points_d, dad3d_stream stream);

/* Live timing of the dominant kernel (the wgmma tile engine) for bench.py's roofline: while on, every conv / linear
 * launch is bracketed by CUDA events on the launching stream.  profile_read synchronises those events and returns their
 * summed duration, the launch count and the ALGORITHMIC FLOPs (2 * true MACs, one product per MAC, no padding) of the
 * recorded launches, then resets the counters. */
DAD3D_API int dad3d_encoder_set_profile(dad3d_encoder* enc, int32_t on);
DAD3D_API int dad3d_encoder_profile_read(dad3d_encoder* enc, double* gemm_ms, long long* gemm_launches,
                                         double* useful_flops);

/* One recorded launch of the current profiling window (call BEFORE dad3d_encoder_profile_read, which clears the window):
 * layer name, device time, useful FLOPs, algorithmic HBM bytes (every operand once), and info8 = {M output pixels, K, N,
 * tensor-core products per MAC, tiles, tile N, pipeline stages, k-blocks per tile}.  Returns DAD3D_ERR_INVALID past the
 * last recorded launch. */
DAD3D_API int dad3d_encoder_profile_layer(dad3d_encoder* enc, int32_t index, char* name, int32_t name_cap, double* ms,
                                          double* useful_flops, double* algo_bytes, int32_t* info8);

/* test hooks: keep_all != 0 disables workspace reuse so that, after a forward, any activation can be read back by the
 * name of the layer that produced it ("stem", "s2u1c3", "b1_p4out", "cat", "fusion", "gap", "heat", "mlp2" ...) as fp32
 * NHWC with channels padded as stored; dims4 receives [N,H,W,C] (pass out_d = NULL to query the shape only). */
DAD3D_API int dad3d_encoder_set_debug(dad3d_encoder* enc, int32_t keep_all);
DAD3D_API int dad3d_encoder_read_activation(dad3d_encoder* enc, const char* name, float* out_d, size_t capacity_floats,
                                            int32_t* dims4, dad3d_stream stream);
/* test hooks for single-step checks of the current plan (the one the last forward built):
 *   describe_plan  writes a NUL-terminated JSON description of every step (kind, layer, variant, the tensors it reads and
 *                  writes with their extents, and the tile-engine geometry of conv steps) into buf[cap]
 *   write_activation  the inverse of read_activation: src_d is fp32 NHWC [N,H,W,C] with channels padded as stored, n its
 *                  element count (must equal the tensor's); piece tensors are split with the library's own RN split, fp32
 *                  tensors are copied raw.  Only with keep_all on (set_debug), where no two tensors share workspace;
 *                  otherwise it fails
 *   run_steps      runs steps [first, first + count) of the plan exactly as dad3d_encoder_forward would (same launches,
 *                  same variant selection by heatmap_d); B and the workspace are those of the plan */
DAD3D_API int dad3d_encoder_describe_plan(dad3d_encoder* enc, char* buf, size_t cap);
DAD3D_API int dad3d_encoder_write_activation(dad3d_encoder* enc, const char* name, const float* src_d, size_t n,
                                             dad3d_stream stream);
DAD3D_API int dad3d_encoder_run_steps(dad3d_encoder* enc, int32_t first, int32_t count, const float* images_d,
                                      float* params_d, float* landmarks_d, float* heatmap_d, dad3d_stream stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Benchmark evaluator hot spots (SURVEY §8f row 1; dad_3dheads_benchmark/benchmark.py, dad_3dheads_benchmark/utils.py),
 * batched over B heads, device pointers, asynchronous on `stream`.
 *   dad3d_eval_chamfer : out[b] = mean_i min_j |a[b,i] - b[b,j]|^2 -- the term the evaluator asks kaolin for
 *                        (utils.py:139: chamfer_distance(gt_face, aligned_pred, 1.0, 0.0)); a [B,na,3], b [B,nb,3].
 *   dad3d_eval_zn      : Z_n ordinal depth accuracy exactly as DADEvaluator.calc_zn computes it (benchmark.py:110-138):
 *                        distances gt->gt (torch.cdist formula), COLUMN-wise argsort, columns 1..top_k of the index matrix,
 *                        mean agreement of the z-order of (i, index[i][j]) between gt and pred.  pred, gt [B,K,3], K <= 4096.
 *   dad3d_eval_align   : out = scale[b] * (verts[b] @ rot[b]) + trans[b] for every vertex (utils.py:178-197; rot [B,3,3]
 *                        row-major, the procrustes tform of the 7 landmark pairs). */
DAD3D_API int dad3d_eval_chamfer(const float* a_d, int32_t na, const float* b_d, int32_t nb, int32_t B, float* out_d,
                                 dad3d_stream stream);
DAD3D_API int dad3d_eval_zn(const float* pred_d, const float* gt_d, int32_t K, int32_t B, int32_t top_k, float* out_d,
                            dad3d_stream stream);
DAD3D_API int dad3d_eval_align(const float* verts_d, int32_t nv, int32_t B, const float* scale_d, const float* rot_d,
                               const float* trans_d, float* out_d, dad3d_stream stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Multi-GPU helpers (SURVEY §8b, §8e): one process per GPU; images are independent, so the only exchanges are the start-up
 * broadcast of the constants and the per-batch all-gather of the outputs, both over NCCL (NVLink 5 / NVSwitch).  libnccl is
 * bound at run time (dlopen: the copy already loaded in the process, e.g. PyTorch's, else the system's).
 *   dad3d_comm_unique_id : rank 0 creates the 128-byte NCCL id; the host distributes it (any side channel, e.g. a
 *                          torch.distributed / MPI broadcast of 128 bytes)
 *   dad3d_comm_init      : every rank joins (collective)
 *   dad3d_bcast_constants: in-place broadcast of `bytes` bytes of device memory from `root` (FLAME bases, packed weights)
 *   dad3d_allgather_outputs: recv_d [world * bytes_per_rank] <- every rank's send_d [bytes_per_rank], rank-major
 *                          (params [B,413], vertices [B,5023,3], landmarks ...) */
typedef struct dad3d_comm dad3d_comm;
DAD3D_API int dad3d_comm_unique_id(uint8_t* id128_h);
DAD3D_API int dad3d_comm_init(dad3d_comm** out, const uint8_t* id128_h, int32_t rank, int32_t world, int32_t device);
DAD3D_API void dad3d_comm_destroy(dad3d_comm* c);
DAD3D_API int dad3d_bcast_constants(dad3d_comm* c, void* buf_d, size_t bytes, int32_t root, dad3d_stream stream);
DAD3D_API int dad3d_allgather_outputs(dad3d_comm* c, const void* send_d, void* recv_d, size_t bytes_per_rank, dad3d_stream stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Rasteriser (SURVEY §8f row 4): the reference's native Sim3DR component (Sim3DR/lib/rasterize_kernel.cpp `_rasterize`
 * :238-292 and `_get_normal` :158-236; callers Sim3DR/Sim3DR.py:8-29, inference/pncc_estimator.py:16-43), bit-exact.
 *   dad3d_rasterize: z-buffer rendering of per-vertex colours with alpha = 1 (what Sim3DR.rasterize uses): vertices_d [nv,3]
 *     (x, y in pixels, z = depth, larger wins), triangles_d [ntri,3], colors_d [nv,c] in [0,1]; image_d [h,w,c] uint8 and
 *     depth_d [h,w] are read-modify-write exactly like the reference's buffers (depth is usually initialised to -1e8);
 *     key_ws_d = h*w 64-bit words of scratch; reverse != 0 flips the image rows.
 *   dad3d_rasterize_batch: the same for `batch` heads of one topology in two launches, replacing a Python loop of
 *     Sim3DR.rasterize calls (Sim3DR/Sim3DR.py:13-29; inference/pncc_estimator.py:16-43,66-68,76-93 per head).
 *     vertices_d [batch,nv,3]; triangles_d [ntri,3] and colors_d [nv,c] are shared by every head.  Outputs, each may be NULL:
 *     image_d [batch,h,w,c] uint8 and depth_d [batch,h,w] fp32 are read-modify-write exactly as in dad3d_rasterize (with
 *     depth_d NULL the z-test threshold is the constant -1e8 of Sim3DR.py:22); tri_index_d [batch,h,w] int32 is written for
 *     every pixel with the winning triangle or -1, in depth-buffer rows (reverse flips only the image).  negate_z != 0 uses -z
 *     as depth (pncc_estimator.py:77 `vertices[:, :, 2] *= -1`; exact, since negation commutes with rounding).  colors_d may
 *     be NULL when image_d is, triangles_d when ntri = 0.  key_ws_d = batch*h*w 64-bit words of scratch.  Every head equals, bit for bit, a
 *     single-head call on that head.  batch = 0 launches nothing; ntri = 0 launches nothing and sets tri_index_d to -1.
 *     dad3d_rasterize is the batch = 1 call of these kernels.
 *   dad3d_rasterize_frames: `batch` heads of one topology drawn into `n_images` shared images (several heads per whole
 *     frame, one z-buffer per frame), with the same two kernels.  image_of_head_d [batch] int32 (device) names each head's
 *     image; a head whose entry is outside [0, n_images) draws nothing (checked on the device, no host read).  Image m equals
 *     the reference's _rasterize (Sim3DR/lib/rasterize_kernel.cpp:238-292, alpha = 1) called once on the union mesh of the
 *     heads mapped to m in head order -- their vertices concatenated, each head's triangles offset by its vertex base -- which
 *     is the reference's per-head call (inference/pncc_estimator.py:16-43,88-101) repeated in head order with the image and
 *     depth buffer carried over.  So the nearest surface wins across heads, and an exact depth tie goes to the lower
 *     (head, triangle) pair, head first.  Outputs, each may be NULL: image_d [n_images,h,w,c] uint8 and depth_d
 *     [n_images,h,w] fp32 read-modify-write as in dad3d_rasterize_batch; tri_index_d [n_images,h,w] int32, the winning
 *     triangle within its head; head_index_d [n_images,h,w] int32, the winning head; both -1 for background.  No reverse.
 *     key_ws_d = n_images*h*w 64-bit words of scratch.  batch * ntri > 2^32 - 2 is DAD3D_ERR_INVALID (the key names a
 *     pair in 32 bits).  batch = 0 or ntri = 0 launches nothing and sets the index maps to -1 (with batch = 0, vertices_d
 *     and image_of_head_d may be NULL).
 *   dad3d_vertex_normals: normalised sum of the incident (un-normalised) face normals per vertex; adj_offsets_d [nv+1] /
 *     adj_triangles_d = CSR list of each vertex's triangles in ascending order (fixed per topology).
 *
 * Lit meshes: the reference's Sim3DR RenderPipeline (Sim3DR/lighting.py:23-71), per-vertex ambient + diffuse + specular
 * light of each head, then the rasteriser above with each head's light as its colours.
 *   dad3d_light_batch: light_d [batch,nv,3] fp32 = RenderPipeline's `light` of every head (vertices_d [batch,nv,3], -z when
 *     negate_z != 0), every float32 operation in the reference's order, round-to-nearest, no contraction: the normal of
 *     dad3d_vertex_normals, norm_vertices from the head's per-axis min / max, the diffuse and specular terms, the final clip
 *     (NaN propagates as np.clip does).  One exception: (v2v * reflection) ** specular_exp is the correctly rounded float32
 *     power, and specular_exp must be an integer in [0, 16] (else DAD3D_ERR_INVALID).  One CTA per head.
 *   dad3d_render_lit: dad3d_light_batch into light_ws_d [batch*nv*3] fp32, then the two raster passes with each head's light
 *     as colours, alpha = 1, into image_d (uint8, c = 3, read-modify-write: zeros or a background).  image_of_head_d NULL:
 *     image_d is [batch,h,w,3], one image per head (n_images ignored); else as dad3d_rasterize_frames, [n_images,h,w,3] with
 *     one z-buffer per image, and batch * ntri must stay <= 2^32 - 2.  key_ws_d = (mapped ? n_images : batch)*h*w 64-bit
 *     words.  Every argument is checked before the first launch. */
typedef struct dad3d_lighting {
  float intensity_ambient, intensity_directional, intensity_specular; /* a term is skipped unless its intensity is > 0 */
  int32_t specular_exp;                                              /* 0..16 */
  float color_ambient[3], color_directional[3], light_pos[3], view_pos[3];
} dad3d_lighting;
DAD3D_API int dad3d_rasterize(const float* vertices_d, const int32_t* triangles_d, const float* colors_d, int32_t ntri,
                              uint8_t* image_d, float* depth_d, unsigned long long* key_ws_d, int32_t h, int32_t w, int32_t c,
                              int32_t reverse, dad3d_stream stream);
DAD3D_API int dad3d_rasterize_batch(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d, int32_t ntri,
                                    const float* colors_d, int32_t c, int32_t h, int32_t w, int32_t reverse, int32_t negate_z,
                                    uint8_t* image_d, float* depth_d, int32_t* tri_index_d, unsigned long long* key_ws_d,
                                    dad3d_stream stream);
DAD3D_API int dad3d_rasterize_frames(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d,
                                     int32_t ntri, const float* colors_d, int32_t c, const int32_t* image_of_head_d,
                                     int32_t n_images, int32_t h, int32_t w, int32_t negate_z, uint8_t* image_d, float* depth_d,
                                     int32_t* tri_index_d, int32_t* head_index_d, unsigned long long* key_ws_d,
                                     dad3d_stream stream);
DAD3D_API int dad3d_vertex_normals(const float* vertices_d, const int32_t* triangles_d, const int32_t* adj_offsets_d,
                                   const int32_t* adj_triangles_d, int32_t nver, float* normals_d, dad3d_stream stream);
DAD3D_API int dad3d_light_batch(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d,
                                const int32_t* adj_offsets_d, const int32_t* adj_triangles_d, int32_t negate_z,
                                dad3d_lighting lighting, float* light_d, dad3d_stream stream);
DAD3D_API int dad3d_render_lit(const float* vertices_d, int32_t nv, int32_t batch, const int32_t* triangles_d, int32_t ntri,
                               const int32_t* adj_offsets_d, const int32_t* adj_triangles_d, int32_t negate_z,
                               dad3d_lighting lighting, const int32_t* image_of_head_d, int32_t n_images, int32_t h, int32_t w,
                               float* light_ws_d, uint8_t* image_d, unsigned long long* key_ws_d, dad3d_stream stream);

/* ---- overlays: the demo's landmark, pose and wireframe drawings, and head pose angles ------------------------------
 * Draws what demo_utils.py's processors draw with cv2 (4.13.0; the rules are restated and pinned in tests/overlay_model.py),
 * byte for byte, into frames the caller has already copied, for R boxes at once, with every box-dependent value read on
 * the device from the dad3d_roi records (see "heads from boxes").  Invalid records draw nothing.
 *   dad3d_pose_geometry  replaces calculate_rpy (model_training/model/flame.py:238-264) for every head, and draw_pose's
 *     float-to-integer geometry (demo_utils.py:68-94).  params_d [R,num_params] fp32; the six rotation parameters start at
 *     rotation_index.  rot_mat_from_6dof (model/utils.py:92-101) in fp32 in torch's CPU operation order (bit-exact; rot_d
 *     [R,3,3] fp32 receives it when not NULL), then scipy 1.18's Rotation.from_matrix(R^T) in fp64 -- the orthogonal polar
 *     factor that scipy takes by SVD, here by three Newton steps (within ~1e-15 of it), then the quaternion -- and
 *     as_euler("xyz", degrees=True), then limit_angle -> rpy_d [R,3] fp64 (roll, pitch, yaw; may be NULL).  With rois_d, pose_d [R,32] int32 records:
 *     [draw, frame, x, y, w, h, thickness, 0, cx, cy, then per arrow (red, green, blue): end x, end y, tip1 x, tip1 y,
 *     tip2 x, tip2 y, then zeros], in the coordinates of the crop view frame[y:y+h, x:x+w] that draw_pose is given: centre
 *     (w // 2, h // 2), size h // 10, thickness int(h * 0.005), ends truncated, tips cvRound of cv2.arrowedLine's fp64
 *     expressions.  draw = 0 for an invalid record, a crop under 200 px high (thickness 0: cv2.arrowedLine refuses it) or
 *     non-finite angles.  rois_d and pose_d are both given or both NULL.  One thread per head.
 *   dad3d_overlay_points  replaces draw_points over draw_landmarks / draw_3d_landmarks (demo_utils.py:22-47): for every
 *     valid record r and l < L, the filled circle (radius, colour color_h[3] RGB bytes) at point index_d[l] (NULL: l) of
 *     head r in points_d [R,n_src,ncomp] (is_float = 0: int64; 1: fp32 truncated toward zero, as astype(int)), drawn into
 *     frames_d [F,H,W,3] frame rois_d[r].frame.  A point that is not finite or whose integers do not fit int32 draws nothing
 *     (cv2 raises there), as does an index outside [0, n_src).  Every write of a call is the same colour, so the order of
 *     the threads does not matter.
 *   dad3d_overlay_pose  replaces draw_pose's three cv2.arrowedLine calls (demo_utils.py:90-92) for every record of
 *     dad3d_pose_geometry, each clipped to its own crop view and to the frame (records from dad3d_roi records of the same
 *     F, H, W always lie inside it): clears key_ws_d [F,H,W] int32, marks every covered pixel with
 *     the largest 3 * box + arrow + 1 (the reference's last writer: box order, then red, green, blue), then writes the
 *     winning arrow's colour over frames_d.  R <= (2^31 - 4) / 3. */
#define DAD3D_POSE_RECORD_INTS 32
DAD3D_API int dad3d_pose_geometry(const float* params_d, int32_t R, int32_t num_params, int32_t rotation_index,
                                  const dad3d_roi* rois_d, double* rpy_d, int32_t* pose_d, float* rot_d,
                                  dad3d_stream stream);
DAD3D_API int dad3d_overlay_points(const void* points_d, int32_t is_float, int32_t R, int32_t n_src, int32_t ncomp,
                                   const int64_t* index_d, int32_t L, const dad3d_roi* rois_d, int32_t radius,
                                   const uint8_t* color_h, uint8_t* frames_d, int32_t F, int32_t H, int32_t W,
                                   dad3d_stream stream);
DAD3D_API int dad3d_overlay_pose(const int32_t* pose_d, int32_t R, int32_t* key_ws_d, uint8_t* frames_d, int32_t F,
                                 int32_t H, int32_t W, dad3d_stream stream);
/*   dad3d_overlay_mesh  replaces draw_mesh (demo_utils.py:50-65): for every valid record r, cv2.line(frame, v[a], v[b],
 *     color_h[3], 1, LINE_AA) for every edge (a, b) of edges_d [E,2] int32 in order, v being head r of vertices_d
 *     [R,nv,ncomp] fp32 (ncomp 2 or 3; x, y truncated toward zero, as astype(int)), drawn into frames_d [F,H,W,3] frame
 *     rois_d[r].frame.  The blends of one pixel come in (box, edge) order, as the reference's loop makes them.  A box draws
 *     nothing when an end point of any edge is not finite or does not fit int32 (cv2 raises), or is outside [0, nv).
 *     ws_d [R,DAD3D_MESH_WS_INTS] int32 is the caller's workspace: per box the frame it draws into (-1: none) and the pixel
 *     box x0, y0, x1, y1 its stamps can touch.  Two kernels, no host synchronisation, 64-bit pixel offsets. */
#define DAD3D_MESH_WS_INTS 5
DAD3D_API int dad3d_overlay_mesh(const float* vertices_d, int32_t R, int32_t nv, int32_t ncomp, const int32_t* edges_d,
                                 int32_t E, const dad3d_roi* rois_d, const uint8_t* color_h, int32_t* ws_d,
                                 uint8_t* frames_d, int32_t F, int32_t H, int32_t W, dad3d_stream stream);

/* number of kernels this library has launched since load (bench.py's gpu_launches) */
DAD3D_API unsigned long long dad3d_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* DAD3D_H_ */
