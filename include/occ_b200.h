/* libocc_b200 -- C ABI of the H100 (sm_90a) camera->occupancy hot path.
 *
 * Every entry point takes plain pointers and sizes (no torch / C++ types) and returns 0 on success;
 * on failure it returns non-zero and occb200_last_error() describes the problem (thread-local).
 * "dev" pointers are CUDA device pointers on the current device; `stream` is a cudaStream_t passed
 * as void* (NULL = default stream).  Calls are asynchronous on `stream` unless stated otherwise.
 * Inputs are borrowed and never mutated; outputs are caller-allocated.
 *
 * Reference interfaces replaced (paths relative to the reference repository root):
 *   [R1] mmcv._ext.ms_deform_attn_forward, bound at
 *        projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py:118-124
 *        (ext loaded at encoder.py:24-25, spatial_cross_attention.py:27-28, temporal_self_attention.py:21-22)
 *   [R2] BEVFormerOccHead.forward + get_occ, projects/mmdet3d_plugin/bevformer/dense_heads/bevformer_occ_head.py:99-160,198-216
 *        -> TransformerOcc.forward (modules/transformer_occ.py:245-321) -> BEVFormerEncoder.forward (modules/encoder.py:153-239)
 *   [R3] dvr.render_forward, tools/ray_iou/lib/dvr/dvr.cpp:39-48 / dvr.cu:329-388
 *   [R4] ray_metrics.process_one_sample + calc_metrics, projects/mmdet3d_plugin/datasets/ray_metrics.py:89-197
 */
#ifndef OCC_B200_H_
#define OCC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* occb200_last_error(void);
/* "occ_b200 <ver> sm_90a" */
const char* occb200_version(void);

/* ---------------------------------------------------------------------------------------------
 * [R1] Multi-scale deformable attention, operator boundary (fp32, mmcv `_ext` argument meaning).
 *   value          dev f32 [B, Nv, M, C]        contiguous
 *   spatial_shapes dev i64 [L, 2] (h, w)        level_start_index dev i64 [L]
 *   sampling_loc   dev f32 [B, Nq, M, L, P, 2]  (x, y) normalised to [0,1]
 *   attn_weight    dev f32 [B, Nq, M, L, P]
 *   out            dev f32 [B, Nq, M*C]
 *   im2col_step is accepted for signature compatibility; mmcv asserts B % min(B, im2col_step) == 0
 *   and so does this entry (error code 1).
 */
int occb200_ms_deform_attn_forward(const float* value, const int64_t* spatial_shapes,
                                   const int64_t* level_start_index, const float* sampling_loc,
                                   const float* attn_weight, int B, int Nv, int M, int C, int Nq, int L, int P,
                                   int im2col_step, float* out, void* stream);

/* Backward of the same operator (mmcv `_ext.ms_deform_attn_backward`, reference call site
 * multi_scale_deformable_attn_function.py:150-160): grad_output dev f32 [B, Nq, M*C]; the three gradient buffers are
 * caller-allocated and PRE-ZEROED (as the reference's autograd Function does, :146-148): grad_value [B,Nv,M,C] is
 * accumulated with atomics, grad_sampling_loc [B,Nq,M,L,P,2] and grad_attn_weight [B,Nq,M,L,P] are written. */
int occb200_ms_deform_attn_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                    const float* sampling_loc, const float* attn_weight, const float* grad_output, int B,
                                    int Nv, int M, int C, int Nq, int L, int P, int im2col_step, float* grad_value,
                                    float* grad_sampling_loc, float* grad_attn_weight, void* stream);

/* ---------------------------------------------------------------------------------------------
 * [R2] Frame engine: packs BEV queries, runs the BEVFormerEncoder layers (temporal self-attention,
 * spatial cross-attention, FFN), the Conv3d voxel decoder and the occupancy / flow heads.
 */
typedef struct occb200_engine occb200_engine;

typedef struct occb200_config {
    int bev_h, bev_w;              /* BEV grid (200 x 200)                     bevformer_base_occ.py:41-42   */
    int embed_dims, num_heads;     /* 256, 8 (only these are supported)                                      */
    int num_layers;                /* encoder layers (4 shipped, 6 BEVFormer-base)          :101             */
    int num_cams;                  /* <= 8                                                                   */
    int num_levels;                /* 4                                                                      */
    int level_h[4], level_w[4];    /* FPN level shapes                                                       */
    int num_points_in_pillar;      /* D in {1,2,4,8}                                        :103             */
    int sca_points, tsa_points;    /* 8, 4                                                  :118, default 4  */
    int ffn_dim;                   /* 512                                                   :125             */
    int pillar_h, out_dim;         /* 16, 32                                                :92, default     */
    int num_classes;               /* 17                                                                     */
    float pc_range[6];
    int precision;                 /* 0 = fp32 storage + fp32 CUDA-core GEMMs (parity config),
                                      1 = bf16 storage, fp32 accumulate (throughput config)                  */
    int use_tensor_cores;          /* 1 = wgmma GEMM / conv kernels where available                         */
    int use_cams_embeds;           /* TransformerOcc(use_cams_embeds=...), transformer_occ.py:214-215; 0 = the
                                      camera embedding is NOT added to the packed features                    */
    int rotate_center[2];          /* TransformerOcc(rotate_center=[100,100]), transformer_occ.py:200: centre
                                      (x, y) of the prev_bev rotation done by occb200_engine_forward_prev      */
} occb200_config;

int occb200_engine_create(const occb200_config* cfg, occb200_engine** out);
void occb200_engine_destroy(occb200_engine* e);

/* Load one parameter by its key in `pts_bbox_head.state_dict()` (e.g.
 * "transformer.encoder.layers.0.attentions.1.output_proj.weight").  `data` is HOST fp32, `numel` its size.
 * Unknown keys return error 3 (so a checkpoint/key-contract mismatch is loud).  Call _finalize afterwards. */
int occb200_engine_load_param(occb200_engine* e, const char* key, const float* data, int64_t numel);
/* Folds BatchNorm, concatenates the offset/weight projections, converts to the storage precision and
 * checks that every parameter the configuration needs was loaded.  Synchronous. */
int occb200_engine_finalize(occb200_engine* e);

/* Camera geometry of the frame(s) to come: cam_mat HOST f32 [num_cams,16] = lidar2img[c] @ ego2lidar (fp32
 * product, encoder.py:126), zs HOST f32 [D] = linspace(.5, Z-.5, D)/Z (encoder.py:66-67), image (h, w) =
 * img_metas[0]['img_shape'][0][:2] (encoder.py:133-134). */
int occb200_engine_set_cameras(occb200_engine* e, const float* cam_mat, const float* zs, int img_h, int img_w);

/* Rotation of the NEXT frames' prev_bev (TransformerOcc.get_bev_features, transformer_occ.py:189-205: torchvision
 * rotate(prev_bev as (C,H,W), can_bus[-1] degrees, center=rotate_center), nearest, zero fill).  A nearest-neighbour
 * rotation is a row permutation of the (Nq, C) BEV: map_host[q] (HOST int32 [Nq]) = source BEV cell of output cell q,
 * -1 = outside (zeros).  The engine applies it while casting prev_bev to the GEMM operand type -- prev_bev is then
 * passed UN-rotated to occb200_engine_forward.  NULL clears it (prev_bev is taken as already rotated).  Synchronous. */
int occb200_engine_set_prev_rotation(occb200_engine* e, const int32_t* map_host);

/* Element type / layout of the feature levels handed to _forward / _forward_host / _submit_host from now on (pointers
 * travel through the same arguments): 0 = fp32 [num_cams, C, h, w] (default, the reference's), 1 = bf16, same layout
 * (half the PCIe bytes for host pipelines that hold bf16 features), 2 = bf16 channels-last [num_cams, h, w, C] -- the
 * native output of occb200_backbone_forward_nhwc_bf16, so images -> voxels never leaves the device or transposes. */
int occb200_engine_set_input_dtype(occb200_engine* e, int feats_bf16);

/* One frame, DEVICE buffers.
 *   feats[l]   dev f32 [num_cams, C, h_l, w_l]  (FPN outputs of one batch item, NCHW)
 *   prev_bev   dev f32 [Nq, C] or NULL          (already rotated; NULL = the reference's only runtime mode)
 * Outputs (any may be NULL to skip):
 *   bev_embed  dev f32 [Nq, C]                   (= reference bev_embed permuted to (Nq, C))
 *   occ_logits dev f32 [X, Y, Z, num_classes]    flow dev f32 [X, Y, Z, 2]
 *   occ_cls_u8 dev u8  [X, Y, Z]                 occ_cls_i64 dev i64 [X, Y, Z]   (argmax, get_occ) */
int occb200_engine_forward(occb200_engine* e, const float* const* feats, const float* prev_bev, float* bev_embed,
                           float* occ_logits, float* flow, uint8_t* occ_cls_u8, int64_t* occ_cls_i64, void* stream);

/* One frame, HOST buffers (pinned recommended): copies feats host->device, runs the frame, copies
 * occ_cls (int64, the reference's LongTensor) / flow back and synchronises.  This is the call the
 * reference-facing detector shell makes (bevformer_occ.py:247-250 returns CPU tensors). */
int occb200_engine_forward_host(occb200_engine* e, const float* const* feats_host, int64_t* occ_cls_i64_host,
                                float* flow_host, void* stream);

/* Pipelined form of the same call for streams of frames: _submit_host enqueues the host->device copy of the
 * frame's features (copy streams; levels above 32 MB are split over OCC_H2D_SPLIT = 1..4 of them, default 2), the
 * frame (caller's stream, after those copies) and the device->host copy of the
 * results (second copy stream) for `slot` in {0,1} and returns; _wait_host blocks until the slot's results are in
 * the host buffers.  With two slots in flight the copies of frame i+1 / i-1 overlap the compute of frame i.
 * Host buffers must be pinned for the copies to be asynchronous. */
int occb200_engine_submit_host(occb200_engine* e, int slot, const float* const* feats_host, int64_t* occ_cls_i64_host,
                               float* flow_host, void* stream);
int occb200_engine_wait_host(occb200_engine* e, int slot);

/* Intermediate taps for parity tests (dev f32, valid after a forward; NULL if not produced):
 *   which: 0 = layer output [Nq,C] of layer `layer`; 1 = TSA output (pre-norm, with residual); 2 = SCA output
 *   (pre-norm, with residual); 3 = voxel features [X,Y,Z,out_dim] (converted to fp32 into `dst`);
 *   4 = packed camera tokens [num_cams, Nv, C] of the last frame (get_bev_features, transformer_occ.py:207-227). */
int occb200_engine_enable_taps(occb200_engine* e, int enable);
int occb200_engine_copy_tap(occb200_engine* e, int which, int layer, float* dst_dev, void* stream);

/* Row a2 on its own: reference_points_cam dev f32 [num_cams, Nq, D, 2], bev_mask dev u8 [num_cams, Nq, D]. */
int occb200_engine_project_pillars(occb200_engine* e, float* ref_cam, uint8_t* mask, void* stream);
/* number of kernels one forward launches (for the benchmark's gpu_launches claim) */
int occb200_engine_launches_per_frame(const occb200_engine* e);
/* Per-kernel-category device timing with CUDA events on the launch stream (benchmark roofline).
 * Categories: 0 pack/prepare, 1 dense GEMM, 2 TSA gather, 3 SCA gather, 4 LayerNorm, 5 bev->voxel, 6 conv3d,
 * 7 occ/flow heads.  _profile(e,1) starts collecting, _profile_read synchronises and returns the summed
 * milliseconds and launch counts since the last read (n >= 8). */
int occb200_engine_profile(occb200_engine* e, int enable);
int occb200_engine_profile_read(occb200_engine* e, float* ms_per_category, int* launches_per_category, int n);

/* ---------------------------------------------------------------------------------------------
 * [R3] dvr.render_forward (phase "test").  sigma dev f32 [N,T,Z,Y,X]; origin dev f32 [N,T,3];
 * points dev f32 [N,M,3]; tindex dev f32 [N,M]; outputs dev f32 pred_dist [N,M], gt_dist [N,M],
 * coord_index [N,M,3] (all written, including the -1 / 0 defaults).
 */
int occb200_render_forward(const float* sigma, const float* origin, const float* points, const float* tindex,
                           int N, int T, int Z, int Y, int X, int64_t M, float* pred_dist, float* gt_dist,
                           float* coord_index, void* stream);

/* [R4] One frame of the Ray-mIoU / mAVE metric on a 200x200x16 grid (0.4 m voxels, range [-40,-40,-1]).
 *   sem_* dev u8 [200,200,16]; flow_* dev f32 [200,200,16,2]; origins dev [T,3] (f32, or f64 if origin_is_f64);
 *   rays dev f32 [M,3] (generate_lidar_rays); counters dev f64 [187] accumulated in place, layout
 *   gt_cnt[17] pred_cnt[17] tp_cnt[3][17] ave[3][17] ave_count[3][17] (ray_metrics.py:149-158);
 *   pcd_pred / pcd_gt dev f32 [T*M,4] optional (process_one_sample rows: class, dist, flow_x, flow_y). */
int occb200_ray_metric_accumulate(const uint8_t* sem_pred, const float* flow_pred, const uint8_t* sem_gt,
                                  const float* flow_gt, const void* origins, int origin_is_f64, int T,
                                  const float* rays, int M, double* counters, float* pcd_pred, float* pcd_gt,
                                  void* stream);

/* ---------------------------------------------------------------------------------------------
 * Building blocks exposed for the module-level API mirror and for kernel tests (dev pointers).
 *   linear: C[M,N] = act(A[M,K] . W[N,K]^T + bias) (+ residual), fp32, act 0 none / 1 relu
 *   layernorm: rows x 256, eps 1e-5 */
int occb200_linear_f32(const float* A, const float* W, const float* bias, const float* residual, float* C, int M,
                       int N, int K, int act, void* stream);
int occb200_layernorm_f32(const float* x, const float* gamma, const float* beta, float* y, int rows, int C,
                          void* stream);
/* tensor-core bf16 GEMM self-test entry: C f32 [M,N] = A bf16 [M,K] . W bf16 [N,K]^T (+bias); used by tests */
int occb200_gemm_bf16_tc(const void* A_bf16, const void* W_bf16, const float* bias, float* C, int M, int N, int K,
                         void* stream);

/* ---------------------------------------------------------------------------------------------
 * Image backbone + neck (SURVEY 8f rank 1, the step immediately BEFORE the hot path); parity vs its oracle:
 * tests/test_backbone_gpu.py (fp32 1e-3 relative to the feature magnitude, bf16 bars stated there).
 * Replaces `self.img_backbone(img)` + `self.img_neck(...)` in BEVFormerOcc.extract_img_feat
 * (detectors/bevformer_occ.py:66-99) for the shipped configuration (bevformer_base_occ.py:48-66): mmdet
 * ResNet(depth=50, out_indices=(1,2,3), style='pytorch', norm_eval=True) + FPN(in_channels=[512,1024,2048],
 * out_channels=256, start_level=0, add_extra_convs='on_output', num_outs=4), eval mode.
 *   precision 0: fp32 storage, CUDA-core GEMMs (parity configuration); 1: bf16 storage (+ tensor-core GEMMs).
 *   Parameters by their key in the detector's state_dict: "img_backbone.conv1.weight", "img_backbone.layer1.0.bn1.
 *   running_mean", "img_neck.lateral_convs.0.conv.bias", ... (HOST fp32; `num_batches_tracked` is not a parameter).
 *   forward: img dev f32 [num_images, 3, H, W] (mean/std-normalised, padded) -> out_l dev f32 [num_images, 256, h_l, w_l]
 *   (any out may be NULL), the layout `extract_img_feat` hands to the head after its view(B, N, C, h, w). */
typedef struct occb200_backbone occb200_backbone;
occb200_backbone* occb200_backbone_create(int num_images, int img_h, int img_w, int precision, int use_tensor_cores);
void occb200_backbone_destroy(occb200_backbone* e);
int occb200_backbone_load_param(occb200_backbone* e, const char* key, const float* data, int64_t numel);
int occb200_backbone_finalize(occb200_backbone* e);
int occb200_backbone_level_shape(const occb200_backbone* e, int level, int* h, int* w);
int occb200_backbone_forward(occb200_backbone* e, const float* img, float* out0, float* out1, float* out2, float* out3,
                             void* stream);
/* Same, precision 1 only: the four FPN outputs are written as bf16 channels-last [num_images, h_l, w_l, 256] straight by
 * the last convolutions (no NCHW fp32 copy): the layout occb200_engine_set_input_dtype(e, 2) consumes. */
int occb200_backbone_forward_nhwc_bf16(occb200_backbone* e, const float* img, void* out0, void* out1, void* out2, void* out3,
                                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OCC_B200_H_ */
