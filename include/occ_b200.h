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
typedef struct occb200_backbone occb200_backbone;   /* image backbone + neck, declared below */

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
                                      (x, y) of the prev_bev rotation by angle (_set_prev_rotation_angle, the
                                      video _angle calls)                                                     */
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
 * passed UN-rotated to occb200_engine_forward.  NULL clears it (prev_bev is taken as already rotated).  Synchronous.
 * The map lives in ONE engine-global device buffer written by a blocking copy: a frame still queued on a non-blocking
 * stream may read the new map, so change it only when no frame is in flight.  The video calls below ignore it (they take a
 * map per frame). */
int occb200_engine_set_prev_rotation(occb200_engine* e, const int32_t* map_host);
/* The same rotation given by its angle: can_bus[-1] degrees about the config's rotate_center.  No map is built, copied or
 * uploaded: the gather computes every cell's source cell on the device (occb200_rotation_coeffs, then torchvision's grid and
 * nearest rounding, bit-identical to the map torchvision's rotate makes of an index image).  The coefficients travel as kernel
 * arguments of each frame, so there is no in-flight hazard.  Host only, no CUDA call.  Between this call and
 * occb200_engine_set_prev_rotation(map or NULL) the last call wins.  A non-finite angle returns 1. */
int occb200_engine_set_prev_rotation_angle(occb200_engine* e, double angle_deg);
/* The six fp32 grid coefficients of torchvision's rotate(img, angle_deg, center=[cx, cy]) on a bev_h x bev_w image, computed
 * as torchvision computes them: _get_inverse_affine_matrix(center - size/2, -angle) in double (cos / sin of angle * pi/180),
 * cast to fp32, divided in fp32 by [bev_w / 2, bev_h / 2].  out[0..2]: g_x = out[0] x + out[1] y + out[2]; out[3..5]: g_y
 * alike, over the base grid x = j - bev_w/2 + 0.5, y = i - bev_h/2 + 0.5.  Host only, no CUDA call. */
int occb200_rotation_coeffs(double angle_deg, int bev_h, int bev_w, int cx, int cy, float out[6]);
/* Debug / test entry: map_dev (dev int32 [Nq]) = the source cell of every BEV cell (-1 = outside) that the rotation gathers
 * compute for angle_deg, written by one kernel on `stream`. */
int occb200_engine_rotation_map(occb200_engine* e, double angle_deg, int32_t* map_dev, void* stream);

/* Element type / layout of the feature levels handed to _forward / _forward_host / _submit_host from now on (pointers
 * travel through the same arguments): 0 = fp32 [num_cams, C, h, w] (default, the reference's), 1 = bf16, same layout
 * (half the PCIe bytes for host pipelines that hold bf16 features), 2 = bf16 channels-last [num_cams, h, w, C] -- the
 * native output of occb200_backbone_forward_nhwc_bf16, so images -> voxels never leaves the device or transposes.
 * 3 = uint8 camera frames: feats[0] is the frame buffer [num_cams, src_h, src_w, 3] of the attached backbone's frame format
 * (occb200_engine_attach_backbone) and feats[1..3] are ignored; a device pointer for _forward, a host pointer for
 * _forward_host / _submit_host.  The backbone runs first, on the same stream; with both precisions bf16 its FPN writes
 * channels-last bf16 levels into engine-owned buffers (code 2's hand-over), otherwise fp32 NCHW levels.  The backbone's
 * workspace and those level buffers are shared by both _submit_host slots: every frame records an event after its last read
 * of them and the next frame's backbone waits for it, so switching streams between submits stays correct.
 * occb200_engine_launches_per_frame then counts the backbone's kernels too.
 * 4 = JPEG camera files: feats[0] points to an occb200_encoded_frame, declared below, holding the num_cams files in HOST memory,
 * for every frame call.  The files are checked and parsed on the host (error 1 before any CUDA call, see occb200_jpeg_*; their
 * size must be the attached backbone's frame format), packed into a pinned staging buffer of the call's buffer set (the
 * device calls' and _forward_host's, or the slot's) and uploaded in one copy (the slot's copy stream, else `stream`); three
 * kernels decode them on `stream` into that set's frame buffer, byte-identical to cv2.imdecode(IMREAD_UNCHANGED), and the
 * frame continues as for 3 with those frames.  The caller may reuse its buffers when the call returns.
 * occb200_engine_launches_per_frame counts the decode's three kernels too. */
int occb200_engine_set_input_dtype(occb200_engine* e, int feats_bf16);
/* Borrowed; NULL detaches.  bb must be finalized, with num_images == num_cams, level shapes equal to the engine's, and a
 * frame format set.  It must outlive the engine's use of it (detach before destroying it). */
int occb200_engine_attach_backbone(occb200_engine* e, occb200_backbone* bb);

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
 * frame's features (copy streams; levels above 32 MB are split over two of them), the
 * frame (caller's stream, after those copies) and the device->host copy of the
 * results (second copy stream) for `slot` in {0,1} and returns; _wait_host blocks until the slot's results are in
 * the host buffers.  With two slots in flight the copies of frame i+1 / i-1 overlap the compute of frame i.
 * Host buffers must be pinned for the copies to be asynchronous. */
int occb200_engine_submit_host(occb200_engine* e, int slot, const float* const* feats_host, int64_t* occ_cls_i64_host,
                               float* flow_host, void* stream);
int occb200_engine_wait_host(occb200_engine* e, int slot);

/* Temporal (video) inference with the BEV history kept inside the engine (BEVFormer's prev_bev, transformer_occ.py:189-205).
 *
 * _set_history(e, 1) allocates the history: ONE [Nq, 256] row-major buffer in the storage precision (bf16; fp32 for
 * precision 0), 20.5 MB / 41 MB at 200 x 200.  _set_history(e, 0) frees it.  Both wait for queued video frames first, and
 * both start a new scene.  Synchronous.
 *
 * Only _forward_video and _submit_host_video read or write the history; _forward, _forward_host and _submit_host never touch
 * it.  A video frame
 *   - runs in self mode (prev_bev = None) when scene_start != 0 or no video frame has run since _set_history(e, 1): bit-identical
 *     to occb200_engine_forward(prev_bev = NULL);
 *   - otherwise takes prev_bev = the history gathered through the rotation map (NULL = no rotation): bit-identical to
 *     occb200_engine_forward(prev_bev = the previous video frame's bev_embed) after occb200_engine_set_prev_rotation(map).
 *     The history holds the last LayerNorm's storage-type copy of bev_embed, which is exactly what that call's gather makes
 *     of the fp32 bev_embed;
 *   - leaves its own final BEV in the history, whether or not bev_embed is requested;
 *   - waits for the previous video frame's history write (an event), so the caller may switch streams between frames.
 * The map is the per-frame form of occb200_engine_set_prev_rotation's (source cell of every cell, -1 = outside); the
 * engine-global map of that call is ignored here.
 *
 * _forward_video: device buffers, the outputs of occb200_engine_forward (any may be NULL).  rot_map_dev: dev int32 [Nq] or
 *   NULL; it is not checked on the host, so an entry outside [-1, Nq) is read as -1 (a row of zeros), never out of bounds.
 * _submit_host_video: the pipelined host-buffer call (occb200_engine_submit_host), completed by occb200_engine_wait_host.
 *   rot_map_host: HOST int32 [Nq] or NULL, checked like occb200_engine_set_prev_rotation's, then staged in a slot-owned pinned
 *   buffer and uploaded on the slot's copy stream: the caller may reuse its array as soon as the call returns.
 * All four input dtypes work (set_input_dtype).  A call without _set_history(e, 1), with a NULL pointer, a bad or busy slot or an
 * out-of-range host map returns 1 before any CUDA call and leaves the history unchanged.  occb200_engine_launches_per_frame
 * counts the video frame's launches. */
int occb200_engine_set_history(occb200_engine* e, int enable);
int occb200_engine_forward_video(occb200_engine* e, const float* const* feats, const int32_t* rot_map_dev, int scene_start,
                                 float* bev_embed, float* occ_logits, float* flow, uint8_t* occ_cls_u8, int64_t* occ_cls_i64,
                                 void* stream);
int occb200_engine_submit_host_video(occb200_engine* e, int slot, const float* const* feats_host, const int32_t* rot_map_host,
                                     int scene_start, int64_t* occ_cls_i64_host, float* flow_host, void* stream);
/* The same two calls with the frame's rotation as an angle (can_bus[-1] degrees about the config's rotate_center) instead of a
 * map: the history gather computes the source cells on the device (see occb200_engine_set_prev_rotation_angle), so there is
 * no map to build, stage or upload and the frame launches the same kernels.  Bit-identical to the map calls with the map
 * torchvision's rotate gives for that angle.  A non-finite angle returns 1 before any CUDA call, like the other rejections. */
int occb200_engine_forward_video_angle(occb200_engine* e, const float* const* feats, double angle_deg, int scene_start,
                                       float* bev_embed, float* occ_logits, float* flow, uint8_t* occ_cls_u8,
                                       int64_t* occ_cls_i64, void* stream);
int occb200_engine_submit_host_video_angle(occb200_engine* e, int slot, const float* const* feats_host, double angle_deg,
                                           int scene_start, int64_t* occ_cls_i64_host, float* flow_host, void* stream);

/* Ray records: what the Occupancy-and-Flow challenge file holds per frame, {pcd_cls int8, pcd_dist fp16, pcd_flow fp16}
 * (datasets/nuscenes_occ.py:189-257), cast inside the frame that predicted the volumes.  T <= 8 lidar origins x M rays go
 * through the predicted 200 x 200 x 16 volume once (ray_metrics.process_one_sample's arithmetic, [R4]); row t * M + m holds the
 * class of the first occupied voxel (the exit voxel, or voxel (0,0,0) for a ray that never enters the grid), its distance in
 * metres (-0.4 for such a ray) and its flow, narrowed as numpy's astype does (round to nearest even, overflow to inf, NaN kept).
 *
 * _set_rays uploads the constant ray bundle (HOST f32 [M,3], generate_lidar_rays) once.  Synchronous; it also disarms.  Change
 * the bundle only when no frame is in flight.
 * _request_rays arms ONE frame: the next frame call of any kind (_forward, _forward_video[_angle], _forward_host,
 *   _submit_host[_video[_angle]]) that passes its own checks consumes the request and, after its head kernel, launches
 *   ray_records_kernel on its stream from the volumes it produced: one kernel more than occb200_engine_launches_per_frame
 *   counts for an unarmed frame.  origins_host: HOST [T,3] f32, or f64 if origin_is_f64 (the arithmetic follows torch's type
 *   promotion); they are copied into the request and travel as a kernel argument, so the caller may reuse the array at once
 *   and frames in flight cannot see each other's origins.  Outputs cls_i8 [T*M], dist_f16 [T*M], flow_f16 [T*M,2]: DEVICE
 *   buffers for the device calls; (pinned) HOST buffers for the host calls, written by the call's device->host copy and
 *   complete when _forward_host returns / at _wait_host.  Host only, no CUDA call.  T = 0 or NULL origins disarms and returns 0.
 *   Rejected with error 1, leaving no request armed: NULL engine, T outside 0..8, a NULL output, a non-finite origin, no ray
 *   bundle set, a grid other than 200 x 200 x 16.  A frame call that is itself rejected leaves the request armed.
 * With a request armed the host calls accept occ_cls_i64_host == NULL and / or flow_host == NULL and skip that 5.12 MB copy;
 * without one NULL is rejected as before.  The caller's own outputs are the same bytes with and without a request. */
int occb200_engine_set_rays(occb200_engine* e, const float* rays_host, int M);
int occb200_engine_request_rays(occb200_engine* e, const void* origins_host, int origin_is_f64, int T, int8_t* cls_i8,
                                void* dist_f16, void* flow_f16);

/* Score a frame against its ground truth inside the frame that predicted it: Ray-mIoU / mAVE counters
 * (datasets/ray_metrics.py:200-257) without the predicted volumes leaving the device.
 * _request_score arms ONE frame, as _request_rays does: the next frame call of any kind that passes its own checks consumes
 *   the request and, after its head kernel, launches ray_score_kernel on its stream: one kernel more than
 *   occb200_engine_launches_per_frame counts for an unarmed frame.  The kernel casts the T x M rays of the _set_rays bundle
 *   through the ground truth and, for rays whose ground-truth hit is not `free`, through the volumes the frame produced, and
 *   adds to counters_dev what occb200_ray_metric_accumulate adds for those volumes (the integer counters bit for bit; the
 *   `ave` sums up to the order of the fp64 additions).
 *   sem_gt u8 [200,200,16], flow_gt f32 [200,200,16,2]: DEVICE pointers for the device calls, borrowed until the frame has
 *   run; HOST pointers for the host calls (pinned for asynchronous copies), uploaded on the slot's copy stream into
 *   slot-owned staging (5.76 MB per slot, allocated on first use; engine-owned staging for _forward_host), reusable after
 *   _forward_host returns / after _wait_host.  counters_dev: DEVICE f64 [187] (gt_cnt[17] pred_cnt[17] tp[3][17] ave[3][17]
 *   ave_count[3][17]), caller-owned, accumulated in place, always a device pointer; complete when the frame is (stream
 *   synchronised / _wait_host).  origins_host: as for _request_rays, copied into the request.
 *   Host only, no CUDA call.  T = 0 or NULL origins disarms and returns 0.  Rejected with error 1, leaving no request armed:
 *   NULL engine, T outside 0..8, NULL sem_gt / flow_gt / counters_dev, a non-finite origin, no ray bundle set, a grid other
 *   than 200 x 200 x 16.  A frame call that is itself rejected leaves the request armed.
 * A score request lets the host calls decline their volumes (NULL) exactly as a ray request does, and both may be armed for
 * the same frame, which then launches both kernels.  The caller's own outputs are the same bytes with and without a request. */
int occb200_engine_request_score(occb200_engine* e, const uint8_t* sem_gt, const float* flow_gt, const void* origins_host,
                                 int origin_is_f64, int T, double* counters_dev);

/* Intermediate taps for parity tests (dev f32, valid after a forward; NULL if not produced):
 *   which: 0 = layer output [Nq,C] of layer `layer`; 1 = TSA output (pre-norm, with residual); 2 = SCA output
 *   (pre-norm, with residual); 3 = voxel features [X,Y,Z,out_dim] (converted to fp32 into `dst`);
 *   4 = packed camera tokens [num_cams, Nv, C] of the last frame (get_bev_features, transformer_occ.py:207-227). */
int occb200_engine_enable_taps(occb200_engine* e, int enable);
int occb200_engine_copy_tap(occb200_engine* e, int which, int layer, float* dst_dev, void* stream);

/* Row a2 on its own: reference_points_cam dev f32 [num_cams, Nq, D, 2], bev_mask dev u8 [num_cams, Nq, D]. */
int occb200_engine_project_pillars(occb200_engine* e, float* ref_cam, uint8_t* mask, void* stream);
/* number of kernels one forward launches (for the benchmark's gpu_launches claim); with input dtype 3 (camera frames) the
 * attached backbone's kernels are included; a frame that consumed a ray request or a score request launched one kernel more
 * for each */
int occb200_engine_launches_per_frame(const occb200_engine* e);
/* Per-kernel-category device timing with CUDA events on the launch stream (benchmark roofline).
 * Categories: 0 pack/prepare, 1 dense GEMM, 2 TSA gather, 3 SCA gather, 4 LayerNorm, 5 bev->voxel, 6 conv3d,
 * 7 occ/flow heads.  _profile(e,1) starts collecting, _profile_read synchronises and returns the summed
 * milliseconds and launch counts since the last read (n >= 8). */
int occb200_engine_profile(occb200_engine* e, int enable);
int occb200_engine_profile_read(occb200_engine* e, float* ms_per_category, int* launches_per_category, int n);

/* ---------------------------------------------------------------------------------------------
 * [R3] dvr.render_forward (phase "test").  sigma dev f32 [N,T,Z,Y,X]; origin dev f32 [N,To,3];
 * points dev f32 [N,M,K], K >= 3 (columns 0..2 are the end point); tindex dev f32 [N,M]; outputs dev f32
 * pred_dist [N,M], gt_dist [N,M], coord_index [N,M,3] (all written, including the -1 / 0 defaults).
 * Ray (n, m) with t = (int)tindex[n][m] >= 0 starts at origin[n][t] and walks sigma[n][T == 1 ? 0 : t], as in the
 * reference; t is checked against neither T nor To (the caller keeps it below both, or below To when T == 1).
 * A NULL pointer, N outside 0..65535, M < 0, T, To, Z, Y or X < 1, or K < 3 returns 1 before any CUDA call.
 */
int occb200_render_forward(const float* sigma, const float* origin, const float* points, const float* tindex,
                           int N, int T, int To, int Z, int Y, int X, int64_t M, int K, float* pred_dist, float* gt_dist,
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

/* The ray-record operator on its own (see occb200_engine_request_rays): sem_u8 dev u8 [200,200,16], flow dev f32
 * [200,200,16,2], origins_host HOST [T,3] (f32, or f64 if origin_is_f64), T in 1..8, rays_dev dev f32 [M,3]; outputs dev
 * cls_i8 [T*M], dist_f16 [T*M], flow_f16 [T*M,2].  One launch of ray_records_kernel on `stream`.  A NULL pointer, T or M out
 * of range or a non-finite origin returns 1 before any CUDA call. */
int occb200_ray_records(const uint8_t* sem_u8, const float* flow, const void* origins_host, int origin_is_f64, int T,
                        const float* rays_dev, int M, int8_t* cls_i8, void* dist_f16, void* flow_f16, void* stream);

/* The score kernel on its own (see occb200_engine_request_score), for tests and timing: all volumes dev, origins_host HOST
 * [T,3] (f32, or f64 if origin_is_f64), T in 1..8, rays_dev dev f32 [M,3], counters_dev dev f64 [187] accumulated in place.
 * One launch of ray_score_kernel on `stream`.  A NULL pointer, T or M out of range or a non-finite origin returns 1 before
 * any CUDA call. */
int occb200_ray_score(const uint8_t* sem_pred, const float* flow_pred, const uint8_t* sem_gt, const float* flow_gt,
                      const void* origins_host, int origin_is_f64, int T, const float* rays_dev, int M, double* counters_dev,
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
/* The tensor-core GEMM (wgmma, bf16 operands, fp32 accumulation) in each of its variants, for operator tests.  Every
 * operand is a dense row-major device array; bias [N] and residual [M,N] are fp32 and may be NULL.  Unsupported shapes,
 * bad codes and NULL required pointers return an error before any CUDA call.
 *   gemm_tc: C [M,N] = act(A . W^T + bias) (+ residual), out_dtype 0 fp32, 1 bf16, 2 fp16; act 0 none / 1 relu.
 *     A bf16 [M,K], or with A2 != NULL the concatenation [A (M x K1) | A2 (M x (K - K1))] along K.  W bf16 [N,K].
 *     M > 0, N % 64 == 0, K % 64 == 0; with A2: K1 % 64 == 0 and 0 < K1 < K. */
int occb200_gemm_tc(const void* A, const void* A2, int K1, const void* W, const float* bias, const float* residual, void* C,
                    int out_dtype, int M, int N, int K, int act, void* stream);
/*   gemm_tc_ln: x = A . W^T + bias + residual, N = 256, y = LayerNorm(x) * gamma + beta (eps 1e-5).  residual, pos and y_f32 are
 *     fp32 in the T32 block layout (32 x 32 blocks of [col % 32 / 4][row % 32][4], rows padded to a multiple of 32); y_bf16 = bf16(y)
 *     and y_pos_bf16 = bf16(y + pos) are row-major [M,256].  Outputs may be NULL; y_pos_bf16 needs pos. */
int occb200_gemm_tc_ln(const void* A, const void* W, const float* bias, const float* residual, const float* gamma,
                       const float* beta, const float* pos, float* y_f32, void* y_bf16, void* y_pos_bf16, int M, int K,
                       void* stream);
/*   gemm_tc_blocked256: C = A . W^T + bias with N % 256 == 0, written as N / 256 bf16 matrices [M,256] at C + i * M * 256. */
int occb200_gemm_tc_blocked256(const void* A, const void* W, const float* bias, void* C, int M, int N, int K, void* stream);
/*   gemm_tc_tsa_inputs: one launch of nv (1 or 2) value problems Cv[i] = bf16(Av[i] . Wv^T + bv) ([M,256], K = 256) and the
 *     projection Cq = fp16([Aq | Aq2] . Wq^T + bq + constant) ([M,Nq], K = Kq, split at K1q when Aq2 != NULL).  The fp32 constant
 *     is rq_t32 (T32 layout) when given and M % 32 == 0, else rq (row-major [M,Nq]); rq_t32 needs rq.  Av, Cv: HOST arrays of nv
 *     device pointers.  bv, bq, rq may be NULL. */
int occb200_gemm_tc_tsa_inputs(const void* const* Av, int nv, const void* Wv, const float* bv, void* const* Cv, const void* Aq,
                               const void* Aq2, int K1q, const void* Wq, const float* bq, const float* rq, const float* rq_t32,
                               void* Cq, int M, int Nq, int Kq, void* stream);
/*   gemm_tc_split3: fp32-grade product C f32 [M,N] = act(S_hi . W_hi^T + S_lo . W_hi^T + S_hi . W_lo^T + bias) (+ residual) from
 *     S = [hi | lo] bf16 [M, 2 Ks] and W3 = [W_hi | W_hi | W_lo] bf16 [N, 3 Ks]; Ks % 64 == 0.
 *   split_bf16: S [rows, 2 (Ka + Kb)] bf16, row r = [hi(a[r]) hi(b[r]) | lo(a[r]) lo(b[r])], hi = bf16(x), lo = bf16(x - hi);
 *     a f32 [rows, Ka], b f32 [rows, Kb] or NULL with Kb = 0; Ka, Kb multiples of 8. */
int occb200_gemm_tc_split3(const void* S, int Ks, const void* W3, const float* bias, const float* residual, float* C, int M, int N,
                           int act, void* stream);
int occb200_split_bf16(const float* a, int Ka, const float* b, int Kb, int64_t rows, void* S, void* stream);

/* The fused deformable-attention gathers of the frame engine, for operator tests: one launch of the kernel the engine launches
 * for the same types.  value_bf16 / qproj_f16 select the storage of the values / outputs (fp32 or bf16) and of the sampling
 * projection (fp32 or fp16); accepted: fp32 / fp32, bf16 / fp32, bf16 / fp16.  All arrays are dense row-major device arrays
 * unless marked HOST.  A NULL required pointer, an unsupported type combination or size returns 1 before any CUDA call.
 *   tsa_gather: v_prev, v_cur [Nq,256] (queue 0 / 1), qproj [Nq,192] = [offsets (head, queue, point, xy) | logits (head,
 *     queue, point)], out [Nq,256] = the mean over the two queues; Nq = bev_h * bev_w, bev_h, bev_w >= 2.
 *   sca_gather: value [num_cams, Nv, 256] (levels in order, Nv = sum h_l * w_l), qproj [Nq,768] = [offsets (head, level, point,
 *     xy) | logits (head, level * point)], out [Nq,256] = the sum over the cameras that see the pillar / max(1, their count),
 *     hits [Nq] (may be NULL) = that count.  cam_mat_host [num_cams,16], zs_host [D], pc_range, the padded image size and the
 *     BEV grid as for occb200_engine_set_cameras; level_hw_host = h0 w0 .. h3 w3.  num_cams in 1..8, D in {1,2,4,8}, every
 *     level at least 2x2, positive image and BEV sizes. */
int occb200_tsa_gather(const void* v_prev, const void* v_cur, int value_bf16, const void* qproj, int qproj_f16, int bev_h,
                       int bev_w, void* out, void* stream);
int occb200_sca_gather(const void* value, int value_bf16, const void* qproj, int qproj_f16, const float* cam_mat_host,
                       const float* zs_host, int num_cams, int D, const float pc_range[6], int img_h, int img_w, int bev_h,
                       int bev_w, const int level_hw_host[8], void* out, uint8_t* hits, void* stream);

/* The voxel decoder's steps, for operator tests: the kernels the frame engine launches for a configuration (precision,
 * use_tensor_cores, num_classes) with pillar_h 16 and out_dim 32, on weights prepared by the engine's own helpers.  Storage is
 * fp32 (precision 0) or bf16 (precision 1); voxels are dense channels-last device arrays [X][Y][16][C].  Every rejection
 * returns 1 before any CUDA call.  Each entry synchronises `stream` and reports the number of kernels it launched.
 *   decoder_lift: vox [W][H][16][16] with vox[x][y][z][cm] = bev[y * W + x][cm * 16 + z] in the storage type, from bev fp32
 *     [H * W, 256] row-major, or with from_t32 (bf16 storage and tensor cores only) in the T32 layout of the residual stream
 *     (32 x 32 blocks of [col % 32 / 4][row % 32][4], rows padded to a multiple of 32).  H * W <= 2^24.
 *   decoder_conv3d: out [X][Y][16][32] = relu(Conv3d 3x3x3, pad 1 (in [X][Y][16][cin]) with BatchNorm3d (eval, eps 1e-5)
 *     folded in), cin 16 or 32, X, Y in [1, 4096].  w_host: HOST fp32 [32][cin][3][3][3] (torch layout, (z, y, x) taps);
 *     bn_host: HOST fp32 [4][32] = gamma | beta | running_mean | running_var.  *path: OCCB200_DECODER_*; the split path
 *     reports 4 launches (the [hi | lo] operand split and three convolution passes).
 *   decoder_head: over vox [nvox][32], occ_logits [nvox][num_classes] = predicter(vox), flow [nvox][2] = flow_predicter(vox),
 *     cls_u8 / cls_i64 [nvox] = the first argmax of the logits; any output may be NULL.  w1 b1 w2 b2 / f1 g1 f2 g2: HOST fp32
 *     predicter.0 / .2 and flow_predicter.0 / .2 weights and biases in torch layout.  num_classes in [1, 32], nvox in
 *     [1, 2^31).  *path: 1 for the tensor-core head (bf16 storage, tensor cores, at most 17 classes), 0 for the CUDA-core one. */
#define OCCB200_DECODER_CUDA_CORES 0   /* conv3d_simt: fp32 weights, fp32 accumulation */
#define OCCB200_DECODER_TC 1           /* conv3d_tc: bf16 weights and operands, fp32 accumulation */
#define OCCB200_DECODER_SPLIT 2        /* conv3d_tc in three passes on bf16 hi / lo splits of fp32 operands and weights */
int occb200_decoder_lift(int precision, int use_tensor_cores, int from_t32, const float* bev, int bev_h, int bev_w, void* vox,
                         int* launches, void* stream);
int occb200_decoder_conv3d(int precision, int use_tensor_cores, const void* in, int X, int Y, int cin, const float* w_host,
                           const float* bn_host, void* out, int* path, int* launches, void* stream);
int occb200_decoder_head(int precision, int use_tensor_cores, int num_classes, const void* vox, int64_t nvox, const float* w1,
                         const float* b1, const float* w2, const float* b2, const float* f1, const float* g1, const float* f2,
                         const float* g2, float* occ_logits, float* flow, uint8_t* cls_u8, int64_t* cls_i64, int* path,
                         int* launches, void* stream);

/* The encoder's unfused kernels, for operator tests: what the frame engine launches for a configuration (precision,
 * use_tensor_cores), on weights prepared by the engine's own helper.  Storage is fp32 (precision 0) or bf16 (precision 1).
 * Every array is a dense row-major device array, 16-byte aligned, unless marked HOST.  Every rejection returns 1 before any
 * CUDA call.  Each entry synchronises `stream`.
 *   encoder_dense: out [M,N] = act([A | A2] . W^T + bias) (+ residual): ReLU (act 1) before the residual add, as every dense
 *     layer of the engine, on the route make_frame_plan's plan picks for the shape.  A: storage type [M,K], or with A2 != NULL
 *     the concatenation [A (M x K1) | A2 (M x (K - K1))], 0 < K1 < K, K1 % 8 == 0 (K1 must be 0 without A2).  w_host: HOST
 *     fp32 [N][K]; bias_host: HOST fp32 [N] or NULL; residual: fp32 [M,N] or NULL.  K % 16 == 0, N % 4 == 0, M >= 0.
 *     out_dtype 0 fp32, 1 bf16, 2 fp16: the storage type or fp32, or fp16 where the plan writes its sampling projections in
 *     fp16 (bf16 storage and tensor cores), on shapes the tensor-core route takes.  *path: OCCB200_DENSE_*; *launches: the
 *     kernels launched (2 on the split route: the entry splits A itself).
 *   encoder_layernorm: LayerNorm over rows x 256 (eps 1e-5) of x fp32: y_f32 fp32, y_t = T(y), y_pos_t = T(y + pos) (the add
 *     in fp32).  Any output may be NULL; y_pos_t needs pos.  rows >= 1.
 *   encoder_pack: tokens [num_cams, Nv, 256] = (level + cams_embeds[cam]) + level_embeds[l] in the storage type, levels in
 *     order, Nv = sum h_l w_l <= 2^24.  layout 0: fp32 NCHW levels [num_cams, 256, h, w]; 1: bf16 NCHW; 2: bf16 NHWC
 *     [num_cams, h, w, 256].  feats_dev: HOST array of num_levels (1..8) device pointers; level_hw_host: HOST h0 w0 h1 w1 ..;
 *     cams_embeds [num_cams,256] or NULL; level_embeds [num_levels,256]; num_cams in 1..8.
 *   encoder_prepare_query: over n (a multiple of 8) floats of q and pos: q_f32 = q (tiled: in the T32 layout of the residual
 *     stream, n a multiple of 256), q_t = T(q), q_pos_t = T(q + pos).  Any output may be NULL.
 *   t32_convert: fp32 [rows, ncols] row-major -> the T32 block layout (32 x 32 blocks of [col % 32 / 4][row % 32][4], rows
 *     padded to a multiple of 32), or back with untile; ncols a positive multiple of 32.  Pad rows are neither read nor
 *     written. */
#define OCCB200_DENSE_CUDA_CORES 0     /* gemm_simt: fp32 weights, fp32 accumulation */
#define OCCB200_DENSE_TC 1             /* gemm_tc: bf16 weights and operands, fp32 accumulation */
#define OCCB200_DENSE_SPLIT 2          /* gemm_tc_split3 on bf16 hi / lo splits of fp32 operands and weights */
int occb200_encoder_dense(int precision, int use_tensor_cores, const void* A, const void* A2, int K1, const float* w_host,
                          const float* bias_host, const float* residual, void* out, int out_dtype, int M, int N, int K, int act,
                          int* path, int* launches, void* stream);
int occb200_encoder_layernorm(int precision, const float* x, const float* gamma, const float* beta, const float* pos, int rows,
                              float* y_f32, void* y_t, void* y_pos_t, void* stream);
int occb200_encoder_pack(int precision, int layout, const void* const* feats_dev, int num_levels, const int* level_hw_host,
                         int num_cams, const float* cams_embeds, const float* level_embeds, void* tokens, void* stream);
int occb200_encoder_prepare_query(int precision, int tiled, const float* q, const float* pos, int64_t n, float* q_f32, void* q_t,
                                  void* q_pos_t, void* stream);
int occb200_t32_convert(const float* src, float* dst, int64_t rows, int untile, int ncols, void* stream);

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
/* Camera frames as the loader produces them: uint8 [num_images, src_h, src_w, 3] (mmcv.imread order, BGR), normalised
 * (to_rgb swap first, then (x - mean[c]) * (1/std[c]) in fp32) and padded bottom/right with 0 to the backbone's H x W
 * inside the stem (NormalizeMultiviewImage + PadMultiViewImage + DefaultFormatBundle3D). src_h <= H, src_w <= W, std != 0.
 * mean / std are indexed in the order of the normalised channels (RGB when to_rgb); 1/std is rounded from double, as
 * mmcv.imnormalize computes it.  Host-side, synchronous; the stem of forward_frames then writes the same im2col operand
 * that _forward writes from the fp32 images the host pipeline would produce, so the outputs are bit-identical to it. */
int occb200_backbone_set_frame_format(occb200_backbone* e, int src_h, int src_w, const float mean[3], const float std[3],
                                      int to_rgb);
/* frames: dev u8 [num_images, src_h, src_w, 3] contiguous (16-byte aligned rows are read with vector loads).
 * out_layout 0: fp32 NCHW (as occb200_backbone_forward, any out may be NULL); 1: bf16 channels-last (as _forward_nhwc_bf16,
 * precision 1 only).  Without a frame format set, or with an out-of-range argument, it returns an error and launches nothing. */
int occb200_backbone_forward_frames(occb200_backbone* e, const uint8_t* frames, void* out0, void* out1, void* out2,
                                    void* out3, int out_layout, void* stream);

/* Single backbone operators, for operator tests: the code the backbone runs, on caller-supplied operands.  Storage is fp32
 * (precision 0) or bf16 (precision 1); tensors are dense NHWC device arrays.  Every rejection returns 1 before any CUDA call.
 *   backbone_conv: out [N, Ho, Wo, cout] = act(conv(in [N, H, W, cin], w) + bias), k x k, `stride`, pad (k - 1) / 2, routed as
 *     the backbone routes the same convolution (use_tensor_cores needs precision 1).  w_host: HOST fp32 [cout][k*k*cin],
 *     BN already folded, tap-major ((ky*k + kx)*cin + ci); rounded to bf16 for the tensor cores as the backbone rounds it.
 *     bias_host: HOST fp32 [cout] or NULL.  residual (NULL, or [N, H, W, cout] with stride 1 and act 1): out = relu(conv + bias
 *     + residual), fused into the convolution where the backbone fuses it, else the convolution rounded to the storage type
 *     and a separate add + ReLU.  cin % 8 == 0 or cin == 3, cout % 8 == 0, k in {1, 3, 7}, stride in {1, 2}.  Synchronises
 *     `stream`.  Reports the path (OCCB200_CONV_*), the number of kernels launched and whether the residual was fused. */
#define OCCB200_CONV_IMPLICIT_TC 1   /* implicit-GEMM tensor-core convolution (conv2d_tc) */
#define OCCB200_CONV_IM2COL_TC 2     /* im2col + tensor-core GEMM */
#define OCCB200_CONV_DIRECT_TC 3     /* tensor-core GEMM on the input as is (1x1, stride 1) */
#define OCCB200_CONV_IM2COL_SIMT 4   /* im2col + CUDA-core GEMM */
#define OCCB200_CONV_DIRECT_SIMT 5   /* CUDA-core GEMM on the input as is */
int occb200_backbone_conv(int precision, int use_tensor_cores, const void* in, int N, int H, int W, int cin, const float* w_host,
                          const float* bias_host, const void* residual, int cout, int k, int stride, int pad, int act, void* out,
                          int* path, int* launches, int* residual_fused, void* stream);
/*   backbone_maxpool: out [N, Ho, Wo, C] = MaxPool2d(3, stride 2, padding 1)(in [N, H, W, C]), C % 8 == 0.
 *   backbone_upsample_add: fine [N, Hf, Wf, C] += F.interpolate(coarse [N, Hc, Wc, C], size (Hf, Wf), mode 'nearest'), the
 *     add in fp32 and rounded to the storage type; C % 8 == 0. */
int occb200_backbone_maxpool(int precision, const void* in, int N, int H, int W, int C, void* out, void* stream);
int occb200_backbone_upsample_add(int precision, void* fine, const void* coarse, int N, int Hf, int Wf, int Hc, int Wc, int C,
                                  void* stream);

/* ---------------------------------------------------------------------------------------------
 * Baseline JPEG decoding on the device, byte-identical to cv2.imdecode(buf, cv2.IMREAD_UNCHANGED) (libjpeg-turbo's default
 * path: ISLOW IDCT, fancy upsampling, integer YCbCr -> BGR), which is what mmcv.imread(name, 'unchanged') runs in
 * LoadMultiViewImageFromFiles.  Supported: SOF0 / SOF1 (sequential Huffman), 8-bit samples and quantisation tables, three
 * YCbCr components in one interleaved scan, 4:2:0 or 4:4:4, any restart interval, any size up to JPEG's 65535 x 65535 with
 * a scan of at most 256 MiB.  Bytes after the last EOI marker are ignored.  Everything else (progressive, arithmetic, 12-bit,
 * 16-bit tables, grayscale, CMYK, Adobe transform, 4:2:2 / 4:4:0 / 4:1:1, several scans, a truncated file, a Huffman table
 * with more codes than its lengths allow) returns 1 on the host, before any CUDA call, with a message naming it.  EXIF orientation is ignored, as IMREAD_UNCHANGED does.
 *
 * _info: host only; the size of one file after the same checks.
 * _decode: n HOST buffers (data[i], sizes[i] bytes); out dev u8 = the n images one after another, image i (h_i, w_i, 3) BGR at
 *   the sum of the earlier images' h * w * 3 bytes; out_bytes must be that total.  The files are parsed on the host, packed
 *   into the decoder's pinned staging buffer (after its previous upload has left it) and uploaded and decoded on `stream`
 *   (three kernels).  The caller's buffers may be reused when the call returns.  Calls on one decoder run in stream order:
 *   use one stream per decoder.
 * _status: after the caller has synchronised the decode's stream, bit i % 32 set = image i's scan was corrupt (an invalid code,
 *   coefficients past the block end, a restart interval that ends early or late, a marker inside the scan).  Such an image
 *   is decoded from zero coefficients (flat grey); nothing is read or written out of bounds, and the next decode is
 *   unaffected. */
typedef struct occb200_jpeg occb200_jpeg;
int occb200_jpeg_create(occb200_jpeg** out);
void occb200_jpeg_destroy(occb200_jpeg* d);
int occb200_jpeg_info(const void* data, int64_t size, int* h, int* w);
int occb200_jpeg_decode(occb200_jpeg* d, int n, const void* const* data, const int64_t* sizes, uint8_t* out, int64_t out_bytes,
                        void* stream);
int occb200_jpeg_status(occb200_jpeg* d, int* status);

/* Input dtype 4 (occb200_engine_set_input_dtype): a frame is the num_cams encoded camera files.  feats[0] points to this HOST
 * descriptor (feats[1..3] are ignored) in every frame call, device or host; data[c] / size[c] are camera c's HOST buffer. */
typedef struct occb200_encoded_frame {
    const void* data[8];
    int64_t size[8];
} occb200_encoded_frame;
/* Status of the last device-call frame (_forward, _forward_video[_angle]) in input dtype 4, once the caller has synchronised
 * its stream: as occb200_jpeg_status.  The host calls check it themselves and return 5 when a camera's scan was corrupt
 * (_forward_host when it returns, _wait_host for a slot). */
int occb200_engine_jpeg_status(occb200_engine* e, int* status);

#ifdef __cplusplus
}
#endif
#endif /* OCC_B200_H_ */
