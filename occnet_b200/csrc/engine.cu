// Host-side frame engine + C ABI (include/occ_b200.h).  One engine = one model replica on one GPU;
// frames are independent (the reference always runs prev_bev=None, bevformer_occ.py:243-244), so the
// multi-GPU story is one engine per rank and no data-path collective.
//
// Per-frame schedule (reference call stack: SURVEY section 3.1):
//   pack_level x4        transformer_occ.py:207-227   (+cams_embeds, +level_embeds, NCHW -> tokens)
//   per encoder layer    encoder.py:356-404           (self_attn, norm, cross_attn, norm, ffn, norm)
//   bev_to_voxel, conv3d x2, occ_head                 transformer_occ.py:305-319, bevformer_occ_head.py:211-212
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/occ_b200.h"
#include "common.cuh"
#include "conv3d_tc.cuh"
#include "gemm_tc.cuh"
#include "jpeg.cuh"
#include "kernels.cuh"

namespace occ {

static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }

namespace {

struct LayerW {
    DevBuf tsa_v_w, tsa_v_b, tsa_q_w, tsa_q_b, tsa_o_w, tsa_o_b;
    DevBuf sca_q_w, sca_q_b, sca_v_w, sca_v_b, sca_o_w, sca_o_b;
    DevBuf ffn1_w, ffn1_b, ffn2_w, ffn2_b;
    DevBuf ln_g[3], ln_b[3];
    // bf16 copies for the tensor-core path
    DevBuf tsa_v_wh, tsa_q_wh, tsa_o_wh, sca_q_wh, sca_v_wh, sca_o_wh, ffn1_wh, ffn2_wh;
    // self mode (prev_bev = None): W1 q + W2 (q + pos) + b == (W1 + W2) q + [W2 pos + b]; the bracket depends on parameters
    // only -> an fp32 [Nq,192] constant per layer, added by the GEMM epilogue (K = 256, weight block resident, A read once)
    DevBuf tsa_q_wh_fold, tsa_q_const, tsa_q_const_t32;   // (_t32: the constant in the T32 block layout, read by the GEMM epilogue)
};

// An armed ray request (occb200_engine_request_rays) and score request (occb200_engine_request_score)
struct RayRequest {
    bool armed = false;
    RayOrigins org;
    int8_t* cls = nullptr;              // device pointers for the device calls, host pointers for the host calls
    void *dist = nullptr, *flow = nullptr;
};
struct ScoreRequest {
    bool armed = false;
    RayOrigins org;
    const uint8_t* sem_gt = nullptr;    // device pointers for the device calls, host pointers for the host calls
    const float* flow_gt = nullptr;
    double* counters = nullptr;         // always a device pointer
};
// what one frame consumes
struct Requests {
    RayRequest rays;
    ScoreRequest score;
};

// The device buffers of a frame: for the host calls the uploaded inputs (four feature levels, or the camera frames in
// feats[0]) and the i64 classes and flow the copies back read; for an armed frame the u8 classes and the flow when the caller
// asked for neither, and for the host calls the staging of a ray request's records and of a score request's ground truth.
// One set for the device calls and _forward_host, one per _submit_host slot (a slot's copies overlap the other slot's kernels).
// Input dtype 4 adds the set's JPEG decoder (its tables, pinned staging and scratch) and the decoded frames it writes.
struct JpegHandle {
    occb200_jpeg* p = nullptr;
    JpegHandle() = default;
    JpegHandle(const JpegHandle&) = delete;
    JpegHandle& operator=(const JpegHandle&) = delete;
    ~JpegHandle() { occb200_jpeg_destroy(p); }
};
struct FrameBufs {
    DevBuf feats[4], occ, flow, sem, rec_cls, rec_dist, rec_flow, gt_sem, gt_flow, frames;
    JpegHandle jpeg;
};

// _submit_host uploads an input buffer above 32 MB in two pieces on two copy streams: when the split was tuned, one
// cudaMemcpyAsync stream reached 46 GB/s of the PCIe link and two reached 50 GB/s.
constexpr int kH2DSplit = 2;

// A frame's outputs on the device (any may be NULL)
struct FrameOut {
    float* bev_embed = nullptr;
    float* occ_logits = nullptr;
    float* flow = nullptr;
    uint8_t* cls_u8 = nullptr;
    int64_t* cls_i64 = nullptr;
};

// Where a frame's previous BEV comes from: none (self mode, prev_bev = None), a caller's fp32 prev_bev [Nq, 256], or the engine
// history (a video frame after the first of its scene).  The rotation applied to it is a device map of source cells (NULL = no
// rotation) or, when `grid` is set, the source cells computed from grid coefficients.  A video frame also writes the history.
struct PrevBev {
    enum Source { NONE, CALLER, HISTORY } src = NONE;
    const float* bev = nullptr;         // CALLER
    const int32_t* map = nullptr;
    const RotGrid* grid = nullptr;
    bool writes_history = false;
};

// The kernel path of every frame, decided once at finalize from the precision, use_tensor_cores and the shapes
// (make_frame_plan).  finalize builds exactly the buffers these fields call for and the frame reads only these fields; what
// varies per frame is the previous BEV, the history write, taps, bev_embed and the input layout.
struct FramePlan {
    // bf16 storage + tensor cores: bf16 weight copies, the SCA value maps of every layer in one launch, and (with taps off)
    // LayerNorm fused into the GEMM epilogues with the fp32 residual stream in the T32 layout and layer 0's operands built once
    bool tc_bf16 = false;
    // fp32 storage + tensor cores: GEMMs on bf16 [hi | lo] operand splits and [W_hi | W_hi | W_lo] weights (fp32-grade), the
    // camera tokens split once per frame
    bool tc_split = false;
    // the sampling-offset / attention-logit projections write fp16 (half the bytes between the projection GEMM and the gather
    // kernel; |offset| is a few pixels, so fp16's 11-bit mantissa keeps locations to < 0.01 px)
    bool qproj_f16 = false;
    // self mode on the fused path: layer 0's TSA + LayerNorm see only parameters and are computed once at finalize
    // (OCC_NO_L0_FOLD=1 at finalize: recomputed every frame instead)
    bool fold_layer0 = false;
    // the two 3-D convolutions: CUDA cores, bf16 tensor cores, or three bf16-split tensor-core passes accumulated in fp32
    enum Conv { CONV_SIMT, CONV_TC, CONV_SPLIT } conv = CONV_SIMT;
    bool head_tc = false;               // occupancy + flow heads in one tensor-core kernel (concatenated weights)
    bool lift_t32 = false;              // the shapes let the voxel lift read the T32 residual stream directly
};

// The voxel decoder's weights on the device, built from the torch-layout parameters by upload_decoder_conv /
// upload_decoder_head for the engine (finalize) and for the occb200_decoder_* test entries alike
struct DecoderConvW {
    DevBuf w, b;                        // BatchNorm folded in: fp32 [27][cin][32] (tap = (dz*3+dy)*3+dx) and [32] (every path)
    DevBuf wh;                          // CONV_TC: bf16 tap-major [27][32][cin] (K-major rows)
    DevBuf wh_hi, wh_lo;                // CONV_SPLIT: the same layout split into bf16 hi + lo
};
struct DecoderHeadW {
    DevBuf w1, b1, w2, b2, fw1, fb1, fw2, fb2;      // predicter / flow_predicter in torch layout, fp32 (CUDA-core head)
    // head_tc: [predicter.0 ; flow_predicter.0] bf16 [128][32], block-diagonal [predicter.2 ; flow_predicter.2] bf16 [32][128]
    // (flow rows at num_classes, num_classes + 1), biases [128] and [num_classes + 2]
    DevBuf w1h, w2h, b1c, b2c;
};

}  // namespace
}  // namespace occ

using namespace occ;

struct occb200_engine {
    occb200_config cfg;
    FramePlan plan;
    int Nq = 0, Nv = 0, C = 256;
    LevelGeom lg;
    ScaParams sp;
    bool cameras_set = false, finalized = false, taps = false;
    // the rotation of occb200_engine_forward's prev_bev, set by the last of occb200_engine_set_prev_rotation (ROT_MAP: source
    // row of every BEV cell, int32, -1 = outside; NULL clears it) and occb200_engine_set_prev_rotation_angle (ROT_GRID)
    enum { ROT_NONE, ROT_MAP, ROT_GRID } rot = ROT_NONE;
    DevBuf rot_map;
    RotGrid rot_grid;
    // occb200_engine_set_history: the last video frame's final BEV [Nq, 256] in the storage type (the bf16 / fp32 copy the last
    // LayerNorm writes), read and written only by the video calls; hist_done is recorded after every video frame
    DevBuf hist;
    bool hist_valid = false;            // a video frame has written it since set_history(e, 1)
    cudaEvent_t hist_done = nullptr;
    bool hist_recorded = false;
    int feats_bf16 = 0;                 // occb200_engine_set_input_dtype: feature levels arrive as bf16 instead of fp32
    // input dtype 3 (uint8 camera frames): the attached backbone (borrowed), the levels it hands over (shared by both host
    // slots, like its workspace) and the event after the last frame that read them
    occb200_backbone* bb = nullptr;
    DevBuf bb_levels[4];
    cudaEvent_t bb_free = nullptr;
    bool bb_free_recorded = false;
    std::map<std::string, std::vector<float>> host_params;
    std::vector<LayerW> layers;
    DevBuf bev_queries, pos, pos_t32, cams_embeds, level_embeds;
    DevBuf qc_f32, qc_t, qc_pos_t;      // parameter-only layer-0 operands (query fp32 T32, bf16 query, bf16 query+pos), built once
    // Self mode (prev_bev = None): layer 0's TemporalSelfAttention + its LayerNorm see only parameters (bev_queries, bev_pos,
    // weights) -- the result is frame-independent and is computed ONCE at finalize by the same kernels (T32 fp32 + bf16 copy)
    DevBuf l0_x_f32, l0_q_t;
    DecoderConvW dec_conv[2];
    DevBuf vox_split;                                    // CONV_SPLIT: the [hi | lo] bf16 voxel operand
    DevBuf sca_v_all_wh, sca_v_all_b, sca_value_all;     // value_proj of every layer, concatenated (tensor-core path)
    // TSA queue 1 with a previous BEV (encoder.py:204-209 stacks the layer-0 query once): value_proj_l(bev_queries) of every
    // layer, [L][Nq,256] in the storage type -- parameters only, computed at finalize by the frame path's own GEMM
    DevBuf tsa_v_query;
    DecoderHeadW head;
    // workspace
    DevBuf tokens, sca_value, q_f32, q_t, q_pos_t, prev_t, tsa_value, qproj, attn_out, x_f32,
        ffn_h, vox0, vox1, vox2, hits;
    DevBuf tap_layer, tap_tsa, tap_sca;
    // fp32-grade tensor-core configuration (precision 0 + use_tensor_cores): bf16 [hi | lo] splits of the GEMM operands
    DevBuf split_ws, tokens_split;
    // ray records (occb200_engine_set_rays / _request_rays): the constant ray bundle, and the request the next frame consumes.
    // The origins travel inside the request and then as a kernel argument, so nothing is uploaded per frame.
    DevBuf rays;
    int rays_M = 0;
    RayRequest ray_req;
    ScoreRequest score_req;             // the frame scores itself against this ground truth into the caller's 187 device counters
    FrameBufs bufs;                     // the device calls' and _forward_host's buffer set
    // pipelined host-buffer variant: 2 slots, copies on their own streams, compute on the caller's stream
    struct Slot {
        FrameBufs bufs;
        DevBuf rot;                     // _submit_host_video: the frame's rotation map, uploaded from rot_pinned on h2d_stream[0]
        int32_t* rot_pinned = nullptr;
        cudaEvent_t h2d_done[kH2DSplit] = {}, compute_done = nullptr, d2h_done = nullptr;
        bool busy = false;
        bool jpeg = false;              // the frame in flight decodes JPEG files: _wait_host checks their status
    } slots[2];
    cudaStream_t h2d_stream[kH2DSplit] = {}, d2h_stream = nullptr;
    int launches = 0;
    // optional per-kernel-category timing (CUDA events on the launch stream)
    bool profiling = false;
    std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> prof_events;
    std::vector<cudaEvent_t> event_pool;
    size_t event_used = 0;
    size_t elt() const { return cfg.precision ? 2 : 4; }
};

namespace {

int upload(DevBuf& b, const float* src, size_t n)
{
    if (b.alloc(n * sizeof(float))) return 2;
    OCC_CUDA(cudaMemcpy(b.p, src, n * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

// [W_hi | W_hi | W_lo] (n x 3k bf16) of an n x k fp32 weight: B operand of gemm_tc_split3
int upload_w3(DevBuf& b, const float* W, size_t n, size_t k)
{
    std::vector<__nv_bfloat16> h(n * 3 * k);
    for (size_t r = 0; r < n; ++r)
        for (size_t j = 0; j < k; ++j) {
            const float w = W[r * k + j];
            const __nv_bfloat16 hi = __float2bfloat16(w);
            const __nv_bfloat16 lo = __float2bfloat16(w - __bfloat162float(hi));
            h[r * 3 * k + j] = hi; h[r * 3 * k + k + j] = hi; h[r * 3 * k + 2 * k + j] = lo;
        }
    if (b.alloc(h.size() * 2)) return 2;
    OCC_CUDA(cudaMemcpy(b.p, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
    return 0;
}

int upload_bf16(DevBuf& b, const float* src, size_t n)
{
    std::vector<__nv_bfloat16> h(n);
    for (size_t i = 0; i < n; ++i) h[i] = __float2bfloat16(src[i]);
    if (b.alloc(n * 2)) return 2;
    OCC_CUDA(cudaMemcpy(b.p, h.data(), n * 2, cudaMemcpyHostToDevice));
    return 0;
}

const std::vector<float>* find(const occb200_engine* e, const std::string& k, size_t numel)
{
    auto it = e->host_params.find(k);
    if (it == e->host_params.end()) { set_last_error("missing parameter: " + k); return nullptr; }
    if (it->second.size() != numel) {
        set_last_error("parameter " + k + " has " + std::to_string(it->second.size()) + " elements, expected " +
                       std::to_string(numel));
        return nullptr;
    }
    return &it->second;
}

// ---- voxel decoder weights (transformer_occ.py:106-141): built here for the engine (finalize) and for the occb200_decoder_*
// test entries alike, so that the operator tests run the kernels on exactly the weights the engine builds
// BatchNorm3d (eval) folded into the bias-free Conv3d in fp32: s = gamma / sqrt(var + 1e-5), wf = w s, bf = beta - mean s;
// torch layout [od][cin][27] -> wf [27][cin][od]
void fold_conv3d_bn(const float* W, const float* gamma, const float* beta, const float* mean, const float* var, int cin, int od,
                    std::vector<float>& wf, std::vector<float>& bf)
{
    wf.assign((size_t)27 * cin * od, 0.f);
    bf.assign(od, 0.f);
    for (int co = 0; co < od; ++co) {
        const float s = gamma[co] / sqrtf(var[co] + 1e-5f);
        bf[co] = beta[co] - mean[co] * s;
        for (int ci = 0; ci < cin; ++ci)
            for (int t = 0; t < 27; ++t) wf[((size_t)t * cin + ci) * od + co] = W[((size_t)co * cin + ci) * 27 + t] * s;
    }
}

// wf [27][cin][od] -> the tensor cores' tap-major [27][od][cin] (K-major rows)
std::vector<float> conv3d_tap_major(const std::vector<float>& wf, int cin, int od)
{
    std::vector<float> wt((size_t)27 * od * cin);
    for (int t = 0; t < 27; ++t)
        for (int co = 0; co < od; ++co)
            for (int ci = 0; ci < cin; ++ci) wt[((size_t)t * od + co) * cin + ci] = wf[((size_t)t * cin + ci) * od + co];
    return wt;
}

// One decoder layer's weights for the plan's convolution path: the folded fp32 weights and bias, and on the tensor cores the
// tap-major bf16 copy (CONV_TC) or its bf16 hi + lo split, lo = bf16(w - hi) (CONV_SPLIT, the 3-pass fp32-grade convolution)
int upload_decoder_conv(DecoderConvW& d, FramePlan::Conv path, const float* W, const float* gamma, const float* beta,
                        const float* mean, const float* var, int cin, int od)
{
    std::vector<float> wf, bf;
    fold_conv3d_bn(W, gamma, beta, mean, var, cin, od, wf, bf);
    if (upload(d.w, wf.data(), wf.size()) || upload(d.b, bf.data(), bf.size())) return 2;
    if (path == FramePlan::CONV_SIMT) return 0;
    const std::vector<float> wt = conv3d_tap_major(wf, cin, od);
    if (path == FramePlan::CONV_TC) return upload_bf16(d.wh, wt.data(), wt.size());
    std::vector<float> hi(wt.size()), lo(wt.size());
    for (size_t i = 0; i < wt.size(); ++i) {
        hi[i] = __bfloat162float(__float2bfloat16(wt[i]));
        lo[i] = wt[i] - hi[i];
    }
    return upload_bf16(d.wh_hi, hi.data(), hi.size()) || upload_bf16(d.wh_lo, lo.data(), lo.size()) ? 2 : 0;
}

// The occupancy / flow heads' weights, torch layout: w1 / f1 [2 od][od], b1 / g1 [2 od], w2 [nc][2 od], b2 [nc], f2 [2][2 od],
// g2 [2].  head_tc adds the concatenated first layer and the block-diagonal second layer (flow rows at nc, nc + 1) in bf16.
int upload_decoder_head(DecoderHeadW& h, bool head_tc, int nc, int od, const float* w1, const float* b1, const float* w2,
                        const float* b2, const float* f1, const float* g1, const float* f2, const float* g2)
{
    const int H = 2 * od;
    if (upload(h.w1, w1, (size_t)H * od) || upload(h.b1, b1, H) || upload(h.w2, w2, (size_t)nc * H) || upload(h.b2, b2, nc) ||
        upload(h.fw1, f1, (size_t)H * od) || upload(h.fb1, g1, H) || upload(h.fw2, f2, (size_t)2 * H) || upload(h.fb2, g2, 2))
        return 2;
    if (!head_tc) return 0;
    std::vector<float> w1c((size_t)2 * H * od), b1c(2 * H), w2c((size_t)32 * 2 * H, 0.f), b2c(nc + 2);
    for (int i = 0; i < H * od; ++i) { w1c[i] = w1[i]; w1c[(size_t)H * od + i] = f1[i]; }
    for (int i = 0; i < H; ++i) { b1c[i] = b1[i]; b1c[H + i] = g1[i]; }
    for (int r = 0; r < nc; ++r)
        for (int k = 0; k < H; ++k) w2c[(size_t)r * 2 * H + k] = w2[(size_t)r * H + k];
    for (int r = 0; r < 2; ++r)
        for (int k = 0; k < H; ++k) w2c[(size_t)(nc + r) * 2 * H + H + k] = f2[(size_t)r * H + k];
    for (int i = 0; i < nc; ++i) b2c[i] = b2[i];
    b2c[nc] = g2[0]; b2c[nc + 1] = g2[1];
    if (upload_bf16(h.w1h, w1c.data(), w1c.size()) || upload_bf16(h.w2h, w2c.data(), w2c.size()) ||
        upload(h.b1c, b1c.data(), b1c.size()) || upload(h.b2c, b2c.data(), b2c.size())) return 2;
    return 0;
}

// ---- geometry of the fused spatial cross-attention gather: built here for the engine (creation, set_cameras) and for the
// occb200_sca_gather test entry alike, so that the operator tests launch the kernels on exactly what the engine builds
// the value-map levels of every camera (four in the engine, up to eight for the occb200_encoder_pack test entry), rows
// [start, start + h*w) of the [Nv, 256] map; *Nv = the total
LevelGeom make_level_geom(const int* level_h, const int* level_w, int* Nv, int num_levels = 4)
{
    LevelGeom lg{};
    lg.num_levels = num_levels;
    int start = 0;
    for (int l = 0; l < num_levels; ++l) {
        lg.h[l] = level_h[l]; lg.w[l] = level_w[l]; lg.start[l] = start;
        start += level_h[l] * level_w[l];
    }
    *Nv = start;
    return lg;
}

// cam_mat [num_cams,16] = lidar2img[c] @ ego2lidar, zs [D] normalised pillar heights, pc_range, padded image size, BEV grid
ScaParams make_sca_params(const float* cam_mat, const float* zs, int num_cams, int D, const float* pc_range, int img_h,
                          int img_w, int bev_h, int bev_w)
{
    ScaParams sp;
    memset(&sp, 0, sizeof(sp));
    for (int i = 0; i < num_cams; ++i)
        for (int k = 0; k < 16; ++k) sp.cam_mat[i][k] = cam_mat[i * 16 + k];
    for (int i = 0; i < D; ++i) sp.zs[i] = zs[i];
    for (int i = 0; i < 3; ++i) {
        sp.pc_scale[i] = (float)((double)pc_range[3 + i] - (double)pc_range[i]);
        sp.pc_min[i] = pc_range[i];
    }
    sp.img_w = (float)img_w; sp.img_h = (float)img_h;
    sp.num_cams = num_cams; sp.D = D; sp.bev_h = bev_h; sp.bev_w = bev_w;
    return sp;
}

#define GETP(var, key, n)                            \
    const std::vector<float>* var = find(e, key, n); \
    if (!var) return 3;

// ---- per-category timing.  Categories: 0 pack/prepare, 1 gemm, 2 tsa gather, 3 sca gather, 4 layernorm,
//      5 bev_to_voxel, 6 conv3d, 7 occ head
enum { CAT_PACK = 0, CAT_GEMM, CAT_TSA, CAT_SCA, CAT_LN, CAT_VOX, CAT_CONV, CAT_HEAD, CAT_COUNT };
struct ProfScope {
    occb200_engine* e; cudaStream_t st; int cat; cudaEvent_t a = nullptr, b = nullptr;
    static cudaEvent_t get(occb200_engine* e) {
        if (e->event_used == e->event_pool.size()) {
            cudaEvent_t ev; cudaEventCreate(&ev); e->event_pool.push_back(ev);
        }
        return e->event_pool[e->event_used++];
    }
    ProfScope(occb200_engine* e_, cudaStream_t st_, int cat_) : e(e_), st(st_), cat(cat_) {
        if (e->profiling) { a = get(e); b = get(e); cudaEventRecord(a, st); }
    }
    ~ProfScope() {
        if (e->profiling) { cudaEventRecord(b, st); e->prof_events.push_back({cat, {a, b}}); }
    }
};

FramePlan make_frame_plan(const occb200_config& c, int Nq)
{
    const int C = 256;
    FramePlan p;
    p.tc_bf16 = c.precision == 1 && c.use_tensor_cores;
    p.tc_split = c.precision == 0 && c.use_tensor_cores;
    p.qproj_f16 = p.tc_bf16 && gemm_tc_supported(Nq, 2 * 8 * c.tsa_points * 3, 2 * C, C) &&
                  gemm_tc_supported(Nq, 8 * c.num_levels * c.sca_points * 3, C, C);
    p.fold_layer0 = p.tc_bf16 && getenv("OCC_NO_L0_FOLD") == nullptr;
    if (p.tc_bf16 && c.pillar_h == 16) p.conv = FramePlan::CONV_TC;
    if (p.tc_split && c.pillar_h == 16 && c.out_dim == 32) p.conv = FramePlan::CONV_SPLIT;
    p.head_tc = p.conv == FramePlan::CONV_TC && c.out_dim == 32 && c.num_classes + 2 <= 19;
    p.lift_t32 = p.tc_bf16 && c.pillar_h == 16;
    return p;
}

// ---- voxel decoder steps (transformer_occ.py:305-319), run by decode_stage and by the occb200_decoder_* test entries.  Each
// enqueues its kernels on `st` and returns how many it launched, or -1 when a launcher failed (its message is set).
// The lift: bev [H*W, 256] fp32 (from_t32: the T32 layout of the residual stream, bf16 voxels, Z = 16) -> vox [W][H][Z][256/Z]
template <typename T>
int decoder_lift(bool from_t32, const float* bev, int bev_h, int bev_w, int Z, T* vox, cudaStream_t st)
{
    if (from_t32) return launch_t32_to_voxel(bev, bev_h, bev_w, reinterpret_cast<bf16*>(vox), st) ? -1 : 1;
    return launch_bev_to_voxel<T>(bev, bev_h, bev_w, Z, 256 / Z, vox, st) ? -1 : 1;
}

// One Conv3d + folded BatchNorm + ReLU layer on the plan's path: in [X][Y][Z][cin] -> out [X][Y][Z][32] in the storage type T.
// CONV_SPLIT (T = float) first splits `in` into the [hi | lo] bf16 workspace `split` [X*Y*Z][2 cin].
template <typename T>
int decoder_conv(FramePlan::Conv path, const T* in, const DecoderConvW& w, int X, int Y, int Z, int cin, T* out, bf16* split,
                 cudaStream_t st)
{
    if (path == FramePlan::CONV_SPLIT) {
        if (launch_split_bf16(reinterpret_cast<const float*>(in), cin, nullptr, 0, (int64_t)X * Y * Z, split, st)) return -1;
        if (launch_conv3d_tc_split(split, w.wh_hi.as<bf16>(), w.wh_lo.as<bf16>(), w.b.as<float>(), X, Y, Z, cin,
                                   reinterpret_cast<float*>(out), st)) return -1;
        return 4;                                                   // the split and the launcher's three passes
    }
    if (path == FramePlan::CONV_TC)
        return launch_conv3d_tc(reinterpret_cast<const bf16*>(in), w.wh.as<bf16>(), w.b.as<float>(), X, Y, Z, cin,
                                reinterpret_cast<bf16*>(out), st) ? -1 : 1;
    return launch_conv3d_simt<T>(in, w.w.as<float>(), w.b.as<float>(), X, Y, Z, cin, out, st) ? -1 : 1;
}

// The occupancy / flow heads and the argmax over vox [nvox][32]; any output may be NULL
template <typename T>
int decoder_head(bool head_tc, const T* vox, const DecoderHeadW& h, int nc, int64_t nvox, float* occ_logits, float* flow,
                 uint8_t* cls_u8, int64_t* cls_i64, cudaStream_t st)
{
    if (head_tc)
        return launch_occ_head_tc(reinterpret_cast<const bf16*>(vox), h.w1h.as<bf16>(), h.w2h.as<bf16>(), h.b1c.as<float>(),
                                  h.b2c.as<float>(), nc, nvox, occ_logits, flow, cls_u8, cls_i64, st) ? -1 : 1;
    const HeadWeights hw{h.w1.as<float>(), h.b1.as<float>(), h.w2.as<float>(), h.b2.as<float>(),
                         h.fw1.as<float>(), h.fb1.as<float>(), h.fw2.as<float>(), h.fb2.as<float>(), nc};
    return launch_occ_head<T>(vox, hw, nvox, occ_logits, flow, cls_u8, cls_i64, st) ? -1 : 1;
}

// the plan of the occb200_decoder_* test entries: a configuration with the engine's decoder shapes (pillar_h 16, out_dim 32)
FramePlan decoder_test_plan(int precision, int use_tensor_cores, int num_classes)
{
    occb200_config c;
    memset(&c, 0, sizeof(c));
    c.precision = precision; c.use_tensor_cores = use_tensor_cores; c.num_classes = num_classes;
    c.pillar_h = 16; c.out_dim = 32;
    return make_frame_plan(c, 1);
}

// the plan of the occb200_encoder_* test entries: a configuration with the engine's attention shapes (4 levels, 8 SCA and 4 TSA
// points), so that the plan's fp16 sampling projections are what a frame gets
FramePlan encoder_test_plan(int precision, int use_tensor_cores)
{
    occb200_config c;
    memset(&c, 0, sizeof(c));
    c.precision = precision; c.use_tensor_cores = use_tensor_cores;
    c.num_levels = 4; c.sca_points = 8; c.tsa_points = 4;
    return make_frame_plan(c, 1);
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// ---- dense layers (nn.Linear, W [n][k]): built here for the engine (finalize) and for the occb200_encoder_dense test entry
// alike.  fp32 W and bias on every route (bias may be NULL); for the plan's tensor-core route `wh` (NULL: none) gets the bf16
// copy (tc_bf16) or [W_hi | W_hi | W_lo] (tc_split).
int upload_dense(const FramePlan& p, DevBuf& w, DevBuf& b, DevBuf* wh, const float* W, const float* B, size_t n, size_t k)
{
    if (upload(w, W, n * k) || (B && upload(b, B, n))) return 2;
    if (p.tc_bf16 && wh && upload_bf16(*wh, W, n * k)) return 2;
    if (p.tc_split && wh && upload_w3(*wh, W, n, k)) return 2;
    return 0;
}

// The route of one dense layer (OCCB200_DENSE_*): the plan's tensor-core GEMM where the shape allows it, the CUDA-core GEMM
// otherwise.  Ka: the width of the first operand block (K without a second block).
template <typename TA, typename TC>
int dense_route(const FramePlan& p, int M, int N, int K, int Ka)
{
    if constexpr (sizeof(TA) == 2)
        if (p.tc_bf16 && gemm_tc_supported(M, N, K, Ka)) return OCCB200_DENSE_TC;
    if constexpr (sizeof(TA) == 4 && std::is_same<TC, float>::value)
        if (p.tc_split && gemm_tc_supported(M, N, 3 * K, 2 * K)) return OCCB200_DENSE_SPLIT;
    return OCCB200_DENSE_CUDA_CORES;
}

// C = act([A | A2] . W^T + bias) (+ residual) on the plan's route, run by the engine's gemm() and by occb200_encoder_dense.
// Enqueues on `st` and returns how many kernels it launched, or -1 when a launcher failed (its message is set).  W: fp32
// [N][K]; Wh: the route's weight copy (upload_dense).  The split route first splits the operand into `split_ws` ([M, 2K]
// bf16) unless `A_split` holds it already split (the camera tokens, once per frame).
template <typename TA, typename TC>
int dense_gemm(const FramePlan& p, const TA* A, const TA* A2, int K1, const float* W, const void* Wh, const float* bias,
               const float* residual, TC* C, int M, int N, int K, int act, bf16* split_ws, cudaStream_t st,
               const bf16* A_split = nullptr)
{
    const int Ka = A2 ? K1 : K;
    const int route = dense_route<TA, TC>(p, M, N, K, Ka);
    if constexpr (sizeof(TA) == 2) {
        if (route == OCCB200_DENSE_TC)
            return gemm_tc<TC>(reinterpret_cast<const bf16*>(A), reinterpret_cast<const bf16*>(A2), K1,
                               reinterpret_cast<const bf16*>(Wh), bias, residual, C, M, N, K, act, st) ? -1 : 1;
    }
    if constexpr (sizeof(TA) == 4 && std::is_same<TC, float>::value) {
        // fp32 storage + tensor cores: operand split into bf16 hi/lo, weights [W_hi | W_hi | W_lo], three passes in one
        // wgmma GEMM (relative error ~2^-16: fp32-grade)
        if (route == OCCB200_DENSE_SPLIT) {
            const bf16* S = A_split;
            if (S == nullptr) {
                if (launch_split_bf16(reinterpret_cast<const float*>(A), Ka, reinterpret_cast<const float*>(A2), K - Ka, M,
                                      split_ws, st)) return -1;
                S = split_ws;
            }
            if (gemm_tc_split3(S, K, reinterpret_cast<const bf16*>(Wh), bias, residual, C, M, N, act, st)) return -1;
            return A_split ? 1 : 2;
        }
    }
    if constexpr (std::is_same<TC, __half>::value) {
        set_last_error("gemm: fp16 outputs exist only on the tensor-core path");
        return -1;
    } else {
        if (gemm_simt<TA, TC>(A, Ka, A2, A2 ? K - K1 : 0, K1, W, bias, residual, N, C, N, M, N, K, act, st)) return -1;
        return M > 0 ? 1 : 0;
    }
}

// ---- the engine's GEMM: dense_gemm on the engine's plan and split workspace, counted and profiled as one GEMM
template <typename TA, typename TC>
int gemm(occb200_engine* e, const TA* A, const TA* A2, int K1, const float* W, const void* Wh, const float* bias,
         const float* residual, TC* C, int M, int N, int K, int act, cudaStream_t st, const bf16* A_split = nullptr)
{
    ProfScope ps(e, st, CAT_GEMM);
    const int n = dense_gemm<TA, TC>(e->plan, A, A2, K1, W, Wh, bias, residual, C, M, N, K, act, e->split_ws.as<bf16>(), st,
                                     A_split);
    if (n < 0) return 2;
    e->launches += n;
    return 0;
}

// y = LayerNorm(A.W^T + b + residual): one wgmma kernel (GEMM with LayerNorm epilogue) on the tensor-core path
int gemm_ln_fused(occb200_engine* e, const bf16* A, const void* Wh, const float* bias, const float* residual,
                  const float* gamma, const float* beta, const float* pos, float* y_f32, bf16* y_t, bf16* y_pos_t, int M,
                  int K, cudaStream_t st)
{
    e->launches++;
    ProfScope ps(e, st, CAT_GEMM);
    return gemm_tc_ln(A, reinterpret_cast<const bf16*>(Wh), bias, residual, gamma, beta, pos, y_f32, y_t, y_pos_t, M, K, st);
}

// TSA's queue-1 value maps value_proj_l(bev_queries) for every layer, with the GEMM the frame path would run on the same
// operand (bf16 tensor cores: rows do not depend on how problems share a launch, so they equal the merged TSA-input launch's)
template <typename T>
int build_tsa_query_values(occb200_engine* e)
{
    const int Nq = e->Nq, C = 256;
    DevBuf q0;
    if (q0.alloc((size_t)Nq * C * sizeof(T)) || e->tsa_v_query.alloc((size_t)e->cfg.num_layers * Nq * C * sizeof(T))) return 2;
    if (launch_cast<T>(e->bev_queries.as<float>(), q0.as<T>(), (int64_t)Nq * C, 0)) return 2;
    for (int l = 0; l < e->cfg.num_layers; ++l) {
        LayerW& w = e->layers[l];
        if (gemm<T, T>(e, q0.as<T>(), nullptr, 0, w.tsa_v_w.as<float>(), w.tsa_v_wh.p, w.tsa_v_b.as<float>(), nullptr,
                       e->tsa_v_query.as<T>() + (size_t)l * Nq * C, Nq, C, C, ACT_NONE, 0)) return 2;
    }
    OCC_CUDA(cudaDeviceSynchronize());
    return 0;
}

// torchvision's rotate(img, angle_deg, center=[cx, cy]) of a bev_h x bev_w image as the six grid coefficients its
// _gen_affine_grid multiplies the base grid with, computed as torchvision computes them: _get_inverse_affine_matrix(center -
// size / 2, -angle) in double (zero translation and shear, scale 1: [cos, sin, t0; -sin, cos, t1] about the centre), cast to
// fp32, then divided in fp32 by [W / 2, H / 2].  out = {row x: r0 r1 r2, row y: r3 r4 r5}.  Host only.
void rotation_coeffs(double angle_deg, int bev_h, int bev_w, int cx, int cy, float out[6])
{
    constexpr double kDegToRad = 3.141592653589793 / 180.0;          // math.radians
    const double rot = -angle_deg * kDegToRad;
    const double c = std::cos(rot), s = std::sin(rot);
    const double ccx = (double)cx - (double)bev_w * 0.5, ccy = (double)cy - (double)bev_h * 0.5;
    double m[6] = {c, s, 0.0, -s, c, 0.0};
    m[2] += m[0] * -ccx + m[1] * -ccy;                                  // inverse rotation of the centred grid ...
    m[5] += m[3] * -ccx + m[4] * -ccy;
    m[2] += ccx;                                                        // ... moved back to the centre
    m[5] += ccy;
    const float sx = (float)(0.5 * bev_w), sy = (float)(0.5 * bev_h);
    for (int k = 0; k < 3; ++k) {
        out[k] = (float)m[k] / sx;
        out[3 + k] = (float)m[3 + k] / sy;
    }
}

RotGrid rotation_grid(const occb200_engine* e, double angle_deg)
{
    RotGrid g;
    rotation_coeffs(angle_deg, e->cfg.bev_h, e->cfg.bev_w, e->cfg.rotate_center[0], e->cfg.rotate_center[1], g.r);
    g.bev_h = e->cfg.bev_h;
    g.bev_w = e->cfg.bev_w;
    return g;
}

// The fp32 residual stream of a frame (T32 layout on the fused path).  `cur` is the stream; the next fused LayerNorm writes
// `next`, which advance() makes the stream.  The stream may start on a parameter-only constant (layer 0's query, or its
// folded TSA output) that is read and never written: `next` and `other` are the two workspace buffers it then alternates
// between.  The unfused path writes each LayerNorm's output back into `cur` and uses `next` for the pre-LayerNorm sum.
struct Residual {
    float* cur;
    float* next;
    float* other;
    void advance() { cur = next; std::swap(next, other); }
};

// ---- camera tokens (transformer_occ.py:207-227: +cams_embeds, +level_embeds, NCHW -> tokens) and, on the split path, their
// bf16 [hi | lo] split, which every layer's SCA value GEMM reads
template <typename T>
int pack_stage(occb200_engine* e, const float* const* feats, int layout, cudaStream_t st)
{
    const int C = 256, ncam = e->cfg.num_cams, Nv = e->Nv;
    T* tokens = e->tokens.as<T>();
    {
        ProfScope ps(e, st, CAT_PACK);
        if (layout == 2) {
            if (launch_pack_levels_nhwc<T>(reinterpret_cast<const void* const*>(feats), e->lg, e->cams_embeds.as<float>(),
                                           e->level_embeds.as<float>(), ncam, C, Nv, tokens, st)) return 2;
        } else if (launch_pack_levels<T>(reinterpret_cast<const void* const*>(feats), layout, e->lg, e->cams_embeds.as<float>(),
                                         e->level_embeds.as<float>(), ncam, C, Nv, tokens, st)) return 2;
        e->launches++;
    }
    if (e->plan.tc_split) {
        ProfScope ps(e, st, CAT_PACK);
        if (launch_split_bf16(reinterpret_cast<const float*>(tokens), C, nullptr, 0, (int64_t)ncam * Nv,
                              e->tokens_split.as<bf16>(), st)) return 2;
        e->launches++;
    }
    return 0;
}

// ---- temporal self-attention of layer l (temporal_self_attention.py:177-272) and its LayerNorm.  q_in / q_pos_in: the
// storage-type query and query + pos; the LayerNorm output goes to the stream and to y_t.  `fuse_ln`: LayerNorm in the GEMM
// epilogues (the plan's tc_bf16 with taps off).  finalize runs layer 0 of self mode through here once to fold it.
template <typename T>
int tsa_stage(occb200_engine* e, bool fuse_ln, bool has_prev, int l, const T* q_in, const T* q_pos_in, Residual& rs, T* y_t,
              cudaStream_t st)
{
    const int Nq = e->Nq, C = 256, nq_tsa = 2 * 8 * e->cfg.tsa_points * 3;     // offsets (x,y) + logits
    const bool q_half = e->plan.qproj_f16;
    LayerW& w = e->layers[l];
    void* qproj = e->qproj.p;
    T* attn_out = e->attn_out.as<T>();
    // one value map per layer and frame: the current query's in self mode (queue 0 = queue 1), prev_bev's with a previous
    // BEV, whose queue-1 map value_proj_l(bev_queries) was computed once at finalize.  The sampling projection reads the same
    // operand (and query + pos).
    const T* a_v = has_prev ? e->prev_t.as<T>() : q_in;
    T* v_prev = e->tsa_value.as<T>();
    const T* v_cur = has_prev ? e->tsa_v_query.as<T>() + (size_t)l * Nq * C : v_prev;
    if (fuse_ln && q_half) {
        // the value map + the sampling projection are independent GEMMs over [Nq,256] operands: ONE launch on disjoint CTA
        // ranges.  Self mode: W1 q + W2 (q + pos) + b == (W1 + W2) q + [W2 pos + b], the bracket a parameter-only constant.
        if constexpr (sizeof(T) == 2) {
            const bf16* Av[1] = {reinterpret_cast<const bf16*>(a_v)};
            bf16* Cv[1] = {reinterpret_cast<bf16*>(v_prev)};
            ProfScope ps(e, st, CAT_GEMM);
            const int rc = !has_prev
                ? gemm_tc_tsa_inputs(Av, 1, w.tsa_v_wh.as<bf16>(), w.tsa_v_b.as<float>(), Cv, reinterpret_cast<const bf16*>(q_in),
                                     nullptr, C, w.tsa_q_wh_fold.as<bf16>(), nullptr, w.tsa_q_const.as<float>(),
                                     w.tsa_q_const_t32.as<float>(), (__half*)qproj, Nq, nq_tsa, C, st)
                : gemm_tc_tsa_inputs(Av, 1, w.tsa_v_wh.as<bf16>(), w.tsa_v_b.as<float>(), Cv, reinterpret_cast<const bf16*>(a_v),
                                     reinterpret_cast<const bf16*>(q_pos_in), C, w.tsa_q_wh.as<bf16>(), w.tsa_q_b.as<float>(),
                                     nullptr, nullptr, (__half*)qproj, Nq, nq_tsa, 2 * C, st);
            if (rc) return 2;
            e->launches++;
        }
    } else {
        if (gemm<T, T>(e, a_v, nullptr, 0, w.tsa_v_w.as<float>(), w.tsa_v_wh.p, w.tsa_v_b.as<float>(), nullptr, v_prev, Nq, C,
                       C, ACT_NONE, st)) return 2;
        const int rc = q_half ? gemm<T, __half>(e, a_v, q_pos_in, C, w.tsa_q_w.as<float>(), w.tsa_q_wh.p, w.tsa_q_b.as<float>(),
                                                nullptr, (__half*)qproj, Nq, nq_tsa, 2 * C, ACT_NONE, st)
                              : gemm<T, float>(e, a_v, q_pos_in, C, w.tsa_q_w.as<float>(), w.tsa_q_wh.p, w.tsa_q_b.as<float>(),
                                               nullptr, (float*)qproj, Nq, nq_tsa, 2 * C, ACT_NONE, st);
        if (rc) return 2;
    }
    {
        ProfScope ps(e, st, CAT_TSA);
        if (launch_tsa_fused<T>(v_prev, v_cur, qproj, q_half, e->cfg.bev_h, e->cfg.bev_w, attn_out, st)) return 2;
        e->launches++;
    }
    if (fuse_ln) {
        if (gemm_ln_fused(e, (const bf16*)attn_out, w.tsa_o_wh.p, w.tsa_o_b.as<float>(), rs.cur, w.ln_g[0].as<float>(),
                          w.ln_b[0].as<float>(), nullptr, rs.next, (bf16*)y_t, nullptr, Nq, C, st)) return 2;
        rs.advance();
        return 0;
    }
    if (gemm<T, float>(e, attn_out, nullptr, 0, w.tsa_o_w.as<float>(), w.tsa_o_wh.p, w.tsa_o_b.as<float>(), rs.cur, rs.next,
                       Nq, C, C, ACT_NONE, st)) return 2;
    if (e->taps)
        OCC_CUDA(cudaMemcpyAsync(e->tap_tsa.as<float>() + (size_t)l * Nq * C, rs.next, (size_t)Nq * C * 4,
                                 cudaMemcpyDeviceToDevice, st));
    ProfScope ps(e, st, CAT_LN);
    if (launch_layernorm<T>(rs.next, w.ln_g[0].as<float>(), w.ln_b[0].as<float>(), nullptr, Nq, C, rs.cur, y_t, (T*)nullptr,
                            st)) return 2;
    e->launches++;
    return 0;
}

// ---- spatial cross-attention of layer l (spatial_cross_attention.py:128-175, :334-393) and its LayerNorm (into the stream
// and q_t).  q_t_in: the storage-type query the sampling projection reads.
template <typename T>
int sca_stage(occb200_engine* e, bool fuse_ln, int l, const T* q_t_in, Residual& rs, cudaStream_t st)
{
    const int Nq = e->Nq, Nv = e->Nv, C = 256, ncam = e->cfg.num_cams;
    const int nq_sca = 8 * e->cfg.num_levels * e->cfg.sca_points * 3;
    const bool q_half = e->plan.qproj_f16;
    LayerW& w = e->layers[l];
    void* qproj = e->qproj.p;
    T* q_t = e->q_t.as<T>();
    T* attn_out = e->attn_out.as<T>();
    const int rc = q_half ? gemm<T, __half>(e, q_t_in, nullptr, 0, w.sca_q_w.as<float>(), w.sca_q_wh.p, w.sca_q_b.as<float>(),
                                            nullptr, (__half*)qproj, Nq, nq_sca, C, ACT_NONE, st)
                          : gemm<T, float>(e, q_t_in, nullptr, 0, w.sca_q_w.as<float>(), w.sca_q_wh.p, w.sca_q_b.as<float>(),
                                           nullptr, (float*)qproj, Nq, nq_sca, C, ACT_NONE, st);
    if (rc) return 2;
    const T* sca_val = e->sca_value.as<T>();
    if (e->plan.tc_bf16) {                  // this layer's slice of the value maps the frame computed for every layer
        sca_val = reinterpret_cast<const T*>(e->sca_value_all.as<bf16>() + (size_t)l * ncam * Nv * C);
    } else if (gemm<T, T>(e, e->tokens.as<T>(), nullptr, 0, w.sca_v_w.as<float>(), w.sca_v_wh.p, w.sca_v_b.as<float>(), nullptr,
                          e->sca_value.as<T>(), ncam * Nv, C, C, ACT_NONE, st,
                          e->plan.tc_split ? e->tokens_split.as<bf16>() : nullptr)) return 2;
    {
        ProfScope ps(e, st, CAT_SCA);
        if (launch_sca_fused<T>(sca_val, qproj, q_half, e->sp, e->lg, Nv, attn_out, e->hits.as<uint8_t>(), st)) return 2;
        e->launches++;
    }
    if (fuse_ln) {
        if (gemm_ln_fused(e, (const bf16*)attn_out, w.sca_o_wh.p, w.sca_o_b.as<float>(), rs.cur, w.ln_g[1].as<float>(),
                          w.ln_b[1].as<float>(), nullptr, rs.next, (bf16*)q_t, nullptr, Nq, C, st)) return 2;
        rs.advance();
        return 0;
    }
    if (gemm<T, float>(e, attn_out, nullptr, 0, w.sca_o_w.as<float>(), w.sca_o_wh.p, w.sca_o_b.as<float>(), rs.cur, rs.next,
                       Nq, C, C, ACT_NONE, st)) return 2;
    if (e->taps)
        OCC_CUDA(cudaMemcpyAsync(e->tap_sca.as<float>() + (size_t)l * Nq * C, rs.next, (size_t)Nq * C * 4,
                                 cudaMemcpyDeviceToDevice, st));
    ProfScope ps(e, st, CAT_LN);
    if (launch_layernorm<T>(rs.next, w.ln_g[1].as<float>(), w.ln_b[1].as<float>(), nullptr, Nq, C, rs.cur, q_t, (T*)nullptr,
                            st)) return 2;
    e->launches++;
    return 0;
}

// ---- FFN of layer l (mmcv FFN: x + W2 relu(W1 x)) and its LayerNorm: into the stream, y_t and (for the next layer's
// unfolded TSA query projection) q_pos_t
template <typename T>
int ffn_stage(occb200_engine* e, bool fuse_ln, bool has_prev, int l, Residual& rs, T* y_t, cudaStream_t st)
{
    const int Nq = e->Nq, C = 256, F = e->cfg.ffn_dim;
    LayerW& w = e->layers[l];
    T* q_t = e->q_t.as<T>();
    T* q_pos_t = e->q_pos_t.as<T>();
    if (gemm<T, T>(e, q_t, nullptr, 0, w.ffn1_w.as<float>(), w.ffn1_wh.p, w.ffn1_b.as<float>(), nullptr, e->ffn_h.as<T>(), Nq, F,
                   C, ACT_RELU, st)) return 2;
    if (fuse_ln) {
        // self mode with the merged TSA launch folds pos into a constant: no LayerNorm has to write q + pos
        const bool need_qpos = has_prev || !e->plan.qproj_f16;
        if (gemm_ln_fused(e, e->ffn_h.as<bf16>(), w.ffn2_wh.p, w.ffn2_b.as<float>(), rs.cur, w.ln_g[2].as<float>(),
                          w.ln_b[2].as<float>(), need_qpos ? e->pos_t32.as<float>() : nullptr, rs.next, (bf16*)y_t,
                          need_qpos ? (bf16*)q_pos_t : nullptr, Nq, F, st)) return 2;
        rs.advance();
        return 0;
    }
    if (gemm<T, float>(e, e->ffn_h.as<T>(), nullptr, 0, w.ffn2_w.as<float>(), w.ffn2_wh.p, w.ffn2_b.as<float>(), rs.cur, rs.next,
                       Nq, C, F, ACT_NONE, st)) return 2;
    ProfScope ps(e, st, CAT_LN);
    if (launch_layernorm<T>(rs.next, w.ln_g[2].as<float>(), w.ln_b[2].as<float>(), e->pos.as<float>(), Nq, C, rs.cur, y_t,
                            q_pos_t, st)) return 2;
    e->launches++;
    return 0;
}

// ---- the final BEV to bev_embed, then the voxel decoder and heads (transformer_occ.py:305-319, bevformer_occ_head.py:211-212)
template <typename T>
int decode_stage(occb200_engine* e, bool fuse_ln, Residual& rs, const FrameOut& out, cudaStream_t st)
{
    const occb200_config& c = e->cfg;
    const FramePlan& p = e->plan;
    const int Nq = e->Nq, C = 256, X = c.bev_w, Y = c.bev_h, Z = c.pillar_h, mid = C / Z;
    const int64_t nvox = (int64_t)X * Y * Z;
    // the voxel lift reads the T32 residual stream directly when bev_embed itself is not an output (one kernel instead of two)
    const bool lift_from_t32 = fuse_ln && p.lift_t32 && out.bev_embed == nullptr;
    if (fuse_ln && !lift_from_t32) {                               // back to row-major for the outputs / voxel decoder
        ProfScope ps(e, st, CAT_PACK);
        if (launch_t32_convert(rs.cur, rs.next, Nq, 1, st)) return 2;
        e->launches++;
        rs.advance();
    }
    if (out.bev_embed)
        OCC_CUDA(cudaMemcpyAsync(out.bev_embed, rs.cur, (size_t)Nq * C * 4, cudaMemcpyDeviceToDevice, st));
    if (!out.occ_logits && !out.flow && !out.cls_u8 && !out.cls_i64) return 0;
    int n;
    {
        ProfScope ps(e, st, CAT_VOX);
        if ((n = decoder_lift<T>(lift_from_t32, rs.cur, c.bev_h, c.bev_w, Z, e->vox0.as<T>(), st)) < 0) return 2;
        e->launches += n;
    }
    bf16* split = e->vox_split.as<bf16>();
    if (p.conv == FramePlan::CONV_SPLIT) {
        ProfScope ps(e, st, CAT_CONV);
        if ((n = decoder_conv<T>(p.conv, e->vox0.as<T>(), e->dec_conv[0], X, Y, Z, mid, e->vox1.as<T>(), split, st)) < 0) return 2;
        e->launches += n;
        if ((n = decoder_conv<T>(p.conv, e->vox1.as<T>(), e->dec_conv[1], X, Y, Z, c.out_dim, e->vox2.as<T>(), split, st)) < 0)
            return 2;
        e->launches += n;
    } else {
        {
            ProfScope ps(e, st, CAT_CONV);
            if ((n = decoder_conv<T>(p.conv, e->vox0.as<T>(), e->dec_conv[0], X, Y, Z, mid, e->vox1.as<T>(), split, st)) < 0)
                return 2;
            e->launches += n;
        }
        ProfScope ps(e, st, CAT_CONV);
        if ((n = decoder_conv<T>(p.conv, e->vox1.as<T>(), e->dec_conv[1], X, Y, Z, c.out_dim, e->vox2.as<T>(), split, st)) < 0)
            return 2;
        e->launches += n;
    }
    ProfScope ps(e, st, CAT_HEAD);
    if ((n = decoder_head<T>(p.head_tc, e->vox2.as<T>(), e->head, c.num_classes, nvox, out.occ_logits, out.flow, out.cls_u8,
                             out.cls_i64, st)) < 0) return 2;
    e->launches += n;
    return 0;
}

// One frame from device feature levels in `layout` (input dtype 0, 1 or 2; see occb200_engine_set_input_dtype).  A frame
// that writes the history has its last LayerNorm write its storage-type copy of the final BEV there.
template <typename T>
int forward_impl(occb200_engine* e, const float* const* feats, int layout, const PrevBev& prev, const FrameOut& out,
                 cudaStream_t st)
{
    const occb200_config& c = e->cfg;
    const int Nq = e->Nq, Nv = e->Nv, C = 256;
    const bool fuse_ln = e->plan.tc_bf16 && !e->taps;
    const bool has_prev = prev.src != PrevBev::NONE;
    const bool fold_l0 = fuse_ln && !has_prev && e->plan.fold_layer0;
    T* q_t = e->q_t.as<T>();
    T* q_pos_t = e->q_pos_t.as<T>();
    e->launches = 0;
    if (pack_stage<T>(e, feats, layout, st)) return 2;
    // Layer-0 operands.  On the fused path they were built once at finalize (parameters only), and so was layer 0's TSA output
    // when it is folded: the stream starts on that constant.
    Residual rs{e->q_f32.as<float>(), e->x_f32.as<float>(), e->q_f32.as<float>()};
    if (fuse_ln) {
        rs = {fold_l0 ? e->l0_x_f32.as<float>() : e->qc_f32.as<float>(), e->q_f32.as<float>(), e->x_f32.as<float>()};
    } else {
        ProfScope ps(e, st, CAT_PACK);
        if (launch_prepare_query<T>(e->bev_queries.as<float>(), e->pos.as<float>(), (int64_t)Nq * C, rs.cur, q_t, q_pos_t, 0,
                                    st)) return 2;
        e->launches++;
    }
    if (has_prev) {
        // encoder.py:204-209: value = stack([prev_bev, bev_query]) built ONCE before the layer loop, so
        // queue 1 keeps seeing the layer-0 query in every layer.
        // (transformer_occ.py:195-205) the rotation of prev_bev about rotate_center is a nearest-neighbour row permutation:
        // applied here, fused with the operand cast, from the frame's index map (or the source cells each thread computes
        // from its grid coefficients).  The history already holds the operand rounding of the previous bev_embed, so
        // gathering it gives the same operand.
        if (prev.src == PrevBev::HISTORY) {
            if (launch_gather_rows_stored<T>(e->hist.as<T>(), prev.map, prev.grid, Nq, C, e->prev_t.as<T>(), st)) return 2;
        } else if (launch_gather_rows<T>(prev.bev, prev.map, prev.grid, Nq, C, e->prev_t.as<T>(), nullptr, st))
            return 2;
        e->launches++;
    }
    if (e->plan.tc_bf16) {
        // SpatialCrossAttention's value_proj input (the camera tokens) does not depend on the layer
        // (spatial_cross_attention.py:334): every layer's value map in one launch
        ProfScope ps(e, st, CAT_GEMM);
        if (gemm_tc_blocked256(e->tokens.as<bf16>(), e->sca_v_all_wh.as<bf16>(), e->sca_v_all_b.as<float>(),
                               e->sca_value_all.as<bf16>(), c.num_cams * Nv, c.num_layers * C, C, st)) return 2;
        e->launches++;
    }
    // per encoder layer (encoder.py:356-404): self_attn, norm, cross_attn, norm, ffn, norm
    for (int l = 0; l < c.num_layers; ++l) {
        const bool l0_const = fuse_ln && l == 0;          // layer 0 reads the operands built at finalize
        if (!(l == 0 && fold_l0) &&
            tsa_stage<T>(e, fuse_ln, has_prev, l, l0_const ? e->qc_t.as<T>() : q_t, l0_const ? e->qc_pos_t.as<T>() : q_pos_t,
                         rs, q_t, st)) return 2;
        if (sca_stage<T>(e, fuse_ln, l, l == 0 && fold_l0 ? e->l0_q_t.as<T>() : q_t, rs, st)) return 2;
        // a video frame's last LayerNorm writes its storage-type copy straight into the history (q_t is not read afterwards)
        T* y_t = prev.writes_history && l == c.num_layers - 1 ? e->hist.as<T>() : q_t;
        if (ffn_stage<T>(e, fuse_ln, has_prev, l, rs, y_t, st)) return 2;
        if (e->taps)
            OCC_CUDA(cudaMemcpyAsync(e->tap_layer.as<float>() + (size_t)l * Nq * C, rs.cur, (size_t)Nq * C * 4,
                                     cudaMemcpyDeviceToDevice, st));
    }
    return decode_stage<T>(e, fuse_ln, rs, out, st);
}

// A backbone the engine can drive for input dtype 3: finalized, one image per camera, the engine's level shapes, frames set.
int check_backbone(const occb200_engine* e, const occb200_backbone* bb)
{
    const BackboneInfo bi = backbone_info(bb);
    OCC_CHECK(bi.finalized, "attach_backbone: backbone_finalize() has not been called");
    OCC_CHECK(bi.num_images == e->cfg.num_cams, "attach_backbone: backbone num_images " + std::to_string(bi.num_images) +
                                                    " != engine num_cams " + std::to_string(e->cfg.num_cams));
    for (int l = 0; l < 4; ++l) {
        int h = 0, w = 0;
        if (occb200_backbone_level_shape(bb, l, &h, &w)) return 1;
        OCC_CHECK(h == e->lg.h[l] && w == e->lg.w[l],
                  "attach_backbone: backbone level " + std::to_string(l) + " is " + std::to_string(h) + "x" +
                      std::to_string(w) + ", the engine's is " + std::to_string(e->lg.h[l]) + "x" + std::to_string(e->lg.w[l]));
    }
    OCC_CHECK(bi.frames_set, "attach_backbone: backbone has no frame format (occb200_backbone_set_frame_format)");
    return 0;
}

// bytes of input buffer l in `layout` (see occb200_engine_set_input_dtype): feature level l of dtype 0 (fp32) or 1 / 2
// (bf16), or for 3 the uint8 frames [num_cams, src_h, src_w, 3] of the attached backbone (l = 0)
size_t input_bytes(const occb200_engine* e, int layout, int l)
{
    if (layout >= 3) {
        const BackboneInfo bi = backbone_info(e->bb);
        return (size_t)e->cfg.num_cams * bi.src_h * bi.src_w * 3;
    }
    return (size_t)e->cfg.num_cams * 256 * e->lg.h[l] * e->lg.w[l] * (layout ? 2 : 4);
}

template <typename T>
int forward_frames_impl(occb200_engine* e, const uint8_t* frames, const PrevBev& prev, const FrameOut& out, cudaStream_t st)
{
    const BackboneInfo bi = backbone_info(e->bb);
    const int layout = e->cfg.precision == 1 && bi.precision == 1 ? 2 : 0;   // bf16 -> bf16: channels-last hand-over
    void* lv[4];
    for (int l = 0; l < 4; ++l) {
        if (ensure(e->bb_levels[l], input_bytes(e, layout, l))) return 2;
        lv[l] = e->bb_levels[l].p;
    }
    if (!e->bb_free) OCC_CUDA(cudaEventCreateWithFlags(&e->bb_free, cudaEventDisableTiming));
    // the backbone workspace and the level buffers are shared by every stream the frames arrive on
    if (e->bb_free_recorded) OCC_CUDA(cudaStreamWaitEvent(st, e->bb_free, 0));
    int rc = occb200_backbone_forward_frames(e->bb, frames, lv[0], lv[1], lv[2], lv[3], layout == 2 ? 1 : 0, st);
    if (rc) return rc;
    const int bb_launches = backbone_info(e->bb).launches;
    const float* feats[4] = {(const float*)lv[0], (const float*)lv[1], (const float*)lv[2], (const float*)lv[3]};
    rc = forward_impl<T>(e, feats, layout, prev, out, st);
    if (rc) return rc;
    OCC_CUDA(cudaEventRecord(e->bb_free, st));
    e->bb_free_recorded = true;
    e->launches += bb_launches;
    return 0;
}

// Host-side checks of a frame's input pointers (device or host): error 1, nothing enqueued.  Input dtype 4 also parses the
// camera files' headers into the decoder of the buffer set `b` the frame will use (host only).
int check_frame(const occb200_engine* e, const float* const* feats, FrameBufs& b)
{
    OCC_CHECK(e->finalized, "engine_finalize() has not been called");
    OCC_CHECK(e->cameras_set, "engine_set_cameras() has not been called");
    if (e->feats_bf16 >= 3) {
        OCC_CHECK(e->bb != nullptr, "input dtypes 3 and 4 (camera frames) need an attached backbone (occb200_engine_attach_backbone)");
        OCC_CHECK(feats[0] != nullptr, "null frame buffer");
        if (check_backbone(e, e->bb)) return 1;
        if (e->feats_bf16 == 3) return 0;
        const auto* f = reinterpret_cast<const occb200_encoded_frame*>(feats[0]);
        for (int c = 0; c < e->cfg.num_cams; ++c) OCC_CHECK(f->data[c] != nullptr, "null camera file " + std::to_string(c));
        if (!b.jpeg.p && occb200_jpeg_create(&b.jpeg.p)) return 1;
        const BackboneInfo bi = backbone_info(e->bb);
        return jpeg_prepare(b.jpeg.p, e->cfg.num_cams, f->data, f->size, bi.src_h, bi.src_w);
    }
    for (int l = 0; l < e->cfg.num_levels; ++l) OCC_CHECK(feats[l] != nullptr, "null feature level");
    return 0;
}

// a frame with a request armed may decline its volumes
bool request_armed(const occb200_engine* e) { return e && (e->ray_req.armed || e->score_req.armed); }

// The requests the next frame consumes, disarmed in the engine: called once every check of the frame call has passed.
Requests take_requests(occb200_engine* e)
{
    const Requests rq{e->ray_req, e->score_req};
    e->ray_req.armed = false;
    e->score_req.armed = false;
    return rq;
}

// A video frame's previous BEV: the history, rotated by `map` (device) or `grid`, unless the scene starts here or no video
// frame has written it since set_history(e, 1) (self mode); either way the frame writes the history.
PrevBev video_prev(const occb200_engine* e, int scene_start, const int32_t* map, const RotGrid* grid)
{
    PrevBev p;
    p.src = scene_start == 0 && e->hist_valid ? PrevBev::HISTORY : PrevBev::NONE;
    p.map = map;
    p.grid = grid;
    p.writes_history = true;
    return p;
}

// Every frame call ends up here, after all of its checks.  The frame consumes `rq`: the head also writes the u8 classes and
// the flow (into `b` when the caller did not ask for them) and ray_records_kernel / ray_score_kernel follow it on the frame's
// stream.  A frame that writes the history waits for the previous one's write (on whatever stream that ran) before it reads
// it, and records hist_done after its own.
int run_frame(occb200_engine* e, const float* const* feats, const PrevBev& prev, FrameOut out, const Requests& rq,
              FrameBufs& b, cudaStream_t st, bool jpeg_uploaded = false)
{
    if (rq.rays.armed || rq.score.armed) {
        const size_t nvox = (size_t)e->cfg.bev_w * e->cfg.bev_h * e->cfg.pillar_h;
        if (out.cls_u8 == nullptr) {
            if (ensure(b.sem, nvox)) return 2;
            out.cls_u8 = b.sem.as<uint8_t>();
        }
        if (out.flow == nullptr) {
            if (ensure(b.flow, nvox * 8)) return 2;
            out.flow = b.flow.as<float>();
        }
    }
    if (prev.writes_history && e->hist_recorded) OCC_CUDA(cudaStreamWaitEvent(st, e->hist_done, 0));
    const bool f32 = e->cfg.precision == 0;
    int rc;
    if (e->feats_bf16 >= 3) {
        const uint8_t* frames = reinterpret_cast<const uint8_t*>(feats[0]);
        if (e->feats_bf16 == 4) {
            // the camera files (parsed by check_frame) are decoded on the frame's stream into the set's frame buffer
            if (ensure(b.frames, input_bytes(e, 4, 0))) return 2;
            if (!jpeg_uploaded && jpeg_upload(b.jpeg.p, st, st)) return 2;
            if (jpeg_decode(b.jpeg.p, b.frames.as<uint8_t>(), st)) return 2;
            frames = b.frames.as<uint8_t>();
        }
        rc = f32 ? forward_frames_impl<float>(e, frames, prev, out, st) : forward_frames_impl<bf16>(e, frames, prev, out, st);
        if (e->feats_bf16 == 4) e->launches += kJpegLaunches;
    } else {
        rc = f32 ? forward_impl<float>(e, feats, e->feats_bf16, prev, out, st)
                 : forward_impl<bf16>(e, feats, e->feats_bf16, prev, out, st);
    }
    if (rc) return rc;
    if (rq.rays.armed) {
        const RayRequest& r = rq.rays;
        e->launches++;
        if (launch_ray_records(out.cls_u8, out.flow, r.org, e->rays.as<float>(), e->rays_M, r.cls, r.dist, r.flow, st)) return 2;
    }
    if (rq.score.armed) {
        const ScoreRequest& s = rq.score;
        e->launches++;
        if (launch_ray_score(out.cls_u8, out.flow, s.sem_gt, s.flow_gt, s.org, e->rays.as<float>(), e->rays_M, s.counters, st))
            return 2;
    }
    if (prev.writes_history) {
        OCC_CUDA(cudaEventRecord(e->hist_done, st));
        e->hist_recorded = true;
        e->hist_valid = true;
    }
    return 0;
}

// error 5 when a camera file of the set's last decode (complete on the host) had a corrupt scan
int check_jpeg_status(const FrameBufs& b)
{
    const int st = jpeg_status_host(b.jpeg.p);
    if (st == 0) return 0;
    set_last_error("corrupt JPEG scan in camera file(s) with bit mask " + std::to_string(st) +
                   " (the frame's outputs are not valid)");
    return 5;
}

// Every host-buffer frame (_forward_host, _submit_host, _submit_host_video[_angle]) after its entry point's own checks, in
// this order: the remaining checks (error 1 before any CUDA call, the requests still armed), the uploads of the inputs and of
// the host rotation map `map_host` (NULL: none), the request staging, the frame, the copies back.  `slot` -1 (_forward_host):
// every copy on the caller's stream, then a stream synchronise.  Slot 0 / 1: uploads on the copy streams, the frame on the
// caller's stream after them, the copies back on d2h_stream; the slot stays busy until _wait_host.
int host_frame(occb200_engine* e, int slot, const float* const* feats_host, PrevBev prev, const int32_t* map_host,
               int64_t* occ_host, float* flow_host, cudaStream_t st)
{
    occb200_engine::Slot* s = slot < 0 ? nullptr : &e->slots[slot];
    OCC_CHECK(s == nullptr || !s->busy, "slot still in flight: call occb200_engine_wait_host first");
    FrameBufs& b = s ? s->bufs : e->bufs;
    if (check_frame(e, feats_host, b)) return 1;
    if (map_host)
        for (int q = 0; q < e->Nq; ++q) OCC_CHECK(map_host[q] >= -1 && map_host[q] < e->Nq, "rotation map entry out of range");

    if (s && !e->d2h_stream) {
        for (cudaStream_t& hs : e->h2d_stream) OCC_CUDA(cudaStreamCreateWithFlags(&hs, cudaStreamNonBlocking));
        OCC_CUDA(cudaStreamCreateWithFlags(&e->d2h_stream, cudaStreamNonBlocking));
    }
    if (s && !s->compute_done) {
        for (cudaEvent_t& ev : s->h2d_done) OCC_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        OCC_CUDA(cudaEventCreateWithFlags(&s->compute_done, cudaEventDisableTiming));
        OCC_CUDA(cudaEventCreateWithFlags(&s->d2h_done, cudaEventDisableTiming));
    }
    if (map_host) {
        // staged in the slot's pinned buffer so that the caller may reuse its array on return; h2d_done[0] covers the upload
        const size_t mb = (size_t)e->Nq * 4;
        if (!s->rot_pinned) OCC_CUDA(cudaMallocHost(&s->rot_pinned, mb));
        if (ensure(s->rot, mb)) return 2;
        OCC_CUDA(cudaEventSynchronize(s->h2d_done[0]));            // the slot's previous upload has left the staging buffer
        memcpy(s->rot_pinned, map_host, mb);
        OCC_CUDA(cudaMemcpyAsync(s->rot.p, s->rot_pinned, mb, cudaMemcpyHostToDevice, e->h2d_stream[0]));
        prev.map = s->rot.as<int32_t>();
    }
    const int layout = e->feats_bf16;
    const float* dev_feats[4] = {nullptr, nullptr, nullptr, nullptr};
    if (layout == 4) {                                                     // the packed camera files, decoded by the frame
        if (jpeg_upload(b.jpeg.p, s ? e->h2d_stream[0] : st, st)) return 2;
        dev_feats[0] = feats_host[0];
    }
    for (int l = 0; l < (layout == 4 ? 0 : layout == 3 ? 1 : 4); ++l) {   // input dtype 3: one buffer, the uint8 frames
        const size_t n = input_bytes(e, layout, l);
        if (ensure(b.feats[l], n)) return 2;
        if (s) {
            const int pieces = n >= (32u << 20) ? kH2DSplit : 1;
            const size_t chunk = ((n / pieces) + 255) & ~(size_t)255;
            for (int i = 0; i < pieces; ++i) {
                const size_t o = (size_t)i * chunk, len = o >= n ? 0 : (n - o < chunk ? n - o : chunk);
                if (len) OCC_CUDA(cudaMemcpyAsync((char*)b.feats[l].p + o, (const char*)feats_host[l] + o, len,
                                                  cudaMemcpyHostToDevice, e->h2d_stream[i]));
            }
        } else {
            OCC_CUDA(cudaMemcpyAsync(b.feats[l].p, feats_host[l], n, cudaMemcpyHostToDevice, st));
        }
        dev_feats[l] = b.feats[l].as<float>();
    }

    // the requests point the frame at device staging: room for a ray request's records (the largest T, so no reallocation
    // between frames), and a score request's ground truth, uploaded after the features
    const Requests host_rq = take_requests(e);
    Requests rq = host_rq;
    const size_t nvox = (size_t)e->cfg.bev_w * e->cfg.bev_h * e->cfg.pillar_h;
    if (rq.rays.armed) {
        const size_t n = (size_t)8 * e->rays_M;
        if (ensure(b.rec_cls, n) || ensure(b.rec_dist, n * 2) || ensure(b.rec_flow, n * 4)) return 2;
        rq.rays.cls = b.rec_cls.as<int8_t>(); rq.rays.dist = b.rec_dist.p; rq.rays.flow = b.rec_flow.p;
    }
    if (rq.score.armed) {
        if (ensure(b.gt_sem, nvox) || ensure(b.gt_flow, nvox * 8)) return 2;
        cudaStream_t copy = s ? e->h2d_stream[0] : st;
        OCC_CUDA(cudaMemcpyAsync(b.gt_sem.p, rq.score.sem_gt, nvox, cudaMemcpyHostToDevice, copy));
        OCC_CUDA(cudaMemcpyAsync(b.gt_flow.p, rq.score.flow_gt, nvox * 8, cudaMemcpyHostToDevice, copy));
        rq.score.sem_gt = b.gt_sem.as<uint8_t>(); rq.score.flow_gt = b.gt_flow.as<float>();
    }
    if (s)
        for (int i = 0; i < kH2DSplit; ++i) {                       // compute waits for this frame's uploads only
            OCC_CUDA(cudaEventRecord(s->h2d_done[i], e->h2d_stream[i]));
            OCC_CUDA(cudaStreamWaitEvent(st, s->h2d_done[i], 0));
        }

    if (occ_host && ensure(b.occ, nvox * 8)) return 2;
    if (ensure(b.flow, nvox * 8)) return 2;
    FrameOut out;
    out.flow = b.flow.as<float>();
    out.cls_i64 = occ_host ? b.occ.as<int64_t>() : nullptr;
    const int rc = run_frame(e, dev_feats, prev, out, rq, b, st, true);
    if (rc) return rc;

    cudaStream_t d2h = st;
    if (s) {
        OCC_CUDA(cudaEventRecord(s->compute_done, st));
        OCC_CUDA(cudaStreamWaitEvent(e->d2h_stream, s->compute_done, 0));
        d2h = e->d2h_stream;
    }
    if (occ_host) OCC_CUDA(cudaMemcpyAsync(occ_host, b.occ.p, nvox * 8, cudaMemcpyDeviceToHost, d2h));
    if (flow_host) OCC_CUDA(cudaMemcpyAsync(flow_host, b.flow.p, nvox * 8, cudaMemcpyDeviceToHost, d2h));
    if (host_rq.rays.armed) {
        const RayRequest& r = host_rq.rays;
        const size_t n = (size_t)r.org.T * e->rays_M;
        OCC_CUDA(cudaMemcpyAsync(r.cls, b.rec_cls.p, n, cudaMemcpyDeviceToHost, d2h));
        OCC_CUDA(cudaMemcpyAsync(r.dist, b.rec_dist.p, n * 2, cudaMemcpyDeviceToHost, d2h));
        OCC_CUDA(cudaMemcpyAsync(r.flow, b.rec_flow.p, n * 4, cudaMemcpyDeviceToHost, d2h));
    }
    if (!s) {
        OCC_CUDA(cudaStreamSynchronize(st));
        return layout == 4 ? check_jpeg_status(b) : 0;
    }
    OCC_CUDA(cudaEventRecord(s->d2h_done, d2h));
    s->busy = true;
    s->jpeg = layout == 4;
    return 0;
}

}  // namespace

extern "C" {

const char* occb200_last_error(void) { return g_last_error.c_str(); }
const char* occb200_version(void) { return "occ_b200 0.1 sm_90a"; }

int occb200_ms_deform_attn_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                   const float* sampling_loc, const float* attn_weight, int B, int Nv, int M, int C,
                                   int Nq, int L, int P, int im2col_step, float* out, void* stream)
{
    OCC_CHECK(B >= 0 && Nv >= 0 && M > 0 && C > 0 && Nq >= 0 && L > 0 && P > 0, "bad sizes");
    if ((int64_t)B * Nq == 0) return 0;                          // empty query set: nothing to write
    OCC_CHECK(value && spatial_shapes && level_start_index && sampling_loc && attn_weight && out, "null pointer");
    const int step = im2col_step < B ? im2col_step : B;
    OCC_CHECK(B == 0 || (step > 0 && B % step == 0), "batch(" + std::to_string(B) + ") must divide im2col_step(" +
                                                         std::to_string(im2col_step) + ")");
    return launch_msda_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, B, Nv, M, C, Nq, L,
                               P, out, (cudaStream_t)stream);
}

int occb200_ms_deform_attn_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                    const float* sampling_loc, const float* attn_weight, const float* grad_output, int B,
                                    int Nv, int M, int C, int Nq, int L, int P, int im2col_step, float* grad_value,
                                    float* grad_sampling_loc, float* grad_attn_weight, void* stream)
{
    OCC_CHECK(B >= 0 && Nv >= 0 && M > 0 && C > 0 && Nq >= 0 && L > 0 && P > 0, "bad sizes");
    if ((int64_t)B * Nq == 0) return 0;
    OCC_CHECK(value && spatial_shapes && level_start_index && sampling_loc && attn_weight && grad_output && grad_value &&
                  grad_sampling_loc && grad_attn_weight, "null pointer");
    const int step = im2col_step < B ? im2col_step : B;
    OCC_CHECK(step > 0 && B % step == 0, "batch(" + std::to_string(B) + ") must divide im2col_step(" +
                                             std::to_string(im2col_step) + ")");
    return launch_msda_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, B, Nv, M,
                                C, Nq, L, P, grad_value, grad_sampling_loc, grad_attn_weight, (cudaStream_t)stream);
}

int occb200_engine_create(const occb200_config* cfg, occb200_engine** out)
{
    OCC_CHECK(cfg && out, "null pointer");
    OCC_CHECK(cfg->embed_dims == 256 && cfg->num_heads == 8, "only embed_dims=256, num_heads=8 are supported");
    OCC_CHECK(cfg->num_levels == 4 && cfg->sca_points == 8 && cfg->tsa_points == 4,
              "only num_levels=4, SCA num_points=8, TSA num_points=4 are supported");
    OCC_CHECK(cfg->num_cams >= 1 && cfg->num_cams <= 8, "num_cams must be in [1,8]");
    OCC_CHECK(cfg->num_points_in_pillar >= 1 && cfg->num_points_in_pillar <= 8 && 8 % cfg->num_points_in_pillar == 0,
              "num_points_in_pillar must be 1, 2, 4 or 8");
    OCC_CHECK(cfg->pillar_h == 16 && cfg->out_dim == 32, "only pillar_h=16, out_dim=32 are supported");
    OCC_CHECK(cfg->ffn_dim % 64 == 0 && cfg->num_classes <= 32 && cfg->num_layers >= 1, "bad ffn_dim/num_classes");
    OCC_CHECK(cfg->precision == 0 || cfg->precision == 1, "precision must be 0 (fp32) or 1 (bf16)");
    int dev_count = 0;
    if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) {
        set_last_error("no CUDA device: libocc_b200 has no CPU fallback");
        return 4;
    }
    auto* e = new occb200_engine();
    e->cfg = *cfg;
    e->Nq = cfg->bev_h * cfg->bev_w;
    e->lg = make_level_geom(cfg->level_h, cfg->level_w, &e->Nv);
    e->layers.resize(cfg->num_layers);
    *out = e;
    return 0;
}

void occb200_engine_destroy(occb200_engine* e)
{
    if (!e) return;
    // the device buffers free themselves; events, streams and pinned staging are released here
    if (e->bb_free) cudaEventDestroy(e->bb_free);
    if (e->hist_done) cudaEventDestroy(e->hist_done);
    for (auto& sl : e->slots) {
        if (sl.rot_pinned) cudaFreeHost(sl.rot_pinned);
        if (sl.compute_done) {
            for (cudaEvent_t ev : sl.h2d_done) cudaEventDestroy(ev);
            cudaEventDestroy(sl.compute_done); cudaEventDestroy(sl.d2h_done);
        }
    }
    if (e->d2h_stream) {
        for (cudaStream_t hs : e->h2d_stream) cudaStreamDestroy(hs);
        cudaStreamDestroy(e->d2h_stream);
    }
    for (cudaEvent_t ev : e->event_pool) cudaEventDestroy(ev);
    delete e;
}

int occb200_engine_load_param(occb200_engine* e, const char* key, const float* data, int64_t numel)
{
    OCC_CHECK(e && key && data && numel >= 0, "null pointer");
    const std::string k(key);
    static const char* known_prefix[] = {"bev_embedding.", "positional_encoding.", "transformer.level_embeds",
                                         "transformer.cams_embeds", "transformer.encoder.layers.",
                                         "transformer.decoder.", "transformer.predicter.", "transformer.flow_predicter."};
    bool ok = false;
    for (const char* p : known_prefix) ok = ok || k.rfind(p, 0) == 0;
    if (!ok) { set_last_error("unknown parameter key: " + k); return 3; }
    e->host_params[k].assign(data, data + numel);
    e->finalized = false;
    return 0;
}

int occb200_engine_finalize(occb200_engine* e)
{
    OCC_CHECK(e, "null engine");
    const occb200_config& c = e->cfg;
    const int C = 256, Nq = e->Nq, F = c.ffn_dim, od = c.out_dim, mid = C / c.pillar_h;
    e->plan = make_frame_plan(c, Nq);
    const FramePlan& p = e->plan;
    {
        GETP(bq, "bev_embedding.weight", (size_t)Nq * C);
        if (upload(e->bev_queries, bq->data(), bq->size())) return 2;
        GETP(re, "positional_encoding.row_embed.weight", (size_t)c.bev_h * (C / 2));
        GETP(ce, "positional_encoding.col_embed.weight", (size_t)c.bev_w * (C / 2));
        DevBuf dre, dce;
        if (upload(dre, re->data(), re->size()) || upload(dce, ce->data(), ce->size())) return 2;
        if (e->pos.alloc((size_t)Nq * C * 4)) return 2;
        if (launch_bev_pos(dre.as<float>(), dce.as<float>(), c.bev_h, c.bev_w, C / 2, e->pos.as<float>(), 0)) return 2;
        if (p.tc_bf16) {                                           // T32 copy of pos for the fused LayerNorm epilogue
            const size_t rows_pad = ((size_t)Nq + 127) / 128 * 128;
            if (e->pos_t32.alloc(rows_pad * C * 4)) return 2;
            OCC_CUDA(cudaMemset(e->pos_t32.p, 0, rows_pad * C * 4));
            if (launch_t32_convert(e->pos.as<float>(), e->pos_t32.as<float>(), Nq, 0, 0)) return 2;
            // bev_queries / pos are parameters: their fp32 (T32) and bf16 operand forms are frame-independent
            if (e->qc_f32.alloc(rows_pad * C * 4) || e->qc_t.alloc((size_t)Nq * C * 2) || e->qc_pos_t.alloc((size_t)Nq * C * 2))
                return 2;
            OCC_CUDA(cudaMemset(e->qc_f32.p, 0, rows_pad * C * 4));
            if (launch_prepare_query<bf16>(e->bev_queries.as<float>(), e->pos.as<float>(), (int64_t)Nq * C, e->qc_f32.as<float>(),
                                           e->qc_t.as<bf16>(), e->qc_pos_t.as<bf16>(), 1, 0)) return 2;
        }
        OCC_CUDA(cudaDeviceSynchronize());
        GETP(le, "transformer.level_embeds", (size_t)c.num_levels * C);
        GETP(cm, "transformer.cams_embeds", (size_t)c.num_cams * C);
        std::vector<float> cams(*cm);
        if (!c.use_cams_embeds) std::fill(cams.begin(), cams.end(), 0.f);    // transformer_occ.py:214-215: added only if set
        if (upload(e->level_embeds, le->data(), le->size()) || upload(e->cams_embeds, cams.data(), cams.size())) return 2;
    }
    for (int l = 0; l < c.num_layers; ++l) {
        LayerW& w = e->layers[l];
        const std::string pre = "transformer.encoder.layers." + std::to_string(l);
        const std::string a0 = pre + ".attentions.0", a1 = pre + ".attentions.1", d = a1 + ".deformable_attention";
        auto up = [&](DevBuf& wbuf, DevBuf& bbuf, DevBuf* wh, const std::string& name, size_t n, size_t k) -> int {
            const std::vector<float>* W = find(e, name + ".weight", n * k);
            const std::vector<float>* B = find(e, name + ".bias", n);
            if (!W || !B) return 3;
            return upload_dense(p, wbuf, bbuf, wh, W->data(), B->data(), n, k);
        };
        auto up_cat = [&](DevBuf& wbuf, DevBuf& bbuf, DevBuf* wh, const std::string& n1, const std::string& n2,
                          size_t r1, size_t r2, size_t k, DevBuf* fold = nullptr, DevBuf* fold_const = nullptr) -> int {
            const std::vector<float>* W1 = find(e, n1 + ".weight", r1 * k);
            const std::vector<float>* B1 = find(e, n1 + ".bias", r1);
            const std::vector<float>* W2 = find(e, n2 + ".weight", r2 * k);
            const std::vector<float>* B2 = find(e, n2 + ".bias", r2);
            if (!W1 || !B1 || !W2 || !B2) return 3;
            std::vector<float> W(*W1), B(*B1);
            W.insert(W.end(), W2->begin(), W2->end());
            B.insert(B.end(), B2->begin(), B2->end());
            if (upload_dense(p, wbuf, bbuf, wh, W.data(), B.data(), r1 + r2, k)) return 2;
            if (p.tc_bf16 && p.qproj_f16 && fold) {              // k = 2C: (W1 + W2) [r, C] bf16 and the constant W2 pos + b
                const size_t half = k / 2, rows = r1 + r2;
                std::vector<float> Wf(rows * half), W2h(rows * half);
                for (size_t r = 0; r < rows; ++r)
                    for (size_t j = 0; j < half; ++j) {
                        Wf[r * half + j] = W[r * k + j] + W[r * k + half + j];
                        W2h[r * half + j] = W[r * k + half + j];
                    }
                if (upload_bf16(*fold, Wf.data(), Wf.size())) return 2;
                DevBuf w2;
                if (upload(w2, W2h.data(), W2h.size())) return 2;
                if (fold_const->alloc((size_t)Nq * rows * 4)) return 2;
                if (gemm_simt<float, float>(e->pos.as<float>(), (int)half, nullptr, 0, (int)half, w2.as<float>(), bbuf.as<float>(),
                                            nullptr, (int)rows, fold_const->as<float>(), (int)rows, Nq, (int)rows, (int)half,
                                            ACT_NONE, 0)) return 2;
                // the same constant in the T32 block layout (rows padded to 32) for the epilogue of the merged launch
                if (rows % 32 == 0) {
                    const size_t rows_pad = ((size_t)Nq + 31) / 32 * 32;
                    if (w.tsa_q_const_t32.alloc(rows_pad * rows * 4)) return 2;
                    OCC_CUDA(cudaMemset(w.tsa_q_const_t32.p, 0, rows_pad * rows * 4));
                    if (launch_t32_convert(fold_const->as<float>(), w.tsa_q_const_t32.as<float>(), Nq, 0, 0, (int)rows)) return 2;
                }
                OCC_CUDA(cudaDeviceSynchronize());
            }
            return 0;
        };
        int rc;
        const size_t tq_off = 2 * 8 * c.tsa_points * 2, tq_w = 2 * 8 * c.tsa_points;
        const size_t sq_off = 8 * c.num_levels * c.sca_points * 2, sq_w = 8 * c.num_levels * c.sca_points;
        if ((rc = up(w.tsa_v_w, w.tsa_v_b, &w.tsa_v_wh, a0 + ".value_proj", C, C))) return rc;
        if ((rc = up_cat(w.tsa_q_w, w.tsa_q_b, &w.tsa_q_wh, a0 + ".sampling_offsets", a0 + ".attention_weights", tq_off,
                         tq_w, 2 * C, &w.tsa_q_wh_fold, &w.tsa_q_const))) return rc;
        if ((rc = up(w.tsa_o_w, w.tsa_o_b, &w.tsa_o_wh, a0 + ".output_proj", C, C))) return rc;
        if ((rc = up_cat(w.sca_q_w, w.sca_q_b, &w.sca_q_wh, d + ".sampling_offsets", d + ".attention_weights", sq_off,
                         sq_w, C))) return rc;
        if ((rc = up(w.sca_v_w, w.sca_v_b, &w.sca_v_wh, d + ".value_proj", C, C))) return rc;
        if ((rc = up(w.sca_o_w, w.sca_o_b, &w.sca_o_wh, a1 + ".output_proj", C, C))) return rc;
        if ((rc = up(w.ffn1_w, w.ffn1_b, &w.ffn1_wh, pre + ".ffns.0.layers.0.0", F, C))) return rc;
        if ((rc = up(w.ffn2_w, w.ffn2_b, &w.ffn2_wh, pre + ".ffns.0.layers.1", C, F))) return rc;
        for (int n = 0; n < 3; ++n) {
            GETP(g, pre + ".norms." + std::to_string(n) + ".weight", (size_t)C);
            GETP(b, pre + ".norms." + std::to_string(n) + ".bias", (size_t)C);
            if (upload(w.ln_g[n], g->data(), C) || upload(w.ln_b[n], b->data(), C)) return 2;
        }
    }
    if (p.tc_bf16) {
        // SpatialCrossAttention's value_proj input (the camera tokens) does not depend on the layer
        // (spatial_cross_attention.py:334): project once with all layers' weights, [L*256, 256].
        std::vector<float> W, B;
        for (int l = 0; l < c.num_layers; ++l) {
            const std::string d = "transformer.encoder.layers." + std::to_string(l) + ".attentions.1.deformable_attention.value_proj";
            const std::vector<float>* w = find(e, d + ".weight", (size_t)C * C);
            const std::vector<float>* b = find(e, d + ".bias", (size_t)C);
            if (!w || !b) return 3;
            W.insert(W.end(), w->begin(), w->end());
            B.insert(B.end(), b->begin(), b->end());
        }
        if (upload_bf16(e->sca_v_all_wh, W.data(), W.size()) || upload(e->sca_v_all_b, B.data(), B.size())) return 2;
        if (e->sca_value_all.alloc((size_t)c.num_layers * c.num_cams * e->Nv * C * 2)) return 2;
        OCC_CUDA(cudaMemset(e->sca_value_all.p, 0, e->sca_value_all.bytes));
    }
    // decoder: BatchNorm3d (eval) folded into the conv weights, laid out for the plan's path; the heads' weights
    for (int i = 0; i < 2; ++i) {
        const int cin = i == 0 ? mid : od;
        const std::string pre = "transformer.decoder." + std::to_string(i);
        GETP(W, pre + ".conv.weight", (size_t)od * cin * 27);
        GETP(g, pre + ".bn.weight", (size_t)od);
        GETP(b, pre + ".bn.bias", (size_t)od);
        GETP(m, pre + ".bn.running_mean", (size_t)od);
        GETP(v, pre + ".bn.running_var", (size_t)od);
        if (upload_decoder_conv(e->dec_conv[i], p.conv, W->data(), g->data(), b->data(), m->data(), v->data(), cin, od)) return 2;
    }
    {
        GETP(w1, "transformer.predicter.0.weight", (size_t)2 * od * od);
        GETP(b1, "transformer.predicter.0.bias", (size_t)2 * od);
        GETP(w2, "transformer.predicter.2.weight", (size_t)c.num_classes * 2 * od);
        GETP(b2, "transformer.predicter.2.bias", (size_t)c.num_classes);
        GETP(f1, "transformer.flow_predicter.0.weight", (size_t)2 * od * od);
        GETP(g1, "transformer.flow_predicter.0.bias", (size_t)2 * od);
        GETP(f2, "transformer.flow_predicter.2.weight", (size_t)2 * 2 * od);
        GETP(g2, "transformer.flow_predicter.2.bias", (size_t)2);
        if (upload_decoder_head(e->head, p.head_tc, c.num_classes, od, w1->data(), b1->data(), w2->data(), b2->data(), f1->data(),
                                g1->data(), f2->data(), g2->data())) return 2;
    }
    // workspace
    const size_t es = e->elt();
    const size_t nvox = (size_t)c.bev_w * c.bev_h * c.pillar_h;
    const size_t ntok = (size_t)c.num_cams * e->Nv;
    int maxq = 8 * c.num_levels * c.sca_points * 3;
    const size_t nq_pad = ((size_t)Nq + 127) / 128 * 128;
    if (e->tokens.alloc(ntok * C * es) || e->sca_value.alloc(ntok * C * es) || e->q_f32.alloc(nq_pad * C * 4) ||
        e->q_t.alloc((size_t)Nq * C * es) || e->q_pos_t.alloc((size_t)Nq * C * es) ||
        e->prev_t.alloc((size_t)Nq * C * es) || e->tsa_value.alloc((size_t)Nq * C * es) ||
        e->qproj.alloc((size_t)Nq * maxq * 4) ||
        e->attn_out.alloc((size_t)Nq * C * es) || e->x_f32.alloc(nq_pad * C * 4) ||
        e->ffn_h.alloc((size_t)Nq * F * es) || e->vox0.alloc(nvox * mid * es) || e->vox1.alloc(nvox * od * es) ||
        e->vox2.alloc(nvox * od * es) || e->hits.alloc(Nq)) return 2;
    OCC_CUDA(cudaMemset(e->q_f32.p, 0, nq_pad * C * 4));
    OCC_CUDA(cudaMemset(e->x_f32.p, 0, nq_pad * C * 4));
    if (p.tc_split) {
        const size_t kmax = (size_t)std::max(2 * C, F);
        if (e->split_ws.alloc((size_t)Nq * 2 * kmax * 2) || e->tokens_split.alloc(ntok * 2 * C * 2)) return 2;
    }
    if (p.conv == FramePlan::CONV_SPLIT && e->vox_split.alloc(nvox * 2 * od * 2)) return 2;
    e->host_params.clear();
    if ((c.precision == 0 ? build_tsa_query_values<float>(e) : build_tsa_query_values<bf16>(e))) return 2;
    if (p.fold_layer0) {
        // Layer 0's TemporalSelfAttention (value_proj, query projection over [bev_queries | pos], gather, output_proj) and
        // its LayerNorm depend on parameters only when prev_bev is None: the frame's own fused TSA stage runs once, here.
        const size_t rows_pad = ((size_t)Nq + 127) / 128 * 128;
        if (e->l0_x_f32.alloc(rows_pad * C * 4) || e->l0_q_t.alloc((size_t)Nq * C * 2)) return 2;
        OCC_CUDA(cudaMemset(e->l0_x_f32.p, 0, rows_pad * C * 4));
        Residual rs{e->qc_f32.as<float>(), e->l0_x_f32.as<float>(), e->l0_x_f32.as<float>()};
        if (tsa_stage<bf16>(e, true, false, 0, e->qc_t.as<bf16>(), e->qc_pos_t.as<bf16>(), rs, e->l0_q_t.as<bf16>(), 0))
            return 2;
        OCC_CUDA(cudaDeviceSynchronize());
    }
    e->finalized = true;
    return 0;
}

int occb200_engine_set_cameras(occb200_engine* e, const float* cam_mat, const float* zs, int img_h, int img_w)
{
    OCC_CHECK(e && cam_mat && zs, "null pointer");
    const occb200_config& c = e->cfg;
    e->sp = make_sca_params(cam_mat, zs, c.num_cams, c.num_points_in_pillar, c.pc_range, img_h, img_w, c.bev_h, c.bev_w);
    e->cameras_set = true;
    return 0;
}

int occb200_engine_forward(occb200_engine* e, const float* const* feats, const float* prev_bev, float* bev_embed,
                           float* occ_logits, float* flow, uint8_t* occ_cls_u8, int64_t* occ_cls_i64, void* stream)
{
    OCC_CHECK(e && feats, "null pointer");
    if (check_frame(e, feats, e->bufs)) return 1;
    PrevBev prev;
    if (prev_bev) {
        prev.src = PrevBev::CALLER;
        prev.bev = prev_bev;
        prev.map = e->rot == occb200_engine::ROT_MAP ? e->rot_map.as<int32_t>() : nullptr;
        prev.grid = e->rot == occb200_engine::ROT_GRID ? &e->rot_grid : nullptr;
    }
    return run_frame(e, feats, prev, {bev_embed, occ_logits, flow, occ_cls_u8, occ_cls_i64}, take_requests(e), e->bufs,
                     (cudaStream_t)stream);
}

int occb200_engine_set_history(occb200_engine* e, int enable)
{
    OCC_CHECK(e, "null engine");
    if (e->hist_recorded) OCC_CUDA(cudaEventSynchronize(e->hist_done));   // a queued video frame may still use the buffer
    e->hist_recorded = false;
    e->hist_valid = false;
    if (!enable) {
        e->hist.release();
        return 0;
    }
    const size_t n = (size_t)e->Nq * 256 * e->elt();
    if (ensure(e->hist, n)) return 2;
    if (!e->hist_done) OCC_CUDA(cudaEventCreateWithFlags(&e->hist_done, cudaEventDisableTiming));
    return 0;
}

int occb200_engine_forward_video(occb200_engine* e, const float* const* feats, const int32_t* rot_map_dev, int scene_start,
                                 float* bev_embed, float* occ_logits, float* flow, uint8_t* occ_cls_u8, int64_t* occ_cls_i64,
                                 void* stream)
{
    OCC_CHECK(feats, "null pointer");
    OCC_CHECK(e, "null engine");
    OCC_CHECK(e->hist.p != nullptr, "history not enabled: call occb200_engine_set_history(e, 1) first");
    if (check_frame(e, feats, e->bufs)) return 1;
    return run_frame(e, feats, video_prev(e, scene_start, rot_map_dev, nullptr),
                     {bev_embed, occ_logits, flow, occ_cls_u8, occ_cls_i64}, take_requests(e), e->bufs, (cudaStream_t)stream);
}

int occb200_engine_forward_video_angle(occb200_engine* e, const float* const* feats, double angle_deg, int scene_start,
                                       float* bev_embed, float* occ_logits, float* flow, uint8_t* occ_cls_u8,
                                       int64_t* occ_cls_i64, void* stream)
{
    OCC_CHECK(std::isfinite(angle_deg), "rotation angle must be finite");
    OCC_CHECK(feats, "null pointer");
    OCC_CHECK(e, "null engine");
    OCC_CHECK(e->hist.p != nullptr, "history not enabled: call occb200_engine_set_history(e, 1) first");
    if (check_frame(e, feats, e->bufs)) return 1;
    const RotGrid g = rotation_grid(e, angle_deg);
    return run_frame(e, feats, video_prev(e, scene_start, nullptr, &g), {bev_embed, occ_logits, flow, occ_cls_u8, occ_cls_i64},
                     take_requests(e), e->bufs, (cudaStream_t)stream);
}

int occb200_engine_forward_host(occb200_engine* e, const float* const* feats_host, int64_t* occ_cls_i64_host,
                                float* flow_host, void* stream)
{
    // with a ray or score request armed the caller may decline either volume (NULL): that 5.12 MB copy is then skipped
    OCC_CHECK(e && feats_host && ((occ_cls_i64_host && flow_host) || request_armed(e)), "null pointer");
    return host_frame(e, -1, feats_host, PrevBev(), nullptr, occ_cls_i64_host, flow_host, (cudaStream_t)stream);
}

int occb200_engine_submit_host(occb200_engine* e, int slot, const float* const* feats_host, int64_t* occ_cls_i64_host,
                               float* flow_host, void* stream)
{
    OCC_CHECK(e && feats_host && ((occ_cls_i64_host && flow_host) || request_armed(e)), "null pointer");
    OCC_CHECK(slot == 0 || slot == 1, "slot must be 0 or 1");
    return host_frame(e, slot, feats_host, PrevBev(), nullptr, occ_cls_i64_host, flow_host, (cudaStream_t)stream);
}

int occb200_engine_submit_host_video(occb200_engine* e, int slot, const float* const* feats_host, const int32_t* rot_map_host,
                                     int scene_start, int64_t* occ_cls_i64_host, float* flow_host, void* stream)
{
    OCC_CHECK(slot == 0 || slot == 1, "slot must be 0 or 1");
    OCC_CHECK(feats_host && ((occ_cls_i64_host && flow_host) || request_armed(e)), "null pointer");
    OCC_CHECK(e, "null engine");
    OCC_CHECK(e->hist.p != nullptr, "history not enabled: call occb200_engine_set_history(e, 1) first");
    return host_frame(e, slot, feats_host, video_prev(e, scene_start, nullptr, nullptr), rot_map_host, occ_cls_i64_host,
                      flow_host, (cudaStream_t)stream);
}

int occb200_engine_submit_host_video_angle(occb200_engine* e, int slot, const float* const* feats_host, double angle_deg,
                                           int scene_start, int64_t* occ_cls_i64_host, float* flow_host, void* stream)
{
    OCC_CHECK(std::isfinite(angle_deg), "rotation angle must be finite");
    OCC_CHECK(slot == 0 || slot == 1, "slot must be 0 or 1");
    OCC_CHECK(feats_host && ((occ_cls_i64_host && flow_host) || request_armed(e)), "null pointer");
    OCC_CHECK(e, "null engine");
    OCC_CHECK(e->hist.p != nullptr, "history not enabled: call occb200_engine_set_history(e, 1) first");
    const RotGrid g = rotation_grid(e, angle_deg);
    return host_frame(e, slot, feats_host, video_prev(e, scene_start, nullptr, &g), nullptr, occ_cls_i64_host, flow_host,
                      (cudaStream_t)stream);
}

int occb200_engine_wait_host(occb200_engine* e, int slot)
{
    OCC_CHECK(e && (slot == 0 || slot == 1), "bad arguments");
    occb200_engine::Slot& s = e->slots[slot];
    if (!s.busy) return 0;
    OCC_CUDA(cudaEventSynchronize(s.d2h_done));
    s.busy = false;
    return s.jpeg ? check_jpeg_status(s.bufs) : 0;
}

int occb200_engine_jpeg_status(occb200_engine* e, int* status)
{
    OCC_CHECK(e && status, "null pointer");
    OCC_CHECK(e->bufs.jpeg.p != nullptr, "no JPEG frame has run on the device calls");
    return occb200_jpeg_status(e->bufs.jpeg.p, status);
}

// origins_host [T,3] (f32, or f64 if is_f64) -> the kernel argument; error 1 for a non-finite coordinate
static int fill_origins(RayOrigins& r, const void* origins_host, int is_f64, int T)
{
    r.T = T;
    r.is_f64 = is_f64 ? 1 : 0;
    for (int i = 0; i < T * 3; ++i) {
        const double v = is_f64 ? static_cast<const double*>(origins_host)[i] : (double)static_cast<const float*>(origins_host)[i];
        OCC_CHECK(std::isfinite(v), "ray origins must be finite");
        r.o[i / 3][i % 3] = v;
    }
    return 0;
}

int occb200_ray_records(const uint8_t* sem_u8, const float* flow, const void* origins_host, int origin_is_f64, int T,
                        const float* rays_dev, int M, int8_t* cls_i8, void* dist_f16, void* flow_f16, void* stream)
{
    OCC_CHECK(T >= 1 && T <= 8, "T (lidar origins) must be in 1..8");
    OCC_CHECK(M >= 1, "M (rays) must be positive");
    OCC_CHECK(sem_u8 && flow && origins_host && rays_dev && cls_i8 && dist_f16 && flow_f16, "null pointer");
    RayOrigins org;
    if (fill_origins(org, origins_host, origin_is_f64, T)) return 1;
    return launch_ray_records(sem_u8, flow, org, rays_dev, M, cls_i8, dist_f16, flow_f16, (cudaStream_t)stream);
}

int occb200_ray_score(const uint8_t* sem_pred, const float* flow_pred, const uint8_t* sem_gt, const float* flow_gt,
                      const void* origins_host, int origin_is_f64, int T, const float* rays_dev, int M, double* counters_dev,
                      void* stream)
{
    OCC_CHECK(T >= 1 && T <= 8, "T (lidar origins) must be in 1..8");
    OCC_CHECK(M >= 1, "M (rays) must be positive");
    OCC_CHECK(sem_pred && flow_pred && sem_gt && flow_gt && origins_host && rays_dev && counters_dev, "null pointer");
    RayOrigins org;
    if (fill_origins(org, origins_host, origin_is_f64, T)) return 1;
    return launch_ray_score(sem_pred, flow_pred, sem_gt, flow_gt, org, rays_dev, M, counters_dev, (cudaStream_t)stream);
}

int occb200_engine_set_rays(occb200_engine* e, const float* rays_host, int M)
{
    OCC_CHECK(e, "null engine");
    OCC_CHECK(rays_host && M >= 1, "set_rays: null ray bundle or M < 1");
    e->ray_req.armed = false;
    e->score_req.armed = false;
    if (upload(e->rays, rays_host, (size_t)M * 3)) return 2;
    e->rays_M = M;
    return 0;
}

int occb200_engine_request_rays(occb200_engine* e, const void* origins_host, int origin_is_f64, int T, int8_t* cls_i8,
                                void* dist_f16, void* flow_f16)
{
    if (e) e->ray_req.armed = false;                               // every rejection below leaves the request disarmed
    OCC_CHECK(T >= 0 && T <= 8, "T (lidar origins) must be in 0..8");
    OCC_CHECK(e, "null engine");
    if (T == 0 || origins_host == nullptr) return 0;
    OCC_CHECK(cls_i8 && dist_f16 && flow_f16, "null pointer");
    OCC_CHECK(e->rays.p != nullptr, "request_rays: occb200_engine_set_rays() has not been called");
    OCC_CHECK(e->cfg.bev_w == 200 && e->cfg.bev_h == 200 && e->cfg.pillar_h == 16,
              "request_rays: the ray caster works on the 200 x 200 x 16 grid only");
    RayRequest rq;
    if (fill_origins(rq.org, origins_host, origin_is_f64, T)) return 1;
    rq.armed = true;
    rq.cls = cls_i8; rq.dist = dist_f16; rq.flow = flow_f16;
    e->ray_req = rq;
    return 0;
}

int occb200_engine_request_score(occb200_engine* e, const uint8_t* sem_gt, const float* flow_gt, const void* origins_host,
                                 int origin_is_f64, int T, double* counters_dev)
{
    if (e) e->score_req.armed = false;                             // every rejection below leaves the request disarmed
    OCC_CHECK(T >= 0 && T <= 8, "T (lidar origins) must be in 0..8");
    OCC_CHECK(e, "null engine");
    if (T == 0 || origins_host == nullptr) return 0;
    OCC_CHECK(sem_gt && flow_gt && counters_dev, "null pointer");
    OCC_CHECK(e->rays.p != nullptr, "request_score: occb200_engine_set_rays() has not been called");
    OCC_CHECK(e->cfg.bev_w == 200 && e->cfg.bev_h == 200 && e->cfg.pillar_h == 16,
              "request_score: the ray caster works on the 200 x 200 x 16 grid only");
    ScoreRequest sq;
    if (fill_origins(sq.org, origins_host, origin_is_f64, T)) return 1;
    sq.armed = true;
    sq.sem_gt = sem_gt; sq.flow_gt = flow_gt; sq.counters = counters_dev;
    e->score_req = sq;
    return 0;
}

int occb200_engine_set_prev_rotation(occb200_engine* e, const int32_t* map_host)
{
    OCC_CHECK(e, "null engine");
    if (map_host == nullptr) { e->rot = occb200_engine::ROT_NONE; return 0; }
    for (int q = 0; q < e->Nq; ++q) OCC_CHECK(map_host[q] >= -1 && map_host[q] < e->Nq, "rotation map entry out of range");
    if (ensure(e->rot_map, (size_t)e->Nq * 4)) return 2;
    OCC_CUDA(cudaMemcpy(e->rot_map.p, map_host, (size_t)e->Nq * 4, cudaMemcpyHostToDevice));
    e->rot = occb200_engine::ROT_MAP;
    return 0;
}

int occb200_engine_set_prev_rotation_angle(occb200_engine* e, double angle_deg)
{
    OCC_CHECK(std::isfinite(angle_deg), "rotation angle must be finite");
    OCC_CHECK(e, "null engine");
    e->rot_grid = rotation_grid(e, angle_deg);
    e->rot = occb200_engine::ROT_GRID;
    return 0;
}

int occb200_engine_rotation_map(occb200_engine* e, double angle_deg, int32_t* map_dev, void* stream)
{
    OCC_CHECK(std::isfinite(angle_deg), "rotation angle must be finite");
    OCC_CHECK(map_dev, "null pointer");
    OCC_CHECK(e, "null engine");
    return launch_rotation_map(rotation_grid(e, angle_deg), map_dev, (cudaStream_t)stream);
}

int occb200_rotation_coeffs(double angle_deg, int bev_h, int bev_w, int cx, int cy, float out[6])
{
    OCC_CHECK(std::isfinite(angle_deg), "rotation angle must be finite");
    OCC_CHECK(out, "null pointer");
    OCC_CHECK(bev_h > 0 && bev_w > 0, "bev_h and bev_w must be positive");
    rotation_coeffs(angle_deg, bev_h, bev_w, cx, cy, out);
    return 0;
}

int occb200_engine_set_input_dtype(occb200_engine* e, int feats_bf16)
{
    OCC_CHECK(e && feats_bf16 >= 0 && feats_bf16 <= 4,
              "input dtype must be 0 (fp32 NCHW), 1 (bf16 NCHW), 2 (bf16 NHWC), 3 (uint8 camera frames) or 4 (JPEG camera files)");
    e->feats_bf16 = feats_bf16;
    return 0;
}

int occb200_engine_attach_backbone(occb200_engine* e, occb200_backbone* bb)
{
    OCC_CHECK(e, "null engine");
    if (bb && check_backbone(e, bb)) return 1;
    if (e->bb_free_recorded) OCC_CUDA(cudaEventSynchronize(e->bb_free));   // the previous backbone may still be running
    e->bb = bb;
    e->bb_free_recorded = false;
    return 0;
}

int occb200_engine_enable_taps(occb200_engine* e, int enable)
{
    OCC_CHECK(e && e->finalized, "engine not finalized");
    e->taps = enable != 0;
    if (e->taps) {
        const size_t n = (size_t)e->cfg.num_layers * e->Nq * 256 * 4;
        if (e->tap_layer.alloc(n) || e->tap_tsa.alloc(n) || e->tap_sca.alloc(n)) return 2;
    }
    return 0;
}

int occb200_engine_copy_tap(occb200_engine* e, int which, int layer, float* dst, void* stream)
{
    OCC_CHECK(e && dst, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)e->Nq * 256;
    if (which >= 0 && which <= 2) {
        OCC_CHECK(e->taps && layer >= 0 && layer < e->cfg.num_layers, "taps not enabled or bad layer");
        const DevBuf& b = which == 0 ? e->tap_layer : (which == 1 ? e->tap_tsa : e->tap_sca);
        OCC_CUDA(cudaMemcpyAsync(dst, b.as<float>() + layer * n, n * 4, cudaMemcpyDeviceToDevice, st));
        return 0;
    }
    if (which == 3) {
        const size_t nv = (size_t)e->cfg.bev_w * e->cfg.bev_h * e->cfg.pillar_h * e->cfg.out_dim;
        if (e->cfg.precision == 0) {
            OCC_CUDA(cudaMemcpyAsync(dst, e->vox2.p, nv * 4, cudaMemcpyDeviceToDevice, st));
            return 0;
        }
        return launch_bf16_to_f32(e->vox2.as<bf16>(), dst, (int64_t)nv, st);
    }
    if (which == 4) {                                            // packed camera tokens [num_cams, Nv, C] (row a9)
        const size_t nt = (size_t)e->cfg.num_cams * e->Nv * 256;
        if (e->cfg.precision == 0) {
            OCC_CUDA(cudaMemcpyAsync(dst, e->tokens.p, nt * 4, cudaMemcpyDeviceToDevice, st));
            return 0;
        }
        return launch_bf16_to_f32(e->tokens.as<bf16>(), dst, (int64_t)nt, st);
    }
    set_last_error("unknown tap");
    return 1;
}

int occb200_engine_project_pillars(occb200_engine* e, float* ref_cam, uint8_t* mask, void* stream)
{
    OCC_CHECK(e && ref_cam && mask && e->cameras_set, "null pointer / cameras not set");
    return launch_project_pillars(e->sp, ref_cam, mask, (cudaStream_t)stream);
}

int occb200_engine_launches_per_frame(const occb200_engine* e) { return e ? e->launches : 0; }

int occb200_engine_profile(occb200_engine* e, int enable)
{
    OCC_CHECK(e, "null engine");
    e->profiling = enable != 0;
    e->prof_events.clear();
    e->event_used = 0;
    return 0;
}

int occb200_engine_profile_read(occb200_engine* e, float* ms_per_category, int* launches_per_category, int n)
{
    OCC_CHECK(e && ms_per_category && launches_per_category && n >= CAT_COUNT, "bad arguments");
    OCC_CUDA(cudaDeviceSynchronize());
    for (int i = 0; i < n; ++i) { ms_per_category[i] = 0.f; launches_per_category[i] = 0; }
    for (auto& pe : e->prof_events) {
        float ms = 0.f;
        OCC_CUDA(cudaEventElapsedTime(&ms, pe.second.first, pe.second.second));
        ms_per_category[pe.first] += ms;
        launches_per_category[pe.first] += 1;
    }
    e->prof_events.clear();
    e->event_used = 0;
    return 0;
}

int occb200_render_forward(const float* sigma, const float* origin, const float* points, const float* tindex, int N,
                           int T, int To, int Z, int Y, int X, int64_t M, int K, float* pred_dist, float* gt_dist,
                           float* coord_index, void* stream)
{
    OCC_CHECK(sigma && origin && points && tindex && pred_dist && gt_dist && coord_index, "null pointer");
    OCC_CHECK(N >= 0 && N <= 65535 && M >= 0, "render_forward: N must be in 0..65535 and M >= 0");
    OCC_CHECK(T >= 1 && To >= 1 && Z >= 1 && Y >= 1 && X >= 1, "render_forward: T, To, Z, Y and X must be positive");
    OCC_CHECK(K >= 3, "render_forward: points need K >= 3 columns");
    return launch_render_forward(sigma, origin, points, tindex, N, T, To, Z, Y, X, M, K, pred_dist, gt_dist, coord_index,
                                 (cudaStream_t)stream);
}

int occb200_ray_metric_accumulate(const uint8_t* sem_pred, const float* flow_pred, const uint8_t* sem_gt,
                                  const float* flow_gt, const void* origins, int origin_is_f64, int T, const float* rays,
                                  int M, double* counters, float* pcd_pred, float* pcd_gt, void* stream)
{
    if (T == 0 || M == 0) return 0;                              // no origins / rays: counters untouched
    OCC_CHECK(sem_pred && flow_pred && sem_gt && flow_gt && origins && rays && counters, "null pointer");
    return launch_ray_metric(sem_pred, flow_pred, sem_gt, flow_gt, origins, origin_is_f64, T, rays, M, counters,
                             pcd_pred, pcd_gt, (cudaStream_t)stream);
}

int occb200_linear_f32(const float* A, const float* W, const float* bias, const float* residual, float* C, int M, int N,
                       int K, int act, void* stream)
{
    OCC_CHECK(A && W && C, "null pointer");
    OCC_CHECK(M >= 0 && N > 0 && K > 0, "linear: bad sizes");
    OCC_CHECK(act == ACT_NONE || act == ACT_RELU, "linear: act must be 0 or 1");
    OCC_CHECK(aligned16(A) && aligned16(W) && aligned16(bias) && aligned16(residual) && aligned16(C),
              "device arrays must be 16-byte aligned");
    return gemm_simt<float, float>(A, K, nullptr, 0, K, W, bias, residual, N, C, N, M, N, K, act, (cudaStream_t)stream);
}

int occb200_layernorm_f32(const float* x, const float* gamma, const float* beta, float* y, int rows, int C, void* stream)
{
    OCC_CHECK(x && gamma && beta && y, "null pointer");
    OCC_CHECK(rows >= 0, "layernorm: rows must be >= 0");
    OCC_CHECK(aligned16(x) && aligned16(gamma) && aligned16(beta) && aligned16(y), "device arrays must be 16-byte aligned");
    if (rows == 0) return 0;
    return launch_layernorm<float>(x, gamma, beta, nullptr, rows, C, y, (float*)nullptr, (float*)nullptr,
                                   (cudaStream_t)stream);
}

int occb200_gemm_bf16_tc(const void* A, const void* W, const float* bias, float* C, int M, int N, int K, void* stream)
{
    OCC_CHECK(A && W && C, "null pointer");
    OCC_CHECK(gemm_tc_supported(M, N, K, K), "shape not supported by the tensor-core GEMM");
    return gemm_tc<float>(reinterpret_cast<const bf16*>(A), nullptr, 0, reinterpret_cast<const bf16*>(W), bias, nullptr,
                          C, M, N, K, ACT_NONE, (cudaStream_t)stream);
}

// ---- tensor-core GEMM variants for kernel tests: argument checks only, every rejection before the first CUDA call
int occb200_gemm_tc(const void* A, const void* A2, int K1, const void* W, const float* bias, const float* residual, void* C,
                    int out_dtype, int M, int N, int K, int act, void* stream)
{
    OCC_CHECK(A && W && C, "null pointer");
    OCC_CHECK(out_dtype >= 0 && out_dtype <= 2, "out_dtype must be 0 (fp32), 1 (bf16) or 2 (fp16)");
    OCC_CHECK(act == ACT_NONE || act == ACT_RELU, "act must be 0 (none) or 1 (relu)");
    OCC_CHECK(K > 0 && (A2 == nullptr || K1 < K) && gemm_tc_supported(M, N, K, A2 ? K1 : K),
              "shape not supported by the tensor-core GEMM (M > 0, N % 64, K % 64, K1 % 64, 0 < K1 < K)");
    const bf16 *a = reinterpret_cast<const bf16*>(A), *a2 = reinterpret_cast<const bf16*>(A2), *w = reinterpret_cast<const bf16*>(W);
    const cudaStream_t st = (cudaStream_t)stream;
    if (out_dtype == 0) return gemm_tc<float>(a, a2, K1, w, bias, residual, reinterpret_cast<float*>(C), M, N, K, act, st);
    if (out_dtype == 1) return gemm_tc<bf16>(a, a2, K1, w, bias, residual, reinterpret_cast<bf16*>(C), M, N, K, act, st);
    return gemm_tc<__half>(a, a2, K1, w, bias, residual, reinterpret_cast<__half*>(C), M, N, K, act, st);
}

int occb200_gemm_tc_ln(const void* A, const void* W, const float* bias, const float* residual, const float* gamma,
                       const float* beta, const float* pos, float* y_f32, void* y_bf16, void* y_pos_bf16, int M, int K,
                       void* stream)
{
    OCC_CHECK(A && W && bias && residual && gamma && beta, "null pointer");
    OCC_CHECK(y_pos_bf16 == nullptr || pos != nullptr, "y_pos_bf16 needs pos");
    OCC_CHECK(M > 0 && K > 0 && K % 64 == 0, "shape not supported by the LayerNorm GEMM (M > 0, K % 64)");
    return gemm_tc_ln(reinterpret_cast<const bf16*>(A), reinterpret_cast<const bf16*>(W), bias, residual, gamma, beta, pos, y_f32,
                      reinterpret_cast<bf16*>(y_bf16), reinterpret_cast<bf16*>(y_pos_bf16), M, K, (cudaStream_t)stream);
}

int occb200_gemm_tc_blocked256(const void* A, const void* W, const float* bias, void* C, int M, int N, int K, void* stream)
{
    OCC_CHECK(A && W && C, "null pointer");
    OCC_CHECK(K > 0 && N % 256 == 0 && gemm_tc_supported(M, N, K, K), "shape not supported (M > 0, N % 256, K % 64)");
    return gemm_tc_blocked256(reinterpret_cast<const bf16*>(A), reinterpret_cast<const bf16*>(W), bias, reinterpret_cast<bf16*>(C),
                              M, N, K, (cudaStream_t)stream);
}

int occb200_gemm_tc_tsa_inputs(const void* const* Av, int nv, const void* Wv, const float* bv, void* const* Cv, const void* Aq,
                               const void* Aq2, int K1q, const void* Wq, const float* bq, const float* rq, const float* rq_t32,
                               void* Cq, int M, int Nq, int Kq, void* stream)
{
    OCC_CHECK(nv >= 1 && nv <= 2, "nv must be 1 or 2");
    OCC_CHECK(Av && Cv && Wv && Aq && Wq && Cq, "null pointer");
    for (int i = 0; i < nv; ++i) OCC_CHECK(Av[i] && Cv[i], "null value operand / output");
    OCC_CHECK(rq_t32 == nullptr || rq != nullptr, "rq_t32 needs the row-major rq (used when M % 32 != 0)");
    OCC_CHECK(gemm_tc_supported(M, 256, 256, 256), "shape not supported (M > 0)");
    OCC_CHECK(Kq > 0 && (Aq2 == nullptr || K1q < Kq) && gemm_tc_supported(M, Nq, Kq, Aq2 ? K1q : Kq),
              "projection shape not supported (Nq % 64, Kq % 64, K1q % 64, 0 < K1q < Kq)");
    return gemm_tc_tsa_inputs(reinterpret_cast<const bf16* const*>(Av), nv, reinterpret_cast<const bf16*>(Wv), bv,
                              reinterpret_cast<bf16* const*>(Cv), reinterpret_cast<const bf16*>(Aq), reinterpret_cast<const bf16*>(Aq2), K1q, reinterpret_cast<const bf16*>(Wq), bq, rq, rq_t32,
                              reinterpret_cast<__half*>(Cq), M, Nq, Kq, (cudaStream_t)stream);
}

int occb200_gemm_tc_split3(const void* S, int Ks, const void* W3, const float* bias, const float* residual, float* C, int M, int N,
                           int act, void* stream)
{
    OCC_CHECK(S && W3 && C, "null pointer");
    OCC_CHECK(act == ACT_NONE || act == ACT_RELU, "act must be 0 (none) or 1 (relu)");
    OCC_CHECK(Ks > 0 && gemm_tc_supported(M, N, 3 * Ks, 2 * Ks), "shape not supported (M > 0, N % 64, Ks % 64)");
    return gemm_tc_split3(reinterpret_cast<const bf16*>(S), Ks, reinterpret_cast<const bf16*>(W3), bias, residual, C, M, N, act,
                          (cudaStream_t)stream);
}

int occb200_split_bf16(const float* a, int Ka, const float* b, int Kb, int64_t rows, void* S, void* stream)
{
    OCC_CHECK(a && S && (Kb == 0 || b), "null pointer");
    OCC_CHECK(rows >= 0 && Ka > 0 && Kb >= 0 && Ka % 8 == 0 && Kb % 8 == 0, "Ka, Kb must be multiples of 8");
    return launch_split_bf16(a, Ka, b, Kb, rows, reinterpret_cast<bf16*>(S), (cudaStream_t)stream);
}

// ---- the fused attention gathers for kernel tests: argument checks only, every rejection before the first CUDA call, then the
// launcher the frame engine calls.  Value / projection types: the three combinations the engine launches.
#define OCC_CHECK_GATHER_TYPES(value_bf16, qproj_f16)                                                                   \
    OCC_CHECK((value_bf16 == 0 || value_bf16 == 1) && (qproj_f16 == 0 || qproj_f16 == 1) && (value_bf16 || !qproj_f16), \
              "value / projection types must be fp32 / fp32, bf16 / fp32 or bf16 / fp16")

int occb200_tsa_gather(const void* v_prev, const void* v_cur, int value_bf16, const void* qproj, int qproj_f16, int bev_h,
                       int bev_w, void* out, void* stream)
{
    OCC_CHECK(v_prev && v_cur && qproj && out, "null pointer");
    OCC_CHECK_GATHER_TYPES(value_bf16, qproj_f16);
    OCC_CHECK(bev_h >= 2 && bev_w >= 2, "the BEV grid must be at least 2x2");
    const cudaStream_t st = (cudaStream_t)stream;
    if (value_bf16)
        return launch_tsa_fused<bf16>(reinterpret_cast<const bf16*>(v_prev), reinterpret_cast<const bf16*>(v_cur), qproj,
                                      qproj_f16 != 0, bev_h, bev_w, reinterpret_cast<bf16*>(out), st);
    return launch_tsa_fused<float>(reinterpret_cast<const float*>(v_prev), reinterpret_cast<const float*>(v_cur), qproj, false,
                                   bev_h, bev_w, reinterpret_cast<float*>(out), st);
}

int occb200_sca_gather(const void* value, int value_bf16, const void* qproj, int qproj_f16, const float* cam_mat_host,
                       const float* zs_host, int num_cams, int D, const float pc_range[6], int img_h, int img_w, int bev_h,
                       int bev_w, const int level_hw_host[8], void* out, uint8_t* hits, void* stream)
{
    OCC_CHECK(value && qproj && cam_mat_host && zs_host && pc_range && level_hw_host && out, "null pointer");
    OCC_CHECK_GATHER_TYPES(value_bf16, qproj_f16);
    OCC_CHECK(num_cams >= 1 && num_cams <= 8, "num_cams must be in [1,8]");
    OCC_CHECK(D == 1 || D == 2 || D == 4 || D == 8, "D (num_points_in_pillar) must be 1, 2, 4 or 8");
    OCC_CHECK(img_h > 0 && img_w > 0, "the image size must be positive");
    OCC_CHECK(bev_h > 0 && bev_w > 0, "the BEV size must be positive");
    int level_h[4], level_w[4];
    for (int l = 0; l < 4; ++l) {
        level_h[l] = level_hw_host[2 * l]; level_w[l] = level_hw_host[2 * l + 1];
        OCC_CHECK(level_h[l] >= 2 && level_w[l] >= 2, "every level must be at least 2x2");
    }
    int Nv = 0;
    const LevelGeom lg = make_level_geom(level_h, level_w, &Nv);
    const ScaParams sp = make_sca_params(cam_mat_host, zs_host, num_cams, D, pc_range, img_h, img_w, bev_h, bev_w);
    const cudaStream_t st = (cudaStream_t)stream;
    if (value_bf16)
        return launch_sca_fused<bf16>(reinterpret_cast<const bf16*>(value), qproj, qproj_f16 != 0, sp, lg, Nv,
                                      reinterpret_cast<bf16*>(out), hits, st);
    return launch_sca_fused<float>(reinterpret_cast<const float*>(value), qproj, false, sp, lg, Nv, reinterpret_cast<float*>(out),
                                   hits, st);
}
#undef OCC_CHECK_GATHER_TYPES

// ---- the voxel decoder's steps for operator tests: the route make_frame_plan picks for (precision, use_tensor_cores,
// num_classes) with pillar_h 16 and out_dim 32, weights built by the engine's helpers, then the step the frame runs.  Every
// rejection returns 1 before the first CUDA call; each entry synchronises `stream` (its weights are freed on return).
#define OCC_CHECK_PLAN_CONFIG(precision, use_tensor_cores)                                 \
    OCC_CHECK(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (bf16)"); \
    OCC_CHECK(use_tensor_cores == 0 || use_tensor_cores == 1, "use_tensor_cores must be 0 or 1")

int occb200_decoder_lift(int precision, int use_tensor_cores, int from_t32, const float* bev, int bev_h, int bev_w, void* vox,
                         int* launches, void* stream)
{
    OCC_CHECK(bev && vox && launches, "null pointer");
    OCC_CHECK_PLAN_CONFIG(precision, use_tensor_cores);
    const FramePlan p = decoder_test_plan(precision, use_tensor_cores, 17);
    OCC_CHECK(from_t32 == 0 || (from_t32 == 1 && p.lift_t32), "from_t32 must be 0, or 1 with bf16 storage and tensor cores");
    OCC_CHECK(bev_h > 0 && bev_w > 0 && (int64_t)bev_h * bev_w <= (1 << 24), "the BEV grid must be positive, at most 2^24 cells");
    const cudaStream_t st = (cudaStream_t)stream;
    const int n = precision ? decoder_lift<bf16>(from_t32 != 0, bev, bev_h, bev_w, 16, reinterpret_cast<bf16*>(vox), st)
                            : decoder_lift<float>(false, bev, bev_h, bev_w, 16, reinterpret_cast<float*>(vox), st);
    if (n < 0) return 2;
    OCC_CUDA(cudaStreamSynchronize(st));
    *launches = n;
    return 0;
}

int occb200_decoder_conv3d(int precision, int use_tensor_cores, const void* in, int X, int Y, int cin, const float* w_host,
                           const float* bn_host, void* out, int* path, int* launches, void* stream)
{
    OCC_CHECK(in && w_host && bn_host && out && path && launches, "null pointer");
    OCC_CHECK_PLAN_CONFIG(precision, use_tensor_cores);
    OCC_CHECK(X >= 1 && X <= 4096 && Y >= 1 && Y <= 4096, "X and Y must be in [1, 4096]");
    OCC_CHECK(cin == 16 || cin == 32, "cin must be 16 or 32");
    const FramePlan p = decoder_test_plan(precision, use_tensor_cores, 17);
    const int od = 32;
    DecoderConvW w;
    if (upload_decoder_conv(w, p.conv, w_host, bn_host, bn_host + od, bn_host + 2 * od, bn_host + 3 * od, cin, od)) return 2;
    DevBuf split;                                                   // CONV_SPLIT: the [hi | lo] operand, as the frame's vox_split
    if (p.conv == FramePlan::CONV_SPLIT && split.alloc((size_t)X * Y * 16 * 2 * cin * 2)) return 2;
    const cudaStream_t st = (cudaStream_t)stream;
    const int n = precision ? decoder_conv<bf16>(p.conv, reinterpret_cast<const bf16*>(in), w, X, Y, 16, cin,
                                                 reinterpret_cast<bf16*>(out), split.as<bf16>(), st)
                            : decoder_conv<float>(p.conv, reinterpret_cast<const float*>(in), w, X, Y, 16, cin,
                                                  reinterpret_cast<float*>(out), split.as<bf16>(), st);
    if (n < 0) return 2;
    OCC_CUDA(cudaStreamSynchronize(st));
    *path = p.conv; *launches = n;
    return 0;
}

int occb200_decoder_head(int precision, int use_tensor_cores, int num_classes, const void* vox, int64_t nvox, const float* w1,
                         const float* b1, const float* w2, const float* b2, const float* f1, const float* g1, const float* f2,
                         const float* g2, float* occ_logits, float* flow, uint8_t* cls_u8, int64_t* cls_i64, int* path,
                         int* launches, void* stream)
{
    OCC_CHECK(vox && w1 && b1 && w2 && b2 && f1 && g1 && f2 && g2 && path && launches, "null pointer");
    OCC_CHECK_PLAN_CONFIG(precision, use_tensor_cores);
    OCC_CHECK(num_classes >= 1 && num_classes <= 32, "num_classes must be in [1, 32]");
    OCC_CHECK(nvox >= 1 && nvox < (1ll << 31), "nvox must be in [1, 2^31)");
    const FramePlan p = decoder_test_plan(precision, use_tensor_cores, num_classes);
    DecoderHeadW h;
    if (upload_decoder_head(h, p.head_tc, num_classes, 32, w1, b1, w2, b2, f1, g1, f2, g2)) return 2;
    const cudaStream_t st = (cudaStream_t)stream;
    const int n = precision ? decoder_head<bf16>(p.head_tc, reinterpret_cast<const bf16*>(vox), h, num_classes, nvox, occ_logits,
                                                 flow, cls_u8, cls_i64, st)
                            : decoder_head<float>(false, reinterpret_cast<const float*>(vox), h, num_classes, nvox, occ_logits,
                                                  flow, cls_u8, cls_i64, st);
    if (n < 0) return 2;
    OCC_CUDA(cudaStreamSynchronize(st));
    *path = p.head_tc ? 1 : 0; *launches = n;
    return 0;
}

// ---- the encoder's unfused kernels for operator tests: the plan make_frame_plan makes for (precision, use_tensor_cores) at the
// engine's attention shapes, dense weights built by the engine's upload_dense, then the GEMM step or launcher the frame runs.
// Every rejection returns 1 before the first CUDA call; each entry synchronises `stream` (its weights are freed on return).
int occb200_encoder_dense(int precision, int use_tensor_cores, const void* A, const void* A2, int K1, const float* w_host,
                          const float* bias_host, const float* residual, void* out, int out_dtype, int M, int N, int K, int act,
                          int* path, int* launches, void* stream)
{
    OCC_CHECK(A && w_host && out && path && launches, "null pointer");
    OCC_CHECK_PLAN_CONFIG(precision, use_tensor_cores);
    OCC_CHECK(act == ACT_NONE || act == ACT_RELU, "act must be 0 (none) or 1 (relu)");
    OCC_CHECK(M >= 0 && N > 0 && N % 4 == 0 && K > 0 && K % 16 == 0, "shape: M >= 0, N a positive multiple of 4, K of 16");
    OCC_CHECK(A2 ? K1 > 0 && K1 < K && K1 % 8 == 0 : K1 == 0,
              "split point: 0 < K1 < K and K1 % 8 == 0 with A2, K1 = 0 without");
    OCC_CHECK(aligned16(A) && aligned16(A2) && aligned16(residual) && aligned16(out), "device arrays must be 16-byte aligned");
    OCC_CHECK(out_dtype == 0 || (out_dtype == 1 && precision == 1) || out_dtype == 2,
              "out_dtype must be 0 (fp32), the storage type (1: bf16) or 2 (fp16)");
    const FramePlan p = encoder_test_plan(precision, use_tensor_cores);
    const int route = precision ? dense_route<bf16, bf16>(p, M, N, K, A2 ? K1 : K) : dense_route<float, float>(p, M, N, K, A2 ? K1 : K);
    OCC_CHECK(out_dtype != 2 || (p.qproj_f16 && route == OCCB200_DENSE_TC),
              "fp16 outputs exist only on the tensor-core route of bf16 storage with tensor cores");
    DevBuf w, b, wh, split;
    if (upload_dense(p, w, b, &wh, w_host, bias_host, N, K)) return 2;
    if (route == OCCB200_DENSE_SPLIT && split.alloc((size_t)M * 2 * K * 2)) return 2;
    const cudaStream_t st = (cudaStream_t)stream;
    const float *wf = w.as<float>(), *bf = b.as<float>();
    bf16* ws = split.as<bf16>();
    int n;
    if (precision == 0) {
        n = dense_gemm<float, float>(p, reinterpret_cast<const float*>(A), reinterpret_cast<const float*>(A2), K1, wf, wh.p, bf,
                                     residual, reinterpret_cast<float*>(out), M, N, K, act, ws, st);
    } else {
        const bf16 *a = reinterpret_cast<const bf16*>(A), *a2 = reinterpret_cast<const bf16*>(A2);
        n = out_dtype == 0 ? dense_gemm<bf16, float>(p, a, a2, K1, wf, wh.p, bf, residual, reinterpret_cast<float*>(out), M, N, K,
                                                     act, ws, st)
          : out_dtype == 1 ? dense_gemm<bf16, bf16>(p, a, a2, K1, wf, wh.p, bf, residual, reinterpret_cast<bf16*>(out), M, N, K,
                                                    act, ws, st)
                           : dense_gemm<bf16, __half>(p, a, a2, K1, wf, wh.p, bf, residual, reinterpret_cast<__half*>(out), M, N,
                                                      K, act, ws, st);
    }
    if (n < 0) return 2;
    OCC_CUDA(cudaStreamSynchronize(st));
    *path = route; *launches = n;
    return 0;
}

int occb200_encoder_layernorm(int precision, const float* x, const float* gamma, const float* beta, const float* pos, int rows,
                              float* y_f32, void* y_t, void* y_pos_t, void* stream)
{
    OCC_CHECK(x && gamma && beta, "null pointer");
    OCC_CHECK(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (bf16)");
    OCC_CHECK(y_pos_t == nullptr || pos != nullptr, "y_pos_t needs pos");
    OCC_CHECK(rows >= 1, "rows must be positive");
    OCC_CHECK(aligned16(x) && aligned16(gamma) && aligned16(beta) && aligned16(pos) && aligned16(y_f32) && aligned16(y_t) &&
                  aligned16(y_pos_t), "device arrays must be 16-byte aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    const int rc = precision ? launch_layernorm<bf16>(x, gamma, beta, pos, rows, 256, y_f32, reinterpret_cast<bf16*>(y_t),
                                                      reinterpret_cast<bf16*>(y_pos_t), st)
                             : launch_layernorm<float>(x, gamma, beta, pos, rows, 256, y_f32, reinterpret_cast<float*>(y_t),
                                                       reinterpret_cast<float*>(y_pos_t), st);
    if (rc) return rc;
    OCC_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int occb200_encoder_pack(int precision, int layout, const void* const* feats_dev, int num_levels, const int* level_hw_host,
                         int num_cams, const float* cams_embeds, const float* level_embeds, void* tokens, void* stream)
{
    OCC_CHECK(feats_dev && level_hw_host && level_embeds && tokens, "null pointer");
    OCC_CHECK(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (bf16)");
    OCC_CHECK(layout >= 0 && layout <= 2, "layout must be 0 (fp32 NCHW), 1 (bf16 NCHW) or 2 (bf16 NHWC)");
    OCC_CHECK(num_levels >= 1 && num_levels <= 8, "num_levels must be in [1, 8]");
    OCC_CHECK(num_cams >= 1 && num_cams <= 8, "num_cams must be in [1, 8]");
    int level_h[8], level_w[8];
    int64_t total = 0;
    for (int l = 0; l < num_levels; ++l) {
        level_h[l] = level_hw_host[2 * l]; level_w[l] = level_hw_host[2 * l + 1];
        OCC_CHECK(level_h[l] >= 1 && level_w[l] >= 1 && (int64_t)level_h[l] * level_w[l] <= (1 << 24),
                  "every level must be at least 1x1, at most 2^24 pixels");
        total += (int64_t)level_h[l] * level_w[l];
        OCC_CHECK(feats_dev[l] != nullptr, "null feature level");
        OCC_CHECK(aligned16(feats_dev[l]), "device arrays must be 16-byte aligned");
    }
    OCC_CHECK(total <= (1 << 24), "the levels must hold at most 2^24 pixels in all");
    OCC_CHECK(aligned16(cams_embeds) && aligned16(level_embeds) && aligned16(tokens), "device arrays must be 16-byte aligned");
    int Nv = 0;
    const LevelGeom lg = make_level_geom(level_h, level_w, &Nv, num_levels);
    const cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if (layout == 2)
        rc = precision ? launch_pack_levels_nhwc<bf16>(feats_dev, lg, cams_embeds, level_embeds, num_cams, 256, Nv,
                                                       reinterpret_cast<bf16*>(tokens), st)
                       : launch_pack_levels_nhwc<float>(feats_dev, lg, cams_embeds, level_embeds, num_cams, 256, Nv,
                                                        reinterpret_cast<float*>(tokens), st);
    else
        rc = precision ? launch_pack_levels<bf16>(feats_dev, layout, lg, cams_embeds, level_embeds, num_cams, 256, Nv,
                                                  reinterpret_cast<bf16*>(tokens), st)
                       : launch_pack_levels<float>(feats_dev, layout, lg, cams_embeds, level_embeds, num_cams, 256, Nv,
                                                   reinterpret_cast<float*>(tokens), st);
    if (rc) return rc;
    OCC_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int occb200_encoder_prepare_query(int precision, int tiled, const float* q, const float* pos, int64_t n, float* q_f32, void* q_t,
                                  void* q_pos_t, void* stream)
{
    OCC_CHECK(q && pos, "null pointer");
    OCC_CHECK(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (bf16)");
    OCC_CHECK(tiled == 0 || tiled == 1, "tiled must be 0 or 1");
    OCC_CHECK(n > 0 && n % 8 == 0 && (!tiled || n % 256 == 0), "n must be a positive multiple of 8 (tiled: of 256)");
    OCC_CHECK(aligned16(q) && aligned16(pos) && aligned16(q_f32) && aligned16(q_t) && aligned16(q_pos_t),
              "device arrays must be 16-byte aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    const int rc = precision ? launch_prepare_query<bf16>(q, pos, n, q_f32, reinterpret_cast<bf16*>(q_t),
                                                          reinterpret_cast<bf16*>(q_pos_t), tiled, st)
                             : launch_prepare_query<float>(q, pos, n, q_f32, reinterpret_cast<float*>(q_t),
                                                           reinterpret_cast<float*>(q_pos_t), tiled, st);
    if (rc) return rc;
    OCC_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int occb200_t32_convert(const float* src, float* dst, int64_t rows, int untile, int ncols, void* stream)
{
    OCC_CHECK(src && dst, "null pointer");
    OCC_CHECK(untile == 0 || untile == 1, "untile must be 0 or 1");
    OCC_CHECK(rows >= 1 && ncols > 0 && ncols % 32 == 0, "rows must be positive, ncols a positive multiple of 32");
    OCC_CHECK(aligned16(src) && aligned16(dst), "device arrays must be 16-byte aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    if (launch_t32_convert(src, dst, rows, untile, st, ncols)) return 2;
    OCC_CUDA(cudaStreamSynchronize(st));
    return 0;
}
#undef OCC_CHECK_PLAN_CONFIG

}  // extern "C"
