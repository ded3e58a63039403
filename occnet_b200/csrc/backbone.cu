// Image backbone + neck engine and its C ABI (include/occ_b200.h, "occb200_backbone_*"): ResNet-50 (style 'pytorch',
// out_indices (1,2,3)) + mmdet FPN (start_level 0, add_extra_convs 'on_output', num_outs 4), i.e. the modules
// bevformer_base_occ.py:48-66 puts in front of the hot path (caller: detectors/bevformer_occ.py:66-99; eval mode:
// GridMask is the identity, BatchNorm uses running statistics).  SURVEY 8f rank 1 ("next").
//
// Checked by tests/test_backbone_gpu.py; default feature extractor of the drop-in detector when it
// is given images.  See backbone_kernels.cu / conv2d_tc.cu for the design (NHWC activations, BatchNorm folded, stride-1
// convolutions on the TMA-im2col implicit-GEMM kernel, the others explicit im2col + the wgmma GEMM; fp32 parity
// configuration: the CUDA-core GEMM).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <map>
#include <string>
#include <vector>

#include "../../include/occ_b200.h"
#include "common.cuh"
#include "conv2d_tc.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"

using namespace occ;

namespace {

struct Buf {
    void* p = nullptr;
    size_t bytes = 0;
    int alloc(size_t n) {
        release();
        if (n == 0) return 0;
        OCC_CUDA(cudaMalloc(&p, n));
        bytes = n;
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    template <typename U> U* as() const { return reinterpret_cast<U*>(p); }
};

struct ConvW {                       // BN-folded, tap-major weights: w[co][(ky*KW + kx)*Cin + c], K zero-padded to kpad
    Buf w, wh, b;
    int cout = 0, cin = 0, kh = 1, kw = 1, stride = 1, pad = 0, kpad = 0;
};

constexpr int STAGE_BLOCKS[4] = {3, 4, 6, 3};
constexpr int STAGE_PLANES[4] = {64, 128, 256, 512};

}  // namespace

struct occb200_backbone {
    int num_images = 0, H = 0, W = 0, precision = 0, use_tc = 0, out_channels = 256;
    bool finalized = false;
    std::map<std::string, std::vector<float>> host_params;
    ConvW stem;
    struct Block { ConvW c1, c2, c3, down; bool has_down = false; int stride = 1; };
    std::vector<Block> blocks[4];
    ConvW lateral[3], fpnc[4];
    // workspace
    Buf img_nhwc, col, ping[2], t1, t2, t3, idn, stage_out[3], lat[3], fo[4];
    size_t elt() const { return precision ? 2 : 4; }
};

namespace {

const std::vector<float>* findp(const occb200_backbone* e, const std::string& k, size_t numel)
{
    auto it = e->host_params.find(k);
    if (it == e->host_params.end()) { set_last_error("backbone: missing parameter: " + k); return nullptr; }
    if (it->second.size() != numel) {
        set_last_error("backbone: parameter " + k + " has " + std::to_string(it->second.size()) + " elements, expected " +
                       std::to_string(numel));
        return nullptr;
    }
    return &it->second;
}

int upload_conv(occb200_backbone* e, ConvW& c, const std::vector<float>& W, const std::vector<float>& B)
{
    if (c.w.alloc(W.size() * 4) || c.b.alloc(B.size() * 4)) return 2;
    OCC_CUDA(cudaMemcpy(c.w.p, W.data(), W.size() * 4, cudaMemcpyHostToDevice));
    OCC_CUDA(cudaMemcpy(c.b.p, B.data(), B.size() * 4, cudaMemcpyHostToDevice));
    if (e->precision && e->use_tc) {
        std::vector<__nv_bfloat16> h(W.size());
        for (size_t i = 0; i < W.size(); ++i) h[i] = __float2bfloat16(W[i]);
        if (c.wh.alloc(h.size() * 2)) return 2;
        OCC_CUDA(cudaMemcpy(c.wh.p, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
    }
    return 0;
}

// conv weight [co][ci][kh][kw] (+ BatchNorm in eval mode, or a conv bias) -> folded tap-major [co][kpad] + bias[co]
int fold_conv(occb200_backbone* e, ConvW& c, const std::string& conv_key, const std::string& bn_key, int cout, int cin,
              int k, int stride, int pad, bool conv_bias)
{
    c.cout = cout; c.cin = cin; c.kh = c.kw = k; c.stride = stride; c.pad = pad;
    const int K = k * k * cin;
    c.kpad = (K + 63) / 64 * 64;
    const std::vector<float>* w = findp(e, conv_key + ".weight", (size_t)cout * cin * k * k);
    if (!w) return 3;
    std::vector<float> scale(cout, 1.f), shift(cout, 0.f);
    if (!bn_key.empty()) {
        const std::vector<float>* g = findp(e, bn_key + ".weight", cout);
        const std::vector<float>* b = findp(e, bn_key + ".bias", cout);
        const std::vector<float>* m = findp(e, bn_key + ".running_mean", cout);
        const std::vector<float>* v = findp(e, bn_key + ".running_var", cout);
        if (!g || !b || !m || !v) return 3;
        for (int o = 0; o < cout; ++o) {
            scale[o] = (*g)[o] / std::sqrt((*v)[o] + 1e-5f);
            shift[o] = (*b)[o] - (*m)[o] * scale[o];
        }
    }
    if (conv_bias) {
        const std::vector<float>* b = findp(e, conv_key + ".bias", cout);
        if (!b) return 3;
        for (int o = 0; o < cout; ++o) shift[o] += (*b)[o] * scale[o];
    }
    std::vector<float> W((size_t)cout * c.kpad, 0.f);
    for (int o = 0; o < cout; ++o)
        for (int ci = 0; ci < cin; ++ci)
            for (int ky = 0; ky < k; ++ky)
                for (int kx = 0; kx < k; ++kx)
                    W[(size_t)o * c.kpad + (size_t)(ky * k + kx) * cin + ci] =
                        (*w)[(((size_t)o * cin + ci) * k + ky) * k + kx] * scale[o];
    return upload_conv(e, c, W, shift);
}

inline int out_size(int in, int k, int stride, int pad) { return (in + 2 * pad - k) / stride + 1; }

// out[M, cout] = act(A[M, kpad] . W^T + b)
template <typename T>
int conv_gemm(occb200_backbone* e, const T* A, int64_t M, const ConvW& c, T* out, int act, cudaStream_t st)
{
    OCC_CHECK(M < (1ll << 31), "backbone: too many pixels for one GEMM");
    if constexpr (sizeof(T) == 2) {
        if (e->use_tc && c.wh.p && gemm_tc_supported((int)M, c.cout, c.kpad, c.kpad))
            return gemm_tc<bf16>(reinterpret_cast<const bf16*>(A), nullptr, 0, c.wh.as<bf16>(), c.b.as<float>(), nullptr,
                                 reinterpret_cast<bf16*>(out), (int)M, c.cout, c.kpad, act, st);
    }
    return gemm_simt<T, T>(A, c.kpad, nullptr, 0, c.kpad, c.w.as<float>(), c.b.as<float>(), nullptr, 0, out, c.cout, (int)M,
                           c.cout, c.kpad, act, st);
}

// Stride-1 3x3 convolutions (and 1x1 + residual) go through the TMA-im2col implicit-GEMM kernel conv2d_tc.cu (the default: it
// skips the im2col round trip through memory); OCC_BACKBONE_IMPLICIT=0 selects the explicit im2col + gemm_tc path for everything.
bool implicit_enabled()
{
    static const bool on = getenv("OCC_BACKBONE_IMPLICIT") == nullptr || atoi(getenv("OCC_BACKBONE_IMPLICIT")) != 0;
    return on;
}

// one convolution on NHWC input [N, H, W, cin] -> out [N, Ho, Wo, cout].  `residual` (same shape as out) is only
// accepted on the implicit-GEMM path, where the add (+ ReLU) is fused into the epilogue; fused_residual reports it.
template <typename T>
int conv(occb200_backbone* e, const T* in, int N, int H, int W, const ConvW& c, T* out, int act, int& Ho, int& Wo,
         cudaStream_t st, const T* residual = nullptr, bool* fused_residual = nullptr)
{
    Ho = out_size(H, c.kh, c.stride, c.pad);
    Wo = out_size(W, c.kw, c.stride, c.pad);
    const int64_t M = (int64_t)N * Ho * Wo;
    if (fused_residual) *fused_residual = false;
    if constexpr (sizeof(T) == 2) {
        if (e->use_tc && implicit_enabled() && c.wh.p && c.stride == 1 && c.kpad == c.kh * c.kw * c.cin &&
            conv2d_tc_supported(c.cin, c.cout, c.kh, c.kw) && (c.kh == 3 || residual != nullptr)) {
            if (fused_residual) *fused_residual = residual != nullptr;
            return conv2d_tc(reinterpret_cast<const bf16*>(in), c.wh.as<bf16>(), c.b.as<float>(),
                             reinterpret_cast<const bf16*>(residual), reinterpret_cast<bf16*>(out), N, H, W, c.cin, c.cout,
                             c.kh, c.kw, c.pad, residual ? ACT_RELU : act, st);
        }
    }
    const T* A = in;
    if (!(c.kh == 1 && c.kw == 1 && c.stride == 1 && c.kpad == c.cin)) {
        OCC_CHECK((size_t)M * c.kpad * sizeof(T) <= e->col.bytes, "backbone: im2col workspace too small");
        if (launch_im2col_nhwc<T>(in, e->col.as<T>(), N, H, W, c.cin, c.kh, c.kw, c.stride, c.pad, Ho, Wo, c.kpad, st)) return 2;
        A = e->col.as<T>();
    }
    return conv_gemm<T>(e, A, M, c, out, act, st);
}

// nhwc_out != nullptr (bf16 only): the FPN output convolutions write the caller's channels-last buffers directly
template <typename T>
int forward_impl(occb200_backbone* e, const float* img, float* const* outs, cudaStream_t st, void* const* nhwc_out = nullptr)
{
    const int N = e->num_images;
    int H = e->H, W = e->W, Ho, Wo;
    if (launch_nchw_to_nhwc_small<T>(img, e->img_nhwc.as<T>(), N, 3, H, W, st)) return 2;
    // stem: conv 7x7 s2 p3 + BN + ReLU, MaxPool 3x3 s2 p1 (mmdet ResNet.forward / torchvision resnet50)
    if (conv<T>(e, e->img_nhwc.as<T>(), N, H, W, e->stem, e->ping[0].as<T>(), ACT_RELU, Ho, Wo, st)) return 2;
    H = Ho; W = Wo;
    const int Hp = out_size(H, 3, 2, 1), Wp = out_size(W, 3, 2, 1);
    if (launch_maxpool3x3s2_nhwc<T>(e->ping[0].as<T>(), e->ping[1].as<T>(), N, H, W, 64, Hp, Wp, st)) return 2;
    H = Hp; W = Wp;
    const T* cur = e->ping[1].as<T>();
    int sh[3], sw[3];
    for (int s = 0; s < 4; ++s) {
        for (size_t b = 0; b < e->blocks[s].size(); ++b) {
            occb200_backbone::Block& blk = e->blocks[s][b];
            int h1, w1, h2, w2, h3, w3;
            if (conv<T>(e, cur, N, H, W, blk.c1, e->t1.as<T>(), ACT_RELU, h1, w1, st)) return 2;
            if (conv<T>(e, e->t1.as<T>(), N, h1, w1, blk.c2, e->t2.as<T>(), ACT_RELU, h2, w2, st)) return 2;
            const T* identity = cur;
            if (blk.has_down) {
                int hd, wd;
                if (conv<T>(e, cur, N, H, W, blk.down, e->idn.as<T>(), ACT_NONE, hd, wd, st)) return 2;
                identity = e->idn.as<T>();
            }
            const bool last = b + 1 == e->blocks[s].size();
            T* dst = (cur == e->ping[0].as<T>()) ? e->ping[1].as<T>() : e->ping[0].as<T>();
            if (last && s >= 1) dst = e->stage_out[s - 1].as<T>();           // C3 / C4 / C5 stay alive for the neck
            // conv3 (1x1): on the implicit-GEMM path the residual add + ReLU ride its epilogue and it writes `dst` directly
            bool fused = false;
            if (implicit_enabled()) {
                if (conv<T>(e, e->t2.as<T>(), N, h2, w2, blk.c3, dst, ACT_NONE, h3, w3, st, identity, &fused)) return 2;
            }
            if (!fused) {
                if (conv<T>(e, e->t2.as<T>(), N, h2, w2, blk.c3, e->t3.as<T>(), ACT_NONE, h3, w3, st)) return 2;
                if (launch_add_relu<T>(e->t3.as<T>(), identity, dst, (int64_t)N * h3 * w3 * blk.c3.cout, st)) return 2;
            }
            cur = dst; H = h3; W = w3;
        }
        if (s >= 1) { sh[s - 1] = H; sw[s - 1] = W; }
    }
    // FPN (mmdet FPN.forward): laterals, top-down nearest upsample + add, 3x3 output convs, extra stride-2 level on the
    // last OUTPUT (add_extra_convs='on_output'; with num_outs = 4 relu_before_extra_convs does not apply)
    int lh[3], lw[3];
    for (int i = 0; i < 3; ++i)
        if (conv<T>(e, e->stage_out[i].as<T>(), N, sh[i], sw[i], e->lateral[i], e->lat[i].as<T>(), ACT_NONE, lh[i], lw[i], st))
            return 2;
    for (int i = 2; i >= 1; --i)
        if (launch_upsample_add_nhwc<T>(e->lat[i - 1].as<T>(), e->lat[i].as<T>(), N, lh[i - 1], lw[i - 1], lh[i], lw[i],
                                        e->out_channels, st)) return 2;
    int oh[4], ow[4];
    T* fo[4];
    for (int i = 0; i < 4; ++i) fo[i] = (nhwc_out && nhwc_out[i]) ? reinterpret_cast<T*>(nhwc_out[i]) : e->fo[i].as<T>();
    for (int i = 0; i < 3; ++i)
        if (conv<T>(e, e->lat[i].as<T>(), N, lh[i], lw[i], e->fpnc[i], fo[i], ACT_NONE, oh[i], ow[i], st)) return 2;
    if (conv<T>(e, fo[2], N, oh[2], ow[2], e->fpnc[3], fo[3], ACT_NONE, oh[3], ow[3], st)) return 2;
    if (nhwc_out) return 0;
    for (int i = 0; i < 4; ++i)
        if (outs[i] && launch_nhwc_to_nchw_f32<T>(e->fo[i].as<T>(), outs[i], N, oh[i] * ow[i], e->out_channels, st)) return 2;
    return 0;
}

}  // namespace

extern "C" {

occb200_backbone* occb200_backbone_create(int num_images, int img_h, int img_w, int precision, int use_tensor_cores)
{
    if (num_images <= 0 || img_h < 64 || img_w < 64 || (precision != 0 && precision != 1)) {
        set_last_error("backbone_create: need num_images > 0, image >= 64x64, precision 0 (fp32) or 1 (bf16)");
        return nullptr;
    }
    occb200_backbone* e = new occb200_backbone();
    e->num_images = num_images; e->H = img_h; e->W = img_w; e->precision = precision;
    e->use_tc = (precision == 1 && use_tensor_cores) ? 1 : 0;
    return e;
}

void occb200_backbone_destroy(occb200_backbone* e)
{
    if (!e) return;
    auto rel = [](ConvW& c) { c.w.release(); c.wh.release(); c.b.release(); };
    rel(e->stem);
    for (auto& st : e->blocks) for (auto& b : st) { rel(b.c1); rel(b.c2); rel(b.c3); rel(b.down); }
    for (auto& c : e->lateral) rel(c);
    for (auto& c : e->fpnc) rel(c);
    Buf* all[] = {&e->img_nhwc, &e->col, &e->ping[0], &e->ping[1], &e->t1, &e->t2, &e->t3, &e->idn, &e->stage_out[0],
                  &e->stage_out[1], &e->stage_out[2], &e->lat[0], &e->lat[1], &e->lat[2], &e->fo[0], &e->fo[1], &e->fo[2],
                  &e->fo[3]};
    for (Buf* b : all) b->release();
    delete e;
}

int occb200_backbone_load_param(occb200_backbone* e, const char* key, const float* data, int64_t numel)
{
    OCC_CHECK(e && key && data && numel > 0, "bad arguments");
    OCC_CHECK(!e->finalized, "backbone already finalized");
    const std::string k(key);
    OCC_CHECK(k.rfind("img_backbone.", 0) == 0 || k.rfind("img_neck.", 0) == 0,
              "backbone_load_param: unknown key (expected img_backbone.* / img_neck.*): " + k);
    e->host_params[k].assign(data, data + numel);
    return 0;
}

int occb200_backbone_finalize(occb200_backbone* e)
{
    OCC_CHECK(e && !e->finalized, "bad arguments");
    const std::string b = "img_backbone.", nk = "img_neck.";
    int rc;
    if ((rc = fold_conv(e, e->stem, b + "conv1", b + "bn1", 64, 3, 7, 2, 3, false))) return rc;
    int inplanes = 64;
    for (int s = 0; s < 4; ++s) {
        e->blocks[s].resize(STAGE_BLOCKS[s]);
        const int planes = STAGE_PLANES[s];
        for (int i = 0; i < STAGE_BLOCKS[s]; ++i) {
            occb200_backbone::Block& blk = e->blocks[s][i];
            const std::string pre = b + "layer" + std::to_string(s + 1) + "." + std::to_string(i) + ".";
            blk.stride = (i == 0 && s > 0) ? 2 : 1;                          // style 'pytorch': the 3x3 conv carries the stride
            blk.has_down = i == 0;
            if ((rc = fold_conv(e, blk.c1, pre + "conv1", pre + "bn1", planes, inplanes, 1, 1, 0, false))) return rc;
            if ((rc = fold_conv(e, blk.c2, pre + "conv2", pre + "bn2", planes, planes, 3, blk.stride, 1, false))) return rc;
            if ((rc = fold_conv(e, blk.c3, pre + "conv3", pre + "bn3", planes * 4, planes, 1, 1, 0, false))) return rc;
            if (blk.has_down &&
                (rc = fold_conv(e, blk.down, pre + "downsample.0", pre + "downsample.1", planes * 4, inplanes, 1, blk.stride, 0,
                                false))) return rc;
            inplanes = planes * 4;
        }
    }
    const int cin[3] = {512, 1024, 2048};
    for (int i = 0; i < 3; ++i)
        if ((rc = fold_conv(e, e->lateral[i], nk + "lateral_convs." + std::to_string(i) + ".conv", "", e->out_channels, cin[i],
                            1, 1, 0, true))) return rc;
    for (int i = 0; i < 4; ++i)
        if ((rc = fold_conv(e, e->fpnc[i], nk + "fpn_convs." + std::to_string(i) + ".conv", "", e->out_channels,
                            e->out_channels, 3, i == 3 ? 2 : 1, 1, true))) return rc;
    // workspace sizes (elements per image), following the shapes through the network
    const size_t es = e->elt(), N = (size_t)e->num_images;
    const int h1 = out_size(e->H, 7, 2, 3), w1 = out_size(e->W, 7, 2, 3);    // stem
    const int h2 = out_size(h1, 3, 2, 1), w2 = out_size(w1, 3, 2, 1);        // maxpool = layer1 resolution
    size_t max_act = (size_t)h1 * w1 * 64, max_col = (size_t)h1 * w1 * e->stem.kpad;
    int h = h2, w = w2;
    size_t stage_elems[4];
    for (int s = 0; s < 4; ++s) {
        const int planes = STAGE_PLANES[s];
        const int ho = s > 0 ? out_size(h, 3, 2, 1) : h, wo = s > 0 ? out_size(w, 3, 2, 1) : w;
        max_act = std::max(max_act, (size_t)h * w * planes);                 // conv1 output at the input resolution
        max_act = std::max(max_act, (size_t)ho * wo * planes * 4);
        max_col = std::max(max_col, (size_t)ho * wo * 9 * planes);           // conv2 im2col
        if (s > 0) max_col = std::max(max_col, (size_t)ho * wo * (size_t)(STAGE_PLANES[s - 1] * 4));   // strided 1x1 downsample
        stage_elems[s] = (size_t)ho * wo * planes * 4;
        h = ho; w = wo;
        if (s >= 1) max_col = std::max(max_col, (size_t)ho * wo * 9 * e->out_channels);   // FPN 3x3 at this level
    }
    if (e->img_nhwc.alloc(N * e->H * e->W * 3 * es) || e->col.alloc(N * max_col * es) || e->ping[0].alloc(N * max_act * es) ||
        e->ping[1].alloc(N * max_act * es) || e->t1.alloc(N * max_act * es) || e->t2.alloc(N * max_act * es) ||
        e->t3.alloc(N * max_act * es) || e->idn.alloc(N * max_act * es)) return 2;
    h = h2; w = w2;
    for (int s = 1; s < 4; ++s) {
        h = out_size(h, 3, 2, 1); w = out_size(w, 3, 2, 1);
        if (e->stage_out[s - 1].alloc(N * stage_elems[s] * es)) return 2;
        const size_t lvl = N * (size_t)h * w * e->out_channels * es;
        if (e->lat[s - 1].alloc(lvl) || e->fo[s - 1].alloc(lvl)) return 2;
    }
    if (e->fo[3].alloc(N * (size_t)out_size(h, 3, 2, 1) * out_size(w, 3, 2, 1) * e->out_channels * es)) return 2;
    e->host_params.clear();
    e->finalized = true;
    return 0;
}

int occb200_backbone_level_shape(const occb200_backbone* e, int level, int* h, int* w)
{
    OCC_CHECK(e && h && w && level >= 0 && level < 4, "bad arguments");
    int hh = out_size(out_size(e->H, 7, 2, 3), 3, 2, 1), ww = out_size(out_size(e->W, 7, 2, 3), 3, 2, 1);
    for (int s = 0; s <= level && s < 3; ++s) { hh = out_size(hh, 3, 2, 1); ww = out_size(ww, 3, 2, 1); }
    if (level == 3) { hh = out_size(hh, 3, 2, 1); ww = out_size(ww, 3, 2, 1); }
    *h = hh; *w = ww;
    return 0;
}

int occb200_backbone_forward(occb200_backbone* e, const float* img, float* out0, float* out1, float* out2, float* out3,
                             void* stream)
{
    OCC_CHECK(e && img, "null pointer");
    OCC_CHECK(e->finalized, "backbone_finalize() has not been called");
    float* outs[4] = {out0, out1, out2, out3};
    return e->precision ? forward_impl<bf16>(e, img, outs, (cudaStream_t)stream)
                        : forward_impl<float>(e, img, outs, (cudaStream_t)stream);
}

int occb200_backbone_forward_nhwc_bf16(occb200_backbone* e, const float* img, void* out0, void* out1, void* out2, void* out3,
                                       void* stream)
{
    OCC_CHECK(e && img && out0 && out1 && out2 && out3, "null pointer");
    OCC_CHECK(e->finalized, "backbone_finalize() has not been called");
    OCC_CHECK(e->precision == 1, "backbone_forward_nhwc_bf16 needs a bf16 backbone (precision 1)");
    void* outs[4] = {out0, out1, out2, out3};
    return forward_impl<bf16>(e, img, nullptr, (cudaStream_t)stream, outs);
}

}  // extern "C"
