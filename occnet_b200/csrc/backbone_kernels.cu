// Layout / data-movement kernels of the image backbone + neck (ResNet-50 + FPN feeding the hot path, SURVEY 8f rank 1;
// reference: detectors/bevformer_occ.py:66-99 with the mmdet modules configured in bevformer_base_occ.py:48-66).
//
// Checked by tests/test_backbone_gpu.py (8 tests against the pinned backbone oracle); the bench's
// `images_to_voxels` leg times it.  The stride-1 3x3 convolutions and the bottleneck's last 1x1 moved to the
// TMA-im2col kernel conv2d_tc.cu; what is described here is the explicit-im2col path that the remaining convolutions still use.
//
// Design of the explicit path: activations are channels-last (NHWC); every convolution is a GEMM on the validated
// wgmma kernel (gemm_tc.cu; CUDA-core gemm_simt.cu in the fp32 parity configuration):
//   1x1 stride 1          : the NHWC tensor IS the [pixels, Cin] operand
//   3x3 / 7x7 / strided   : explicit im2col into a [pixels_out, K] operand (K = KH*KW*Cin zero-padded to 64)
// BatchNorm is folded into the weights at finalize, ReLU rides the GEMM epilogue, the bottleneck's residual add and
// the FPN top-down add are small elementwise kernels.  The explicit im2col costs ~10 GB of extra traffic per
// 6-camera frame; replacing it by TMA im2col inside the GEMM producer (as conv3d_tc.cu does) is the planned next step.
#include "common.cuh"
#include "kernels.cuh"

namespace occ {

namespace {

// image [N, C, H, W] fp32 -> [N, H, W, C] T   (C = 3: no vector path needed, 26 MB per 6-camera frame)
template <typename T>
__global__ void nchw_to_nhwc_small_kernel(const float* __restrict__ src, T* __restrict__ dst, int N, int C, int H, int W)
{
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // over N*H*W pixels
    const int64_t hw = (int64_t)H * W;
    if (idx >= (int64_t)N * hw) return;
    const int64_t n = idx / hw, p = idx % hw;
    for (int c = 0; c < C; ++c) dst[idx * C + c] = from_f32<T>(__ldg(src + (n * C + c) * hw + p));
}

// im2col on channels-last data: out[m][k], m = (n, yo, xo), k = (ky*KW + kx)*C + c, zero outside the image and for
// k >= KH*KW*C (padding of K up to Kpad).  VEC = 8 (C % 8 == 0, 16-byte accesses for bf16) or 1.
template <typename T, int VEC>
__global__ void im2col_nhwc_kernel(const T* __restrict__ in, T* __restrict__ out, int N, int H, int W, int C, int KH,
                                   int KW, int stride, int pad, int Ho, int Wo, int Kpad)
{
    const int kv = Kpad / VEC;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)N * Ho * Wo * kv;
    if (idx >= total) return;
    const int k = (int)(idx % kv) * VEC;
    const int64_t m = idx / kv;
    const int xo = (int)(m % Wo), yo = (int)((m / Wo) % Ho), n = (int)(m / ((int64_t)Wo * Ho));
    T* o = out + m * Kpad + k;
    const int tap = k / C, c = k % C;                          // VEC == 8: C % 8 == 0 keeps the 8 values inside one tap
    const int ky = tap / KW, kx = tap % KW;
    const int y = yo * stride + ky - pad, x = xo * stride + kx - pad;
    const bool inside = tap < KH * KW && y >= 0 && y < H && x >= 0 && x < W;
    if constexpr (VEC == 8) {
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (inside) load8(in + (((int64_t)n * H + y) * W + x) * C + c, v);
        store8(o, v);
    } else {
        o[0] = inside ? in[(((int64_t)n * H + y) * W + x) * C + c] : from_f32<T>(0.f);
    }
}

// Any C (the 7x7 stem: C = 3): 8 consecutive k per thread, ONE 16-byte store, (tap, c) advanced incrementally.  The element-per-
// thread form (VEC = 1) spends its time in five 64-bit divisions per 2-byte element.
template <typename T>
__global__ void im2col_nhwc_any_kernel(const T* __restrict__ in, T* __restrict__ out, int N, int H, int W, int C, int KH,
                                       int KW, int stride, int pad, int Ho, int Wo, int Kpad)
{
    const unsigned kv = (unsigned)Kpad / 8u;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;          // (launcher guarantees N*Ho*Wo*kv < 2^32)
    const unsigned total = (unsigned)N * Ho * Wo * kv;
    if (idx >= total) return;
    const unsigned m = idx / kv;
    const int k0 = (int)(idx - m * kv) * 8;
    const int xo = (int)(m % (unsigned)Wo);
    const unsigned my = m / (unsigned)Wo;
    const int yo = (int)(my % (unsigned)Ho), n = (int)(my / (unsigned)Ho);
    int tap = k0 / C, c = k0 - tap * C;
    int ky = tap / KW, kx = tap - ky * KW;
    const T* img = in + (int64_t)n * H * W * C;
    const int y_base = yo * stride - pad, x_base = xo * stride - pad;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int y = y_base + ky, x = x_base + kx;
        const bool inside = ky < KH && y >= 0 && y < H && x >= 0 && x < W;
        v[j] = inside ? to_f32(img[((int64_t)y * W + x) * C + c]) : 0.f;
        if (++c == C) { c = 0; if (++kx == KW) { kx = 0; ++ky; } }
    }
    store8(out + (int64_t)m * Kpad + k0, v);
}

// Small-C im2col through shared memory (the 7x7 / stride-2 stem, C = 3): one CTA = 128 output pixels of one output row.  The KH
// input rows it needs ((127*stride + KW) * C elements each) are staged once with coalesced loads; every thread then assembles
// 16-byte chunks (8 consecutive k) of the output rows from shared memory and writes them coalesced (855 MB of im2col rows for
// 6 x 928 x 1600 images: an element-per-thread gather from global memory was the slowest step of the backbone).
constexpr int STEM_TW = 128, STEM_MAX_KH = 7, STEM_MAX_SPAN = 1024;
template <typename T>
__global__ void __launch_bounds__(256)
im2col_smallc_kernel(const T* __restrict__ in, T* __restrict__ out, int N, int H, int W, int C, int KH, int KW, int stride,
                     int pad, int Ho, int Wo, int Kpad)
{
    __shared__ T rows[STEM_MAX_KH][STEM_MAX_SPAN];
    const int x0 = blockIdx.x * STEM_TW, yo = blockIdx.y, n = blockIdx.z;
    const int span = ((STEM_TW - 1) * stride + KW) * C;         // elements of one staged row
    const int gx0 = (x0 * stride - pad) * C;                    // element offset of the staged span inside the image row
    for (int ky = 0; ky < KH; ++ky) {
        const int y = yo * stride + ky - pad;
        const T* src = in + ((int64_t)n * H + y) * W * C;
        for (int e = threadIdx.x; e < span; e += 256) {
            const int g = gx0 + e;
            rows[ky][e] = (y >= 0 && y < H && g >= 0 && g < W * C) ? src[g] : from_f32<T>(0.f);
        }
    }
    __syncthreads();
    const int kv = Kpad / 8, kwc = KW * C, ktot = KH * kwc;
    const int64_t m0 = ((int64_t)n * Ho + yo) * Wo + x0;
    for (int id = threadIdx.x; id < STEM_TW * kv; id += 256) {
        const int px = id / kv, k0 = (id - px * kv) * 8;
        if (x0 + px >= Wo) break;
        int ky = k0 / kwc, r = k0 - ky * kwc;
        const int base = px * stride * C;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            v[j] = (k0 + j < ktot) ? to_f32(rows[ky][base + r]) : 0.f;
            if (++r == kwc) { r = 0; ++ky; }
        }
        store8(out + (m0 + px) * Kpad + k0, v);
    }
}

// MaxPool2d(kernel 3, stride 2, padding 1) on NHWC, 8 channels per thread (padding behaves as -inf)
template <typename T>
__global__ void maxpool3x3s2_nhwc_kernel(const T* __restrict__ in, T* __restrict__ out, int N, int H, int W, int C, int Ho,
                                         int Wo)
{
    const int cv = C / 8;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)N * Ho * Wo * cv) return;
    const int c = (int)(idx % cv) * 8;
    const int64_t m = idx / cv;
    const int xo = (int)(m % Wo), yo = (int)((m / Wo) % Ho), n = (int)(m / ((int64_t)Wo * Ho));
    float best[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) best[i] = -INFINITY;
    for (int ky = 0; ky < 3; ++ky) {
        const int y = yo * 2 + ky - 1;
        if (y < 0 || y >= H) continue;
        for (int kx = 0; kx < 3; ++kx) {
            const int x = xo * 2 + kx - 1;
            if (x < 0 || x >= W) continue;
            float v[8];
            load8(in + (((int64_t)n * H + y) * W + x) * C + c, v);
#pragma unroll
            for (int i = 0; i < 8; ++i) best[i] = fmaxf(best[i], v[i]);
        }
    }
    store8(out + m * C + c, best);
}

// out = relu(a + b), 8 elements per thread (bottleneck: out = relu(conv3 + identity))
template <typename T>
__global__ void add_relu_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, int64_t n8)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n8) return;
    float x[8], y[8];
    load8(a + i * 8, x);
    load8(b + i * 8, y);
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = fmaxf(x[k] + y[k], 0.f);
    store8(out + i * 8, x);
}

// FPN top-down path: fine[n, y, x, :] += coarse[n, sy, sx, :] with F.interpolate(mode='nearest', size=(Hf, Wf)):
// s = min(floor(dst * (float)in / out), in - 1)   (PyTorch's legacy nearest index rule, float scale)
template <typename T>
__global__ void upsample_add_nhwc_kernel(T* __restrict__ fine, const T* __restrict__ coarse, int N, int Hf, int Wf, int Hc,
                                         int Wc, int C)
{
    const int cv = C / 8;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)N * Hf * Wf * cv) return;
    const int c = (int)(idx % cv) * 8;
    const int64_t m = idx / cv;
    const int x = (int)(m % Wf), y = (int)((m / Wf) % Hf), n = (int)(m / ((int64_t)Wf * Hf));
    const float sh = (float)Hc / (float)Hf, sw = (float)Wc / (float)Wf;
    const int sy = min((int)floorf((float)y * sh), Hc - 1), sx = min((int)floorf((float)x * sw), Wc - 1);
    float a[8], b[8];
    load8(fine + m * C + c, a);
    load8(coarse + (((int64_t)n * Hc + sy) * Wc + sx) * C + c, b);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] += b[k];
    store8(fine + m * C + c, a);
}

// [N, H*W, C] T -> [N, C, H*W] fp32 (the reference's FPN output layout), 32x32 tiles through shared memory
template <typename T>
__global__ void nhwc_to_nchw_f32_kernel(const T* __restrict__ src, float* __restrict__ dst, int HW, int C)
{
    __shared__ float tile[32][33];
    const int n = blockIdx.z, p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 256 threads: 8 rows per pass
    for (int r = ty; r < 32; r += 8) {
        const int p = p0 + r, c = c0 + tx;
        tile[r][tx] = (p < HW && c < C) ? to_f32(src[((int64_t)n * HW + p) * C + c]) : 0.f;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int c = c0 + r, p = p0 + tx;
        if (p < HW && c < C) dst[((int64_t)n * C + c) * HW + p] = tile[tx][r];
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------ launchers
template <typename T>
int launch_nchw_to_nhwc_small(const float* src, T* dst, int N, int C, int H, int W, cudaStream_t stream)
{
    const int64_t total = (int64_t)N * H * W;
    nchw_to_nhwc_small_kernel<T><<<ceil_div(total, 256), 256, 0, stream>>>(src, dst, N, C, H, W);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template <typename T>
int launch_im2col_nhwc(const T* in, T* out, int N, int H, int W, int C, int KH, int KW, int stride, int pad, int Ho, int Wo,
                       int Kpad, cudaStream_t stream)
{
    OCC_CHECK(Kpad >= KH * KW * C && Kpad % 8 == 0, "im2col: Kpad must cover KH*KW*C and be a multiple of 8");
    if (C % 8 == 0) {
        const int64_t total = (int64_t)N * Ho * Wo * (Kpad / 8);
        im2col_nhwc_kernel<T, 8><<<ceil_div(total, 256), 256, 0, stream>>>(in, out, N, H, W, C, KH, KW, stride, pad, Ho, Wo, Kpad);
    } else if (KH <= STEM_MAX_KH && ((STEM_TW - 1) * stride + KW) * C <= STEM_MAX_SPAN && N <= 65535 && Ho <= 65535) {
        dim3 grid(ceil_div(Wo, STEM_TW), Ho, N);
        im2col_smallc_kernel<T><<<grid, 256, 0, stream>>>(in, out, N, H, W, C, KH, KW, stride, pad, Ho, Wo, Kpad);
    } else if ((int64_t)N * Ho * Wo * (Kpad / 8) < (1ll << 32) - 256) {
        const int64_t total = (int64_t)N * Ho * Wo * (Kpad / 8);
        im2col_nhwc_any_kernel<T><<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(in, out, N, H, W, C, KH, KW, stride, pad, Ho, Wo, Kpad);
    } else {
        const int64_t total = (int64_t)N * Ho * Wo * Kpad;
        im2col_nhwc_kernel<T, 1><<<ceil_div(total, 256), 256, 0, stream>>>(in, out, N, H, W, C, KH, KW, stride, pad, Ho, Wo, Kpad);
    }
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template <typename T>
int launch_maxpool3x3s2_nhwc(const T* in, T* out, int N, int H, int W, int C, int Ho, int Wo, cudaStream_t stream)
{
    OCC_CHECK(C % 8 == 0, "maxpool: C must be a multiple of 8");
    const int64_t total = (int64_t)N * Ho * Wo * (C / 8);
    maxpool3x3s2_nhwc_kernel<T><<<ceil_div(total, 256), 256, 0, stream>>>(in, out, N, H, W, C, Ho, Wo);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template <typename T>
int launch_add_relu(const T* a, const T* b, T* out, int64_t n, cudaStream_t stream)
{
    OCC_CHECK(n % 8 == 0, "add_relu: size must be a multiple of 8");
    add_relu_kernel<T><<<ceil_div(n / 8, 256), 256, 0, stream>>>(a, b, out, n / 8);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template <typename T>
int launch_upsample_add_nhwc(T* fine, const T* coarse, int N, int Hf, int Wf, int Hc, int Wc, int C, cudaStream_t stream)
{
    OCC_CHECK(C % 8 == 0, "upsample_add: C must be a multiple of 8");
    const int64_t total = (int64_t)N * Hf * Wf * (C / 8);
    upsample_add_nhwc_kernel<T><<<ceil_div(total, 256), 256, 0, stream>>>(fine, coarse, N, Hf, Wf, Hc, Wc, C);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template <typename T>
int launch_nhwc_to_nchw_f32(const T* src, float* dst, int N, int HW, int C, cudaStream_t stream)
{
    dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), N);
    nhwc_to_nchw_f32_kernel<T><<<grid, 256, 0, stream>>>(src, dst, HW, C);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

#define OCC_INST(T)                                                                                                       \
    template int launch_nchw_to_nhwc_small<T>(const float*, T*, int, int, int, int, cudaStream_t);                       \
    template int launch_im2col_nhwc<T>(const T*, T*, int, int, int, int, int, int, int, int, int, int, int, cudaStream_t); \
    template int launch_maxpool3x3s2_nhwc<T>(const T*, T*, int, int, int, int, int, int, cudaStream_t);                  \
    template int launch_add_relu<T>(const T*, const T*, T*, int64_t, cudaStream_t);                                      \
    template int launch_upsample_add_nhwc<T>(T*, const T*, int, int, int, int, int, int, cudaStream_t);                  \
    template int launch_nhwc_to_nchw_f32<T>(const T*, float*, int, int, int, cudaStream_t);
OCC_INST(float)
OCC_INST(bf16)
#undef OCC_INST

}  // namespace occ
