// Implicit-GEMM 2-D convolution (stride 1) on the tensor cores for the image backbone / neck (sm_90a):
//     out[n, y, x, co] = act( sum_{ky,kx,ci} in[n, y+ky-pad, x+kx-pad, ci] * w[co][(ky*KW+kx)*Cin + ci] + bias[co]
//                             (+ residual[n, y, x, co]) ),      NHWC bf16 tensors, fp32 accumulation in registers.
// Used for the 3x3 convolutions of ResNet-50 / FPN and (KH = KW = 1) for the bottleneck's last 1x1 convolution with the
// residual add + ReLU fused (reference: mmdet ResNet / FPN as configured in bevformer_base_occ.py:48-66).
//
// Same skeleton as gemm_tc.cu (persistent, one CTA per SM, warp-specialised), with im2col done by TMA as in conv3d_tc.cu:
//   M tile  = 128 output pixels = 8 rows x 16 columns of one image; K loop = taps x (Cin / 64)
//   warps 8-11 producer warpgroup (warp 8 issues): per k-block one 4-D box {64 ch, 16 x, 8 y, 1 n} of the input at the tap's (ky,kx) offset
//                             (out-of-bounds pixels zero-filled by the TMA unit = the conv's zero padding) + the weight
//                             k-block [BN x 64]; 128B swizzle; 2-6 stage mbarrier ring
//   warps 0-7  two consumer warpgroups: wgmma.m64n64k16 over 64 pixels each, then +bias (+residual) -> ReLU -> bf16 stores
// Checked by tests/test_backbone_ops_gpu.py through occb200_backbone_conv: bit-exact on integer and one-hot operands at every
// backbone shape and at edge shapes (partial tiles, N, Cin, each BN with several n-tiles, m-tile splits, bias / residual /
// ReLU), and against fp64 at production size.
#include <cstdlib>

#include "common.cuh"
#include "conv2d_tc.cuh"
#include "tc_common.cuh"

namespace occ {

namespace {

constexpr int BLOCK_M = 128, BLOCK_K = 64, A_TILE_BYTES = BLOCK_M * BLOCK_K * 2, TILE_W = 16, TILE_H = 8;
constexpr int NUM_THREADS = 384, MAX_STAGES = 6;      // 2 consumer warpgroups + 1 producer warpgroup
constexpr int SMEM_MAX = 232448 - 1024;
constexpr int SMEM_TAIL = 256 + 1024;                     // barriers + per-column bias

struct Geom { int N, H, W, Cin, Cout, KH, KW, pad; };

__global__ void __launch_bounds__(NUM_THREADS, 1)
conv2d_tc_kernel(const __grid_constant__ CUtensorMap tmIn, const __grid_constant__ CUtensorMap tmW,
                 const float* __restrict__ bias, const bf16* __restrict__ residual, bf16* __restrict__ out, Geom g, int BN,
                 int stages, int act)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t w_tile_bytes = BN * BLOCK_K * 2;
    const uint32_t stage_bytes = A_TILE_BYTES + w_tile_bytes;
    const uint32_t ring_base = smem_base;
    const uint32_t bar_base = ring_base + stages * stage_bytes;
    auto full_bar = [&](int s) { return bar_base + s * 8; };
    auto empty_bar = [&](int s) { return bar_base + (MAX_STAGES + s) * 8; };
    float* const cvec = reinterpret_cast<float*>(smem_raw + (bar_base + 256 - tc::smem_u32(smem_raw)));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles = g.Cout / BN;
    const int tiles_x = (g.W + TILE_W - 1) / TILE_W, tiles_y = (g.H + TILE_H - 1) / TILE_H;
    const int m_tiles = g.N * tiles_y * tiles_x;
    const int n_blk = blockIdx.x % n_tiles;
    const int grp = blockIdx.x / n_tiles, ngrp = gridDim.x / n_tiles;
    const int t_begin = (int)(((long long)m_tiles * grp) / ngrp), t_end = (int)(((long long)m_tiles * (grp + 1)) / ngrp);
    const int taps = g.KH * g.KW, ncb = g.Cin / BLOCK_K, nk = taps * ncb;

    if (warp == 8 && lane == 0) {
        tc::tma_prefetch_desc(&tmIn); tc::tma_prefetch_desc(&tmW);
        for (int s = 0; s < stages; ++s) { tc::mbar_init(full_bar(s), 1); tc::mbar_init(empty_bar(s), 2); }
        tc::mbar_fence_init();
    }
    if (threadIdx.x < BN) cvec[threadIdx.x] = bias ? __ldg(bias + n_blk * BN + threadIdx.x) : 0.f;
    __syncthreads();

    auto decode = [&](int t, int& n, int& y0, int& x0) {
        const int tx = t % tiles_x, ty = (t / tiles_x) % tiles_y;
        n = t / (tiles_x * tiles_y); y0 = ty * TILE_H; x0 = tx * TILE_W;
    };

    if (warp >= 8) {
        tc::setmaxnreg_dec<40>();                                 // producer warpgroup: registers go to the consumers
        if (warp == 8 && lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int t = t_begin; t < t_end; ++t) {
                int n, y0, x0;
                decode(t, n, y0, x0);
                for (int tap = 0; tap < taps; ++tap) {
                    const int ky = tap / g.KW, kx = tap % g.KW;
                    for (int cb = 0; cb < ncb; ++cb) {
                        tc::mbar_wait(empty_bar(s), ph ^ 1);
                        tc::mbar_arrive_expect_tx(full_bar(s), stage_bytes);
                        const uint32_t a_dst = ring_base + s * stage_bytes;
                        tc::tma_load_4d(a_dst, &tmIn, full_bar(s), cb * BLOCK_K, x0 + kx - g.pad, y0 + ky - g.pad, n);
                        tc::tma_load_2d(a_dst + A_TILE_BYTES, &tmW, full_bar(s), tap * g.Cin + cb * BLOCK_K, n_blk * BN);
                        if (++s == stages) { s = 0; ph ^= 1; }
                    }
                }
            }
        }
        return;
    }

    tc::setmaxnreg_inc<232>();
    const int wg = warp >> 2, wl = warp & 3;
    const int nsubs = BN >> 6;
    const int quad_col = 2 * (lane & 3);
    int s = 0; uint32_t ph = 0;
    for (int t = t_begin; t < t_end; ++t) {
        int n, y0, x0;
        decode(t, n, y0, x0);
        float acc[4][32];
        for (int kb = 0; kb < nk; ++kb) {
            tc::mbar_wait(full_bar(s), ph);
            const uint32_t a_addr = ring_base + s * stage_bytes + wg * (64 * 128);
            const uint32_t b_addr = ring_base + s * stage_bytes + A_TILE_BYTES;
            switch (nsubs) {
            case 4: tc::wgmma_kblock<4>(acc, a_addr, b_addr, kb == 0); break;
            case 2: tc::wgmma_kblock<2>(acc, a_addr, b_addr, kb == 0); break;
            default: tc::wgmma_kblock<1>(acc, a_addr, b_addr, kb == 0); break;
            }
            if ((threadIdx.x & 127) == 0) tc::mbar_arrive(empty_bar(s));
            if (++s == stages) { s = 0; ph ^= 1; }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wg * 64 + 16 * wl + (lane >> 2) + 8 * h;     // tile row = 16 * (y - y0) + (x - x0)
            const int y = y0 + (r >> 4), x = x0 + (r & 15);
            if (y >= g.H || x >= g.W) continue;
            const size_t pix = (((size_t)n * g.H + y) * g.W + x) * g.Cout + n_blk * BN;
#pragma unroll
            for (int ns = 0; ns < 4; ++ns) {
                if (ns >= nsubs) break;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int cl = ns * 64 + 8 * j + quad_col;
                    float v0 = acc[ns][4 * j + 2 * h] + cvec[cl], v1 = acc[ns][4 * j + 2 * h + 1] + cvec[cl + 1];
                    if (residual) {
                        const uint32_t q = __ldg(reinterpret_cast<const unsigned int*>(residual + pix + cl));
                        v0 += __uint_as_float(q << 16); v1 += __uint_as_float(q & 0xffff0000u);
                    }
                    if (act == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    *reinterpret_cast<uint32_t*>(out + pix + cl) = pack_bf16x2(v0, v1);
                }
            }
        }
    }
}

}  // namespace

bool conv2d_tc_supported(int Cin, int Cout, int KH, int KW)
{
    return Cin % 64 == 0 && Cout % 64 == 0 && KH == KW && (KH == 1 || KH == 3);
}

int conv2d_tc(const bf16* in, const bf16* w_tap_major, const float* bias, const bf16* residual, bf16* out, int N, int H,
              int W, int Cin, int Cout, int KH, int KW, int pad, int act, cudaStream_t stream)
{
    OCC_CHECK(conv2d_tc_supported(Cin, Cout, KH, KW), "conv2d_tc: Cin, Cout multiples of 64; 1x1 or 3x3");
    OCC_CHECK(N > 0 && H > 0 && W > 0, "conv2d_tc: empty input");
    const int BN = Cout % 256 == 0 ? 256 : (Cout % 128 == 0 ? 128 : 64);
    const int stage = A_TILE_BYTES + BN * BLOCK_K * 2;
    int stages = (SMEM_MAX - SMEM_TAIL) / stage;
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    OCC_CHECK(stages >= 2, "conv2d_tc: not enough shared memory for two stages");
    const int smem = 1024 + stages * stage + SMEM_TAIL;
    CUtensorMap tmIn, tmW;
    {
        const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
        const uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        const uint32_t box[4] = {BLOCK_K, TILE_W, TILE_H, 1};
        if (make_tensor_map_bf16(&tmIn, in, 4, dims, strides, box, 128)) return 1;
    }
    {
        const uint64_t dims[2] = {(uint64_t)KH * KW * Cin, (uint64_t)Cout}, strides[1] = {(uint64_t)KH * KW * Cin * 2};
        const uint32_t box[2] = {BLOCK_K, (uint32_t)BN};
        if (make_tensor_map_bf16(&tmW, w_tap_major, 2, dims, strides, box, 128)) return 1;
    }
    const int num_sms = sm_count_current_device();
    OCC_CUDA(cudaFuncSetAttribute(conv2d_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));   // per device
    const int m_tiles = N * ((H + TILE_H - 1) / TILE_H) * ((W + TILE_W - 1) / TILE_W), n_tiles = Cout / BN;
    int per_n = num_sms / n_tiles;
    if (per_n < 1) per_n = 1;
    if (per_n > m_tiles) per_n = m_tiles;
    const Geom g{N, H, W, Cin, Cout, KH, KW, pad};
    conv2d_tc_kernel<<<per_n * n_tiles, NUM_THREADS, smem, stream>>>(tmIn, tmW, bias, residual, out, g, BN, stages, act);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace occ
