// Voxel decoder on the tensor cores (sm_90a): 3x3x3 Conv3d (pad 1, no bias) + folded
// BatchNorm3d + ReLU as an implicit GEMM.   Reference: TransformerOcc.decoder (use_3d),
// projects/mmdet3d_plugin/bevformer/modules/transformer_occ.py:106-131, applied at :305-308.
//
// Tensors are channels-last bf16 [X][Y][Z][C] (see decoder_simt.cu for the layout rationale).
//   M tile  = 128 voxels = 8 (y) x 16 (z, the whole pillar) at one x
//   N       = 32 output channels,  K = 27 taps x Cin
// im2col is done by TMA: one 4-D box load {Cin, 16 z, 8 + 2 y, 1 x} per (plane, dz) with the dz offset in the
// coordinates and a one-row y halo on both sides, so the three dy shifts are SUB-VIEWS of the same shared-memory tile
// (row offset dy * 16, a multiple of the 8-row swizzle atom); out-of-bounds rows are zero-filled by the TMA unit, which
// IS the conv's zero padding (including the z = -1 / z = 16 halo).  All 27 weight tiles stay resident in shared memory.
//   warp 8: TMA producer (8-stage ring)
//   warps 0-7: two consumer warpgroups, each owning 64 of the tile's 128 voxels (4 y rows x 16 z)
//
// Plane-major schedule: an input tile (plane x = p, shift (dz,dy)) is the A operand of three taps -- dx = 0, 1, 2 of
// the outputs x = p+1, p, p-1 -- so it is loaded ONCE (~9 instead of 27 tile loads per output tile) and multiplied into the
// three live accumulators with ONE wgmma of N = 96: the weight tiles of a (dz,dy) pair are resident in the order dx = 2, 1, 0,
// so accumulator columns [0,32) belong to output p-1, [32,64) to p and [64,96) to p+1.  After plane p the output p-1 is
// complete: it is written out and the accumulator window slides by 32 columns (register moves).
// Each CTA owns a contiguous range of the (y_tile, x) tile sequence, cut into segments of constant y_tile; a segment
// [xa, xb) streams the planes max(xa-1,0) .. min(xb, X-1).
// EPI: 0 = bf16 out = relu(acc + bias) (the bf16 configuration); fp32-storage configuration, one of three split passes
// (hi.W_hi, lo.W_hi, hi.W_lo of the bf16 split of an fp32 input, relative error ~2^-16 like gemm_tc_split3):
// 1 = out_f32 = acc, 2 = out_f32 += acc, 3 = out_f32 = relu(out_f32 + acc + bias).  Every output element is owned by one thread
// per pass, so the fp32 accumulation across passes needs no atomics.
#include <cstdlib>

#include "common.cuh"
#include "conv3d_tc.cuh"
#include "tc_common.cuh"

namespace occ {

namespace {

constexpr int STAGES = 8, TILE_Y = 8, TILE_Z = 16, COUT = 32, TAPS = 27;
constexpr int HALO_ROWS = (TILE_Y + 2) * TILE_Z;          // rows of one staged tile: y0-1 .. y0+8, all 16 z
constexpr int NUM_THREADS = 288;
constexpr int BAR_BYTES = 512;

template <int CIN, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv3d_tc_kernel(const __grid_constant__ CUtensorMap tmIn, const __grid_constant__ CUtensorMap tmW,
                 const float* __restrict__ bias, bf16* __restrict__ out, float* __restrict__ out_f32, int X, int Y)
{
    constexpr int ROW_BYTES = CIN * 2;                       // 32 (SWIZZLE_32B) or 64 (SWIZZLE_64B)
    constexpr int A_BYTES = HALO_ROWS * ROW_BYTES;           // 5 / 10 KB per stage (three dy sub-views of 128 rows)
    constexpr int DY_BYTES = TILE_Z * ROW_BYTES;             // one y row of the tile
    constexpr int W_TAP_BYTES = COUT * ROW_BYTES;            // 1 / 2 KB per tap
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t w_base = smem_base;                                       // 27 weight tiles, resident
    const uint32_t a_base = smem_base + ((TAPS * W_TAP_BYTES + 1023) & ~1023);
    const uint32_t bar_base = a_base + STAGES * A_BYTES;
    auto full_bar = [&](int s) { return bar_base + s * 8; };
    auto empty_bar = [&](int s) { return bar_base + (STAGES + s) * 8; };
    const uint32_t w_bar = bar_base + (2 * STAGES) * 8;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int y_tiles = (Y + TILE_Y - 1) / TILE_Y;
    const long long total = (long long)X * y_tiles;
    const int t_begin = (int)(total * blockIdx.x / gridDim.x), t_end = (int)(total * (blockIdx.x + 1) / gridDim.x);

    if (warp == 8 && lane == 0) {
        tc::tma_prefetch_desc(&tmIn); tc::tma_prefetch_desc(&tmW);
        for (int s = 0; s < STAGES; ++s) { tc::mbar_init(full_bar(s), 1); tc::mbar_init(empty_bar(s), 2); }
        tc::mbar_init(w_bar, 1);
        tc::mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            tc::mbar_arrive_expect_tx(w_bar, TAPS * W_TAP_BYTES);
            for (int t = 0; t < TAPS; ++t)                   // global tap order is (dz,dy,dx); resident order (dz,dy,2-dx)
                tc::tma_load_2d(w_base + ((t / 3) * 3 + (2 - t % 3)) * W_TAP_BYTES, &tmW, w_bar, 0, t * COUT);
            int s = 0; uint32_t ph = 0;
            for (int t = t_begin; t < t_end;) {
                const int yt = t / X, xa = t % X;
                const int xb = min(X, xa + (t_end - t));
                const int y0 = yt * TILE_Y;
                const int p_lo = max(xa - 1, 0), p_hi = min(xb, X - 1);
                for (int p = p_lo; p <= p_hi; ++p) {
                    for (int dz = 0; dz < 3; ++dz) {
                        tc::mbar_wait(empty_bar(s), ph ^ 1);
                        tc::mbar_arrive_expect_tx(full_bar(s), A_BYTES);
                        tc::tma_load_4d(a_base + s * A_BYTES, &tmIn, full_bar(s), 0, dz - 1, y0 - 1, p);
                        if (++s == STAGES) { s = 0; ph ^= 1; }
                    }
                }
                t += xb - xa;
            }
        }
        return;
    }

    const int wg = warp >> 2, wl = warp & 3;
    const int quad_col = 2 * (lane & 3);
    float b[8];                                              // bias of this thread's 8 output channels 8 j + quad_col + e
#pragma unroll
    for (int j = 0; j < 4; ++j) { b[2 * j] = __ldg(bias + 8 * j + quad_col); b[2 * j + 1] = __ldg(bias + 8 * j + quad_col + 1); }
    const uint64_t da0 = tc::make_smem_desc(a_base + wg * 64 * ROW_BYTES, ROW_BYTES), db0 = tc::make_smem_desc(w_base, ROW_BYTES);
    tc::mbar_wait(w_bar, 0);
    int s = 0; uint32_t ph = 0;
    for (int t = t_begin; t < t_end;) {
        const int yt = t / X, xa = t % X;
        const int xb = min(X, xa + (t_end - t));
        const int y0 = yt * TILE_Y;
        float acc[48];                                       // outputs p-1 | p | p+1 of the current plane p
#pragma unroll
        for (int i = 0; i < 48; ++i) acc[i] = 0.f;
        for (int p = xa - 1; p <= xb; ++p) {
            if (p >= 0 && p < X) {                           // planes outside the volume are the zero padding
                for (int dz = 0; dz < 3; ++dz) {
                    tc::mbar_wait(full_bar(s), ph);
                    const uint64_t da = da0 + (uint64_t)((s * A_BYTES) >> 4);
                    tc::wgmma_fence();
#pragma unroll
                    for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
                        for (int k = 0; k < CIN / 16; ++k)
                            tc::wgmma_m64n96(acc, da + (uint64_t)((dy * DY_BYTES) >> 4) + 2 * k,
                                             db0 + (uint64_t)(((dz * 3 + dy) * 3 * W_TAP_BYTES) >> 4) + 2 * k, 1);
                    }
                    tc::wgmma_commit();
                    tc::wgmma_wait_all();
                    tc::reg_fence(acc);
                    if ((threadIdx.x & 127) == 0) tc::mbar_arrive(empty_bar(s));
                    if (++s == STAGES) { s = 0; ph ^= 1; }
                }
            }
            const int x = p - 1;                              // complete: accumulator columns [0, 32)
            if (x >= xa) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = wg * 64 + 16 * wl + (lane >> 2) + 8 * h;
                    const int y = y0 + row / TILE_Z, z = row % TILE_Z;
                    if (y >= Y) continue;
                    const size_t vox = (((size_t)x * Y + y) * TILE_Z + z) * COUT;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int c = 8 * j + quad_col;
                        const float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
                        if constexpr (EPI == 0) {
                            *reinterpret_cast<uint32_t*>(out + vox + c) =
                                pack_bf16x2(fmaxf(a0 + b[2 * j], 0.f), fmaxf(a1 + b[2 * j + 1], 0.f));
                        } else {
                            float2* op = reinterpret_cast<float2*>(out_f32 + vox + c);
                            float2 v = make_float2(a0, a1);
                            if constexpr (EPI >= 2) { const float2 q = *op; v.x += q.x; v.y += q.y; }
                            if constexpr (EPI == 3) { v.x = fmaxf(v.x + b[2 * j], 0.f); v.y = fmaxf(v.y + b[2 * j + 1], 0.f); }
                            *op = v;
                        }
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = acc[i + 16];   // slide the window: p | p+1 | 0
#pragma unroll
            for (int i = 32; i < 48; ++i) acc[i] = 0.f;
        }
        t += xb - xa;
    }
}

}  // namespace

namespace {
// in_pitch: elements between consecutive voxels of `in` (Cin for a dense tensor, 2*Cin for one half of a [hi | lo] split)
template <int EPI>
int launch_conv3d_tc_impl(const bf16* in, int in_pitch, const bf16* w_tap_major, const float* bias, int X, int Y, int Z, int Cin,
                          bf16* out, float* out_f32, cudaStream_t stream)
{
    OCC_CHECK(Z == TILE_Z && (Cin == 16 || Cin == 32), "conv3d_tc: Z must be 16 and Cin in {16, 32}");
    const int row_bytes = Cin * 2;
    CUtensorMap tmIn, tmW;
    {
        const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Z, (uint64_t)Y, (uint64_t)X};
        const uint64_t strides[3] = {(uint64_t)in_pitch * 2, (uint64_t)Z * in_pitch * 2, (uint64_t)Y * Z * in_pitch * 2};
        const uint32_t box[4] = {(uint32_t)Cin, (uint32_t)TILE_Z, (uint32_t)(TILE_Y + 2), 1u};
        if (make_tensor_map_bf16(&tmIn, in, 4, dims, strides, box, row_bytes)) return 1;
    }
    {
        const uint64_t dims[2] = {(uint64_t)Cin, (uint64_t)TAPS * COUT};
        const uint64_t strides[1] = {(uint64_t)Cin * 2};
        const uint32_t box[2] = {(uint32_t)Cin, (uint32_t)COUT};
        if (make_tensor_map_bf16(&tmW, w_tap_major, 2, dims, strides, box, row_bytes)) return 1;
    }
    const int a_bytes = HALO_ROWS * row_bytes, w_bytes = (TAPS * COUT * row_bytes + 1023) & ~1023;
    const int smem = 1024 + w_bytes + STAGES * a_bytes + BAR_BYTES;
    const int num_sms = sm_count_current_device();
    const int tiles = X * ((Y + TILE_Y - 1) / TILE_Y);
    const int grid = tiles < num_sms ? tiles : num_sms;
#define OCC_CONV_LAUNCH(C)                                                                                          \
    do {                                                                                                            \
        OCC_CUDA(cudaFuncSetAttribute(conv3d_tc_kernel<C, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
        conv3d_tc_kernel<C, EPI><<<grid, NUM_THREADS, smem, stream>>>(tmIn, tmW, bias, out, out_f32, X, Y);         \
    } while (0)
    if (Cin == 16) OCC_CONV_LAUNCH(16); else OCC_CONV_LAUNCH(32);
#undef OCC_CONV_LAUNCH
    OCC_CUDA(cudaGetLastError());
    return 0;
}
}  // namespace

int launch_conv3d_tc(const bf16* in, const bf16* w_tap_major, const float* bias, int X, int Y, int Z, int Cin,
                     bf16* out, cudaStream_t stream)
{
    return launch_conv3d_tc_impl<0>(in, Cin, w_tap_major, bias, X, Y, Z, Cin, out, nullptr, stream);
}

// fp32-grade convolution on the tensor cores: split = [hi | lo] bf16 halves of the fp32 input ([nvox][2*Cin], launch_split_bf16),
// w_hi / w_lo = bf16 split of the BN-folded fp32 weights ([27][32][Cin] each); out_f32 = relu(hi.W_hi + lo.W_hi + hi.W_lo + bias)
// accumulated in fp32 over three passes of the same kernel (the lo.lo term, 2^-16 relative, is dropped)
int launch_conv3d_tc_split(const bf16* split, const bf16* w_hi, const bf16* w_lo, const float* bias, int X, int Y, int Z, int Cin,
                           float* out_f32, cudaStream_t stream)
{
    if (launch_conv3d_tc_impl<1>(split, 2 * Cin, w_hi, bias, X, Y, Z, Cin, nullptr, out_f32, stream)) return 1;
    if (launch_conv3d_tc_impl<2>(split + Cin, 2 * Cin, w_hi, bias, X, Y, Z, Cin, nullptr, out_f32, stream)) return 1;
    return launch_conv3d_tc_impl<3>(split, 2 * Cin, w_lo, bias, X, Y, Z, Cin, nullptr, out_f32, stream);
}

}  // namespace occ
