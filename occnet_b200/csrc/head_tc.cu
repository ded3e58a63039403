// Occupancy + flow heads on the tensor cores (sm_90a).  Reference: TransformerOcc.predicter /
// flow_predicter (transformer_occ.py:132-141, applied :318-319) and BEVFormerOccHead.get_occ
// (bevformer_occ_head.py:211-212; argmax of the logits == argmax of their softmax).
//
// Per 128-voxel tile, a chain of two wgmma GEMMs with the activations kept on chip.  Each of the two consumer warpgroups owns
// 64 voxels of the tile:
//   GEMM1  [64 x 32] . [32 x 128]   hidden = [ predicter.0 | flow_predicter.0 ]          (registers)
//   epilogue A: +bias, Softplus (cols 0-63) / ReLU (cols 64-127), bf16, written to the warpgroup's shared-memory buffer in
//               the 128B-swizzled K-major layout the tensor core reads (generic-proxy stores + fence.proxy.async)
//   GEMM2  [64 x 128] . [128 x 32]  block-diagonal [ predicter.2 (17) ; flow_predicter.2 (2) ; 0-pad ]
//   epilogue B: +bias, argmax over the 17 classes (reduced over the 4 threads of a quad), logits / class / flow
// Warp 8 streams the voxel tiles through a 4-stage TMA ring; the weights stay resident.
#include "common.cuh"
#include "conv3d_tc.cuh"
#include "tc_common.cuh"

namespace occ {

namespace {

constexpr int A_STAGES = 4, BLOCK_M = 128, HID = 128, NOUT = 32;
constexpr int A_BYTES = BLOCK_M * 64;                 // 128 rows x 32 bf16
constexpr int W1_BYTES = HID * 64;                    // 128 rows x 32 bf16
constexpr int W2_CHUNK_BYTES = NOUT * 128;            // 32 rows x 64 bf16
constexpr int H_CHUNK_BYTES = 64 * 128;               // 64 rows x 64 bf16 (one warpgroup)
constexpr int NUM_THREADS = 288;                     // 2 consumer warpgroups + 1 TMA warp
constexpr int MAX_CLS = 19;                           // 17 classes + 2 flow channels live in the 32 GEMM2 columns

// Softplus with ONE MUFU op: softplus(x) = max(x, 0) + log1p(t), t = exp(-|x|) in (0, 1], and log1p(t) = t * P(t) with a degree-5
// minimax polynomial (|P - log1p(t)/t| <= 7.2e-6 on [0,1], so the result is within 7.2e-6 RELATIVE of softplus everywhere -- the
// hidden activations are then rounded to bf16, 2^-9).  The form log(1 + exp(x)) needs ex2 AND lg2 and is bound by the MUFU pipe.
__device__ __forceinline__ float softplus1(float x)
{
    constexpr float C0 = 0.9999929070472717f, C1 = -0.4994262754917145f, C2 = 0.32572421431541443f, C3 = -0.211494579911232f,
                    C4 = 0.10287206619977951f, C5 = -0.024528255686163902f;
    float t;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(-fabsf(x) * 1.4426950408889634f));
    float p = fmaf(C5, t, C4);
    p = fmaf(p, t, C3);
    p = fmaf(p, t, C2);
    p = fmaf(p, t, C1);
    p = fmaf(p, t, C0);
    return fmaf(t, p, fmaxf(x, 0.f));
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
head_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW1,
               const __grid_constant__ CUtensorMap tmW2, const float* __restrict__ b1cat,
               const float* __restrict__ b2cat, int ncls, int64_t nvox, float* __restrict__ occ_logits,
               float* __restrict__ flow, uint8_t* __restrict__ cls_u8, int64_t* __restrict__ cls_i64)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - tc::smem_u32(smem_raw));
    const uint32_t w1_base = smem_base;                                  // 8 KB
    const uint32_t w2_base = w1_base + W1_BYTES;                         // 2 x 4 KB
    const uint32_t a_base = w2_base + 2 * W2_CHUNK_BYTES;                // 4 x 8 KB
    const uint32_t h_base = a_base + A_STAGES * A_BYTES;                 // 2 warpgroups x 2 chunks x 8 KB
    const uint32_t bias_base = h_base + 4 * H_CHUNK_BYTES;               // 128 + 32 floats: b1cat | b2cat
    const uint32_t bar_base = bias_base + (HID + NOUT) * 4 + 64;
    auto a_full = [&](int s) { return bar_base + s * 8; };
    auto a_empty = [&](int s) { return bar_base + (A_STAGES + s) * 8; };
    const uint32_t w_bar = bar_base + (2 * A_STAGES) * 8;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_tiles = (int)((nvox + BLOCK_M - 1) / BLOCK_M);

    if (warp == 8 && lane == 0) {
        tc::tma_prefetch_desc(&tmA); tc::tma_prefetch_desc(&tmW1); tc::tma_prefetch_desc(&tmW2);
        for (int s = 0; s < A_STAGES; ++s) { tc::mbar_init(a_full(s), 1); tc::mbar_init(a_empty(s), 2); }
        tc::mbar_init(w_bar, 1);
        tc::mbar_fence_init();
    }
    float* const sbias = reinterpret_cast<float*>(smem_gen + (bias_base - smem_base));
    if (threadIdx.x < HID + NOUT) {
        const int t = threadIdx.x;
        sbias[t] = t < HID ? __ldg(b1cat + t) : (t - HID < ncls + 2 ? __ldg(b2cat + t - HID) : 0.f);
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            tc::mbar_arrive_expect_tx(w_bar, W1_BYTES + 2 * W2_CHUNK_BYTES);
            tc::tma_load_2d(w1_base, &tmW1, w_bar, 0, 0);
            tc::tma_load_2d(w2_base, &tmW2, w_bar, 0, 0);
            tc::tma_load_2d(w2_base + W2_CHUNK_BYTES, &tmW2, w_bar, 64, 0);
            int s = 0; uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                tc::mbar_wait(a_empty(s), ph ^ 1);
                tc::mbar_arrive_expect_tx(a_full(s), A_BYTES);
                tc::tma_load_2d(a_base + s * A_BYTES, &tmA, a_full(s), 0, tile * BLOCK_M);
                if (++s == A_STAGES) { s = 0; ph ^= 1; }
            }
        }
        return;
    }

    const int wg = warp >> 2, wl = warp & 3;
    const int quad_col = 2 * (lane & 3);
    const uint32_t hbuf = h_base + wg * 2 * H_CHUNK_BYTES;
    tc::mbar_wait(w_bar, 0);
    int s = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        // ---- GEMM1: hidden = A . W1cat^T (K = 32: two K = 16 steps inside the 64-byte swizzle atom)
        float hid[64];
        tc::mbar_wait(a_full(s), ph);
        {
            const uint64_t da = tc::make_smem_desc(a_base + s * A_BYTES + wg * (64 * 64), 64);
            const uint64_t db = tc::make_smem_desc(w1_base, 64);
            tc::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 2; ++k) tc::wgmma_m64n128(hid, da + 2 * k, db + 2 * k, k != 0);
            tc::wgmma_commit();
            tc::wgmma_wait_all();
            tc::reg_fence(hid);
        }
        if ((threadIdx.x & 127) == 0) tc::mbar_arrive(a_empty(s));
        if (++s == A_STAGES) { s = 0; ph ^= 1; }
        // ---- epilogue A: activations -> bf16 -> swizzled K-major A operand of GEMM2 (chunk c = hidden columns [64c, 64c+64))
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");  // the previous tile's GEMM2 is done with the buffer
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int col = 8 * j + quad_col, row = 16 * wl + (lane >> 2) + 8 * h;
                const float x0 = hid[4 * j + 2 * h] + sbias[col], x1 = hid[4 * j + 2 * h + 1] + sbias[col + 1];
                const float v0 = j < 8 ? softplus1(x0) : fmaxf(x0, 0.f), v1 = j < 8 ? softplus1(x1) : fmaxf(x1, 0.f);
                const uint32_t addr = hbuf + (j >> 3) * H_CHUNK_BYTES + row * 128 + (((j & 7) ^ (row & 7)) << 4) + quad_col * 2;
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_bf16x2(v0, v1)) : "memory");
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy writes -> visible to wgmma
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        // ---- GEMM2: logits = hidden . W2cat^T (K = 128: two 64-column chunks of four K = 16 steps)
        float lg[16];
        tc::wgmma_fence();
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const uint64_t da = tc::make_smem_desc(hbuf + c * H_CHUNK_BYTES, 128);
            const uint64_t db = tc::make_smem_desc(w2_base + c * W2_CHUNK_BYTES, 128);
#pragma unroll
            for (int k = 0; k < 4; ++k) tc::wgmma_m64n32(lg, da + 2 * k, db + 2 * k, (c | k) != 0);
        }
        tc::wgmma_commit();
        tc::wgmma_wait_all();
        tc::reg_fence(lg);
        // ---- epilogue B: +bias, logits, argmax (first maximum, as torch.argmax), flow
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t v = (int64_t)tile * BLOCK_M + wg * 64 + 16 * wl + (lane >> 2) + 8 * h;
            float best = -INFINITY; int arg = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = 8 * j + quad_col + e;
                    const float a = lg[4 * j + 2 * h + e] + sbias[HID + c];
                    if (c < ncls) {
                        if (a > best) { best = a; arg = c; }
                        if (occ_logits && v < nvox) occ_logits[v * ncls + c] = a;
                    } else if (c < ncls + 2 && flow && v < nvox) {
                        flow[v * 2 + (c - ncls)] = a;
                    }
                }
            }
#pragma unroll
            for (int d = 1; d <= 2; d <<= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, d);
                const int oa = __shfl_xor_sync(0xffffffffu, arg, d);
                if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
            }
            if ((lane & 3) == 0 && v < nvox) {
                if (cls_u8) cls_u8[v] = (uint8_t)arg;
                if (cls_i64) cls_i64[v] = arg;
            }
        }
    }
}

}  // namespace

int launch_occ_head_tc(const bf16* vox, const bf16* w1cat, const bf16* w2cat, const float* b1cat, const float* b2cat,
                       int ncls, int64_t nvox, float* occ_logits, float* flow, uint8_t* cls_u8, int64_t* cls_i64,
                       cudaStream_t stream)
{
    OCC_CHECK(ncls + 2 <= MAX_CLS, "occ_head_tc: at most 17 classes");
    CUtensorMap tmA, tmW1, tmW2;
    {
        const uint64_t dims[2] = {32, (uint64_t)nvox}, strides[1] = {64};
        const uint32_t box[2] = {32, BLOCK_M};
        if (make_tensor_map_bf16(&tmA, vox, 2, dims, strides, box, 64)) return 1;
    }
    {
        const uint64_t dims[2] = {32, HID}, strides[1] = {64};
        const uint32_t box[2] = {32, HID};
        if (make_tensor_map_bf16(&tmW1, w1cat, 2, dims, strides, box, 64)) return 1;
    }
    {
        const uint64_t dims[2] = {HID, NOUT}, strides[1] = {HID * 2};
        const uint32_t box[2] = {64, NOUT};
        if (make_tensor_map_bf16(&tmW2, w2cat, 2, dims, strides, box, 128)) return 1;
    }
    const int smem = 1024 + W1_BYTES + 2 * W2_CHUNK_BYTES + A_STAGES * A_BYTES + 4 * H_CHUNK_BYTES + (HID + NOUT) * 4 + 64 + 256;
    const int num_sms = sm_count_current_device();
    const int tiles = (int)((nvox + BLOCK_M - 1) / BLOCK_M);
    const int grid = tiles < num_sms ? tiles : num_sms;
    OCC_CUDA(cudaFuncSetAttribute(head_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    head_tc_kernel<<<grid, NUM_THREADS, smem, stream>>>(tmA, tmW1, tmW2, b1cat, b2cat, ncls, nvox, occ_logits, flow,
                                                       cls_u8, cls_i64);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace occ
