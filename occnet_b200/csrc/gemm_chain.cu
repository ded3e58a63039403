// Chained wgmma GEMMs: several dense layers of the encoder in ONE persistent launch.
//
// Every nn.Linear of the encoder is row-wise independent (output row r depends on input row r only), and the launch-per-layer
// schedule of gemm_tc.cu gives each CTA only ~2 tiles per launch: its kernels are start-up + a latency chain, and a large share
// of the dense-layer time is spent ramping up and draining.  Here a CTA keeps its row range [row_begin, row_end) and walks a
// LIST of ops over it:
//
//     chain A (per encoder layer):  SCA output_proj + LayerNorm  ->  FFN linear 1 (ReLU)  ->  FFN linear 2 + LayerNorm
//                                   ->  next layer's TSA value_proj  ->  next layer's TSA sampling projection
//     chain B (per encoder layer):  TSA output_proj + LayerNorm  ->  SCA sampling projection
//
// (reference: custom_base_transformer_layer.py:150-165, temporal_self_attention.py:198-211,267, spatial_cross_attention.py:173,
// 338-348).  An op whose A operand is produced by the previous op waits, per tile, on a shared-memory counter that the consumer
// warps bump after their global writes of that tile are visible to the async proxy; nothing crosses CTAs, so there is no grid-wide
// synchronisation.  While the consumers run the epilogue of op k, the producer already loads op k+1's first tiles.
//
// Roles as in gemm_tc.cu: warps 0-7 two consumer warpgroups (wgmma.m64n64k16, accumulators in registers, epilogue from the
// accumulator fragment), warps 8-11 the producer warpgroup (warp 8 issues the TMA loads).  Two epilogue kinds:
//   kind 0  16-bit output (bf16 / fp16): bias (+ fp32 T32 constant) (+ ReLU)
//   kind 1  fused LayerNorm (N = 256): x = acc + bias + residual, row statistics over the 4 threads of a quad; fp32 residual
//           stream (T32 layout) + bf16 operand copy (+ bf16 copy of y + pos)
// Weights of an n-block stay resident in shared memory when they fit next to the ring (<= 128 KB), else a W k-block travels with
// every A stage.  N > 256 is walked as n-blocks (outer loop) x tiles (inner loop).
#include <cstdlib>
#include <cstring>

#include "gemm_tc.cuh"
#include "tc_common.cuh"

namespace occ {

int cached_map_2d(const void* base, uint64_t inner, uint64_t rows, uint32_t box_inner, uint32_t box_rows, CUtensorMap* out, uint64_t ld);

namespace {

constexpr int BLOCK_M = 128, BLOCK_K = 64, A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int NUM_THREADS = 384;                           // 2 consumer warpgroups + 1 producer warpgroup
constexpr int SMEM_TOTAL = 232448;                           // 227 KB opt-in maximum
// fixed tail at the END of the dynamic shared memory: barriers 512 B | done counters 64 B | constants 3 KB
constexpr int TAIL_BYTES = 512 + 64 + 3072;
constexpr int MAX_STAGES = 6;

struct ChainOp {
    CUtensorMap tmA, tmA2, tmW;
    void* C;                                                 // 16-bit output [M, N] (kind 0)
    const float* bias; const float* res_t32;
    const float* residual; const float* gamma; const float* beta; const float* pos;
    float* y_f32; bf16* y_bf16; bf16* y_pos_bf16;
    int kind;                                                // 0: 16-bit epilogue, 1: LayerNorm epilogue
    int N, BN, nk, nk1, act, out_half, w_resident;
    int dep;                                                 // A rows are written by the previous op of this chain
    int signal;                                              // the next op depends on this one: publish tile completions
};
struct ChainArgs { ChainOp op[GEMM_CHAIN_MAX_OPS]; int n_ops, M, stages; };

__device__ __forceinline__ int ld_acquire_shared(uint32_t addr)
{
    int v;
    asm volatile("ld.acquire.cta.shared::cta.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_shared_add(uint32_t addr, int v)
{
    asm volatile("red.release.cta.shared::cta.add.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_shared(uint32_t addr, int v)
{
    asm volatile("st.release.cta.shared::cta.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_chain_kernel(const __grid_constant__ ChainArgs args)
{
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t smem_end = tc::smem_u32(smem_raw) + SMEM_TOTAL;
    const uint32_t tail_base = (smem_end - TAIL_BYTES) & ~15u;
    const uint32_t bar_base = tail_base;                          // 512 B of mbarriers
    const uint32_t done_base = tail_base + 512;                   // int done[GEMM_CHAIN_MAX_OPS]: tiles of op i fully written
    const uint32_t cvec_base = done_base + 64;                    // float [3][256] bias / gamma / beta of the current op
    const int stages = args.stages;
    auto full_bar = [&](int s) { return bar_base + s * 8; };
    auto empty_bar = [&](int s) { return bar_base + (MAX_STAGES + s) * 8; };
    auto w_bar = [&](int kb) { return bar_base + (2 * MAX_STAGES + (kb < 7 ? kb : 7)) * 8; };
    const uint32_t wfree_bar = bar_base + (2 * MAX_STAGES + 8) * 8;   // every MMA of the (op, n-block) has completed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int M = args.M;
    const int nb32 = (M + 31) >> 5;
    const int row_begin = (int)(((long long)nb32 * blockIdx.x) / gridDim.x) << 5;
    const int row_end = min(M, (int)(((long long)nb32 * (blockIdx.x + 1)) / gridDim.x) << 5);
    const int n_tiles_m = (row_end - row_begin + BLOCK_M - 1) / BLOCK_M;

    if (warp == 8 && lane == 0) {
        for (int o = 0; o < args.n_ops; ++o) {
            tc::tma_prefetch_desc(&args.op[o].tmA); tc::tma_prefetch_desc(&args.op[o].tmW);
        }
        for (int s = 0; s < stages; ++s) { tc::mbar_init(full_bar(s), 1); tc::mbar_init(empty_bar(s), 2); }
        for (int kb = 0; kb < 8; ++kb) tc::mbar_init(w_bar(kb), 1);
        tc::mbar_init(wfree_bar, 2);
        for (int o = 0; o < GEMM_CHAIN_MAX_OPS; ++o) st_release_shared(done_base + 4 * o, 0);
        tc::mbar_fence_init();
    }
    __syncthreads();

    if (warp >= 8) {
        // ================================================================= TMA producer warpgroup (warp 8 issues)
        tc::setmaxnreg_dec<40>();                                 // registers go to the consumers
        if (warp == 8 && lane == 0) {
            int s = 0; uint32_t ph = 0; uint32_t wfree_ph = 0;
            bool first_block = true;
            asm volatile("griddepcontrol.wait;" ::: "memory");
            for (int o = 0; o < args.n_ops; ++o) {
                const ChainOp& op = args.op[o];
                const int BN = op.BN, nk = op.nk, n_blks = op.N / BN;
                const uint32_t w_tile_bytes = BN * BLOCK_K * 2;
                const uint32_t stage_bytes = A_TILE_BYTES + (op.w_resident ? 0 : w_tile_bytes);
                const uint32_t ring_base = smem_base + (op.w_resident ? nk * w_tile_bytes : 0);
                for (int nb = 0; nb < n_blks; ++nb) {
                    // the weight region / the re-carved ring may only be overwritten once every MMA issued so far has completed
                    if (!first_block) { tc::mbar_wait(wfree_bar, wfree_ph); wfree_ph ^= 1; }
                    first_block = false;
                    if (op.w_resident) {
                        for (int kb = 0; kb < nk && kb < 8; ++kb)
                            tc::mbar_arrive_expect_tx(w_bar(kb), kb < 7 ? w_tile_bytes : (nk - 7) * w_tile_bytes);
                        for (int kb = 0; kb < nk; ++kb)
                            tc::tma_load_2d(smem_base + kb * w_tile_bytes, &op.tmW, w_bar(kb), kb * BLOCK_K, nb * BN);
                    }
                    for (int t = 0; t < n_tiles_m; ++t) {
                        const int m_row = row_begin + t * BLOCK_M;
                        if (op.dep) {                             // rows of this tile written (and visible) by the previous op?
                            uint32_t spins = 0;
                            while (ld_acquire_shared(done_base + 4 * (o - 1)) < 8 * (t + 1)) {
                                __nanosleep(32);
                                if (++spins > 50000000u) { asm volatile("trap;"); }
                            }
                            asm volatile("fence.proxy.async.global;" ::: "memory");
                        }
                        for (int kb = 0; kb < nk; ++kb) {
                            tc::mbar_wait(empty_bar(s), ph ^ 1);
                            tc::mbar_arrive_expect_tx(full_bar(s), stage_bytes);
                            const uint32_t a_dst = ring_base + s * stage_bytes;
                            if (kb < op.nk1) tc::tma_load_2d(a_dst, &op.tmA, full_bar(s), kb * BLOCK_K, m_row);
                            else             tc::tma_load_2d(a_dst, &op.tmA2, full_bar(s), (kb - op.nk1) * BLOCK_K, m_row);
                            if (!op.w_resident)
                                tc::tma_load_2d(a_dst + A_TILE_BYTES, &op.tmW, full_bar(s), kb * BLOCK_K, nb * BN);
                            if (++s == stages) { s = 0; ph ^= 1; }
                        }
                    }
                }
            }
        }
        return;
    }

    // ================================================================= consumer warpgroups
    tc::setmaxnreg_inc<232>();
    const int wg = warp >> 2, wl = warp & 3;
    const int quad_col = 2 * (lane & 3);
    float* const cvec = reinterpret_cast<float*>(smem_raw + (cvec_base - tc::smem_u32(smem_raw)));
    int s = 0; uint32_t ph = 0;
    uint32_t wmask = 0;                                          // phase parity of each weight barrier (bit kb)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int o = 0; o < args.n_ops; ++o) {
        const ChainOp& op = args.op[o];
        const int BN = op.BN, nk = op.nk, n_blks = op.N / BN, N = op.N;
        const int nsubs = BN >> 6;
        const uint32_t w_tile_bytes = BN * BLOCK_K * 2;
        const uint32_t stage_bytes = A_TILE_BYTES + (op.w_resident ? 0 : w_tile_bytes);
        const uint32_t ring_base = smem_base + (op.w_resident ? nk * w_tile_bytes : 0);
        const bool ln = op.kind == 1;
        for (int nb = 0; nb < n_blks; ++nb) {
            // per-column constants of this (op, n-block) -> shared memory (both warpgroups are past the previous block's reads)
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (threadIdx.x < BN) {
                const int t = threadIdx.x;
                cvec[t] = op.bias ? __ldg(op.bias + nb * BN + t) : 0.f;
                if (ln) { cvec[256 + t] = __ldg(op.gamma + t); cvec[512 + t] = __ldg(op.beta + t); }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            for (int t = 0; t < n_tiles_m; ++t) {
                const int m_row = row_begin + t * BLOCK_M;
                float acc[4][32];
                for (int kb = 0; kb < nk; ++kb) {
                    if (op.w_resident && t == 0) tc::mbar_wait(w_bar(kb), (wmask >> (kb < 7 ? kb : 7)) & 1u);
                    tc::mbar_wait(full_bar(s), ph);
                    const uint32_t a_addr = ring_base + s * stage_bytes + wg * (64 * 128);
                    const uint32_t b_addr = op.w_resident ? smem_base + kb * w_tile_bytes : ring_base + s * stage_bytes + A_TILE_BYTES;
                    switch (nsubs) {
                    case 4: tc::wgmma_kblock<4>(acc, a_addr, b_addr, kb == 0); break;
                    case 3: tc::wgmma_kblock<3>(acc, a_addr, b_addr, kb == 0); break;
                    case 2: tc::wgmma_kblock<2>(acc, a_addr, b_addr, kb == 0); break;
                    default: tc::wgmma_kblock<1>(acc, a_addr, b_addr, kb == 0); break;
                    }
                    if ((threadIdx.x & 127) == 0) tc::mbar_arrive(empty_bar(s));
                    if (++s == stages) { s = 0; ph ^= 1; }
                }
                // last tile of this (op, n-block): the weights and the ring may be recarved
                if (t == n_tiles_m - 1 && (threadIdx.x & 127) == 0) tc::mbar_arrive(wfree_bar);
                const int r0 = m_row + wg * 64 + wl * 16 + (lane >> 2);
                if (ln) {
                    tc::ln_epilogue(acc, r0, row_end, quad_col, cvec, op.residual, op.pos, op.y_f32, op.y_bf16, op.y_pos_bf16);
                } else {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = r0 + 8 * h;
                        if (row >= row_end) continue;
#pragma unroll
                        for (int ns = 0; ns < 4; ++ns) {
                            if (ns >= nsubs) break;
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                const int col = nb * BN + ns * 64 + 8 * j + quad_col, cl = col - nb * BN;
                                float x0 = acc[ns][4 * j + 2 * h] + cvec[cl], x1 = acc[ns][4 * j + 2 * h + 1] + cvec[cl + 1];
                                if (op.res_t32) {
                                    const float2 q = __ldg(reinterpret_cast<const float2*>(op.res_t32 + tc::t32_index(row, col, N)));
                                    x0 += q.x; x1 += q.y;
                                }
                                if (op.act == ACT_RELU) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                                *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(op.C) + (size_t)row * N + col) =
                                    tc::pack_16(x0, x1, op.out_half != 0);
                            }
                        }
                    }
                }
                // Tile t of this op is complete once its LAST n-block is written: make this thread's global writes visible to
                // the async proxy (the producer's TMA loads of the next op), then one arrival per warp (8 per tile)
                if (op.signal && nb == n_blks - 1) {
                    asm volatile("fence.proxy.async.global;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) red_release_shared_add(done_base + 4 * o, 1);
                }
            }
            if (op.w_resident) wmask ^= (1u << (nk < 8 ? nk : 8)) - 1u;
        }
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------- host side
int gemm_chain_launch(const GemmChainOp* ops, int n_ops, int M, cudaStream_t stream)
{
    OCC_CHECK(n_ops >= 1 && n_ops <= GEMM_CHAIN_MAX_OPS && M > 0, "gemm_chain: 1..GEMM_CHAIN_MAX_OPS ops");
    ChainArgs a;
    memset(&a, 0, sizeof(a));
    a.n_ops = n_ops; a.M = M;
    const int avail = SMEM_TOTAL - 1024 - TAIL_BYTES - 16;
    int stages = MAX_STAGES;
    for (int i = 0; i < n_ops; ++i) {
        const GemmChainOp& g = ops[i];
        ChainOp& o = a.op[i];
        OCC_CHECK(g.K % 64 == 0 && g.K1 % 64 == 0 && g.K1 > 0 && g.K1 <= g.K && g.N % 32 == 0, "gemm_chain: unsupported shape");
        int BN = 0;
        if (g.ln) { OCC_CHECK(g.N == 256, "gemm_chain: LayerNorm ops have N = 256"); BN = 256; }
        else { for (int bn : {256, 192, 128, 64}) if (g.N % bn == 0) { BN = bn; break; } }
        OCC_CHECK(BN > 0, "gemm_chain: N must be a multiple of 64");
        o.kind = g.ln ? 1 : 0; o.N = g.N; o.BN = BN; o.nk = g.K / BLOCK_K; o.nk1 = g.K1 / BLOCK_K; o.act = g.act;
        o.out_half = g.out_half; o.dep = (i > 0 && g.dep) ? 1 : 0;
        const int w_bytes = BN * g.K * 2;
        o.w_resident = w_bytes <= 131072 && (avail - w_bytes) / A_TILE_BYTES >= 3;
        const int stage = A_TILE_BYTES + (o.w_resident ? 0 : BN * BLOCK_K * 2);
        const int st = (avail - (o.w_resident ? w_bytes : 0)) / stage;
        OCC_CHECK(st >= 2, "gemm_chain: not enough shared memory for the operand ring");
        stages = st < stages ? st : stages;
        if (cached_map_2d(g.A, (uint64_t)g.K1, (uint64_t)M, BLOCK_K, BLOCK_M, &o.tmA, 0)) return 1;
        if (g.A2) { if (cached_map_2d(g.A2, (uint64_t)(g.K - g.K1), (uint64_t)M, BLOCK_K, BLOCK_M, &o.tmA2, 0)) return 1; }
        else o.tmA2 = o.tmA;
        if (cached_map_2d(g.W, (uint64_t)g.K, (uint64_t)g.N, BLOCK_K, (uint32_t)BN, &o.tmW, 0)) return 1;
        if (!g.ln) {
            OCC_CHECK(g.C != nullptr, "gemm_chain: output pointer");
        } else {
            OCC_CHECK(g.bias && g.residual && g.gamma && g.beta && g.y_f32, "gemm_chain: LayerNorm op needs bias, residual, gamma, beta, y_f32");
            OCC_CHECK(g.y_pos_bf16 == nullptr || g.pos != nullptr, "gemm_chain: pos required for y_pos");
        }
        o.C = g.C;
        o.signal = (i + 1 < n_ops && ops[i + 1].dep) ? 1 : 0;
        o.bias = g.bias; o.res_t32 = g.res_t32; o.residual = g.residual; o.gamma = g.gamma; o.beta = g.beta; o.pos = g.pos;
        o.y_f32 = g.y_f32; o.y_bf16 = g.y_bf16; o.y_pos_bf16 = g.y_pos_bf16;
    }
    a.stages = stages;
    OCC_CUDA(cudaFuncSetAttribute(gemm_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
    const int num_sms = sm_count_current_device();
    const int nb32 = (M + 31) / 32;
    const int grid = num_sms < nb32 ? num_sms : nb32;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = SMEM_TOTAL; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    OCC_CUDA(cudaLaunchKernelEx(&cfg, gemm_chain_kernel, a));
    OCC_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace occ
