// wgmma / TMA bf16 GEMM for the dense layers of the encoder (sm_90a):
//     C[M,N] = act(A[M,K] . W[N,K]^T + bias[N]) (+ residual[M,N]),   fp32 accumulation in registers.
// Every nn.Linear on the path has this shape (reference: temporal_self_attention.py:99-104,
// spatial_cross_attention.py:67,245-249, mmcv FFN) with K in {256,512}, N in {192,256,512,768}.
//
// Persistent, warp-specialised kernel, one CTA per SM; every CTA owns one n-block and a contiguous range of rows
// (dealt in 32-row blocks so that all CTAs move the same number of bytes):
//   warps 0-7  two consumer warpgroups: warpgroup g multiplies rows [64 g, 64 g + 64) of each 128-row tile with
//              wgmma.m64n64k16 (BN / 64 of them per K = 16 step), accumulators in registers, then runs the epilogue
//              straight from the accumulator fragment.  Per-column constants (bias; gamma, beta) are staged in shared
//              memory once per CTA.  Three variants: 16-bit output (bias, optional fp32 T32 constant, ReLU), fused
//              LayerNorm (row statistics reduced over the 4 threads of a quad), fp32 output (+ residual).
//   warps 8-11 producer warpgroup (setmaxnreg: its registers go to the consumers); warp 8 issues the TMA loads:
//              the CTA's weight block once (resident, <= 128 KB, one mbarrier per k-block) or a W
//              k-block per stage; A tiles 128x64 (bf16, 128B swizzle) through a 2-6 stage mbarrier ring.
// Programmatic dependent launch: the prologue (barriers, weights, constants) does not wait for the previous grid.
// The A operand may be the concatenation of two matrices along K (TSA's cat([value, query+pos]),
// temporal_self_attention.py:197) -- two tensor maps, no materialised concat.
#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>

#include "gemm_tc.cuh"
#include "tc_common.cuh"

namespace occ {

// ------------------------------------------------------------------------------------------------ host helpers
PFN_encodeTiled get_encode_tiled()
{
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

int make_tensor_map_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                         const uint32_t* box, int swizzle_bytes)
{
    PFN_encodeTiled enc = get_encode_tiled();
    OCC_CHECK(enc != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
    cuuint64_t gdim[5], gstr[5];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr,
                           bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    OCC_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
    return 0;
}

namespace {

constexpr int BLOCK_M = 128, BLOCK_K = 64, A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int NUM_THREADS = 384;                          // 2 consumer warpgroups + 1 producer warpgroup
constexpr int SMEM_TAIL = 3072 + 256;                     // per-column constants (bias | gamma | beta) + barriers
constexpr int SMEM_MAX = 232448 - 1024;                   // 227 KB opt-in maximum minus alignment slack
constexpr int MAX_STAGES = 6;

struct LnArgs {                                           // fused LayerNorm epilogue (N == BN == 256)
    const float* gamma; const float* beta; const float* pos;
    float* y_f32; bf16* y_bf16; bf16* y_pos_bf16;
};

// One GEMM problem of a launch.  A launch carries up to MAX_PROBS INDEPENDENT problems (e.g. TSA's value projection and
// sampling-offset projection of the same query tensor): the CTAs [cta_begin, cta_begin + cta_count) work on problem p.  These
// GEMMs have only ~2 tiles per CTA, so their duration is start-up + a latency chain, not bandwidth: two problems on
// half the CTAs each finish in about the time ONE took on all of them.
// w_resident: all nk weight k-blocks of this CTA's n-block stay in shared memory for the CTA's lifetime and the
// ring only carries A tiles; otherwise each stage carries an A tile and a W k-block.
constexpr int MAX_PROBS = 3;
struct GemmProb {
    CUtensorMap tmA, tmA2, tmW;
    const float* bias; const float* residual; void* C;
    const float* res_t32;                                     // optional fp32 epilogue constant [M,N] in the T32 block layout
                                                              // (never together with residual: the epilogue loads one of them)
    long long ldc, nblk_stride;                               // C offset of (row, column c of n-block b): b * nblk_stride + row * ldc + c
    int head_major;                                           // always 0 (see the 16-bit epilogue)
    int M, N, BN, nk, nk1, act, w_resident, stages;
    int out_half;                                             // 16-bit outputs as fp16 instead of bf16 (runtime, per problem)
    int cta_begin, cta_count;
};
struct GemmProbs { GemmProb p[MAX_PROBS]; int n; };

template <typename TC, bool LN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ GemmProbs probs, LnArgs ln)
{
    int pi = 0;
    while (pi + 1 < probs.n && (int)blockIdx.x >= probs.p[pi + 1].cta_begin) ++pi;
    const GemmProb& P = probs.p[pi];
    const float* __restrict__ residual = P.residual;
    const float* __restrict__ res_t32 = P.res_t32;
    const int M = P.M, N = P.N, BN = P.BN, nk = P.nk, nk1 = P.nk1, act = P.act;
    const int w_resident = P.w_resident, stages = P.stages;
    const bool out_half = std::is_same<TC, __half>::value || P.out_half != 0;
    const int bid = (int)blockIdx.x - P.cta_begin, nctas = P.cta_count;
    // Programmatic dependent launch: let the next kernel in the stream start its prologue while this grid drains,
    // and (below) only wait for the PREVIOUS grid right before touching data it produced.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t w_tile_bytes = BN * BLOCK_K * 2;
    const uint32_t w_region = w_resident ? nk * w_tile_bytes : 0;
    const uint32_t stage_bytes = A_TILE_BYTES + (w_resident ? 0 : w_tile_bytes);
    const uint32_t ring_base = smem_base + w_region;
    const uint32_t cvec_base = ring_base + stages * stage_bytes;
    const uint32_t bar_base = cvec_base + 3072;
    auto full_bar = [&](int s) { return bar_base + s * 8; };
    auto empty_bar = [&](int s) { return bar_base + (MAX_STAGES + s) * 8; };
    // one barrier per resident weight k-block (the last one collects every block >= 7): the first MMA starts as soon
    // as ITS slice has landed instead of waiting for the whole block
    auto w_bar = [&](int kb) { return bar_base + (2 * MAX_STAGES + (kb < 7 ? kb : 7)) * 8; };
    float* const cvec = reinterpret_cast<float*>(smem_raw + (cvec_base - tc::smem_u32(smem_raw)));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles = N / BN;
    // CTA -> (fixed n block, contiguous row range): a resident weight block serves every tile of the CTA, and the
    // rows are dealt out in 32-row blocks so that every CTA gets (almost) the same number of ROWS; the last tile of a
    // CTA is partial and its epilogue only touches the rows it owns.
    const int n_blk = bid % n_tiles;
    const int grp = bid / n_tiles, ngrp = nctas / n_tiles;
    const int nb32 = (M + 31) >> 5;
    const int row_begin = (int)(((long long)nb32 * grp) / ngrp) << 5;
    const int row_end = min(M, (int)(((long long)nb32 * (grp + 1)) / ngrp) << 5);

    if (warp == 8 && lane == 0) {
        tc::tma_prefetch_desc(&P.tmA); tc::tma_prefetch_desc(&P.tmA2); tc::tma_prefetch_desc(&P.tmW);
        for (int s = 0; s < stages; ++s) { tc::mbar_init(full_bar(s), 1); tc::mbar_init(empty_bar(s), 2); }
        for (int kb = 0; kb < 8; ++kb) tc::mbar_init(w_bar(kb), 1);
        tc::mbar_fence_init();
    }
    if (threadIdx.x < BN) {                                       // parameters: no dependency on the previous grid
        const int t = threadIdx.x;
        cvec[t] = P.bias ? __ldg(P.bias + n_blk * BN + t) : 0.f;
        if constexpr (LN) { cvec[256 + t] = __ldg(ln.gamma + t); cvec[512 + t] = __ldg(ln.beta + t); }
    }
    __syncthreads();

    if (warp >= 8) {
        tc::setmaxnreg_dec<40>();                                 // producer warpgroup: registers go to the consumers
        if (warp == 8 && lane == 0) {
            if (w_resident) {
                for (int kb = 0; kb < nk && kb < 8; ++kb)
                    tc::mbar_arrive_expect_tx(w_bar(kb), kb < 7 ? w_tile_bytes : (nk - 7) * w_tile_bytes);
                for (int kb = 0; kb < nk; ++kb)
                    tc::tma_load_2d(smem_base + kb * w_tile_bytes, &P.tmW, w_bar(kb), kb * BLOCK_K, n_blk * BN);
            }
            int s = 0; uint32_t ph = 0;
            asm volatile("griddepcontrol.wait;" ::: "memory");    // A (and residual) come from the previous kernel
            for (int m_row = row_begin; m_row < row_end; m_row += BLOCK_M) {
                for (int kb = 0; kb < nk; ++kb) {
                    tc::mbar_wait(empty_bar(s), ph ^ 1);
                    tc::mbar_arrive_expect_tx(full_bar(s), stage_bytes);
                    const uint32_t a_dst = ring_base + s * stage_bytes;
                    if (kb < nk1) tc::tma_load_2d(a_dst, &P.tmA, full_bar(s), kb * BLOCK_K, m_row);
                    else          tc::tma_load_2d(a_dst, &P.tmA2, full_bar(s), (kb - nk1) * BLOCK_K, m_row);
                    if (!w_resident)
                        tc::tma_load_2d(a_dst + A_TILE_BYTES, &P.tmW, full_bar(s), kb * BLOCK_K, n_blk * BN);
                    if (++s == stages) { s = 0; ph ^= 1; }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumer warpgroups
    tc::setmaxnreg_inc<232>();
    const int wg = warp >> 2, wl = warp & 3;
    const int nsubs = BN >> 6;                                    // 64-column wgmma sub-tiles (1..4)
    const int quad_col = 2 * (lane & 3);
    int s = 0; uint32_t ph = 0;
    int tcount = 0;
    asm volatile("griddepcontrol.wait;" ::: "memory");            // before the first global read / write of this role
    for (int m_row = row_begin; m_row < row_end; m_row += BLOCK_M, ++tcount) {
        float acc[4][32];
        for (int kb = 0; kb < nk; ++kb) {
            if (w_resident && tcount == 0) tc::mbar_wait(w_bar(kb), 0);      // weight slice kb resident
            tc::mbar_wait(full_bar(s), ph);
            const uint32_t a_addr = ring_base + s * stage_bytes + wg * (64 * 128);
            const uint32_t b_addr = w_resident ? smem_base + kb * w_tile_bytes : ring_base + s * stage_bytes + A_TILE_BYTES;
            switch (nsubs) {
            case 4: tc::wgmma_kblock<4>(acc, a_addr, b_addr, kb == 0); break;
            case 3: tc::wgmma_kblock<3>(acc, a_addr, b_addr, kb == 0); break;
            case 2: tc::wgmma_kblock<2>(acc, a_addr, b_addr, kb == 0); break;
            default: tc::wgmma_kblock<1>(acc, a_addr, b_addr, kb == 0); break;
            }
            if ((threadIdx.x & 127) == 0) tc::mbar_arrive(empty_bar(s));   // this warpgroup is done with the stage
            if (++s == stages) { s = 0; ph ^= 1; }
        }
        const int r0 = m_row + wg * 64 + wl * 16 + (lane >> 2);        // rows r0 (h = 0) and r0 + 8 (h = 1)
        if constexpr (LN) {
            tc::ln_epilogue(acc, r0, row_end, quad_col, cvec, residual, ln.pos, ln.y_f32, ln.y_bf16, ln.y_pos_bf16);
        } else {
            // Column cl = ns * 64 + 8 j + quad_col lies in 32-column block 2 ns + j / 4 at offset 8 (j % 4) + quad_col, so every
            // address below is a per-row base plus a compile-time multiple of a per-launch stride.  The fp32 epilogue operand
            // (res_t32 or residual, never both) of a row is loaded in full before its first use: the loads are in flight
            // together instead of one latency per column pair.  Per element the arithmetic is unchanged.
            const bool has_t32 = res_t32 != nullptr, has_res = residual != nullptr, relu = act == ACT_RELU;
            const float* __restrict__ qsrc = has_t32 ? res_t32 : residual;
            const int q_blk = has_t32 ? 1024 : 32, q_j = has_t32 ? 256 : 8;           // operand offset per 32 / per 8 columns
            // Output offset per 32 columns.  The head_major arm is never taken, but without this run-time select nvcc 12.9 schedules
            // the epilogue differently and the dense layers got 4-5 % slower on an H100 (400 W); it goes with the epilogue rework.
            const size_t o_blk = P.head_major ? (size_t)M * 32 : 32;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h;
                if (row >= row_end) continue;
                const float* const qrow =
                    qsrc + (has_t32 ? ((((size_t)(row >> 5) * (N >> 5) + n_blk * (BN >> 5)) * 256 + (quad_col >> 2) * 32 + (row & 31)) << 2) +
                                          (quad_col & 3)
                                    : (size_t)row * N + n_blk * BN + quad_col);
                float2 q[4][8];
                if (qsrc) {
#pragma unroll
                    for (int ns = 0; ns < 4; ++ns) {
                        if (ns >= nsubs) break;
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            q[ns][j] = __ldg(reinterpret_cast<const float2*>(qrow + (2 * ns + j / 4) * q_blk + (j & 3) * q_j));
                    }
                }
                TC* const orow = reinterpret_cast<TC*>(P.C) +
                                 (P.head_major ? ((size_t)n_blk * (BN >> 5) * M + row) * 32 + quad_col
                                               : (size_t)n_blk * P.nblk_stride + (size_t)row * P.ldc + quad_col);
#pragma unroll
                for (int ns = 0; ns < 4; ++ns) {
                    if (ns >= nsubs) break;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int cl = ns * 64 + 8 * j + quad_col;
                        float x0 = acc[ns][4 * j + 2 * h] + cvec[cl], x1 = acc[ns][4 * j + 2 * h + 1] + cvec[cl + 1];
                        if (has_t32) { x0 += q[ns][j].x; x1 += q[ns][j].y; }
                        if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                        if (has_res) { x0 += q[ns][j].x; x1 += q[ns][j].y; }
                        TC* const o = orow + (2 * ns + j / 4) * o_blk + 8 * (j & 3);
                        if constexpr (sizeof(TC) == 4)
                            *reinterpret_cast<float2*>(o) = make_float2(x0, x1);
                        else
                            *reinterpret_cast<uint32_t*>(o) = tc::pack_16(x0, x1, out_half);
                    }
                }
            }
        }
    }
}

// tile-N choice: prefer a weight block that fits resident (<= 128 KB) next to >= 4 A stages
struct Plan { int BN, resident, stages, smem; };

Plan make_plan(int N, int K, bool ln)
{
    const int SMEM_LIMIT = SMEM_MAX - SMEM_TAIL;
    Plan p{0, 0, 0, 0};
    const int cands[] = {256, 192, 128, 64};                  // multiples of the 64-column wgmma sub-tile
    if (ln) {
        p.BN = 256;
    } else {
        for (int bn : cands) {
            if (N % bn != 0 || bn > N) continue;
            if ((long)bn * K * 2 <= 131072) { p.BN = bn; break; }
        }
        if (K > 512 && p.BN != 0 && p.BN < 128) p.BN = 0;     // split-operand GEMMs (K' = 3K): a 64-wide resident block would
                                                              // re-read A once per 64 columns; stream W with a wide tile instead
        if (p.BN == 0) {                                      // no resident candidate: largest tile that divides N
            for (int bn : cands) if (N % bn == 0 && bn <= N) { p.BN = bn; break; }
        }
    }
    if (p.BN == 0) return p;
    const int w_bytes = p.BN * K * 2;
    p.resident = w_bytes <= 131072;
    const int stage = A_TILE_BYTES + (p.resident ? 0 : p.BN * BLOCK_K * 2);
    const int avail = SMEM_LIMIT - (p.resident ? w_bytes : 0);
    p.stages = avail / stage;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    p.smem = 1024 + (p.resident ? w_bytes : 0) + p.stages * stage + SMEM_TAIL;
    return p;
}

struct MapKey {
    const void* p; uint64_t d0, d1, ld; uint32_t b0, b1;
    bool operator<(const MapKey& o) const { return std::tie(p, d0, d1, ld, b0, b1) < std::tie(o.p, o.d0, o.d1, o.ld, o.b0, o.b1); }
};

// row-major bf16 [rows, inner] with a row pitch of `ld` elements (0 = dense)
int cached_map_2d(const void* base, uint64_t inner, uint64_t rows, uint32_t box_inner, uint32_t box_rows, CUtensorMap* out,
                  uint64_t ld = 0)
{
    static std::map<MapKey, CUtensorMap> cache;
    static std::mutex mu;
    std::lock_guard<std::mutex> g(mu);
    if (ld == 0) ld = inner;
    const MapKey k{base, inner, rows, ld, box_inner, box_rows};
    auto it = cache.find(k);
    if (it == cache.end()) {
        CUtensorMap m;
        const uint64_t dims[2] = {inner, rows}, strides[1] = {ld * 2};
        const uint32_t box[2] = {box_inner, box_rows};
        if (make_tensor_map_bf16(&m, base, 2, dims, strides, box, 128)) return 1;
        if (cache.size() > 4096) cache.clear();
        it = cache.emplace(k, m).first;
    }
    *out = it->second;
    return 0;
}

// Fills one problem (tensor maps, plan, CTA share).  ctas = number of CTAs this problem may use (0: all SMs).
template <typename TC, bool LN>
int build_prob(GemmProb& P, int& smem, const bf16* A, const bf16* A2, int K1, const bf16* W, const float* bias, const float* residual,
               TC* C, int M, int N, int K, int act, bool blocked_out, int lda, int lda2, int ctas, int cta_begin)
{
    if (A2 == nullptr) K1 = K;
    const Plan p = make_plan(N, K, LN);
    OCC_CHECK(p.BN > 0 && p.stages >= 2 && K % 64 == 0 && K1 % 64 == 0 && M > 0, "gemm_tc: unsupported shape");
    if (cached_map_2d(A, (uint64_t)K1, (uint64_t)M, BLOCK_K, BLOCK_M, &P.tmA, (uint64_t)lda)) return 1;
    if (A2) { if (cached_map_2d(A2, (uint64_t)(K - K1), (uint64_t)M, BLOCK_K, BLOCK_M, &P.tmA2, (uint64_t)lda2)) return 1; }
    else P.tmA2 = P.tmA;
    if (cached_map_2d(W, (uint64_t)K, (uint64_t)N, BLOCK_K, (uint32_t)p.BN, &P.tmW)) return 1;
    if (ctas <= 0) ctas = sm_count_current_device();
    const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M, n_tiles = N / p.BN;
    int per_n = ctas / n_tiles;
    if (per_n > m_tiles) per_n = m_tiles;                        // (row ranges are dealt in 32-row blocks: >= 1 per CTA)
    OCC_CHECK(per_n >= 1, "gemm_tc: fewer CTAs than n-blocks");
    P.bias = bias; P.residual = residual; P.C = C; P.res_t32 = nullptr;
    P.ldc = blocked_out ? (long long)p.BN : (long long)N;
    P.nblk_stride = blocked_out ? (long long)M * p.BN : (long long)p.BN;
    P.head_major = 0;
    P.M = M; P.N = N; P.BN = p.BN; P.nk = K / BLOCK_K; P.nk1 = K1 / BLOCK_K; P.act = act;
    P.w_resident = p.resident; P.stages = p.stages;
    P.out_half = std::is_same<TC, __half>::value ? 1 : 0;
    P.cta_begin = cta_begin; P.cta_count = per_n * n_tiles;
    smem = p.smem;
    return 0;
}

template <typename TC, bool LN>
int launch_probs(const GemmProbs& probs, int smem, LnArgs ln, cudaStream_t stream)
{
    // per-device attribute (cheap): a process-wide `static bool` would leave a second device without the opt-in
    OCC_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<TC, LN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    const GemmProb& last = probs.p[probs.n - 1];
    const int grid = last.cta_begin + last.cta_count;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    OCC_CUDA(cudaLaunchKernelEx(&cfg, gemm_tc_kernel<TC, LN>, probs, ln));
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template <typename TC, bool LN>
int launch(const bf16* A, const bf16* A2, int K1, const bf16* W, const float* bias, const float* residual, TC* C,
           LnArgs ln, int M, int N, int K, int act, cudaStream_t stream, bool blocked_out = false, int lda = 0, int lda2 = 0)
{
    GemmProbs probs;
    probs.n = 1;
    int smem = 0;
    if (build_prob<TC, LN>(probs.p[0], smem, A, A2, K1, W, bias, residual, C, M, N, K, act, blocked_out, lda, lda2, 0, 0))
        return 1;
    return launch_probs<TC, LN>(probs, smem, ln, stream);
}

}  // namespace

bool gemm_tc_supported(int M, int N, int K, int K1)
{
    const Plan p = make_plan(N, K, false);
    return M > 0 && p.BN >= 64 && p.BN % 64 == 0 && p.stages >= 2 && K % 64 == 0 && K1 % 64 == 0 && K1 > 0 && K1 <= K;
}

template <typename TC>
int gemm_tc(const bf16* A, const bf16* A2, int K1, const bf16* W, const float* bias, const float* residual, TC* C,
            int M, int N, int K, int act, cudaStream_t stream)
{
    return launch<TC, false>(A, A2, K1, W, bias, residual, C, LnArgs{}, M, N, K, act, stream);
}

// fp32-grade GEMM on the tensor cores: S = [hi | lo] (bf16 split of an fp32 operand, row pitch 2*Ks), W3 = [W_hi | W_hi | W_lo]
// (N x 3*Ks).  C = hi.W_hi + lo.W_hi + hi.W_lo  (the lo.lo term, 2^-16 relative, is dropped) as ONE GEMM with K' = 3*Ks whose
// A operand is the concatenation [S (2*Ks columns) | first Ks columns of S again] -- two tensor maps over the same buffer.
int gemm_tc_split3(const bf16* S, int Ks, const bf16* W3, const float* bias, const float* residual, float* C, int M, int N,
                   int act, cudaStream_t stream)
{
    return launch<float, false>(S, S, 2 * Ks, W3, bias, residual, C, LnArgs{}, M, N, 3 * Ks, act, stream, false, 2 * Ks, 2 * Ks);
}

int gemm_tc_blocked256(const bf16* A, const bf16* W, const float* bias, bf16* C, int M, int N, int K, cudaStream_t stream)
{
    const Plan p = make_plan(N, K, false);
    OCC_CHECK(p.BN == 256 && N % 256 == 0, "gemm_tc_blocked256: N must be a multiple of 256 with 256-wide tiles");
    return launch<bf16, false>(A, nullptr, 0, W, bias, nullptr, C, LnArgs{}, M, N, K, ACT_NONE, stream, true);
}

// residual, y_f32 and pos are in the T32 block layout (elementwise.cu), rows padded to a multiple of 32
int gemm_tc_ln(const bf16* A, const bf16* W, const float* bias, const float* residual, const float* gamma,
               const float* beta, const float* pos, float* y_f32, bf16* y_bf16, bf16* y_pos_bf16, int M, int K,
               cudaStream_t stream)
{
    OCC_CHECK(bias && residual && gamma && beta, "gemm_tc_ln: bias, residual, gamma, beta are required");
    OCC_CHECK(y_pos_bf16 == nullptr || pos != nullptr, "gemm_tc_ln: pos required for y_pos");
    return launch<float, true>(A, nullptr, 0, W, bias, residual, (float*)nullptr, LnArgs{gamma, beta, pos, y_f32, y_bf16, y_pos_bf16},
                               M, 256, K, ACT_NONE, stream);
}

// Two (or three) independent 16-bit-output GEMMs in ONE launch: the CTAs are shared out in proportion to N.K.
//   value problems: Cv[i] = Av[i].Wv^T + bv (bf16, [M,256]), i < nv <= 2  (TSA value_proj of each queue entry)
//   projection    : Cq = [Aq | Aq2].Wq^T + bq (+ rq, fp32 [M,Nq]) as fp16   (sampling offsets + attention logits)
int gemm_tc_tsa_inputs(const bf16* const* Av, int nv, const bf16* Wv, const float* bv, bf16* const* Cv, const bf16* Aq,
                       const bf16* Aq2, int K1q, const bf16* Wq, const float* bq, const float* rq, const float* rq_t32, __half* Cq,
                       int M, int Nq, int Kq, cudaStream_t stream)
{
    OCC_CHECK(nv >= 1 && nv <= 2, "gemm_tc_tsa_inputs: 1 or 2 value problems");
    const int num_sms = sm_count_current_device();
    const double wv = 256.0 * 256.0, wq = (double)Nq * Kq, tot = nv * wv + wq;
    int cq = (int)(num_sms * wq / tot + 0.5);
    const int nq_tiles = Nq / make_plan(Nq, Kq, false).BN;
    if (cq < nq_tiles) cq = nq_tiles;
    const int cv = (num_sms - cq) / nv;
    OCC_CHECK(cv >= 1, "gemm_tc_tsa_inputs: not enough SMs");
    GemmProbs probs;
    probs.n = nv + 1;
    int smem = 0, sm = 0, begin = 0;
    for (int i = 0; i < nv; ++i) {
        if (build_prob<bf16, false>(probs.p[i], sm, Av[i], nullptr, 0, Wv, bv, nullptr, Cv[i], M, 256, 256, ACT_NONE, false, 0, 0,
                                    cv, begin)) return 1;
        begin += probs.p[i].cta_count;
        smem = sm > smem ? sm : smem;
    }
    // (built through the bf16 instantiation: out_half selects the fp16 packing at run time)
    // rq_t32: the epilogue constant in the T32 layout, added before the 16-bit rounding; otherwise the row-major fp32 rq
    const bool t32 = rq_t32 != nullptr && M % 32 == 0;
    if (build_prob<bf16, false>(probs.p[nv], sm, Aq, Aq2, K1q, Wq, bq, t32 ? nullptr : rq, reinterpret_cast<bf16*>(Cq), M, Nq, Kq,
                                ACT_NONE, false, 0, 0, cq, begin)) return 1;
    probs.p[nv].out_half = 1;
    if (t32) probs.p[nv].res_t32 = rq_t32;
    smem = sm > smem ? sm : smem;
    return launch_probs<bf16, false>(probs, smem, LnArgs{}, stream);
}

template int gemm_tc<float>(const bf16*, const bf16*, int, const bf16*, const float*, const float*, float*, int, int,
                            int, int, cudaStream_t);
template int gemm_tc<bf16>(const bf16*, const bf16*, int, const bf16*, const float*, const float*, bf16*, int, int, int,
                           int, cudaStream_t);
template int gemm_tc<__half>(const bf16*, const bf16*, int, const bf16*, const float*, const float*, __half*, int, int, int,
                             int, cudaStream_t);

}  // namespace occ
