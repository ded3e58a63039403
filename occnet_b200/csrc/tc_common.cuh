// Hopper (sm_90a) primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma (warpgroup MMA with register accumulators) and its shared-memory operand descriptors.
// Hand-written inline PTX; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace occ {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded spin: a protocol bug must not hang the GPU -- trap instead.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > 20000000u) { asm volatile("trap;"); }
    }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* desc)
{
    asm volatile("prefetch.tensormap [%0];" ::"l"(desc) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* desc, uint32_t bar, int c0, int c1)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(desc), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* desc, uint32_t bar, int c0, int c1, int c2, int c3)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(desc), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, sm_90a)
// D[regs] (+)= A[smem] . B[smem]^T, bf16 inputs, fp32 accumulators in the registers of the issuing warpgroup (4 aligned warps,
// all 128 threads execute the instruction).  Accumulator fragment of m64nN: thread t = 32 w + l holds rows 16 w + l / 4 (+ 8) and
// columns 8 j + 2 (l % 4) (+ 1):  d[4 j + 2 h + e] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + e].
// Register budget of a warpgroup (all its warps execute it): the producer warpgroup gives registers back, the consumer
// warpgroups take them (12 warps x 168 at launch; 2 x 4 warps x 232 + 4 x 40 after).
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keep the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// output operands d[i] .. d[i + 7] of a wgmma wrapper
#define OCC_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : OCC_ACC8(0), OCC_ACC8(8)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : OCC_ACC8(0), OCC_ACC8(8), OCC_ACC8(16), OCC_ACC8(24)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n96(float (&d)[48], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
        : OCC_ACC8(0), OCC_ACC8(8), OCC_ACC8(16), OCC_ACC8(24), OCC_ACC8(32), OCC_ACC8(40)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : OCC_ACC8(0), OCC_ACC8(8), OCC_ACC8(16), OCC_ACC8(24), OCC_ACC8(32), OCC_ACC8(40), OCC_ACC8(48), OCC_ACC8(56)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}

// ---------------------------------------------------------------- descriptors
// K-major operand tile whose rows are `row_bytes` (32 / 64 / 128) wide and swizzled with the matching TMA swizzle mode:
// 8-row core groups are 8 * row_bytes apart (SBO); LBO is unused for swizzled K-major tiles.  A K = 16 step inside the
// swizzle atom advances the start address by 32 bytes (+2 in the descriptor).  sm_90 layout: bits [62,64) 1/2/3 = 128/64/32 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t row_bytes)
{
    const uint64_t layout = row_bytes == 128 ? 1 : (row_bytes == 64 ? 2 : 3);
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);            // start address, bits [0,14)
    d |= (uint64_t)1 << 16;                                 // leading byte offset (unused)
    d |= (uint64_t)((8 * row_bytes) >> 4) << 32;            // stride byte offset, bits [32,46)
    d |= layout << 62;                                      // swizzle mode, bits [62,64)
    return d;
}

// float offset of (row, col) in the T32 block layout of an [rows, ncols] fp32 matrix (elementwise.cu): 32 x 32 blocks, inside a
// block float4 piece j = (col % 32) / 4 of row r at (j * 32 + r)
__device__ __forceinline__ size_t t32_index(int row, int col, int ncols)
{
    return ((((size_t)(row >> 5) * (ncols >> 5) + (col >> 5)) * 256 + ((col & 31) >> 2) * 32 + (row & 31)) << 2) + (col & 3);
}

__device__ __forceinline__ uint32_t pack_16(float a, float b, bool half)
{
    if (half) {
        const __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<const uint32_t*>(&h);
    }
    return pack_bf16x2(a, b);
}

// LayerNorm epilogue of a 64 x 256 warpgroup tile (acc: 4 x wgmma.m64n64 fragments; rows r0 and r0 + 8 of this thread, columns
// 8 j + quad_col (+ 1) of every 64-column sub-tile).  x = acc + bias + residual (T32), y = LN(x) over the 256 columns of a row,
// whose statistics are reduced over the 4 threads of a quad (one pass, or two where the mean is large against the spread);
// cvec = [bias | gamma | beta] in shared memory.  Writes y (fp32 T32),
// bf16 y and bf16 y + pos (row-major [M, 256]) where the pointers are set.  The residual is read with plain (coherent) loads:
// it may have been written earlier in the same launch.
constexpr float LN_ONE_PASS_R2 = 16.f;
__device__ __forceinline__ void ln_epilogue(float (&acc)[4][32], int r0, int row_end, int quad_col, const float* cvec,
                                            const float* residual, const float* pos, float* y_f32, bf16* y_bf16, bf16* y_pos_bf16)
{
    auto ld2 = [](const float* p) {
        float2 v;
        asm volatile("ld.global.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
        return v;
    };
    float mean[2], rstd[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        float sum = 0.f, sumsq = 0.f;
#pragma unroll
        for (int ns = 0; ns < 4; ++ns) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = ns * 64 + 8 * j + quad_col;
                const float2 q = row < row_end ? ld2(residual + t32_index(row, c, 256)) : make_float2(0.f, 0.f);
                const float x0 = acc[ns][4 * j + 2 * h] + cvec[c] + q.x, x1 = acc[ns][4 * j + 2 * h + 1] + cvec[c + 1] + q.y;
                acc[ns][4 * j + 2 * h] = x0; acc[ns][4 * j + 2 * h + 1] = x1;
                sum += x0 + x1;
                sumsq = fmaf(x0, x0, fmaf(x1, x1, sumsq));
            }
        }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1); sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        sumsq += __shfl_xor_sync(0xffffffffu, sumsq, 1); sumsq += __shfl_xor_sync(0xffffffffu, sumsq, 2);
        mean[h] = sum * (1.f / 256.f);
        float var = fmaxf(sumsq * (1.f / 256.f) - mean[h] * mean[h], 0.f);
        // The one-pass variance cancels when |mean| >> std: its relative error grows like (mean / std)^2.  Rows with
        // mean^2 > 16 var take a second pass over the registers, sum((x - mean)^2) as layernorm256 computes it; below that
        // bound the one-pass error stays under 3e-5 relative.  The branch is warp-uniform (the quad shuffles need the whole
        // warp), so warps without such a row skip the second pass.
        const bool two_pass = mean[h] * mean[h] > LN_ONE_PASS_R2 * var;
        if (__any_sync(0xffffffffu, two_pass)) {
            float ss = 0.f;
#pragma unroll
            for (int ns = 0; ns < 4; ++ns) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float d0 = acc[ns][4 * j + 2 * h] - mean[h], d1 = acc[ns][4 * j + 2 * h + 1] - mean[h];
                    ss = fmaf(d0, d0, fmaf(d1, d1, ss));
                }
            }
            ss += __shfl_xor_sync(0xffffffffu, ss, 1); ss += __shfl_xor_sync(0xffffffffu, ss, 2);
            if (two_pass) var = ss * (1.f / 256.f);
        }
        rstd[h] = rsqrtf(var + 1e-5f);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (row >= row_end) continue;
#pragma unroll
        for (int ns = 0; ns < 4; ++ns) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = ns * 64 + 8 * j + quad_col;
                const float y0 = (acc[ns][4 * j + 2 * h] - mean[h]) * rstd[h] * cvec[256 + c] + cvec[512 + c];
                const float y1 = (acc[ns][4 * j + 2 * h + 1] - mean[h]) * rstd[h] * cvec[256 + c + 1] + cvec[512 + c + 1];
                const size_t ti = t32_index(row, c, 256);
                if (y_f32) *reinterpret_cast<float2*>(y_f32 + ti) = make_float2(y0, y1);
                if (y_bf16) *reinterpret_cast<uint32_t*>(y_bf16 + (size_t)row * 256 + c) = pack_bf16x2(y0, y1);
                if (y_pos_bf16) {
                    const float2 p = __ldg(reinterpret_cast<const float2*>(pos + ti));
                    *reinterpret_cast<uint32_t*>(y_pos_bf16 + (size_t)row * 256 + c) = pack_bf16x2(y0 + p.x, y1 + p.y);
                }
            }
        }
    }
}

// one 64-deep k-block (128-byte rows) of a warpgroup's 64-row slice: A (64 x 64, 128B swizzle) times the NS 64-row sub-tiles of the weight
// k-block, then wait for the MMAs (the stage may be released afterwards)
template <int NS>
__device__ __forceinline__ void wgmma_kblock(float (&acc)[4][32], uint32_t a_addr, uint32_t b_addr, bool first)
{
    const uint64_t da = make_smem_desc(a_addr, 128);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {                     // +32 bytes (>>4 = 2) per K = 16 step inside the swizzle atom
#pragma unroll
        for (int ns = 0; ns < NS; ++ns)
            wgmma_m64n64(acc[ns], da + 2 * k, make_smem_desc(b_addr + ns * (64 * 128), 128) + 2 * k, !(first && k == 0));
    }
    wgmma_commit();
    wgmma_wait_all();
#pragma unroll
    for (int ns = 0; ns < NS; ++ns) reg_fence(acc[ns]);
}

}  // namespace tc

// ---------------------------------------------------------------- host: per-device launch facts
// (one process may drive engines on several devices: nothing here may be cached process-wide)
inline int sm_count_current_device()
{
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cache[dev] == 0) cudaDeviceGetAttribute(&cache[dev], cudaDevAttrMultiProcessorCount, dev);
    return cache[dev] > 0 ? cache[dev] : 132;
}

// ---------------------------------------------------------------- host: tensor-map encoding without linking libcuda
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();
// bf16 tensor of `rank` dims (dims[0] innermost / contiguous), strides in BYTES for dims 1..rank-1
int make_tensor_map_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                         const uint32_t* box, int swizzle_bytes);

}  // namespace occ
