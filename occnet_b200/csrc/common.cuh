// Shared device/host helpers for libocc_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace occ {

// ---- error plumbing: every C-ABI entry returns 0 on success, non-zero + message otherwise
void set_last_error(const std::string& msg);
#define OCC_CHECK(cond, msg)                                                              \
    do {                                                                                  \
        if (!(cond)) {                                                                    \
            occ::set_last_error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + \
                                ": " + (msg));                                            \
            return 1;                                                                     \
        }                                                                                 \
    } while (0)
#define OCC_CUDA(expr)                                                                    \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            occ::set_last_error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + \
                                ": CUDA error: " + cudaGetErrorString(_e));               \
            return 2;                                                                     \
        }                                                                                 \
    } while (0)

// ---- one device allocation, freed by its destructor (movable, not copyable)
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept
    {
        if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
        return *this;
    }
    ~DevBuf() { release(); }
    int alloc(size_t n)
    {
        release();
        if (n == 0) return 0;
        OCC_CUDA(cudaMalloc(&p, n));
        bytes = n;
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    template <typename U> U* as() const { return reinterpret_cast<U*>(p); }
};

// allocate `b` to exactly n bytes unless it already has that size (contents are kept then)
inline int ensure(DevBuf& b, size_t n) { return b.bytes != n && b.alloc(n) ? 2 : 0; }

typedef __nv_bfloat16 bf16;

// ---- storage-type helpers: T in {float, bf16}; arithmetic is always fp32
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f32<bf16>(float v) { return __float2bfloat16_rn(v); }

// load 8 consecutive channels (16-byte aligned for bf16, 32-byte for fp32) as fp32
__device__ __forceinline__ void load8(const float* __restrict__ p, float (&v)[8]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void load8(const bf16* __restrict__ p, float (&v)[8]) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    v[0] = __uint_as_float(u.x << 16); v[1] = __uint_as_float(u.x & 0xffff0000u);
    v[2] = __uint_as_float(u.y << 16); v[3] = __uint_as_float(u.y & 0xffff0000u);
    v[4] = __uint_as_float(u.z << 16); v[5] = __uint_as_float(u.z & 0xffff0000u);
    v[6] = __uint_as_float(u.w << 16); v[7] = __uint_as_float(u.w & 0xffff0000u);
}
__device__ __forceinline__ void store8(float* __restrict__ p, const float (&v)[8]) {
    reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void store8(bf16* __restrict__ p, const float (&v)[8]) {
    uint4 u;
    u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
    u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(p) = u;
}

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- geometry of one multi-scale value map (<= 8 levels), passed by value to kernels
struct LevelGeom {
    int num_levels;
    int h[8];
    int w[8];
    int start[8];
};

// ---- kernel launchers shared between translation units (implemented in the .cu files) ----
enum Act { ACT_NONE = 0, ACT_RELU = 1 };

// C[M,N] = act(A[M,K] . W[N,K]^T + bias[N]) (+ residual[M,N]);  A may be split in two column
// blocks (A1: k < K1 from `A`, A2: k >= K1 from `A2`), used for TSA's cat([q, q+pos]).
// TA/TC in {float, bf16}; weights and bias fp32; accumulation fp32.  SIMT (CUDA-core) path.
template <typename TA, typename TC>
int gemm_simt(const TA* A, int lda, const TA* A2, int lda2, int K1, const float* W, const float* bias,
              const float* residual, int ldr, TC* C, int ldc, int M, int N, int K, int act,
              cudaStream_t stream);

}  // namespace occ
