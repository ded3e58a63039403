// CUDA-core (SIMT) GEMM used for the fp32 parity configuration and as the bring-up path:
//   C[M,N] = act(A[M,K] . W[N,K]^T + bias[N]) (+ residual[M,N])
// Every dense layer of the path is an nn.Linear (weight [N,K], K contiguous), reference:
//   temporal_self_attention.py:99-104, spatial_cross_attention.py:245-249,:67, mmcv FFN.
// fp32 accumulation; A fp32 with C fp32, or A bf16 with C fp32 or bf16.  The tensor-core (wgmma) path
// in gemm_tc.cu replaces this for the bf16 configurations.
#include "common.cuh"

namespace occ {

namespace {

constexpr int BM = 128, BN = 64, BK = 16, LDS_A = BM + 4, LDS_W = BN + 4;

template <typename TA, typename TC>
__global__ void __launch_bounds__(256)
gemm_simt_kernel(const TA* __restrict__ A, int lda, const TA* __restrict__ A2, int lda2, int K1,
                 const float* __restrict__ W, const float* __restrict__ bias,
                 const float* __restrict__ residual, int ldr, TC* __restrict__ C, int ldc,
                 int M, int N, int K, int act)
{
    __shared__ __align__(16) float As[2][BK][LDS_A];
    __shared__ __align__(16) float Ws[2][BK][LDS_W];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int tx = tid & 15, ty = tid >> 4;               // 16 x 16 threads -> 4 cols x 8 rows each
    const int a_row = tid >> 1, a_k = (tid & 1) * 8;      // A tile: 128 rows x 16 k, 8 k per thread
    const int w_row = tid >> 2, w_k = (tid & 3) * 4;      // W tile: 64 rows x 16 k, 4 k per thread

    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    float ra[8];
    float4 rw;
    auto fetch = [&](int k0) {
        const int gm = m0 + a_row;
        if (gm < M) {
            const int kk = k0 + a_k;
            if (kk < K1) load8(A + (size_t)gm * lda + kk, ra);
            else         load8(A2 + (size_t)gm * lda2 + (kk - K1), ra);
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) ra[i] = 0.f;
        }
        const int gn = n0 + w_row;
        rw = (gn < N) ? __ldg(reinterpret_cast<const float4*>(W + (size_t)gn * K + k0 + w_k))
                      : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto stash = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 8; ++i) As[buf][a_k + i][a_row] = ra[i];
        Ws[buf][w_k + 0][w_row] = rw.x; Ws[buf][w_k + 1][w_row] = rw.y;
        Ws[buf][w_k + 2][w_row] = rw.z; Ws[buf][w_k + 3][w_row] = rw.w;
    };

    fetch(0);
    stash(0);
    __syncthreads();
    const int nk = K / BK;
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) fetch((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Ws[buf][k][tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (kt + 1 < nk) {
            stash(buf ^ 1);
            __syncthreads();
        }
    }

    const int gn = n0 + tx * 4;
    if (gn >= N) return;
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (bias) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(bias + gn));
        bv[0] = b.x; bv[1] = b.y; bv[2] = b.z; bv[3] = b.w;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int gm = m0 + ty * 8 + i;
        if (gm >= M) break;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            v[j] = acc[i][j] + bv[j];
            if (act == ACT_RELU) v[j] = fmaxf(v[j], 0.f);
        }
        if (residual) {
            const float4 r = __ldg(reinterpret_cast<const float4*>(residual + (size_t)gm * ldr + gn));
            v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
        }
        if constexpr (sizeof(TC) == 4) {
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(C) + (size_t)gm * ldc + gn) =
                make_float4(v[0], v[1], v[2], v[3]);
        } else {
            uint2 u;
            u.x = pack_bf16x2(v[0], v[1]);
            u.y = pack_bf16x2(v[2], v[3]);
            *reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(C) + (size_t)gm * ldc + gn) = u;
        }
    }
}

}  // namespace

template <typename TA, typename TC>
int gemm_simt(const TA* A, int lda, const TA* A2, int lda2, int K1, const float* W, const float* bias,
              const float* residual, int ldr, TC* C, int ldc, int M, int N, int K, int act,
              cudaStream_t stream)
{
    OCC_CHECK(K % BK == 0 && N % 4 == 0, "gemm_simt: K must be a multiple of 16 and N of 4");
    if (A2 == nullptr) { A2 = A; lda2 = lda; K1 = K; }
    OCC_CHECK(K1 % 8 == 0, "gemm_simt: split point must be a multiple of 8");
    if (M == 0) return 0;
    dim3 grid(ceil_div(M, BM), ceil_div(N, BN));
    gemm_simt_kernel<TA, TC><<<grid, 256, 0, stream>>>(A, lda, A2, lda2, K1, W, bias, residual, ldr, C, ldc,
                                                      M, N, K, act);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template int gemm_simt<float, float>(const float*, int, const float*, int, int, const float*, const float*,
                                     const float*, int, float*, int, int, int, int, int, cudaStream_t);
template int gemm_simt<bf16, float>(const bf16*, int, const bf16*, int, int, const float*, const float*,
                                    const float*, int, float*, int, int, int, int, int, cudaStream_t);
template int gemm_simt<bf16, bf16>(const bf16*, int, const bf16*, int, int, const float*, const float*,
                                   const float*, int, bf16*, int, int, int, int, int, cudaStream_t);

}  // namespace occ
