// Memory-bound glue kernels of the path: camera-feature packing (transformer_occ.py:207-227),
// BEV positional encoding (mmdet LearnedPositionalEncoding), LayerNorm (encoder norms), casts.
#include "common.cuh"
#include "kernels.cuh"

namespace occ {

namespace {

// [cam][C][hw] f32 -> [cam][Nv][C] T (+ cams_embeds[cam][c], then + level_embed[c]; same order as the reference).
// 64 (pixels) x 64 (channels) tile per CTA: float4 reads along the pixel axis, 16-byte (8 x bf16) writes along C.
// All FPN levels in one launch: blockIdx.x walks the 64-pixel tiles of level 0, then level 1, ...
template <typename T, typename TI>
__global__ void __launch_bounds__(256)
pack_levels_kernel(PackLevels pl, const float* __restrict__ cams_embeds, const float* __restrict__ level_embeds, int C,
                   int Nv, T* __restrict__ tokens)
{
    // fp32 features: [channel][pixel] fp32 tile, padded.  bf16 features (the throughput configuration): the transpose is done on
    // the 16-bit values -- [pixel][channel] bf16 tile, 8-channel groups XOR-swizzled by pixel/8: 2-byte stores on the way in,
    // ONE 16-byte load per 8 output channels on the way out, both conflict-free (the fp32 tile made this kernel shared-memory
    // bound: L1 data pipe 85 %, 63 us for 189 MB)
    constexpr bool BF = sizeof(TI) == 2;
    __shared__ float tile[BF ? 1 : 64][BF ? 1 : 65];
    __shared__ __align__(16) bf16 tileb[BF ? 64 * 64 : 8];
    int lvl = 0;
#pragma unroll
    for (int l = 1; l < 8; ++l) if (l < pl.num_levels && (int)blockIdx.x >= pl.tile_begin[l]) lvl = l;
    const void* feat_v = nullptr; int hw = 0, start = 0, tb = 0;
#pragma unroll
    for (int l = 0; l < 8; ++l)                                // static selects (no dynamically indexed parameter copy)
        if (l == lvl) { feat_v = pl.feat[l]; hw = pl.hw[l]; start = pl.start[l]; tb = pl.tile_begin[l]; }
    const TI* feat = reinterpret_cast<const TI*>(feat_v);
    const float* level_embed = level_embeds + lvl * C;
    const int cam = blockIdx.z;
    const int p0 = ((int)blockIdx.x - tb) * 64, c0 = blockIdx.y * 64;
    const int tid = threadIdx.x;
    const TI* src = feat + (int64_t)cam * C * hw;
    if constexpr (sizeof(TI) == 4) {
        const bool vec_ok = (hw & 3) == 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {                          // 64 channels x 16 float4 = 1024 float4, 4 per thread
            const int idx = tid + i * 256;
            const int c = idx >> 4, p4 = (idx & 15) * 4;
            const float* sp = src + (int64_t)(c0 + c) * hw + p0 + p4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (vec_ok && p0 + p4 + 3 < hw) v = __ldg(reinterpret_cast<const float4*>(sp));
            else {
                if (p0 + p4 + 0 < hw) v.x = __ldg(sp + 0);
                if (p0 + p4 + 1 < hw) v.y = __ldg(sp + 1);
                if (p0 + p4 + 2 < hw) v.z = __ldg(sp + 2);
                if (p0 + p4 + 3 < hw) v.w = __ldg(sp + 3);
            }
            tile[c][p4 + 0] = v.x; tile[c][p4 + 1] = v.y; tile[c][p4 + 2] = v.z; tile[c][p4 + 3] = v.w;
        }
    } else {                                                   // bf16 features (what an on-device backbone hands over)
        const bool vec_ok = (hw & 7) == 0;
#pragma unroll
        for (int i = 0; i < 2; ++i) {                          // 64 channels x 8 uint4 (8 pixels each), 2 per thread
            const int idx = tid + i * 256;
            const int c = idx >> 3, p8 = (idx & 7) * 8;
            const bf16* sp = src + (int64_t)(c0 + c) * hw + p0 + p8;
            bf16 v[8];
            if (vec_ok && p0 + p8 + 7 < hw) *reinterpret_cast<uint4*>(v) = __ldg(reinterpret_cast<const uint4*>(sp));
            else {
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = (p0 + p8 + k < hw) ? sp[k] : __float2bfloat16(0.f);
            }
            const int gp = p8 >> 3;                               // = pixel / 8 for all 8 pixels of this thread
#pragma unroll
            for (int k = 0; k < 8; ++k) tileb[(p8 + k) * 64 + ((((c >> 3) ^ gp) << 3) | (c & 7))] = v[k];
        }
    }
    __syncthreads();
    if constexpr (BF) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {                          // 64 pixels x 8 channel-octets = 512 stores, 2 per thread
            const int idx = tid + i * 256;
            const int p = idx >> 3, c8 = (idx & 7) * 8;
            if (p0 + p < hw) {
                const uint4 raw = *reinterpret_cast<const uint4*>(&tileb[p * 64 + (((c8 >> 3) ^ (p >> 3)) << 3)]);
                const bf16* xb = reinterpret_cast<const bf16*>(&raw);
                float v[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    float x = __bfloat162float(xb[k]);
                    if (cams_embeds) x = x + cams_embeds[cam * C + c0 + c8 + k];
                    v[k] = x + level_embed[c0 + c8 + k];
                }
                store8(tokens + ((int64_t)cam * Nv + start + p0 + p) * C + c0 + c8, v);
            }
        }
        return;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {                              // 64 pixels x 8 channel-octets = 512 stores, 2 per thread
        const int idx = tid + i * 256;
        const int p = idx >> 3, c8 = (idx & 7) * 8;
        if (p0 + p < hw) {
            float v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float x = tile[c8 + k][p];
                if (cams_embeds) x = x + cams_embeds[cam * C + c0 + c8 + k];
                v[k] = x + level_embed[c0 + c8 + k];
            }
            store8(tokens + ((int64_t)cam * Nv + start + p0 + p) * C + c0 + c8, v);
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
layernorm256_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                    const float* __restrict__ pos, int rows, float* __restrict__ y_f32, T* __restrict__ y_t,
                    T* __restrict__ y_pos_t)
{
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float* xr = x + (int64_t)row * 256 + lane * 8;
    float v[8];
    load8(xr, v);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += v[i];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.f / 256.f);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float d = v[i] - mean; ss = fmaf(d, d, ss); }
#pragma unroll
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss * (1.f / 256.f) + 1e-5f);
    float g[8], b[8], y[8];
    load8(gamma + lane * 8, g);
    load8(beta + lane * 8, b);
#pragma unroll
    for (int i = 0; i < 8; ++i) y[i] = (v[i] - mean) * rstd * g[i] + b[i];
    const int64_t o = (int64_t)row * 256 + lane * 8;
    if (y_f32) store8(y_f32 + o, y);
    if (y_t) store8(y_t + o, y);
    if (y_pos_t) {
        float pv[8];
        load8(pos + o, pv);
#pragma unroll
        for (int i = 0; i < 8; ++i) pv[i] += y[i];
        store8(y_pos_t + o, pv);
    }
}

// "T32" layout of a [rows, 256] fp32 matrix used for the residual stream on the tensor-core path: 32x32 blocks,
// inside a block [piece j = (col%32)/4][row%32][4 floats].  A thread that owns one ROW of a tile (the shape
// of the LayerNorm rows) then reads / writes 16 bytes per instruction with the 32 lanes of a warp contiguous.
__device__ __forceinline__ int64_t t32_index(int64_t row, int col)
{
    return ((((row >> 5) * 8 + (col >> 5)) * 8 + ((col & 31) >> 2)) * 32 + (row & 31)) * 4 + (col & 3);
}

template <typename T>
__global__ void prepare_query_kernel(const float* __restrict__ q, const float* __restrict__ pos, int64_t n8,
                                     float* __restrict__ q_f32, T* __restrict__ q_t, T* __restrict__ q_pos_t, int tiled)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n8) return;
    float v[8], p[8];
    load8(q + i * 8, v);
    load8(pos + i * 8, p);
    if (q_f32 && tiled) {
        const int64_t row = (i * 8) >> 8; const int col = (int)((i * 8) & 255);
        *reinterpret_cast<float4*>(q_f32 + t32_index(row, col)) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(q_f32 + t32_index(row, col + 4)) = make_float4(v[4], v[5], v[6], v[7]);
    } else
    if (q_f32) store8(q_f32 + i * 8, v);
    if (q_t) store8(q_t + i * 8, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) p[k] += v[k];
    if (q_pos_t) store8(q_pos_t + i * 8, p);
}

__global__ void bev_pos_kernel(const float* __restrict__ row_embed, const float* __restrict__ col_embed, int bev_h,
                               int bev_w, int half, float* __restrict__ pos)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int C = 2 * half;
    if (i >= (int64_t)bev_h * bev_w * C) return;
    const int c = (int)(i % C);
    const int q = (int)(i / C);
    const int x = q % bev_w, y = q / bev_w;
    pos[i] = (c < half) ? col_embed[x * half + c] : row_embed[y * half + (c - half)];
}

// row-major [rows,ncols] <-> T32 (dir 0: tile, 1: untile); one thread per 4 floats; ncols a multiple of 32 (256: the residual stream)
__global__ void t32_convert_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t rows, int dir, int ncols)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int q4 = ncols >> 2;
    if (i >= rows * q4) return;
    const int64_t row = i / q4; const int col = (int)(i % q4) * 4;
    const int64_t a = row * ncols + col;
    const int64_t b = ((((row >> 5) * (ncols >> 5) + (col >> 5)) * 8 + ((col & 31) >> 2)) * 32 + (row & 31)) * 4 + (col & 3);
    if (dir == 0) *reinterpret_cast<float4*>(dst + b) = __ldg(reinterpret_cast<const float4*>(src + a));
    else          *reinterpret_cast<float4*>(dst + a) = __ldg(reinterpret_cast<const float4*>(src + b));
}

template <typename T>
__global__ void cast_kernel(const float* __restrict__ s, T* __restrict__ d, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) d[i] = from_f32<T>(s[i]);
}

}  // namespace

template <typename T>
int launch_pack_levels(const void* const* feats, int feats_bf16, const LevelGeom& lg, const float* cams_embeds,
                       const float* level_embeds, int num_cams, int C, int Nv, T* tokens, cudaStream_t stream)
{
    OCC_CHECK(C % 64 == 0, "pack_levels: C must be a multiple of 64");
    OCC_CHECK(lg.num_levels >= 1 && lg.num_levels <= 8, "pack_levels: 1..8 levels");
    PackLevels pl{};
    pl.num_levels = lg.num_levels;
    int tiles = 0;
    for (int l = 0; l < lg.num_levels; ++l) {
        pl.feat[l] = feats[l]; pl.hw[l] = lg.h[l] * lg.w[l]; pl.start[l] = lg.start[l]; pl.tile_begin[l] = tiles;
        tiles += ceil_div(pl.hw[l], 64);
    }
    dim3 grid(tiles, C / 64, num_cams);
    if (feats_bf16) pack_levels_kernel<T, bf16><<<grid, 256, 0, stream>>>(pl, cams_embeds, level_embeds, C, Nv, tokens);
    else            pack_levels_kernel<T, float><<<grid, 256, 0, stream>>>(pl, cams_embeds, level_embeds, C, Nv, tokens);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
template int launch_pack_levels<float>(const void* const*, int, const LevelGeom&, const float*, const float*, int, int, int,
                                       float*, cudaStream_t);
template int launch_pack_levels<bf16>(const void* const*, int, const LevelGeom&, const float*, const float*, int, int, int,
                                      bf16*, cudaStream_t);

template <typename T>
int launch_layernorm(const float* x, const float* gamma, const float* beta, const float* pos, int rows, int C,
                     float* y_f32, T* y_t, T* y_pos_t, cudaStream_t stream)
{
    OCC_CHECK(C == 256, "layernorm: embed_dims must be 256");
    layernorm256_kernel<T><<<ceil_div(rows, 8), 256, 0, stream>>>(x, gamma, beta, pos, rows, y_f32, y_t, y_pos_t);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
template int launch_layernorm<float>(const float*, const float*, const float*, const float*, int, int, float*,
                                     float*, float*, cudaStream_t);
template int launch_layernorm<bf16>(const float*, const float*, const float*, const float*, int, int, float*, bf16*,
                                    bf16*, cudaStream_t);

template <typename T>
int launch_prepare_query(const float* bev_queries, const float* pos, int64_t n, float* q_f32, T* q_t, T* q_pos_t,
                         int tiled, cudaStream_t stream)
{
    OCC_CHECK(n % 8 == 0, "prepare_query: size must be a multiple of 8");
    prepare_query_kernel<T><<<ceil_div(n / 8, 256), 256, 0, stream>>>(bev_queries, pos, n / 8, q_f32, q_t, q_pos_t, tiled);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
template int launch_prepare_query<float>(const float*, const float*, int64_t, float*, float*, float*, int, cudaStream_t);
template int launch_prepare_query<bf16>(const float*, const float*, int64_t, float*, bf16*, bf16*, int, cudaStream_t);

int launch_bev_pos(const float* row_embed, const float* col_embed, int bev_h, int bev_w, int half, float* pos,
                   cudaStream_t stream)
{
    const int64_t n = (int64_t)bev_h * bev_w * 2 * half;
    bev_pos_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(row_embed, col_embed, bev_h, bev_w, half, pos);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

int launch_t32_convert(const float* src, float* dst, int64_t rows, int untile, cudaStream_t stream, int ncols)
{
    OCC_CHECK(ncols > 0 && ncols % 32 == 0, "t32_convert: ncols must be a multiple of 32");
    t32_convert_kernel<<<ceil_div(rows * (ncols / 4), 256), 256, 0, stream>>>(src, dst, rows, untile, ncols);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

template <typename T>
int launch_cast(const float* src, T* dst, int64_t n, cudaStream_t stream)
{
    cast_kernel<T><<<ceil_div(n, 256), 256, 0, stream>>>(src, dst, n);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
template int launch_cast<float>(const float*, float*, int64_t, cudaStream_t);
template int launch_cast<bf16>(const float*, bf16*, int64_t, cudaStream_t);

}  // namespace occ

#include "gemm_tc.cuh"
namespace occ {
namespace {
__global__ void bf16_to_f32_kernel(const bf16* __restrict__ s, float* __restrict__ d, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) d[i] = __bfloat162float(s[i]);
}
}  // namespace
int launch_bf16_to_f32(const bf16* src, float* dst, int64_t n, cudaStream_t stream)
{
    bf16_to_f32_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(src, dst, n);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
}  // namespace occ

// ---- bf16 split of fp32 GEMM operands (fp32-grade tensor-core configuration): x = hi + lo + O(2^-17 |x|)
namespace occ {
namespace {
// one thread = 8 consecutive elements of one source row; Ka, Kb multiples of 8
__global__ void split_bf16_kernel(const float* __restrict__ a, int Ka, const float* __restrict__ b, int Kb, int64_t rows,
                                  bf16* __restrict__ S)
{
    const int K = Ka + Kb, per_row = K >> 3;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * per_row) return;
    const int64_t r = i / per_row;
    const int c = (int)(i % per_row) * 8;
    const float* src = c < Ka ? a + r * Ka + c : b + r * Kb + (c - Ka);
    float v[8], hi[8], lo[8];
    load8(src, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float h = __bfloat162float(__float2bfloat16_rn(v[k]));
        hi[k] = h; lo[k] = v[k] - h;                           // exact in fp32 (Sterbenz-style: |lo| <= 2^-9 |x|)
    }
    bf16* row = S + r * (2 * (int64_t)K);
    store8(row + c, hi);
    store8(row + K + c, lo);
}
}  // namespace
int launch_split_bf16(const float* a, int Ka, const float* b, int Kb, int64_t rows, bf16* S, cudaStream_t stream)
{
    OCC_CHECK(a && Ka % 8 == 0 && Kb % 8 == 0 && (Kb == 0 || b), "split_bf16: operands must be multiples of 8 wide");
    const int64_t n = rows * ((Ka + Kb) >> 3);
    if (n == 0) return 0;
    split_bf16_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(a, Ka, b, Kb, rows, S);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
}  // namespace occ

// ---- prev_bev rotation as a row gather (transformer_occ.py:195-205: torchvision `rotate`, nearest, zero fill): the host
//      hands over the index map source_row[q] (-1 = outside), or the rotation's six grid coefficients from which every
//      thread computes its source row; this kernel applies it while producing the GEMM operand copy
namespace occ {
namespace {
// Source cell of BEV cell q under the rotation `g`, or -1 outside: torchvision's rotate(center=...) with nearest
// interpolation, operation for operation (_gen_affine_grid + grid_sample(align_corners=False, padding_mode='zeros')):
//   base grid  x = j - W/2 + 0.5, y = i - H/2 + 0.5                  (half-integers: exact in fp32)
//   grid       g = (x * r0 + y * r1) + r2 with the y term fused       (the rounding torch's CPU bmm produces)
//   unnormalise ix = ((g_x + 1) * W - 1) / 2, iy alike with H
//   nearest    rint (half to even), cells outside the image read the zero fill.
// Every step is an explicitly rounded intrinsic, so -fmad cannot contract a different rounding into it.
__device__ __forceinline__ int rotation_source(int q, const RotGrid& g)
{
    const int i = q / g.bev_w, j = q - i * g.bev_w;
    const float x = 0.5f * (float)(2 * j - g.bev_w + 1), y = 0.5f * (float)(2 * i - g.bev_h + 1);
    const float gx = __fadd_rn(__fmaf_rn(y, g.r[1], __fmul_rn(x, g.r[0])), g.r[2]);
    const float gy = __fadd_rn(__fmaf_rn(y, g.r[4], __fmul_rn(x, g.r[3])), g.r[5]);
    const float ix = rintf(__fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)g.bev_w), 1.f), 2.f));
    const float iy = rintf(__fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)g.bev_h), 1.f), 2.f));
    if (!(ix >= 0.f && ix < (float)g.bev_w && iy >= 0.f && iy < (float)g.bev_h)) return -1;
    return (int)iy * g.bev_w + (int)ix;
}

// kGrid: source rows from rotation_source(grid); otherwise from `map` (host-checked, NULL = identity)
template <typename T, bool kGrid>
__global__ void gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ map, RotGrid grid, int rows,
                                   int C, T* __restrict__ dst, float* __restrict__ dst_f32)
{
    const int per_row = C >> 3;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)rows * per_row) return;
    const int r = (int)(i / per_row), c = (int)(i % per_row) * 8;
    const int sr = kGrid ? rotation_source(r, grid) : (map ? map[r] : r);
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (sr >= 0) load8(src + (int64_t)sr * C + c, v);
    if (dst) store8(dst + (int64_t)r * C + c, v);
    if (dst_f32) store8(dst_f32 + (int64_t)r * C + c, v);
}

__global__ void rotation_map_kernel(RotGrid grid, int rows, int32_t* __restrict__ map)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < rows) map[q] = rotation_source(q, grid);
}
}  // namespace
template <typename T>
int launch_gather_rows(const float* src, const int32_t* map, const RotGrid* grid, int rows, int C, T* dst, float* dst_f32,
                       cudaStream_t stream)
{
    OCC_CHECK(C % 8 == 0, "gather_rows: C must be a multiple of 8");
    OCC_CHECK(grid == nullptr || grid->bev_h * grid->bev_w == rows, "gather_rows: rotation grid size != rows");
    const int64_t n = (int64_t)rows * (C >> 3);
    if (grid)
        gather_rows_kernel<T, true><<<ceil_div(n, 256), 256, 0, stream>>>(src, nullptr, *grid, rows, C, dst, dst_f32);
    else
        gather_rows_kernel<T, false><<<ceil_div(n, 256), 256, 0, stream>>>(src, map, RotGrid{}, rows, C, dst, dst_f32);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
template int launch_gather_rows<float>(const float*, const int32_t*, const RotGrid*, int, int, float*, float*, cudaStream_t);
template int launch_gather_rows<bf16>(const float*, const int32_t*, const RotGrid*, int, int, bf16*, float*, cudaStream_t);

int launch_rotation_map(const RotGrid& grid, int32_t* map, cudaStream_t stream)
{
    const int rows = grid.bev_h * grid.bev_w;
    if (rows == 0) return 0;
    rotation_map_kernel<<<ceil_div(rows, 256), 256, 0, stream>>>(grid, rows, map);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

// ---- the same rotation from the engine-owned BEV history, already in the storage type: a pure row permutation (16 bytes
//      per thread, no conversion).  The map may come straight from the caller's device memory, so an entry outside
//      [-1, rows) reads as -1 (zeros) instead of out of bounds.
namespace {
// kGrid: source rows from rotation_source(grid) instead of the map
template <bool kGrid>
__global__ void gather_rows16_kernel(const uint4* __restrict__ src, const int32_t* __restrict__ map, RotGrid grid, int rows,
                                     int per_row, uint4* __restrict__ dst)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)rows * per_row) return;
    const int r = (int)(i / per_row), c = (int)(i % per_row);
    const int sr = kGrid ? rotation_source(r, grid) : (map ? __ldg(map + r) : r);
    dst[i] = (sr >= 0 && sr < rows) ? __ldg(src + (int64_t)sr * per_row + c) : make_uint4(0u, 0u, 0u, 0u);
}
}  // namespace
template <typename T>
int launch_gather_rows_stored(const T* src, const int32_t* map, const RotGrid* grid, int rows, int C, T* dst,
                              cudaStream_t stream)
{
    OCC_CHECK((C * sizeof(T)) % 16 == 0, "gather_rows_stored: rows must be a multiple of 16 bytes");
    OCC_CHECK(grid == nullptr || grid->bev_h * grid->bev_w == rows, "gather_rows_stored: rotation grid size != rows");
    const int per_row = (int)(C * sizeof(T) / 16);
    const int64_t n = (int64_t)rows * per_row;
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(dst);
    if (grid)
        gather_rows16_kernel<true><<<ceil_div(n, 256), 256, 0, stream>>>(s, nullptr, *grid, rows, per_row, d);
    else
        gather_rows16_kernel<false><<<ceil_div(n, 256), 256, 0, stream>>>(s, map, RotGrid{}, rows, per_row, d);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
template int launch_gather_rows_stored<float>(const float*, const int32_t*, const RotGrid*, int, int, float*, cudaStream_t);
template int launch_gather_rows_stored<bf16>(const bf16*, const int32_t*, const RotGrid*, int, int, bf16*, cudaStream_t);
}  // namespace occ

// ---- feature packing from channels-last bf16 levels [num_cams, h, w, C] (what occb200_backbone_forward_nhwc_bf16 writes):
//      no transpose left -- tokens[cam][start_l + p][:] = feat_l[cam][p][:] + cams_embeds[cam] + level_embeds[l]
namespace occ {
namespace {
template <typename T>
__global__ void __launch_bounds__(256)
pack_levels_nhwc_kernel(PackLevels pl, const float* __restrict__ cams_embeds, const float* __restrict__ level_embeds, int C,
                        int Nv, int num_cams, T* __restrict__ tokens)
{
    const int per_row = C >> 3;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)num_cams * Nv * per_row) return;
    const int c8 = (int)(i % per_row) * 8;
    const int64_t row = i / per_row;                            // cam * Nv + token
    const int cam = (int)(row / Nv), tok = (int)(row % Nv);
    int lvl = 0;
#pragma unroll
    for (int l = 1; l < 8; ++l) if (l < pl.num_levels && tok >= pl.start[l]) lvl = l;
    const void* feat_v = nullptr; int hw = 0, start = 0;
#pragma unroll
    for (int l = 0; l < 8; ++l) if (l == lvl) { feat_v = pl.feat[l]; hw = pl.hw[l]; start = pl.start[l]; }
    const bf16* src = reinterpret_cast<const bf16*>(feat_v) + ((int64_t)cam * hw + (tok - start)) * C + c8;
    float v[8];
    load8(src, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        float x = v[k];
        if (cams_embeds) x = x + cams_embeds[cam * C + c8 + k];
        v[k] = x + level_embeds[lvl * C + c8 + k];
    }
    store8(tokens + row * C + c8, v);
}
}  // namespace
template <typename T>
int launch_pack_levels_nhwc(const void* const* feats, const LevelGeom& lg, const float* cams_embeds, const float* level_embeds,
                            int num_cams, int C, int Nv, T* tokens, cudaStream_t stream)
{
    OCC_CHECK(C % 8 == 0 && lg.num_levels >= 1 && lg.num_levels <= 8, "pack_levels_nhwc: C % 8, 1..8 levels");
    PackLevels pl{};
    pl.num_levels = lg.num_levels;
    for (int l = 0; l < lg.num_levels; ++l) { pl.feat[l] = feats[l]; pl.hw[l] = lg.h[l] * lg.w[l]; pl.start[l] = lg.start[l]; }
    const int64_t n = (int64_t)num_cams * Nv * (C >> 3);
    pack_levels_nhwc_kernel<T><<<ceil_div(n, 256), 256, 0, stream>>>(pl, cams_embeds, level_embeds, C, Nv, num_cams, tokens);
    OCC_CUDA(cudaGetLastError());
    return 0;
}
template int launch_pack_levels_nhwc<float>(const void* const*, const LevelGeom&, const float*, const float*, int, int, int, float*,
                                            cudaStream_t);
template int launch_pack_levels_nhwc<bf16>(const void* const*, const LevelGeom&, const float*, const float*, int, int, int, bf16*,
                                           cudaStream_t);
}  // namespace occ
