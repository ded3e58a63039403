// Ray-casting metric for sm_90a (SURVEY rows a14 / a15).
//   render_forward_kernel <- tools/ray_iou/lib/dvr/dvr.cu:69-319 ("test" phase) + host wrapper :329-388
//   ray_metric_kernel     <- datasets/ray_metrics.py process_one_sample :89-143 + calc_metrics :146-189
// The traversal arithmetic is double precision with the reference's comparison order, so voxel
// indices are bit-exact.  The reference walks the whole grid recording a path (52 KB of local
// memory per thread) and scans it afterwards; here the first sigma > 0.5 voxel is latched during
// the walk, which needs no path storage.  The fused kernel casts all T origins x M rays through
// the predicted and the ground-truth volume in one launch and reduces the 187 counters on device.
//   ray_records_kernel    <- datasets/nuscenes_occ.py format_results :230-255: the same rays through the predicted volume only,
//                            written as the challenge file's records (int8 class, fp16 distance, fp16 flow)
//   ray_score_kernel      <- ray_metric_kernel for a frame the engine has just predicted: origins by value, the ground truth
//                            walked first and the prediction only for rays that count
#include <float.h>

#include "common.cuh"
#include "kernels.cuh"

namespace occ {

namespace {

constexpr int MAX_STEP = 1000;

struct Hit { double dist; int x, y, z; bool any; };

// occupied(x,y,z) -> bool.  Returns first-hit (or exit) distance and voxel; any == false when the ray
// never enters the grid (the reference then leaves pred_dist = -1 and coord_index = 0).
template <typename Occ>
__device__ __forceinline__ Hit dda_first_hit(double xo, double yo, double zo, double xe, double ye, double ze,
                                             int vxsize, int vysize, int vzsize, double& gt_d, Occ occupied)
{
    int vx = (int)xo, vy = (int)yo, vz = (int)zo;
    const double rx = xe - xo, ry = ye - yo, rz = ze - zo;
    gt_d = sqrt(rx * rx + ry * ry + rz * rz);
    const double dx = rx / gt_d, dy = ry / gt_d, dz = rz / gt_d;
    const int stepX = (dx >= 0) ? 1 : -1, stepY = (dy >= 0) ? 1 : -1, stepZ = (dz >= 0) ? 1 : -1;
    const double nbx = vx + (stepX < 0 ? 0 : 1), nby = vy + (stepY < 0 ? 0 : 1), nbz = vz + (stepZ < 0 ? 0 : 1);
    double tMaxX = (dx != 0) ? (nbx - xo) / dx : DBL_MAX;
    double tMaxY = (dy != 0) ? (nby - yo) / dy : DBL_MAX;
    double tMaxZ = (dz != 0) ? (nbz - zo) / dz : DBL_MAX;
    const double tDeltaX = (dx != 0) ? stepX / dx : DBL_MAX;
    const double tDeltaY = (dy != 0) ? stepY / dy : DBL_MAX;
    const double tDeltaZ = (dz != 0) ? stepZ / dz : DBL_MAX;
    Hit h; h.dist = 0.0; h.x = h.y = h.z = 0; h.any = false;
    bool was_inside = false, hit = false;
    int step = 0;
    while (true) {
        const bool inside = (0 <= vx && vx < vxsize) && (0 <= vy && vy < vysize) && (0 <= vz && vz < vzsize);
        const int cx = vx, cy = vy, cz = vz;
        if (inside) was_inside = true;
        else if (was_inside) break;
        double d;
        if (tMaxX < tMaxY) {
            if (tMaxX < tMaxZ) { d = tMaxX; vx += stepX; tMaxX += tDeltaX; }
            else               { d = tMaxZ; vz += stepZ; tMaxZ += tDeltaZ; }
        } else {
            if (tMaxY < tMaxZ) { d = tMaxY; vy += stepY; tMaxY += tDeltaY; }
            else               { d = tMaxZ; vz += stepZ; tMaxZ += tDeltaZ; }
        }
        if (inside && !hit) {
            h.any = true; h.dist = d; h.x = cx; h.y = cy; h.z = cz;     // last in-grid voxel so far
            if (occupied(cx, cy, cz)) { hit = true; break; }             // later voxels cannot change the answer
        }
        ++step;
        if (step > MAX_STEP) break;
    }
    return h;
}

__global__ void render_forward_kernel(const float* __restrict__ sigma, const float* __restrict__ origin,
                                      const float* __restrict__ points, const float* __restrict__ tindex, int T,
                                      int vzsize, int vysize, int vxsize, int64_t M, float* __restrict__ pred_dist,
                                      float* __restrict__ gt_dist, float* __restrict__ coord_index)
{
    const int n = blockIdx.y;
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= M) return;
    const int64_t rc = (int64_t)n * M + c;
    pred_dist[rc] = -1.f; gt_dist[rc] = -1.f;
    coord_index[rc * 3] = 0.f; coord_index[rc * 3 + 1] = 0.f; coord_index[rc * 3 + 2] = 0.f;
    const float tf = tindex[rc];
    if (tf < 0) return;
    const int t = (int)tf;
    const int ts = (T == 1) ? 0 : t;
    const float* o = origin + ((int64_t)n * T + t) * 3;
    const float* p = points + rc * 3;
    const float* sg = sigma + ((int64_t)n * T + ts) * vzsize * vysize * vxsize;
    double gt_d;
    const Hit h = dda_first_hit(o[0], o[1], o[2], p[0], p[1], p[2], vxsize, vysize, vzsize, gt_d,
                                [&](int x, int y, int z) {
                                    return (double)sg[((int64_t)z * vysize + y) * vxsize + x] > 0.5;
                                });
    if (h.any) {
        pred_dist[rc] = (float)h.dist;
        gt_dist[rc] = (float)gt_d;
        coord_index[rc * 3] = (float)h.x; coord_index[rc * 3 + 1] = (float)h.y; coord_index[rc * 3 + 2] = (float)h.z;
    }
}

constexpr int NCLS = 17, FREE = 16, NFLOW = 8, NCNT = 11 * NCLS;
constexpr int GX = 200, GY = 200, GZ = 16;

// Voxel-unit origin og / end point en of one metric ray, exactly as ray_metrics.py:102-112.  torch type promotion: with the
// dataset's float64 origins (ego_pose_extractor.py:108-119) the arithmetic is double and rounded once by `.float()`; with
// float32 origins (o holds their exact values) every step is fp32.
__device__ __forceinline__ void voxel_ray(const double (&o)[3], int origin_is_f64, const float* __restrict__ ray,
                                          float (&og)[3], float (&en)[3])
{
    const float off[3] = {-40.f, -40.f, -1.f};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (origin_is_f64) {
            const double e = (double)ray[k] + o[k];
            og[k] = (float)((o[k] - (double)off[k]) / (double)0.4f);
            en[k] = (float)((e - (double)off[k]) / (double)0.4f);
        } else {
            const float of = (float)o[k];
            const float e = __fadd_rn(ray[k], of);
            og[k] = __fdiv_rn(__fsub_rn(of, off[k]), 0.4f);
            en[k] = __fdiv_rn(__fsub_rn(e, off[k]), 0.4f);
        }
    }
}

// process_one_sample's row of one ray through one volume: {class, distance in metres, flow x, flow y} of the first occupied
// voxel; the exit voxel for a ray that hits nothing, voxel (0,0,0) and -0.4 m for a ray that never enters the grid
__device__ __forceinline__ void ray_row(const uint8_t* __restrict__ sem, const float* __restrict__ flow, const float (&og)[3],
                                        const float (&en)[3], float (&row)[4])
{
    double gt_d;
    const Hit h = dda_first_hit(og[0], og[1], og[2], en[0], en[1], en[2], GX, GY, GZ, gt_d,
                                [&](int x, int y, int z) { return sem[((int64_t)x * GY + y) * GZ + z] != FREE; });
    const int64_t vi = ((int64_t)h.x * GY + h.y) * GZ + h.z;
    row[0] = (float)sem[vi]; row[1] = (h.any ? (float)h.dist : -1.f) * 0.4f; row[2] = flow[vi * 2]; row[3] = flow[vi * 2 + 1];
}

// calc_metrics' update for one ray (ray_metrics.py:146-189, 218-220) from its predicted and ground-truth rows, into the CTA's
// shared counters
__device__ __forceinline__ void score_ray(double* s_cnt, const float (&pred)[4], const float (&gt)[4])
{
    const int cp = (int)pred[0], cg = (int)gt[0];
    if (cg != FREE) {                                                  // ray_metrics.py:218-220
        if (cg < NCLS) atomicAdd(&s_cnt[cg], 1.0);
        if (cp < NCLS) atomicAdd(&s_cnt[NCLS + cp], 1.0);
        if (cg == cp && cg < NCLS) {
            const float l1 = fabsf(pred[1] - gt[1]);
            const float fx = gt[2] - pred[2], fy = gt[3] - pred[3];
            const float err = sqrtf(fx * fx + fy * fy);
            const float thr[3] = {1.f, 2.f, 4.f};
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                if (l1 < thr[j]) {
                    atomicAdd(&s_cnt[2 * NCLS + j * NCLS + cg], 1.0);
                    if (cg < NFLOW) {
                        atomicAdd(&s_cnt[5 * NCLS + j * NCLS + cg], (double)err);
                        atomicAdd(&s_cnt[8 * NCLS + j * NCLS + cg], 1.0);
                    }
                }
            }
        }
    }
}

// one thread = one (origin t, ray m); casts through pred and gt, updates the counters
__global__ void __launch_bounds__(128)
ray_metric_kernel(const uint8_t* __restrict__ sem_pred, const float* __restrict__ flow_pred,
                  const uint8_t* __restrict__ sem_gt, const float* __restrict__ flow_gt,
                  const void* __restrict__ origins, int origin_is_f64, int T, const float* __restrict__ rays,
                  int M, double* __restrict__ counters, float* __restrict__ pcd_pred, float* __restrict__ pcd_gt)
{
    __shared__ double s_cnt[NCNT];
    for (int i = threadIdx.x; i < NCNT; i += blockDim.x) s_cnt[i] = 0.0;
    __syncthreads();
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < (int64_t)T * M) {
        const int t = (int)(idx / M), m = (int)(idx % M);
        const double* od = reinterpret_cast<const double*>(origins) + t * 3;
        const float* of = reinterpret_cast<const float*>(origins) + t * 3;
        const double o[3] = {origin_is_f64 ? od[0] : (double)of[0], origin_is_f64 ? od[1] : (double)of[1],
                             origin_is_f64 ? od[2] : (double)of[2]};
        float og[3], en[3];
        voxel_ray(o, origin_is_f64, rays + m * 3, og, en);
        float row[2][4];
        ray_row(sem_pred, flow_pred, og, en, row[0]);
        ray_row(sem_gt, flow_gt, og, en, row[1]);
        if (pcd_pred) *reinterpret_cast<float4*>(pcd_pred + idx * 4) = make_float4(row[0][0], row[0][1], row[0][2], row[0][3]);
        if (pcd_gt) *reinterpret_cast<float4*>(pcd_gt + idx * 4) = make_float4(row[1][0], row[1][1], row[1][2], row[1][3]);
        score_ray(s_cnt, row[0], row[1]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < NCNT; i += blockDim.x)
        if (s_cnt[i] != 0.0) atomicAdd(&counters[i], s_cnt[i]);
}

// ray_metric_kernel's counters for the volumes a frame has just predicted.  The origins arrive by value, so a frame uploads
// none.  The ground truth is walked first: a ray whose ground-truth row is `free` adds to no counter (ray_metrics.py:218-220),
// so its walk through the prediction is skipped -- the metric's upward rays, a large share of a real scene.
__global__ void __launch_bounds__(128)
ray_score_kernel(const uint8_t* __restrict__ sem_pred, const float* __restrict__ flow_pred,
                 const uint8_t* __restrict__ sem_gt, const float* __restrict__ flow_gt, const RayOrigins org,
                 const float* __restrict__ rays, int M, double* __restrict__ counters)
{
    __shared__ double s_cnt[NCNT];
    for (int i = threadIdx.x; i < NCNT; i += blockDim.x) s_cnt[i] = 0.0;
    __syncthreads();
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < (int64_t)org.T * M) {
        const int t = (int)(idx / M), m = (int)(idx % M);
        const double o[3] = {org.o[t][0], org.o[t][1], org.o[t][2]};
        float og[3], en[3], gt[4];
        voxel_ray(o, org.is_f64, rays + m * 3, og, en);
        ray_row(sem_gt, flow_gt, og, en, gt);
        if ((int)gt[0] != FREE) {
            float pred[4];
            ray_row(sem_pred, flow_pred, og, en, pred);
            score_ray(s_cnt, pred, gt);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < NCNT; i += blockDim.x)
        if (s_cnt[i] != 0.0) atomicAdd(&counters[i], s_cnt[i]);
}

// numpy's astype(np.float16) of a float32: round to nearest even, overflow to inf; a NaN keeps its sign and the top ten
// payload bits (cvt.rn.f16.f32 would give the canonical NaN 0x7fff instead, and the file would differ in those bytes)
__device__ __forceinline__ uint16_t half_bits(float v)
{
    if (v != v) {
        const uint32_t u = __float_as_uint(v);
        uint16_t h = (uint16_t)(0x7c00u | ((u & 0x007fffffu) >> 13));
        if (h == 0x7c00u) h = 0x7c01u;                                  // the payload was all in the dropped bits
        return (uint16_t)(h | ((u >> 16) & 0x8000u));
    }
    return __half_as_ushort(__float2half_rn(v));
}

// one thread = one (origin t, ray m): one walk through the predicted volume, one record
__global__ void __launch_bounds__(128)
ray_records_kernel(const uint8_t* __restrict__ sem, const float* __restrict__ flow, const RayOrigins org,
                   const float* __restrict__ rays, int M, int8_t* __restrict__ pcd_cls, uint16_t* __restrict__ pcd_dist,
                   uint16_t* __restrict__ pcd_flow)
{
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)org.T * M) return;
    const int t = (int)(idx / M), m = (int)(idx % M);
    const double o[3] = {org.o[t][0], org.o[t][1], org.o[t][2]};
    float og[3], en[3];
    voxel_ray(o, org.is_f64, rays + m * 3, og, en);
    double gt_d;
    const Hit h = dda_first_hit(og[0], og[1], og[2], en[0], en[1], en[2], GX, GY, GZ, gt_d,
                                [&](int x, int y, int z) { return sem[((int64_t)x * GY + y) * GZ + z] != FREE; });
    const float dist = (h.any ? (float)h.dist : -1.f) * 0.4f;
    const int64_t vi = ((int64_t)h.x * GY + h.y) * GZ + h.z;           // voxel (0,0,0) for a ray that never enters
    pcd_cls[idx] = (int8_t)sem[vi];
    pcd_dist[idx] = half_bits(dist);
    pcd_flow[idx * 2] = half_bits(flow[vi * 2]);
    pcd_flow[idx * 2 + 1] = half_bits(flow[vi * 2 + 1]);
}

}  // namespace

int launch_render_forward(const float* sigma, const float* origin, const float* points, const float* tindex,
                          int N, int T, int Z, int Y, int X, int64_t M, float* pred_dist, float* gt_dist,
                          float* coord_index, cudaStream_t stream)
{
    if (N == 0 || M == 0) return 0;
    dim3 grid(ceil_div(M, 128), N);
    render_forward_kernel<<<grid, 128, 0, stream>>>(sigma, origin, points, tindex, T, Z, Y, X, M, pred_dist, gt_dist,
                                                    coord_index);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

int launch_ray_metric(const uint8_t* sem_pred, const float* flow_pred, const uint8_t* sem_gt, const float* flow_gt,
                      const void* origins, int origin_is_f64, int T, const float* rays, int M, double* counters,
                      float* pcd_pred, float* pcd_gt, cudaStream_t stream)
{
    if (T == 0 || M == 0) return 0;
    ray_metric_kernel<<<ceil_div((int64_t)T * M, 128), 128, 0, stream>>>(sem_pred, flow_pred, sem_gt, flow_gt, origins,
                                                                        origin_is_f64, T, rays, M, counters, pcd_pred,
                                                                        pcd_gt);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

int launch_ray_score(const uint8_t* sem_pred, const float* flow_pred, const uint8_t* sem_gt, const float* flow_gt,
                     const RayOrigins& org, const float* rays, int M, double* counters, cudaStream_t stream)
{
    if (org.T == 0 || M == 0) return 0;
    ray_score_kernel<<<ceil_div((int64_t)org.T * M, 128), 128, 0, stream>>>(sem_pred, flow_pred, sem_gt, flow_gt, org, rays, M,
                                                                           counters);
    OCC_CUDA(cudaGetLastError());
    return 0;
}

int launch_ray_records(const uint8_t* sem, const float* flow, const RayOrigins& org, const float* rays, int M, int8_t* pcd_cls,
                       void* pcd_dist, void* pcd_flow, cudaStream_t stream)
{
    if (org.T == 0 || M == 0) return 0;
    ray_records_kernel<<<ceil_div((int64_t)org.T * M, 128), 128, 0, stream>>>(
        sem, flow, org, rays, M, pcd_cls, reinterpret_cast<uint16_t*>(pcd_dist), reinterpret_cast<uint16_t*>(pcd_flow));
    OCC_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace occ
