/* ORACLE (test infrastructure only -- never linked into the product library).
 *
 * Plain-C restatement of the reference's ray-casting kernel in "test" phase:
 *   tools/ray_iou/lib/dvr/dvr.cu:69-319 of the reference tree  (render_forward_cuda_kernel)
 *   host wrapper dvr.cu:329-388 (outputs pre-filled with -1 / 0)
 * One call == one `dvr.render_forward(sigma, origin, points, tindex, grid, "test")` with the reference's full argument
 * meaning: sigma [N][T][Z][Y][X], origin [N][To][3], points [N][M][K] (K >= 3, columns 0..2 read, as the accessor
 * points[n][c][0..2] reads them), tindex [N][M] (float; negative = padded point).  Ray (n, c) with t = (int)tindex[n][c]
 * starts at origin[n][t] -- indexed through origin's own To -- and walks sigma[n][ts], ts = T == 1 ? 0 : t.  All
 * traversal arithmetic is double, exactly as in the kernel; inputs and outputs are float (the reference dispatches on
 * sigma's dtype, which is float32 at its only call site, datasets/ray_metrics.py:116-123).
 *
 * The kernel records the whole in-grid path and afterwards scans it for the first voxel
 * with sigma > 0.5; here the scan is folded into the walk (first hit wins, later voxels
 * cannot change the result) but the walk still continues to the exit so that `d[count-1]`
 * (the no-hit answer) and the MAX_STEP cut-off behave identically.
 *
 * The norm.  nvcc contracts by default, and both GPU kernels contract rx*rx + ry*ry + rz*rz the same way: the SASS of
 * the reference's render_forward_cuda_kernel<float> (oracle/_ref/dvr_ref.so) and of the product's render_forward_kernel
 * and metric kernels (libocc_b200.so, sm_90a) is DMUL rx*rx, DFMA ry*ry + that, DFMA rz*rz + that, then the correctly
 * rounded DSQRT sequence.  This file is built with -ffp-contract=off, so the same evaluation is spelled out with fma():
 * without it gt_d (and through dx = rx / gt_d every tMax) can differ from the kernels' in the last bit.  The divisions
 * and additions have no contraction to make.
 *
 * Parity status: validated on the GPU against the reference kernel itself
 * (oracle/_ref/dvr_ref*.so, built from the reference sources by oracle/build_ref.py).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>

#define MAX_STEP 1000

/* pred_dist, gt_dist: [N][M]; coord_index: [N][M][3] */
void oracle_render_forward(const float* sigma, const float* origin, const float* points, const float* tindex,
                           int N, int T, int To, int vzsize, int vysize, int vxsize, int64_t M, int K,
                           float* pred_dist, float* gt_dist, float* coord_index)
{
    for (int64_t n = 0; n < N; ++n)
    for (int64_t c = 0; c < M; ++c) {
        const int64_t rc = n * M + c;
        pred_dist[rc] = -1.0f; gt_dist[rc] = -1.0f;
        coord_index[3 * rc + 0] = 0.0f; coord_index[3 * rc + 1] = 0.0f; coord_index[3 * rc + 2] = 0.0f;
        const float tf = tindex[rc];
        if (tf < 0) continue;                                   /* padded point (dvr.cu:105) */
        const int t = (int)tf;                                  /* float used as an index (dvr.cu:94,114) */
        const int ts = (T == 1) ? 0 : t;
        const float* o = origin + (n * To + t) * 3;             /* origin[n][t] (dvr.cu:114-116) */
        const float* p = points + rc * K;                       /* points[n][c] (dvr.cu:119-121) */
        const double xo = o[0], yo = o[1], zo = o[2];
        const double xe = p[0], ye = p[1], ze = p[2];
        int vx = (int)xo, vy = (int)yo, vz = (int)zo;
        const double rx = xe - xo, ry = ye - yo, rz = ze - zo;
        double gt_d = sqrt(fma(rz, rz, fma(ry, ry, rx * rx)));  /* the kernels' contraction, see the header */
        const double dx = rx / gt_d, dy = ry / gt_d, dz = rz / gt_d;
        const int stepX = (dx >= 0) ? 1 : -1, stepY = (dy >= 0) ? 1 : -1, stepZ = (dz >= 0) ? 1 : -1;
        const double nbx = vx + (stepX < 0 ? 0 : 1), nby = vy + (stepY < 0 ? 0 : 1), nbz = vz + (stepZ < 0 ? 0 : 1);
        double tMaxX = (dx != 0) ? (nbx - xo) / dx : DBL_MAX;
        double tMaxY = (dy != 0) ? (nby - yo) / dy : DBL_MAX;
        double tMaxZ = (dz != 0) ? (nbz - zo) / dz : DBL_MAX;
        const double tDeltaX = (dx != 0) ? stepX / dx : DBL_MAX;
        const double tDeltaY = (dy != 0) ? stepY / dy : DBL_MAX;
        const double tDeltaZ = (dz != 0) ? stepZ / dz : DBL_MAX;
        int step = 0, count = 0, was_inside = 0, hit = 0;
        double last_in_d = 0.0, hit_d = 0.0;
        int lx = 0, ly = 0, lz = 0, hx = 0, hy = 0, hz = 0;
        const float* sg = sigma + (n * T + ts) * vzsize * vysize * vxsize;
        while (1) {
            const int inside = (0 <= vx && vx < vxsize) && (0 <= vy && vy < vysize) && (0 <= vz && vz < vzsize);
            const int cx = vx, cy = vy, cz = vz;
            if (inside) was_inside = 1;
            else if (was_inside) break;
            double _d;
            if (tMaxX < tMaxY) {
                if (tMaxX < tMaxZ) { _d = tMaxX; vx += stepX; tMaxX += tDeltaX; }
                else               { _d = tMaxZ; vz += stepZ; tMaxZ += tDeltaZ; }
            } else {
                if (tMaxY < tMaxZ) { _d = tMaxY; vy += stepY; tMaxY += tDeltaY; }
                else               { _d = tMaxZ; vz += stepZ; tMaxZ += tDeltaZ; }
            }
            if (inside) {
                last_in_d = _d; lx = cx; ly = cy; lz = cz;
                if (!hit) {
                    const double occ = sg[((int64_t)cz * vysize + cy) * vxsize + cx];
                    if (occ > 0.5) { hit = 1; hit_d = _d; hx = cx; hy = cy; hz = cz; }
                }
                count++;
            }
            step++;
            if (step > MAX_STEP) break;
        }
        if (count > 0) {
            pred_dist[rc] = (float)(hit ? hit_d : last_in_d);
            gt_dist[rc] = (float)gt_d;                           /* test phase: not clamped */
            coord_index[3 * rc + 0] = (float)(hit ? hx : lx);
            coord_index[3 * rc + 1] = (float)(hit ? hy : ly);
            coord_index[3 * rc + 2] = (float)(hit ? hz : lz);
        }
    }
}
