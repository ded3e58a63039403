/* ORACLE (test infrastructure only -- never linked into the product library).
 *
 * Plain-C restatement of the reference's ray-casting kernel in "test" phase:
 *   tools/ray_iou/lib/dvr/dvr.cu:69-319 of the reference tree  (render_forward_cuda_kernel)
 *   host wrapper dvr.cu:329-388 (outputs pre-filled with -1 / 0)
 * One call == one `dvr.render_forward(sigma, origin, points, tindex, grid, "test")`
 * with N == 1.  All traversal arithmetic is double, exactly as in the kernel; inputs
 * and outputs are float (the reference dispatches on sigma's dtype, which is float32
 * at its only call site, datasets/ray_metrics.py:116-123).
 *
 * The kernel records the whole in-grid path and afterwards scans it for the first voxel
 * with sigma > 0.5; here the scan is folded into the walk (first hit wins, later voxels
 * cannot change the result) but the walk still continues to the exit so that `d[count-1]`
 * (the no-hit answer) and the MAX_STEP cut-off behave identically.
 *
 * Parity status: validated on the GPU against the reference kernel itself
 * (oracle/_ref/dvr_ref*.so, built from the reference sources by oracle/build_ref.py).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>

#define MAX_STEP 1000

/* sigma: [T][Z][Y][X] float; origin: [T][3]; points: [M][3]; tindex: [M] float
 * pred_dist, gt_dist: [M]; coord_index: [M][3]                                  */
void oracle_render_forward(const float* sigma, const float* origin, const float* points,
                           const float* tindex, int T, int vzsize, int vysize, int vxsize,
                           int64_t M, float* pred_dist, float* gt_dist, float* coord_index)
{
    for (int64_t c = 0; c < M; ++c) {
        pred_dist[c] = -1.0f; gt_dist[c] = -1.0f;
        coord_index[3 * c + 0] = 0.0f; coord_index[3 * c + 1] = 0.0f; coord_index[3 * c + 2] = 0.0f;
        const float tf = tindex[c];
        if (tf < 0) continue;                                   /* padded point (dvr.cu:102) */
        const int t = (int)tf;                                  /* float used as an index (dvr.cu:94,114) */
        const int ts = (T == 1) ? 0 : t;
        const double xo = origin[3 * t + 0], yo = origin[3 * t + 1], zo = origin[3 * t + 2];
        const double xe = points[3 * c + 0], ye = points[3 * c + 1], ze = points[3 * c + 2];
        int vx = (int)xo, vy = (int)yo, vz = (int)zo;
        const double rx = xe - xo, ry = ye - yo, rz = ze - zo;
        double gt_d = sqrt(rx * rx + ry * ry + rz * rz);
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
        const float* sg = sigma + (int64_t)ts * vzsize * vysize * vxsize;
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
            pred_dist[c] = (float)(hit ? hit_d : last_in_d);
            gt_dist[c] = (float)gt_d;                            /* test phase: not clamped */
            coord_index[3 * c + 0] = (float)(hit ? hx : lx);
            coord_index[3 * c + 1] = (float)(hit ? hy : ly);
            coord_index[3 * c + 2] = (float)(hit ? hz : lz);
        }
    }
}
