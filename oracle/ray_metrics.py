"""ORACLE (test infrastructure only -- never imported by the product path).

Restatement of the reference's Ray-mIoU / mAVE metric (SURVEY rows a14, a15):
  projects/mmdet3d_plugin/datasets/ray_metrics.py (reference tree)
     generate_lidar_rays :63-86, process_one_sample :89-143, calc_metrics :146-197, main :200-257
The voxel traversal is the C restatement in oracle/ray_dda.c (of tools/ray_iou/lib/dvr/dvr.cu:69-319).

Parity status: python logic pinned against the unmodified reference functions
(tests/golden/gen_golden.py -> tests/golden/ref_metric.npz); DDA pinned on the GPU against the
reference kernel's outputs (tests/golden/ref_dvr.npz, and oracle/_ref when it is built).
"""
import ctypes
import math
import os
import subprocess

import numpy as np

_PC_RANGE = [-40, -40, -1.0, 40, 40, 5.4]
_VOXEL_SIZE = 0.4
NUM_CLASSES = 17
FREE_ID = 16
FLOW_CLASSES = 8        # class ids 0..7 carry flow (ray_metrics.py:26-29)
THRESHOLDS = (1, 2, 4)

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build_dda(force=False):
    """gcc oracle/ray_dda.c -> oracle/_build/libray_dda.so (the checker, not the product)."""
    out_dir = os.path.join(_HERE, '_build')
    so = os.path.join(out_dir, 'libray_dda.so')
    src = os.path.join(_HERE, 'ray_dda.c')
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(['gcc', '-O2', '-fPIC', '-shared', '-ffp-contract=off', '-o', so, src, '-lm'])
    return so


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build_dda())
        f32p = ctypes.POINTER(ctypes.c_float)
        i = ctypes.c_int
        _LIB.oracle_render_forward.argtypes = [f32p, f32p, f32p, f32p, i, i, i, i, i, i, ctypes.c_int64, i, f32p, f32p, f32p]
        _LIB.oracle_render_forward.restype = None
    return _LIB


def render_forward(sigma, origin, points, tindex):
    """dvr.render_forward(sigma, origin, points, tindex, grid, 'test') in double (oracle/ray_dda.c).

    Batched, the reference's full argument meaning: sigma (N,T,Z,Y,X), origin (N,To,3), points (N,M,K) with K >= 3,
    tindex (N,M) -> pred_dist (N,M), gt_dist (N,M), coord (N,M,3).  Unbatched (N = 1 dropped): sigma (T,Z,Y,X),
    origin (To,3), points (M,K), tindex (M,) -> (M,), (M,), (M,3).  tindex must stay below To (and below T when T > 1):
    like the reference, nothing here checks it."""
    sigma = np.ascontiguousarray(sigma, np.float32)
    batched = sigma.ndim == 5
    if not batched:
        sigma, origin, points, tindex = sigma[None], np.asarray(origin)[None], np.asarray(points)[None], np.asarray(tindex)[None]
    origin = np.ascontiguousarray(origin, np.float32)
    points = np.ascontiguousarray(points, np.float32)
    tindex = np.ascontiguousarray(tindex, np.float32)
    N, T, Z, Y, X = sigma.shape
    _, M, K = points.shape
    To = origin.shape[1]
    assert origin.shape == (N, To, 3) and To >= 1 and K >= 3 and points.shape[0] == N and tindex.shape == (N, M)
    ok = tindex[tindex >= 0].astype(np.int64)
    assert (ok < To).all() and (T == 1 or (ok < T).all()), 'tindex points past origin or sigma'
    pd = np.empty((N, M), np.float32); gd = np.empty((N, M), np.float32); ci = np.empty((N, M, 3), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    _lib().oracle_render_forward(p(sigma), p(origin), p(points), p(tindex), N, T, To, Z, Y, X, M, K, p(pd), p(gd), p(ci))
    return (pd, gd, ci) if batched else (pd[0], gd[0], ci[0])


def generate_lidar_rays():
    """ray_metrics.py:63-86 -> (14040, 3) float32."""
    pitch_angles = []
    for k in range(10):
        pitch_angles.append(-(math.pi / 2 - math.atan(k + 1)))
    while pitch_angles[-1] < 0.21:
        pitch_angles.append(pitch_angles[-1] + (pitch_angles[-1] - pitch_angles[-2]))
    rays = []
    for pitch in pitch_angles:
        for az in np.arange(0, 360, 1):
            az = np.deg2rad(az)
            rays.append((np.cos(pitch) * np.cos(az), np.cos(pitch) * np.sin(az), np.sin(pitch)))
    return np.array(rays, dtype=np.float32)


def process_one_sample(sem, lidar_rays, output_origin, flow):
    """ray_metrics.py:89-143.  sem (200,200,16) int, flow (200,200,16,2), origins (1,T,3) -> (T*M, 4) f32
    rows = [class, dist (m), flow_x, flow_y]."""
    T = output_origin.shape[1]
    occ = np.where(sem < FREE_ID, 1, 0).astype(np.float32)
    sigma = np.ascontiguousarray(occ.transpose(2, 1, 0))[None]                   # (1, Z, Y, X)
    offset = np.asarray(_PC_RANGE[:3], np.float32)[None, None, :]
    scaler = np.asarray([_VOXEL_SIZE] * 3, np.float32)[None, None, :]
    lidar_rays = np.asarray(lidar_rays, np.float32)
    tindex = np.zeros(lidar_rays.shape[0], np.float32)
    out = []
    for t in range(T):
        lidar_origin = np.asarray(output_origin[:, t:t + 1, :], np.float32)      # (1,1,3)
        lidar_endpts = lidar_rays[None] + lidar_origin                            # fp32 add (torch semantics)
        o_r = ((lidar_origin - offset) / scaler).astype(np.float32)
        p_r = ((lidar_endpts - offset) / scaler).astype(np.float32)
        pd, _, ci = render_forward(sigma[0][None], o_r[0], p_r[0], tindex)
        pd = pd * np.float32(_VOXEL_SIZE)
        ci = ci.astype(np.int32)
        lab = sem[ci[:, 0], ci[:, 1], ci[:, 2]].astype(np.float32)[:, None]
        fl = flow[ci[:, 0], ci[:, 1], ci[:, 2]].astype(np.float32)
        out.append(np.concatenate([lab, pd[:, None], fl], -1))
    return np.concatenate(out, 0).astype(np.float32)


def new_counters():
    ave = np.zeros([3, NUM_CLASSES])
    ave[:, FLOW_CLASSES:] = np.nan                                                # ray_metrics.py:153-156
    return dict(gt_cnt=np.zeros(NUM_CLASSES), pred_cnt=np.zeros(NUM_CLASSES), tp_cnt=np.zeros([3, NUM_CLASSES]),
                ave=ave, ave_count=np.zeros([3, NUM_CLASSES]))


def accumulate(cnt, pcd_pred, pcd_gt):
    """ray_metrics.py:160-189 for one frame (rays with free GT already dropped)."""
    for j, thr in enumerate(THRESHOLDS):
        l1 = np.abs(pcd_pred[:, 1] - pcd_gt[:, 1])
        tp_dist = l1 < thr
        for i in range(NUM_CLASSES):
            mp = pcd_pred[:, 0] == i
            mg = pcd_gt[:, 0] == i
            if j == 0:
                cnt['gt_cnt'][i] += mg.sum()
                cnt['pred_cnt'][i] += mp.sum()
            tp = np.logical_and(mg & mp, tp_dist)
            cnt['tp_cnt'][j][i] += tp.sum()
            if i < FLOW_CLASSES and tp.sum() > 0:
                err = np.linalg.norm(pcd_gt[tp, 2:4] - pcd_pred[tp, 2:4], axis=1)
                cnt['ave'][j][i] += np.sum(err)
                cnt['ave_count'][j][i] += err.shape[0]
    return cnt


def finalize(cnt):
    """ray_metrics.py:191-195, 248-253 -> dict(iou (3,16), ave (16,), miou, mave, score)."""
    with np.errstate(divide='ignore', invalid='ignore'):
        iou = np.stack([(cnt['tp_cnt'][j] / (cnt['gt_cnt'] + cnt['pred_cnt'] - cnt['tp_cnt'][j]))[:-1]
                        for j in range(3)])
        ave = cnt['ave'][1][:-1] / cnt['ave_count'][1][:-1]
        miou = np.nanmean(iou)
        mave = np.nanmean(ave)
    score = miou * 0.9 + max(1 - mave, 0.0) * 0.1
    return dict(iou=iou, ave=ave, miou=miou, mave=mave, score=score)


def counters_to_vector(cnt):
    """187 doubles in the all-reduce order (SURVEY 8e); NaN slots of `ave` travel as 0."""
    return np.concatenate([cnt['gt_cnt'], cnt['pred_cnt'], cnt['tp_cnt'].ravel(),
                           np.nan_to_num(cnt['ave']).ravel(), cnt['ave_count'].ravel()])


def vector_to_counters(v):
    v = np.asarray(v, np.float64)
    n = NUM_CLASSES
    cnt = dict(gt_cnt=v[:n].copy(), pred_cnt=v[n:2 * n].copy(), tp_cnt=v[2 * n:5 * n].reshape(3, n).copy(),
               ave=v[5 * n:8 * n].reshape(3, n).copy(), ave_count=v[8 * n:11 * n].reshape(3, n).copy())
    cnt['ave'][:, FLOW_CLASSES:] = np.nan
    return cnt


def main(sem_pred_list, sem_gt_list, flow_pred_list, flow_gt_list, lidar_origin_list):
    """ray_metrics.py:200-257 without the table printing."""
    rays = generate_lidar_rays()
    cnt = new_counters()
    for sp, sg, fp, fg, orig in zip(sem_pred_list, sem_gt_list, flow_pred_list, flow_gt_list, lidar_origin_list):
        sp = np.reshape(sp, [200, 200, 16]); sg = np.reshape(sg, [200, 200, 16])
        fp = np.reshape(fp, [200, 200, 16, 2]); fg = np.reshape(fg, [200, 200, 16, 2])
        pp = process_one_sample(sp, rays, orig, fp)
        pg = process_one_sample(sg, rays, orig, fg)
        valid = pg[:, 0].astype(np.int32) != FREE_ID
        accumulate(cnt, pp[valid], pg[valid])
    return finalize(cnt), cnt
