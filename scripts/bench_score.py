#!/usr/bin/env python
"""A frame scored inside the frame engine against the evaluation loop that copies the volumes out and calls the metric
afterwards, at the shipped size (6 cameras, 200 x 200 BEV, 6 encoder layers, bf16 + tensor cores as bench.py's headline,
synthetic weights), for T = 8 and T = 1 lidar origins.  Prints one JSON line and a table.  It needs a CUDA device.

    python scripts/bench_score.py [--frames 24] [--runs 3]

Per run and T (the variants alternate inside every run; wall clock around work that ends synchronised, pinned host buffers):
  host_add_frame : stream_host returning the volumes (10.24 MB per frame to the host), then RayMetric.add_frame per frame,
                   which uploads prediction and ground truth and launches ray_metric_kernel (the current loop)
  host_main      : the same volumes through datasets/ray_metrics.main called per frame (the reference-signature entry: numpy
                   casts, a RayMetric and a finalize per call)
  host_score     : stream_host with a score request per frame and volumes=False: 5.76 MB of ground truth per frame go up,
                   nothing comes back
  det_volumes    : BEVFormerOcc.forward_test (engine_history=True) on img_feats scoring itself, volumes still returned
  det_score_only : the same detector with score_only=True
  kernel         : ray_metric_kernel and ray_score_kernel alone on the metric fixture (CUDA events over 200 launches); its
                   ground truth leaves about half of the rays free, whose prediction walk ray_score_kernel skips
Also: host<->device bytes per frame counted from the shapes, the share of free rays, and whether host_add_frame and
host_score end with the same counters.  The card's name, power limit and SM clock are read (nvidia-smi queries only) in the
same call."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from occnet_b200 import fixtures, ops                                       # noqa: E402
from occnet_b200.engine import OccEngine                                    # noqa: E402
from occnet_b200.metric import RayMetric                                    # noqa: E402
from projects.mmdet3d_plugin.datasets import ray_metrics                    # noqa: E402

M = 14040
NVOX = 200 * 200 * 16


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        f = [x.strip() for x in out.split(',')]
        return dict(name=f[0], power_limit_w=float(f[1]), sm_mhz=float(f[2]), sm_max_mhz=float(f[3]))
    except Exception as e:                                                   # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), error=f'nvidia-smi: {e}'[:200])


def wall(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn(n)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n, out


def events(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def metric_fixture():
    """the repository's metric fixture: a synthetic scene and a shifted, noisy prediction of it"""
    sem_gt, flow_gt = fixtures.make_occ_scene(seed=4)
    rng = np.random.RandomState(5)
    sem_pred = np.roll(sem_gt, 1, axis=0).copy()
    flip = rng.rand(*sem_pred.shape) < 0.03
    sem_pred[flip] = rng.randint(0, 17, int(flip.sum())).astype(np.uint8)
    flow_pred = (np.roll(flow_gt, 1, axis=0) + rng.normal(0, 0.5, flow_gt.shape)).astype(np.float32)
    return sem_pred, flow_pred, sem_gt, flow_gt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=24, help='frames per timed variant')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--layers', type=int, default=6)
    args = ap.parse_args()
    cfg = fixtures.make_cfg('full', num_layers=args.layers)
    fixture = metric_fixture()
    orgs = {T: fixtures.make_ray_origins(T=T).astype(np.float64) for T in (8, 1)}     # the dataset's origins are float64
    if not torch.cuda.is_available():
        raise SystemExit('bench_score needs a GPU: no CUDA device found, nothing was timed')
    dev = torch.device('cuda:0')
    params = fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS)
    metas = fixtures.make_img_metas(cfg, bs=1)
    feats = [fixtures.make_feats(cfg, bs=1, seed=100 + i) for i in range(3)]
    fr_dev = [[f[0].to(dev) for f in fr] for fr in feats]
    fr_host = [[f[0].contiguous().pin_memory() for f in fr] for fr in feats]
    del feats
    eng = OccEngine(cfg, params, precision='bf16', use_tensor_cores=True, device=str(dev))
    eng.set_cameras(metas)
    gt_host = (torch.from_numpy(fixture[2]).pin_memory(), torch.from_numpy(fixture[3]).pin_memory())
    gt_dev = tuple(t.to(dev) for t in gt_host)

    loop_rm = RayMetric(dev)                                         # one metric for the loops, reset per run

    def host_add_frame(T):
        def run(n):
            rm = loop_rm
            rm.reset()
            for occ, flow in eng.stream_host(fr_host[i % 3] for i in range(n)):
                rm.add_frame(occ.to(torch.uint8), flow, gt_host[0], gt_host[1], torch.as_tensor(orgs[T]))
            return rm.counters.cpu().numpy()
        return run

    def host_main(T):
        def run(n):
            for occ, flow in eng.stream_host(fr_host[i % 3] for i in range(n)):
                ray_metrics.main([occ.numpy()], [fixture[2]], [flow.numpy()], [fixture[3]], [orgs[T]], device=str(dev),
                                 verbose=False)
        return run

    def host_score(T):
        def run(n):
            rm = loop_rm
            rm.reset()
            for _ in eng.stream_host((fr_host[i % 3] for i in range(n)), score=((*gt_host, orgs[T]) for _ in range(n)),
                                     metric=rm, volumes=False):
                pass
            return rm.counters.cpu().numpy()
        return run

    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200.mmcv_shim import build_detector
    dets = {}
    for score_only in (False, True):
        d = build_detector(dict(type='BEVFormerOcc', video_test_mode=True, temporal_test=True, engine_history=True,
                                score_only=score_only,
                                pts_bbox_head=dict(fixtures.head_cfg(cfg), precision='bf16', test_logits=False)))
        d = d.to(dev).eval()
        d.pts_bbox_head.load_state_dict(params, strict=True)
        dets[score_only] = d
    det_feats = [[f[None] for f in fr] for fr in fr_dev]
    det_meta = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=1.5)
    det_meta[0]['scene_token'] = 'bench'

    def det(score_only):
        def mk(T):
            def run(n):
                loop_rm.reset()
                for i in range(n):
                    dets[score_only](return_loss=False, img_feats=det_feats[i % 3], img_metas=[det_meta], lidar_origins=orgs[T],
                                     gt_semantics=gt_dev[0], gt_flow=gt_dev[1], ray_metric=loop_rm)
            return run
        return mk

    # the two kernels alone, on the metric fixture
    fx_dev = [torch.from_numpy(a).to(dev) for a in fixture]
    rm = RayMetric(dev)
    cnt = torch.zeros(187, dtype=torch.float64, device=dev)

    def kernel_metric(T):
        o = torch.as_tensor(orgs[T])
        return lambda: rm.add_frame(fx_dev[0], fx_dev[1], fx_dev[2], fx_dev[3], o)

    def kernel_score(T):
        return lambda: ops.ray_score(fx_dev[0], fx_dev[1], fx_dev[2], fx_dev[3], orgs[T], cnt)

    free_share = {}
    for T in (8, 1):
        _, pg = RayMetric(dev).add_frame(*fx_dev, torch.as_tensor(orgs[T]), return_pcd=True)
        free_share[f'T{T}'] = round(float((pg[:, 0] == 16).float().mean()), 4)

    variants = {'host_add_frame': host_add_frame, 'host_main': host_main, 'host_score': host_score,
                'det_volumes': det(False), 'det_score_only': det(True)}
    for T in (8, 1):                                                   # warm-up: every path and shape
        for mk in variants.values():
            mk(T)(4)
        for mk in (kernel_metric, kernel_score):
            for _ in range(10):
                mk(T)()
    torch.cuda.synchronize()

    info_before = card()
    runs, same = [], True
    for _ in range(args.runs):
        r = {}
        for T in (8, 1):
            got = {}
            for name, mk in variants.items():
                ms, got[name] = wall(mk(T), args.frames)
                r[f'{name}_T{T}_ms'] = round(ms, 4)
            a, b = got['host_add_frame'], got['host_score']
            same = same and np.array_equal(a[:85], b[:85]) and np.array_equal(a[136:], b[136:]) \
                and np.allclose(a[85:136], b[85:136], rtol=1e-12, atol=0)
            r[f'kernel_metric_T{T}_ms'] = round(events(kernel_metric(T), 200), 5)
            r[f'kernel_score_T{T}_ms'] = round(events(kernel_score(T), 200), 5)
        runs.append(r)
    info_after = card()

    med = {k: sorted(r[k] for r in runs)[len(runs) // 2] for k in runs[0]}
    vol, gt = NVOX * 8 + NVOX * 8, NVOX + NVOX * 8
    result = {'what': 'a frame scored inside the frame engine vs volumes out + the metric afterwards; full size, bf16 + tensor cores',
              'layers': args.layers, 'frames_per_variant': args.frames, 'runs': runs, 'median_ms': med,
              'bytes_per_frame': {'host_add_frame': {'d2h': vol, 'h2d': NVOX + NVOX * 8 + gt},   # prediction up again as u8 + fp32
                                  'host_score': {'d2h': 0, 'h2d': gt}},
              'free_ray_share_of_the_kernel_fixture': free_share,
              'counters_equal_host_add_frame_vs_host_score': bool(same),
              'card_before': info_before, 'card_after': info_after}
    print(json.dumps(result))
    print(f"\n{info_before.get('name')}, power limit {info_before.get('power_limit_w')} W; median of {args.runs} runs, "
          f'{args.frames} frames per variant, ms per frame')
    print(f"{'variant':<52}{'T = 8':>10}{'T = 1':>10}")
    rows = [('stream_host volumes + RayMetric.add_frame', 'host_add_frame'), ('stream_host volumes + ray_metrics.main per frame', 'host_main'),
            ('stream_host score request, volumes=False', 'host_score'), ('forward_test scoring itself, volumes returned', 'det_volumes'),
            ('forward_test score_only', 'det_score_only'), ('ray_metric_kernel alone (metric fixture)', 'kernel_metric'),
            ('ray_score_kernel alone (metric fixture)', 'kernel_score')]
    for label, key in rows:
        print(f"{label:<52}{med[f'{key}_T8_ms']:>10.3f}{med[f'{key}_T1_ms']:>10.3f}")
    if not same:
        raise SystemExit('the counters differ between the two host paths')


if __name__ == '__main__':
    main()
