#!/usr/bin/env python
"""Ray records cast inside the frame engine against the ray cast `format_results` does afterwards, at the shipped size
(6 cameras, 200 x 200 BEV, 6 encoder layers, bf16 + tensor cores as bench.py's headline, synthetic weights), for T = 8 and
T = 1 lidar origins.  Prints one JSON line and a table.  It needs a CUDA device.

    python scripts/bench_ray_records.py [--frames 24] [--runs 3]

Per run and T (the variants alternate inside every run; wall clock around work that ends synchronised, pinned host buffers):
  host_volumes   : stream_host returning the volumes (10.24 MB per frame to the host), then today's format_results ray cast
                   per frame: volumes uploaded again, ray_metric_kernel with the prediction as "pred" and "gt", (T*M,4) fp32
                   rows downloaded and narrowed by numpy
  host_records   : stream_host with a ray request per frame and volumes=False: T*M*7 bytes per frame to the host
  det_volumes    : BEVFormerOcc.forward_test (engine_history=True) on img_feats, then the same format_results ray cast
  det_records    : the same detector with ray_only=True and lidar_origins per frame
  kernel         : ray_records_kernel alone against ray_metric_kernel called as process_one_sample calls it (CUDA events)
Also: device->host bytes per frame counted from the shapes, and whether host_volumes and host_records give byte-identical
records.  The card's name, power limit and SM clock are read (nvidia-smi queries only) in the same call."""
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
from occnet_b200.metric import RayMetric, generate_lidar_rays               # noqa: E402
from projects.mmdet3d_plugin.datasets.ray_metrics import process_one_sample  # noqa: E402

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


def narrow(pcd):
    """format_results' narrowing of process_one_sample's rows"""
    return (pcd[:, 0].astype(np.int8), pcd[:, 1].astype(np.float16), pcd[:, 2:4].astype(np.float16))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=24, help='frames per timed variant')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--layers', type=int, default=6)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ray_records needs a CUDA device')
    dev = torch.device('cuda:0')
    cfg = fixtures.make_cfg('full', num_layers=args.layers)
    params = fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS)
    metas = fixtures.make_img_metas(cfg, bs=1)
    feats = [fixtures.make_feats(cfg, bs=1, seed=100 + i) for i in range(3)]
    fr_dev = [[f[0].to(dev) for f in fr] for fr in feats]
    fr_host = [[f[0].contiguous().pin_memory() for f in fr] for fr in feats]
    del feats
    eng = OccEngine(cfg, params, precision='bf16', use_tensor_cores=True, device=str(dev))
    eng.set_cameras(metas)
    rays = generate_lidar_rays()
    orgs = {T: fixtures.make_ray_origins(T=T).astype(np.float64) for T in (8, 1)}     # the dataset's origins are float64

    def host_volumes(T):
        def run(n):
            last = None
            for occ, flow in eng.stream_host(fr_host[i % 3] for i in range(n)):
                last = narrow(process_one_sample(occ.numpy(), rays, orgs[T], flow.numpy(), device=str(dev)))
            return last
        return run

    def host_records(T):
        def run(n):
            last = None
            for _, _, rec in eng.stream_host((fr_host[i % 3] for i in range(n)), ray_origins=(orgs[T] for _ in range(n)),
                                             volumes=False):
                last = tuple(rec[k].numpy().copy() for k in ('ray_cls', 'ray_dist', 'ray_flow'))
            return last
        return run

    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200.mmcv_shim import build_detector
    dets = {}
    for ray_only in (False, True):
        d = build_detector(dict(type='BEVFormerOcc', video_test_mode=True, temporal_test=True, engine_history=True,
                                ray_only=ray_only,
                                pts_bbox_head=dict(fixtures.head_cfg(cfg), precision='bf16', test_logits=False)))
        d = d.to(dev).eval()
        d.pts_bbox_head.load_state_dict(params, strict=True)
        dets[ray_only] = d
    det_feats = [[f[None] for f in fr] for fr in fr_dev]
    det_meta = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=1.5)
    det_meta[0]['scene_token'] = 'bench'

    def det_volumes(T):
        def run(n):
            for i in range(n):
                r = dets[False](return_loss=False, img_feats=det_feats[i % 3], img_metas=[det_meta])
                narrow(process_one_sample(r['occ_results'].numpy().reshape(200, 200, 16), rays, orgs[T],
                                          r['flow_results'].numpy().reshape(200, 200, 16, 2), device=str(dev)))
        return run

    def det_records(T):
        def run(n):
            for i in range(n):
                dets[True](return_loss=False, img_feats=det_feats[i % 3], img_metas=[det_meta], lidar_origins=orgs[T])
        return run

    # the two kernels alone, on one predicted frame
    out = eng.forward(fr_dev[0], want=('flow', 'occ_cls'))
    sem, flow = out['occ_cls'], out['flow']
    rm = RayMetric(dev)

    def kernel_metric(T):
        o = torch.as_tensor(orgs[T])
        return lambda: rm.add_frame(sem, flow, sem, flow, o, return_pcd=True)

    def kernel_records(T):
        return lambda: ops.ray_records(sem, flow, orgs[T])

    variants = {'host_volumes': host_volumes, 'host_records': host_records, 'det_volumes': det_volumes, 'det_records': det_records}
    for T in (8, 1):                                                   # warm-up: every path and shape
        for mk in variants.values():
            mk(T)(4)
        for mk in (kernel_metric, kernel_records):
            for _ in range(10):
                mk(T)()
    torch.cuda.synchronize()

    info_before = card()
    runs, identical = [], True
    for _ in range(args.runs):
        r = {}
        for T in (8, 1):
            got = {}
            for name, mk in variants.items():
                ms, got[name] = wall(mk(T), args.frames)
                r[f'{name}_T{T}_ms'] = round(ms, 4)
            identical = identical and all(a.tobytes() == b.tobytes() for a, b in zip(got['host_volumes'], got['host_records']))
            r[f'kernel_metric_T{T}_ms'] = round(events(kernel_metric(T), 200), 5)
            r[f'kernel_records_T{T}_ms'] = round(events(kernel_records(T), 200), 5)
        runs.append(r)
    info_after = card()

    med = {k: sorted(r[k] for r in runs)[len(runs) // 2] for k in runs[0]}
    d2h = {'volumes': NVOX * 8 + NVOX * 8, 'rows_fp32_T8': 8 * M * 16, 'rows_fp32_T1': M * 16,
           'records_T8': 8 * M * 7, 'records_T1': M * 7}
    result = {'what': 'ray records inside the frame engine vs format_results ray cast; full size, bf16 + tensor cores',
              'layers': args.layers, 'frames_per_variant': args.frames, 'runs': runs, 'median_ms': med,
              'd2h_bytes_per_frame': {'host_volumes_T8': d2h['volumes'] + d2h['rows_fp32_T8'],
                                      'host_volumes_T1': d2h['volumes'] + d2h['rows_fp32_T1'],
                                      'host_records_T8': d2h['records_T8'], 'host_records_T1': d2h['records_T1']},
              'h2d_bytes_per_frame_re_uploaded_by_format_results': NVOX + NVOX * 8 + M * 12,
              'records_identical_host_volumes_vs_host_records': identical,
              'card_before': info_before, 'card_after': info_after}
    print(json.dumps(result))
    print(f"\n{info_before.get('name')}, power limit {info_before.get('power_limit_w')} W; median of {args.runs} runs, "
          f'{args.frames} frames per variant, ms per frame')
    print(f"{'variant':<44}{'T = 8':>10}{'T = 1':>10}")
    rows = [('stream_host volumes + format_results ray cast', 'host_volumes'), ('stream_host ray request, volumes=False', 'host_records'),
            ('forward_test volumes + format_results ray cast', 'det_volumes'), ('forward_test ray_only, lidar_origins', 'det_records'),
            ('ray_metric_kernel alone (pred as pred and gt)', 'kernel_metric'), ('ray_records_kernel alone', 'kernel_records')]
    for label, key in rows:
        print(f"{label:<44}{med[f'{key}_T8_ms']:>10.3f}{med[f'{key}_T1_ms']:>10.3f}")
    if not identical:
        raise SystemExit('records differ between the two host paths')


if __name__ == '__main__':
    main()
