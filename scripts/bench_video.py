#!/usr/bin/env python
"""Temporal (video) inference with the BEV history inside the engine, against the explicit prev_bev path, at the shipped size
(6 cameras, 200 x 200 BEV, 6 encoder layers, bf16 + tensor cores as bench.py's headline, synthetic weights).  Prints one
JSON line.

    python scripts/bench_video.py [--frames 32] [--runs 3]

Per run (the variants alternate inside every run):
  device   (CUDA events, features on the device)
    explicit           : forward(prev_bev = previous bev_embed) with one global rotation map (3 degrees), as bench.py's
                         temporal_config leg; the caller carries bev_embed
    video_fixed        : forward_video with the host index map of 3 degrees every frame (range-checked and uploaded per frame)
    video_per_frame    : forward_video cycling through the host maps of 8 angles (rotation_index_map's host cache)
    video_unique       : forward_video with a new angle every frame, as real can_bus[-1] values are, as a host map: every
                         frame pays the host torchvision rotate of rotation_index_map and the map upload
    video_unique_angle : the same new angle every frame handed over as the angle: the engine computes the source cells on
                         the device inside the history gather (no host work, no upload)
    self_mode          : forward(prev_bev = None): the ceiling, no temporal attention
  host     (wall clock, ends synchronised; pinned fp32 features, two frames in flight)
    stream_host_video with the 8 cycling host maps, with a new angle every frame as a host map and as the angle, against
    stream_host (self mode)
  detector (wall clock, BEVFormerOcc.forward_test on img_feats, results copied to the host as forward_test returns them)
    temporal_test with the prev_bev cache (explicit) against engine_history=True, a new angle every frame
Also: whether explicit and video paths (angles) give byte-identical occ_cls / flow / bev_embed over a frame sequence with
per-frame angles, and the launches per frame of each variant.  The card's name, power limit and SM clock are read
(nvidia-smi queries only) in the same call.
"""
import argparse
import itertools
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from occnet_b200 import fixtures                                # noqa: E402
from occnet_b200.engine import OccEngine, rotation_index_map    # noqa: E402

ANGLES = [3.0, -1.5, 2.25, 0.5, -2.75, 1.0, 4.5, -0.25]


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        f = [x.strip() for x in out.split(',')]
        return dict(name=f[0], power_limit_w=float(f[1]), sm_mhz=float(f[2]), sm_max_mhz=float(f[3]))
    except Exception as e:                                                   # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), error=f'nvidia-smi: {e}'[:200])


def timed(fn, n):
    """device ms per call over n calls (CUDA events on the current stream)"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for i in range(n):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def wall(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(n)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def detector(cfg, params, fr_dev):
    """BEVFormerOcc(temporal_test=True, video_test_mode=True) with the benchmark engine's configuration and weights; one
    scene, so every frame after the first has a previous BEV"""
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200.mmcv_shim import build_detector
    det = build_detector(dict(type='BEVFormerOcc', video_test_mode=True, temporal_test=True,
                              pts_bbox_head=dict(fixtures.head_cfg(cfg), precision='bf16', test_logits=False)))
    det = det.to(fr_dev[0][0].device).eval()
    det.pts_bbox_head.load_state_dict(params, strict=True)
    feats = [[f[None] for f in fr] for fr in fr_dev]
    metas = []
    for _ in range(3):
        m = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=0.0)
        m[0]['scene_token'] = 'bench'
        metas.append(m)
    return det, feats, metas


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=32, help='frames per timed variant')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--layers', type=int, default=6)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_video needs a CUDA device')
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
    eng.set_history(True)
    center = cfg.get('rotate_center', [100, 100])
    fixed_map = rotation_index_map(cfg['bev_h'], cfg['bev_w'], 3.0, center)
    X, Y, Z = eng.vox_shape
    want_video = ('flow', 'occ_cls')
    fresh = (5.0 + 0.0123 * k for k in itertools.count())          # angles never seen before: no cache hits
    per_frame_maps = [rotation_index_map(cfg['bev_h'], cfg['bev_w'], a, center) for a in ANGLES]

    def fresh_map():
        return rotation_index_map(cfg['bev_h'], cfg['bev_w'], next(fresh), center)
    state = {'prev': None}

    def explicit(i):
        state['prev'] = eng.forward(fr_dev[i % 3], prev_bev=state['prev'], want=('bev_embed', 'flow', 'occ_cls'))['bev_embed']

    variants = {
        'explicit': explicit,
        'video_fixed': lambda i: eng.forward_video(fr_dev[i % 3], rotation=fixed_map, want=want_video),
        'video_per_frame': lambda i: eng.forward_video(fr_dev[i % 3], rotation=per_frame_maps[i % len(ANGLES)], want=want_video),
        'video_unique': lambda i: eng.forward_video(fr_dev[i % 3], rotation=fresh_map(), want=want_video),
        'video_unique_angle': lambda i: eng.forward_video(fr_dev[i % 3], rotation=next(fresh), want=want_video),
        'self_mode': lambda i: eng.forward(fr_dev[i % 3], want=want_video),
    }

    def host_video(n):
        for _ in eng.stream_host_video((fr_host[i % 3], per_frame_maps[i % len(ANGLES)], False) for i in range(n)):
            pass

    def host_video_unique(n):
        for _ in eng.stream_host_video((fr_host[i % 3], fresh_map(), False) for i in range(n)):
            pass

    def host_video_unique_angle(n):
        for _ in eng.stream_host_video((fr_host[i % 3], next(fresh), False) for i in range(n)):
            pass

    def host_self(n):
        for _ in eng.stream_host(fr_host[i % 3] for i in range(n)):
            pass

    # warm-up: every path, the history primed, the 8 cycling angles' host maps computed
    eng.set_prev_rotation(fixed_map)
    for name, fn in variants.items():
        for i in range(len(ANGLES)):
            fn(i)
    host_video(4)
    host_video_unique(4)
    host_video_unique_angle(4)
    host_self(4)
    det, det_feats, det_metas = detector(cfg, params, fr_dev)

    def det_run(engine_history):
        def run(n):
            det.engine_history = engine_history
            for i in range(n):
                det_metas[i % 3][0]['can_bus'][-1] = next(fresh)
                det(return_loss=False, img_feats=det_feats[i % 3], img_metas=[det_metas[i % 3]])
        return run
    det_run(False)(4)
    det_run(True)(4)
    torch.cuda.synchronize()
    launches = {}
    for name, fn in variants.items():
        fn(0)
        launches[name] = eng.launches_per_frame

    info_before = card()
    runs = []
    for _ in range(args.runs):
        r = {}
        for name, fn in variants.items():
            r[name + '_ms'] = round(timed(fn, args.frames), 4)
        r['host_video_ms'] = round(wall(host_video, args.frames), 4)
        r['host_video_unique_ms'] = round(wall(host_video_unique, args.frames), 4)
        r['host_video_unique_angle_ms'] = round(wall(host_video_unique_angle, args.frames), 4)
        r['host_self_ms'] = round(wall(host_self, args.frames), 4)
        r['detector_explicit_ms'] = round(wall(det_run(False), args.frames), 4)
        r['detector_engine_history_ms'] = round(wall(det_run(True), args.frames), 4)
        runs.append(r)
    info_after = card()

    # outputs: explicit (global map set per frame, synchronous) against the video path, per-frame angles, a scene reset
    starts = [True] + [False] * 5 + [True, False]
    want = ('bev_embed', 'flow', 'occ_cls')
    ref, prev = [], None
    for i, s in enumerate(starts):
        if s:
            prev = None
        eng.set_prev_rotation(rotation_index_map(cfg['bev_h'], cfg['bev_w'], ANGLES[i], center) if prev is not None else None)
        o = {k: v.clone() for k, v in eng.forward(fr_dev[i % 3], prev_bev=prev, want=want).items()}
        ref.append(o)
        prev = o['bev_embed']
    eng.set_prev_rotation(None)
    eng.set_history(True)
    identical = True
    for i, s in enumerate(starts):
        o = eng.forward_video(fr_dev[i % 3], rotation=ANGLES[i], scene_start=s, want=want)
        identical = identical and all(torch.equal(o[k], ref[i][k]) for k in want)
    eng.set_history(True)
    host = [(o.clone(), f.clone()) for o, f in
            eng.stream_host_video((fr_host[i % 3], ANGLES[i], s) for i, s in enumerate(starts))]
    host_identical = all(torch.equal(o, ref[i]['occ_cls'].cpu().long()) and torch.equal(f, ref[i]['flow'].cpu())
                         for i, (o, f) in enumerate(host))

    med = {k: sorted(r[k] for r in runs)[len(runs) // 2] for k in runs[0]}
    result = {
        'what': 'temporal (video) inference: engine-held BEV history vs explicit prev_bev; full size, bf16 + tensor cores',
        'layers': args.layers, 'frames_per_variant': args.frames, 'runs': runs, 'median_ms': med,
        'video_fixed_vs_explicit_speedup': round(med['explicit_ms'] / med['video_fixed_ms'], 4),
        'video_per_frame_vs_explicit_speedup': round(med['explicit_ms'] / med['video_per_frame_ms'], 4),
        'video_unique_angle_vs_host_map_speedup': round(med['video_unique_ms'] / med['video_unique_angle_ms'], 4),
        'host_video_unique_angle_vs_host_map_speedup': round(med['host_video_unique_ms'] / med['host_video_unique_angle_ms'], 4),
        'detector_engine_history_vs_explicit_speedup': round(med['detector_explicit_ms'] / med['detector_engine_history_ms'], 4),
        'launches_per_frame': launches,
        'outputs_identical_explicit_vs_video': identical, 'outputs_identical_explicit_vs_host_video': host_identical,
        'card_before': info_before, 'card_after': info_after,
    }
    print(json.dumps(result))


if __name__ == '__main__':
    main()
