#!/usr/bin/env python
"""uint8 camera frames -> voxels against fp32 normalised images -> voxels, at the shipped size (6 x 900 x 1600 frames padded
to 928 x 1600, 6 encoder layers as bench.py, synthetic weights).  Prints one JSON line.

    python scripts/bench_camera_frames.py [--frames 24] [--runs 3] [--dump-outputs DIR]

Per precision (bf16 + tensor cores; fp32 storage on CUDA cores) and per run (the variants alternate inside every run):
  device  : frames on the device -> engine input dtype 3 (backbone stem normalises / pads) -> voxels, against fp32 images on
            the device -> BackboneEngine.forward -> OccEngine.forward (bench.py's images_to_voxels dataflow); backbone-only
            ms per frame both ways.  CUDA events.
  host    : pinned uint8 frames through submit_host / wait_host with two frames in flight, against a Python loop that uploads
            pinned fp32 images on a side stream (double-buffered) and runs the same chain.  Wall clock, ends synchronised.
Also: bytes uploaded per frame (from shapes), the host CPU cost of the preprocessing the frames path removes (the numpy
restatement in oracle/image_pipeline.py, one thread), and whether the two paths' occ_cls / flow are byte-identical.
The card's name, power limit and SM clock are read (nvidia-smi queries only) in the same call.
"""
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

from occnet_b200 import fixtures                  # noqa: E402
from occnet_b200.backbone import BackboneEngine   # noqa: E402
from occnet_b200.engine import OccEngine          # noqa: E402
from oracle import image_pipeline as IP           # noqa: E402

SRC_HW, NC = (900, 1600), 6
MEAN, STD, TO_RGB = IP.SHIPPED_NORM['mean'], IP.SHIPPED_NORM['std'], IP.SHIPPED_NORM['to_rgb']
WANT = ('flow', 'occ_cls_i64')


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


class Variant:
    def __init__(self, precision, cfg, params, metas, frames_u8, imgs_f32, dev):
        tc = precision == 'bf16'
        self.cl = tc                                                         # bf16 -> bf16: channels-last hand-over
        self.be = BackboneEngine(fixtures.init_backbone_params(seed=5), NC, cfg['img_shape'][:2], precision=precision,
                                 use_tensor_cores=tc, device=str(dev))
        self.be.set_frame_format(SRC_HW, MEAN, STD, TO_RGB)
        self.eng = OccEngine(cfg, params, precision=precision, use_tensor_cores=tc, device=str(dev))
        self.eng.set_cameras(metas)
        self.eng.attach_backbone(self.be)
        self.fr_dev = [f.to(dev) for f in frames_u8]
        self.im_dev = [f.to(dev) for f in imgs_f32]
        self.fr_host = [f.pin_memory() for f in frames_u8]
        self.im_host = [f.pin_memory() for f in imgs_f32]
        self.dev = dev

    def images_mode(self):
        self.eng.set_input_dtype(torch.bfloat16 if self.cl else torch.float32, channels_last=self.cl)

    def frames_mode(self):
        self.eng.set_input_dtype(torch.uint8)

    def run_images(self, i):
        return self.eng.forward(self.be.forward(self.im_dev[i % 3], channels_last_bf16=self.cl), want=WANT)

    def run_frames(self, i):
        return self.eng.forward(self.fr_dev[i % 3], want=WANT)

    def host_frames(self, n):
        for _ in self.eng.stream_host(self.fr_host[i % 3] for i in range(n)):
            pass

    def host_images(self, n):
        """pinned fp32 images -> device on a copy stream, double-buffered; chain + result copies on the compute stream"""
        comp, copy = torch.cuda.current_stream(), torch.cuda.Stream(device=self.dev)
        if not hasattr(self, '_bufs'):
            X, Y, Z = self.eng.vox_shape
            self._bufs = [torch.empty_like(self.im_dev[0]) for _ in range(2)]
            self._outs = [(torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(), torch.empty((X, Y, Z, 2)).pin_memory())
                          for _ in range(2)]
        up = [torch.cuda.Event() for _ in range(2)]
        free = [torch.cuda.Event() for _ in range(2)]
        for i in range(n):
            s = i & 1
            with torch.cuda.stream(copy):
                if i >= 2:
                    copy.wait_event(free[s])
                self._bufs[s].copy_(self.im_host[i % 3], non_blocking=True)
                up[s].record(copy)
            comp.wait_event(up[s])
            o = self.eng.forward(self.be.forward(self._bufs[s], channels_last_bf16=self.cl), want=WANT)
            free[s].record(comp)
            self._outs[s][0].copy_(o['occ_cls_i64'], non_blocking=True)
            self._outs[s][1].copy_(o['flow'], non_blocking=True)

    def measure(self, n):
        r = {}
        self.images_mode()
        r['device_images_ms'] = timed(self.run_images, n)
        r['backbone_images_ms'] = timed(lambda i: self.be.forward(self.im_dev[i % 3], channels_last_bf16=self.cl), n)
        r['host_images_ms'] = wall(self.host_images, n)
        self.frames_mode()
        r['device_frames_ms'] = timed(self.run_frames, n)
        r['backbone_frames_ms'] = timed(lambda i: self.be.forward_frames(self.fr_dev[i % 3], channels_last_bf16=self.cl), n)
        r['host_frames_ms'] = wall(self.host_frames, n)
        return r

    def outputs(self):
        """occ_cls (int64) and flow of frame 0 through the images path, the frames path and the pinned-frames host path"""
        self.images_mode()
        a = {k: v.cpu() for k, v in self.run_images(0).items()}
        self.frames_mode()
        b = {k: v.cpu() for k, v in self.run_frames(0).items()}
        occ_h, flow_h = self.eng.forward_host(self.fr_host[0])
        c = {'occ_cls_i64': occ_h.clone(), 'flow': flow_h.clone()}
        return a, b, c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=24, help='frames per timed leg (bf16; fp32 runs a quarter of them)')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--layers', type=int, default=6)
    ap.add_argument('--dump-outputs', metavar='DIR', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_camera_frames needs a CUDA device')
    dev = torch.device('cuda:0')
    cfg = fixtures.make_cfg('full', num_layers=args.layers)
    params = fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS)
    metas = fixtures.make_img_metas(cfg)
    rng = np.random.default_rng(7)
    frames_np = [rng.integers(0, 256, size=(NC,) + SRC_HW + (3,), dtype=np.uint8) for _ in range(3)]
    # host CPU cost of the preprocessing the frames path removes (numpy normalise + pad + HWC->CHW, one thread)
    cpu_ms, imgs = [], []
    for f in frames_np:
        t0 = time.perf_counter()
        im, pm = IP.pipeline(f, MEAN, STD, TO_RGB, size_divisor=32)
        cpu_ms.append((time.perf_counter() - t0) * 1e3)
        imgs.append(torch.from_numpy(im))
    assert tuple(pm['img_shape'][0][:2]) == tuple(cfg['img_shape'][:2])
    frames = [torch.from_numpy(f) for f in frames_np]
    info_before = card()
    variants = {p: Variant(p, cfg, params, metas, frames, imgs, dev) for p in ('bf16', 'fp32')}
    nframes = {'bf16': args.frames, 'fp32': max(4, args.frames // 4)}
    for p, v in variants.items():                                          # warm-up: every shape and path once
        v.measure(2)
    runs = {p: [] for p in variants}
    for _ in range(args.runs):
        for p, v in variants.items():
            runs[p].append(v.measure(nframes[p]))
    info_after = card()
    result = dict(metric='camera frames (uint8) vs fp32 images -> 200x200x16 voxels', card=info_before,
                  card_after=info_after, src_hw=SRC_HW, padded_hw=tuple(cfg['img_shape'][:2]), num_cams=NC,
                  layers=args.layers, runs=args.runs,
                  upload_bytes_per_frame=dict(frames_u8=NC * SRC_HW[0] * SRC_HW[1] * 3,
                                              images_f32=NC * 3 * cfg['img_shape'][0] * cfg['img_shape'][1] * 4),
                  host_preprocess_ms_per_frame=dict(median=round(float(np.median(cpu_ms)), 1),
                                                    all=[round(x, 1) for x in cpu_ms], threads=1,
                                                    what='oracle.image_pipeline (numpy fp32 normalise + pad + transpose)'))
    for p, rs in runs.items():
        med = {k: float(np.median([r[k] for r in rs])) for k in rs[0]}
        rng_ = {k: [round(min(r[k] for r in rs), 3), round(max(r[k] for r in rs), 3)] for k in rs[0]}
        result[p] = dict(
            frames_per_leg=nframes[p],
            device=dict(frames_samples_s=round(1e3 / med['device_frames_ms'], 2),
                        images_samples_s=round(1e3 / med['device_images_ms'], 2),
                        backbone_frames_ms=round(med['backbone_frames_ms'], 3),
                        backbone_images_ms=round(med['backbone_images_ms'], 3)),
            host_pinned=dict(frames_samples_s=round(1e3 / med['host_frames_ms'], 2),
                             images_samples_s=round(1e3 / med['host_images_ms'], 2)),
            ms_median=dict((k, round(x, 3)) for k, x in med.items()), ms_range=rng_)
        a, b, c = variants[p].outputs()
        same = {k: a[k].numpy().tobytes() == b[k].numpy().tobytes() and a[k].numpy().tobytes() == c[k].numpy().tobytes()
                for k in WANT}
        result[p]['outputs_byte_identical'] = same
        if args.dump_outputs:
            os.makedirs(args.dump_outputs, exist_ok=True)
            for tag, d in (('images', a), ('frames', b), ('frames_host', c)):
                for k, t in d.items():
                    np.save(os.path.join(args.dump_outputs, f'{p}_{tag}_{k}.npy'), t.numpy())
    print(json.dumps(result))


if __name__ == '__main__':
    main()
