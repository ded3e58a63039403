"""JPEG camera files decoded on the GPU against cv2.imdecode on the host, at the shipped size (6 x 900 x 1600 camera files,
padded to 928 x 1600, 6 encoder layers, bf16 + tensor cores, synthetic weights).  Prints one JSON line.

    python scripts/bench_jpeg.py [--frames 24] [--runs 3]

Per run (the variants alternate inside every run):
  decode  : device ms of one 6-camera frame through JpegDecoder (CUDA events over --frames frames, host parsing and the
            upload included in the stream), at qualities 75 and 95, without restart markers and with one per MCU row;
            compressed bytes per frame.  The content is synthetic (`camera`: a smooth gradient with +-6 noise): real camera
            files may compress differently, and the decode time follows the compressed size.
  host    : host ms of one JpegDecoder.decode call with the GPU idle: header parsing (twice: once for the output size,
            once into the tables), the copy of the compressed bytes into the pinned staging buffer, the upload and the
            kernel launches being enqueued (perf_counter around the call; the median of the frames).
  cv2     : cv2.imdecode of the same frame on one host core, and over all host cores with a thread pool.
  stream  : frames/s end to end through OccEngine.stream_host with the backbone attached: JPEG bytes in host memory (input
            'jpeg'), against the current path, cv2 decode in a thread pool feeding stream_host with pinned uint8 frames.
            Bytes uploaded per frame both ways, and whether the two paths' occ_cls / flow are byte-identical.
The card's name, power limit and SM clock are read (nvidia-smi queries only) in the same call.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from occnet_b200 import fixtures                  # noqa: E402
from occnet_b200.backbone import BackboneEngine   # noqa: E402
from occnet_b200.engine import OccEngine          # noqa: E402
from occnet_b200.jpeg import JpegDecoder          # noqa: E402
from oracle import image_pipeline as IP           # noqa: E402
from oracle import jpeg_decode as J               # noqa: E402

SRC_HW, NC = (900, 1600), 6
MEAN, STD, TO_RGB = IP.SHIPPED_NORM['mean'], IP.SHIPPED_NORM['std'], IP.SHIPPED_NORM['to_rgb']
VARIANTS = [(75, 0), (75, 'row'), (95, 0), (95, 'row')]


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        f = [x.strip() for x in out.split(',')]
        return dict(name=f[0], power_limit_w=float(f[1]), sm_mhz=float(f[2]), sm_max_mhz=float(f[3]))
    except Exception as e:                                                   # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), error=f'nvidia-smi: {e}'[:200])


def frame_files(quality, restart, k):
    return [J.encode(J.make_image('camera', *SRC_HW, seed=100 * k + c), quality, '420', restart) for c in range(NC)]


def decode_ms(dec, files, n):
    for f in files:                                                          # warm-up: scratch allocated, modules loaded
        dec.decode(f)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for i in range(n):
        dec.decode(files[i % len(files)])
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def host_ms(dec, files):
    t = []
    for f in files:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dec.decode(f)
        t.append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    return float(np.median(t))


def cv2_ms(files, pool=None):
    t0 = time.perf_counter()
    if pool is None:
        for f in files:
            J.cv2_decode(f)
    else:
        list(pool.map(J.cv2_decode, files))
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=24)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--layers', type=int, default=6)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    cores = os.cpu_count()
    pool = ThreadPoolExecutor(cores)
    files = {v: [frame_files(*v, k) for k in range(3)] for v in VARIANTS}
    dec = JpegDecoder(str(dev))

    cfg = fixtures.make_cfg('full', num_layers=args.layers)
    params = fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS)
    be = BackboneEngine(fixtures.init_backbone_params(seed=5), NC, cfg['img_shape'][:2], precision='bf16',
                        use_tensor_cores=True, device=str(dev))
    be.set_frame_format(SRC_HW, MEAN, STD, TO_RGB)
    eng = OccEngine(cfg, params, precision='bf16', use_tensor_cores=True, device=str(dev))
    eng.set_cameras(fixtures.make_img_metas(cfg))
    eng.attach_backbone(be)
    stream_files = files[(95, 0)]

    def run_jpeg(n):
        eng.set_input_dtype('jpeg')
        last = None
        for occ, flow in eng.stream_host(stream_files[i % 3] for i in range(n)):
            last = (occ.clone(), flow.clone())
        return last

    def run_cv2(n):
        """the current path: the six files of each frame decoded by cv2 in the thread pool while the GPU runs the frames
        submitted before it"""
        eng.set_input_dtype(torch.uint8)
        pinned = [torch.empty((NC, *SRC_HW, 3), dtype=torch.uint8).pin_memory() for _ in range(3)]

        def decoded(i):
            out = pinned[i % 3]
            for c, img in enumerate(pool.map(J.cv2_decode, stream_files[i % 3])):
                out[c].copy_(torch.from_numpy(img))
            return out

        last = None
        for occ, flow in eng.stream_host(decoded(i) for i in range(n)):
            last = (occ.clone(), flow.clone())
        return last

    # warm-up of both stream paths, and the identity check on the last frame of each
    a, b = run_jpeg(3), run_cv2(3)
    identical = bool(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]))

    res = {f'q{q}_rst_{r}': dict(decode_ms=[], host_ms=[], cv2_1core_ms=[], cv2_pool_ms=[],
                                 bytes_per_frame=int(np.mean([sum(map(len, f)) for f in files[(q, r)]])))
           for q, r in VARIANTS}
    stream = dict(jpeg_fps=[], cv2_pool_fps=[])
    for _ in range(args.runs):
        for q, r in VARIANTS:
            d = res[f'q{q}_rst_{r}']
            d['decode_ms'].append(round(decode_ms(dec, files[(q, r)], args.frames), 3))
            d['host_ms'].append(round(host_ms(dec, files[(q, r)]), 3))
            d['cv2_1core_ms'].append(round(cv2_ms(files[(q, r)][0]), 2))
            d['cv2_pool_ms'].append(round(cv2_ms(files[(q, r)][0], pool), 2))
        for name, fn in (('jpeg_fps', run_jpeg), ('cv2_pool_fps', run_cv2)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(args.frames)
            torch.cuda.synchronize()
            stream[name].append(round(args.frames / (time.perf_counter() - t0), 2))
    torch.cuda.synchronize()
    assert dec.status() == 0
    stream.update(jpeg_upload_bytes_per_frame=res['q95_rst_0']['bytes_per_frame'], u8_upload_bytes_per_frame=NC * SRC_HW[0] *
                  SRC_HW[1] * 3, outputs_byte_identical=identical)
    print(json.dumps(dict(card=card(), host_cores=cores, frames=args.frames, runs=args.runs, layers=args.layers,
                          content='synthetic camera-like gradient + noise, 4:2:0', decode=res, stream_host=stream)))


if __name__ == '__main__':
    main()
