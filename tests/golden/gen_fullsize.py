"""Full-size goldens (BASELINE configs[1]/[3]: 6 cams, 200x200 BEV, 6 encoder layers, 200x200x16 voxels).

    python tests/golden/gen_fullsize.py          # ~1 min on 8 threads; writes full6_fp32.npz, full6_bf16.npz

The oracle finishes a full frame in ~15 s, but GPU-box minutes are budgeted, so the `-m gpu` tests compare against
these committed vectors instead of re-running the oracle there:

  full6_fp32.npz   oracle/bevformer_occ.py (pinned bit-exactly against the unmodified reference modules by
                   gen_golden.py): seeded subsamples of every per-layer tap (TSA out, SCA out, layer out), bev_embed,
                   voxel features, occ logits, flow; the full argmax class volume (uint8) and flow volume (fp16);
                   the 187 Ray-mIoU counters of (oracle prediction vs the synthetic GT scene).
  full6_bf16.npz   oracle/bf16_model.py (same algorithm, rounded at the bf16 engine's storage points): subsamples of
                   bev_embed / voxel / occ / flow, the full class volume, the counters.

Inputs are regenerated from seeds on the test side (fixtures.make_feats(seed=100), init_params(seed=2, FREE_BIAS)).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from occnet_b200 import fixtures                    # noqa: E402
from oracle import bevformer_occ as O               # noqa: E402
from oracle import bf16_model as B                  # noqa: E402
from oracle import ray_metrics as ORM               # noqa: E402

from sampling import N_OUT, N_TAP, sub_idx         # noqa: E402  (tests/golden/sampling.py)


def case(prev=False):
    cfg = fixtures.make_cfg('full', num_layers=6)
    params = fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS)
    feats = fixtures.make_feats(cfg, bs=1, seed=100)
    metas = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=3.0 if prev else None)
    pb = None
    if prev:
        pb = torch.randn(1, cfg['bev_h'] * cfg['bev_w'], cfg['embed_dims'], generator=torch.Generator().manual_seed(3))
    return cfg, params, feats, metas, pb


def sub(key, t, n):
    flat = t.reshape(-1)
    return flat[torch.from_numpy(sub_idx(key, flat.numel(), n))].numpy().astype(np.float32)


def ray_counters(occ_cls, flow):
    sem_gt, flow_gt = fixtures.make_occ_scene(seed=4)
    orig = fixtures.make_ray_origins(T=8)
    fin, cnt = ORM.main([occ_cls.astype(np.uint8)], [sem_gt], [flow.astype(np.float32)], [flow_gt], [orig])
    return ORM.counters_to_vector(cnt), fin


def pack_outputs(out, d):
    for k in ('bev_embed', 'occ', 'flow'):
        d[k + '_sub'] = sub(k, out[k], N_OUT)
        d[k + '_shape'] = np.asarray(out[k].shape)
    cls = out['occ'].argmax(-1)[0].numpy().astype(np.uint8)
    d['occ_cls'] = cls
    # the metric reads the reference flow only at voxels whose class carries flow (ray_metrics.py:26-29, 178-185): stored there
    flow = out['flow'][0].numpy()
    d['flow_f16'] = np.where(cls[..., None] < ORM.FLOW_CLASSES, flow, 0).astype(np.float16)
    d['counters'], fin = ray_counters(cls, out['flow'][0].numpy())
    d['miou'], d['mave'] = fin['miou'], fin['mave']
    return fin


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    for prev in (False, True):
        tag = '_prev' if prev else ''
        cfg, params, feats, metas, pb = case(prev)
        taps = {}
        with torch.no_grad():
            want = O.head_forward(params, cfg, feats, metas, prev_bev=None if pb is None else pb.clone(), taps=taps)
        d = {}
        for l in range(cfg['num_layers']):
            for name in ('tsa', 'sca', ''):
                key = f'layer{l}' + ('_' + name if name else '')
                d[key + '_sub'] = sub(key, taps[key][0], N_TAP)
        d['voxel_sub'] = sub('voxel', taps['voxel_feats'][0], N_OUT)
        fin = pack_outputs(want, d)
        if prev:                                                   # the temporal golden only pins the outputs
            d = {k: v for k, v in d.items() if not k.startswith('layer') and k not in ('flow_f16',)}
        np.savez_compressed(os.path.join(HERE, f'full6{tag}_fp32.npz'), **d)
        hist = np.bincount(d['occ_cls'].reshape(-1), minlength=17)
        print(f'fp32{tag}: free voxels {hist[16] / hist.sum():.3f}, miou vs GT scene {fin["miou"]:.4f}, mave {fin["mave"]:.4f}')
        got = B.head_forward(params, cfg, feats, metas, prev_bev=pb, quant=True)
        e = {}
        e['voxel_sub'] = sub('voxel', got['voxel'][0], N_OUT)
        fin = pack_outputs(got, e)
        e.pop('flow_f16')
        np.savez_compressed(os.path.join(HERE, f'full6{tag}_bf16.npz'), **e)
        agree = (e['occ_cls'] == d['occ_cls']).mean()
        print(f'bf16 model{tag}: max|bev - fp32| {(got["bev_embed"] - want["bev_embed"]).abs().max():.4f}, '
              f'max|occ - fp32| {(got["occ"] - want["occ"]).abs().max():.4f}, class agreement {agree:.4f}, '
              f'miou vs GT scene {fin["miou"]:.4f}')


if __name__ == '__main__':
    main()
