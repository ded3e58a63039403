"""One-encoder-layer goldens at FULL size (6 cams, 200x200 BEV, 200x200x16 voxels) for the bf16 / tensor-core configuration.

    python tests/golden/gen_onelayer.py          # ~20 s; writes full1_bf16.npz, full1_prev_bf16.npz

Why: over SIX layers the bf16 path is chaotic in the rounding sense -- a 1-ulp difference in an fp32 accumulation order flips a
bf16 rounding somewhere, and that flip propagates as bf16-sized noise -- so against the storage-rounding model
(oracle/bf16_model.py) a six-layer engine run can only agree to about the model's own distance from the fp32 oracle.
After ONE layer few roundings have happened, so the
same comparison is tight and a wrong constant / index / layout in the fused path cannot hide behind the 6e-2 bar.
Both files hold seeded subsamples (tests/golden/sampling.py) of bev_embed / occ / flow from the fp32 oracle AND the model.
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
from sampling import N1, sub_idx                    # noqa: E402


def case(prev):
    cfg = fixtures.make_cfg('full', num_layers=1)
    params = fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS)
    feats = fixtures.make_feats(cfg, bs=1, seed=100)
    metas = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=3.0 if prev else None)
    pb = None
    if prev:
        pb = torch.randn(1, cfg['bev_h'] * cfg['bev_w'], cfg['embed_dims'], generator=torch.Generator().manual_seed(3))
    return cfg, params, feats, metas, pb


def sub(key, t):
    flat = t.reshape(-1)
    return flat[torch.from_numpy(sub_idx(key, flat.numel(), N1))].numpy().astype(np.float32)


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    for prev in (False, True):
        cfg, params, feats, metas, pb = case(prev)
        with torch.no_grad():
            want = O.head_forward(params, cfg, feats, metas, prev_bev=None if pb is None else pb.clone())
        got = B.head_forward(params, cfg, feats, metas, prev_bev=pb, quant=True)
        d = {}
        for k in ('bev_embed', 'occ', 'flow'):
            d[k + '_fp32_sub'] = sub(k, want[k])
            d[k + '_bf16_sub'] = sub(k, got[k])
            print(f'prev={prev} {k}: model vs fp32 max {np.abs(d[k + "_fp32_sub"] - d[k + "_bf16_sub"]).max():.4f} '
                  f'mean {np.abs(d[k + "_fp32_sub"] - d[k + "_bf16_sub"]).mean():.5f}')
        d['occ_cls_bf16'] = got['occ'].argmax(-1)[0].numpy().astype(np.uint8)
        d['occ_cls_fp32'] = want['occ'].argmax(-1)[0].numpy().astype(np.uint8)
        np.savez_compressed(os.path.join(HERE, 'full1_prev_bf16.npz' if prev else 'full1_bf16.npz'), **d)


if __name__ == '__main__':
    main()
