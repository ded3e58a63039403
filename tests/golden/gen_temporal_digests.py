"""SHA-256 digests of the explicit temporal path's outputs (occb200_engine_forward with a prev_bev and a rotation map) on
seeded inputs, written to tests/golden/temporal_digests.json and checked by tests/test_video_engine_gpu.py.

The digests were produced by the engine that still ran TSA's queue-1 value_proj(bev_queries) in every layer of every frame,
so the check shows that computing those maps once at finalize changes no output bit.  Run on an H100 from the repository
root:  python tests/golden/gen_temporal_digests.py [out.json]
"""
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from occnet_b200 import fixtures                                 # noqa: E402
from occnet_b200.engine import OccEngine, rotation_index_map     # noqa: E402

KEYS = ('bev_embed', 'occ', 'flow', 'occ_cls_i64')
# (name, config, precision, tensor cores, angles; frame 0 starts the scene, the others take the previous bev_embed)
CASES = [
    ('small6_fp32', dict(base='small6', num_layers=2, rotate_center=[20, 20]), 'fp32', False, [0.0, 2.0, -3.0]),
    ('small6_fp32_tc', dict(base='small6', num_layers=2, rotate_center=[20, 20]), 'fp32', True, [0.0, 2.0, -3.0]),
    ('small6_bf16_tc', dict(base='small6', num_layers=2, rotate_center=[20, 20]), 'bf16', True, [0.0, 2.0, -3.0]),
    ('full6_bf16_tc', dict(base='full', num_layers=6), 'bf16', True, [0.0, 3.0]),
]


def digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def run_case(kw, precision, tc, angles):
    kw = dict(kw)
    cfg = fixtures.make_cfg(kw.pop('base'), **kw)
    eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2), precision=precision, use_tensor_cores=tc, device='cuda:0')
    eng.set_cameras(fixtures.make_img_metas(cfg, bs=1))
    out, prev = [], None
    for i, a in enumerate(angles):
        feats = [f[0].to('cuda:0') for f in fixtures.make_feats(cfg, bs=1, seed=400 + i)]
        eng.set_prev_rotation(None if prev is None else rotation_index_map(cfg['bev_h'], cfg['bev_w'], a,
                                                                          cfg.get('rotate_center', [100, 100])))
        o = eng.forward(feats, prev_bev=prev, want=KEYS)
        out.append({k: digest(o[k]) for k in KEYS})
        prev = o['bev_embed'].clone()
    return out


def main():
    res = {name: run_case(kw, p, tc, a) for name, kw, p, tc, a in CASES}
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden', 'temporal_digests.json')
    with open(path, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
