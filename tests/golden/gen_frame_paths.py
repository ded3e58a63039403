"""Digests and launch schedules of every frame path of the engine, written to tests/golden/frame_paths.json and checked by
tests/test_frame_paths_gpu.py.

Each configuration runs one seeded sequence of frames through the public OccEngine API: self mode with and without
bev_embed, an explicit prev_bev rotated by a map and by an angle, a video run on the engine history (scene start, angle,
map), for bf16 a channels-last bf16 input frame, and for small6 a self frame and a prev_bev frame with taps on.  Every frame
records the SHA-256 of each output (and of each tap), launches_per_frame and the per-category launch counts of profile_read.
Run on an H100 from the repository root:  python tests/golden/gen_frame_paths.py [out.json]
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

ALL = ('bev_embed', 'occ', 'flow', 'occ_cls', 'occ_cls_i64')
NO_BEV = ('occ', 'flow', 'occ_cls', 'occ_cls_i64')
SMALL6 = dict(base='small6', num_layers=2, rotate_center=[20, 20])
# (name, config, precision, tensor cores)
CASES = [
    ('small6_fp32', SMALL6, 'fp32', False),
    ('small6_fp32_tc', SMALL6, 'fp32', True),
    ('small6_bf16', SMALL6, 'bf16', False),
    ('small6_bf16_tc', SMALL6, 'bf16', True),
    ('full6_bf16_tc', dict(base='full', num_layers=6), 'bf16', True),
]


def digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def run_case(kw, precision, tc):
    """-> {frame name: {'out': {output: sha256}, 'launches': n, 'categories': {category: launches}}}"""
    kw = dict(kw)
    small = kw['base'] == 'small6'
    cfg = fixtures.make_cfg(kw.pop('base'), **kw)
    eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2), precision=precision, use_tensor_cores=tc, device='cuda:0')
    eng.set_cameras(fixtures.make_img_metas(cfg, bs=1))
    eng.profile(True)
    rot_map = rotation_index_map(cfg['bev_h'], cfg['bev_w'], 2.0, cfg.get('rotate_center', [100, 100]))
    seed = iter(range(500, 600))
    res = {}

    def feats():
        return [f[0].to('cuda:0') for f in fixtures.make_feats(cfg, bs=1, seed=next(seed))]

    def record(name, out, taps=False):
        rec = {'out': {k: digest(v) for k, v in sorted(out.items())}, 'launches': eng.launches_per_frame,
               'categories': {k: n for k, (_, n) in eng.profile_read().items()}}
        if taps:
            for which in ('layer', 'tsa', 'sca'):
                for l in range(cfg['num_layers']):
                    rec['out'][f'tap_{which}{l}'] = digest(eng.tap(which, l))
        res[name] = rec
        return out

    prev = record('self', eng.forward(feats(), want=ALL))['bev_embed'].clone()
    record('self_no_bev', eng.forward(feats(), want=NO_BEV))
    eng.set_prev_rotation(rot_map)
    record('prev_map', eng.forward(feats(), prev_bev=prev, want=ALL))
    eng.set_prev_rotation(-3.0)
    record('prev_angle', eng.forward(feats(), prev_bev=prev, want=ALL))
    eng.set_prev_rotation(None)
    eng.set_history(True)
    record('video_start', eng.forward_video(feats(), scene_start=True, want=ALL))
    record('video_angle', eng.forward_video(feats(), rotation=1.5, want=NO_BEV))
    record('video_map', eng.forward_video(feats(), rotation=rot_map, want=ALL))
    eng.set_history(False)
    if precision == 'bf16':
        eng.set_input_dtype(torch.bfloat16, channels_last=True)
        nhwc = [f.to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2) for f in feats()]
        record('nhwc_bf16', eng.forward(nhwc, want=ALL))
        eng.set_input_dtype(torch.float32)
    if small:
        eng.enable_taps(True)
        record('taps_self', eng.forward(feats(), want=ALL), taps=True)
        eng.set_prev_rotation(rot_map)
        record('taps_prev', eng.forward(feats(), prev_bev=prev, want=ALL), taps=True)
        eng.enable_taps(False)
    return res


def main():
    res = {name: run_case(kw, p, tc) for name, kw, p, tc in CASES}
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden', 'frame_paths.json')
    with open(path, 'w') as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(json.dumps({n: {f: (r['launches'], r['categories']) for f, r in c.items()} for n, c in res.items()}))


if __name__ == '__main__':
    main()
