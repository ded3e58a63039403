"""The prev_bev rotation computed on the device from an angle (occb200_engine_rotation_map, _forward_video_angle,
_submit_host_video_angle, _set_prev_rotation_angle) against the same rotation given as torchvision's index map
(`rotation_index_map`).  Maps must be equal cell for cell; frames byte for byte (torch.equal)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occnet_b200 import fixtures
from occnet_b200.engine import rotation_index_map

import test_rotation_cpu as RC
import test_video_engine_gpu as V

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'

# a new angle every frame, scene A: frames 0-4, scene B: frames 5-8
ANGLES = [0.37, 2.71, -3.14, 11.5, -0.004, 179.999, -90.0, 4.2, -17.25]
STARTS = [True, False, False, False, False, True, False, False, False]
WANT = ('bev_embed', 'occ', 'flow', 'occ_cls_i64')


def _isolated(call, timeout=900):
    """tensor-core runs happen in a child process: a device fault there must not poison this session's context"""
    code = f"import sys; sys.path.insert(0, 'tests'); import test_rotation_gpu as t; t.{call}; print('OK')"
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and 'OK' in r.stdout, f'child failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'


def _maps(cfg, angles):
    return [rotation_index_map(cfg['bev_h'], cfg['bev_w'], a, cfg.get('rotate_center', [100, 100])) for a in angles]


# ------------------------------------------------------------------------------------------------ 1. the device map
def test_device_rotation_map_equals_torchvision_and_golden():
    from occnet_b200.engine import OccEngine
    for h, w, center, angles, digests in RC.golden_cases():
        cfg = fixtures.make_cfg('toy', bev_h=h, bev_w=w, rotate_center=list(center))
        eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2), precision='fp32', device=DEV)
        extra = RC.angle_set(21 + h, 300, 200) if h == 200 else []
        for k, a in enumerate(list(angles) + list(extra)):
            got = eng.rotation_map(a).cpu().numpy()
            want = rotation_index_map(h, w, float(a), center)
            assert np.array_equal(got, want), (float(a), h, w, center, RC._mismatch(got, want, w))
            if k < len(digests):
                assert RC.map_digest(got) == digests[k], (float(a), h, w, center)


# ----------------------------------------------------------------------------------- 2. device video path, small6
def check_video_angle_equals_map(precision, tc):
    cfg, eng, frames = V._small6(precision, tc, n=len(ANGLES))
    maps = [torch.from_numpy(m).to(DEV) for m in _maps(cfg, ANGLES)]
    eng.set_history(True)
    by_map = [V._clone(eng.forward_video(fr, rotation=m, scene_start=s, want=WANT)) for fr, m, s in zip(frames, maps, STARTS)]
    n_map = eng.launches_per_frame
    by_angle = V.video_loop(eng, frames, ANGLES, STARTS)
    assert eng.launches_per_frame == n_map
    V.assert_frames_equal(by_angle, by_map, WANT)
    # host numpy maps (uploaded per frame) agree too, and the angles are not all the identity
    eng.set_history(True)
    host = [V._clone(eng.forward_video(fr, rotation=m, scene_start=s, want=WANT))
            for fr, m, s in zip(frames, _maps(cfg, ANGLES), STARTS)]
    V.assert_frames_equal(host, by_map, WANT)
    eng.set_history(True)
    unrotated = [V._clone(eng.forward_video(fr, scene_start=s, want=WANT)) for fr, s in zip(frames, STARTS)]
    assert not torch.equal(unrotated[3]['bev_embed'], by_angle[3]['bev_embed'])


@pytest.mark.parametrize('precision,tc', [('fp32', False), ('fp32', True), ('bf16', False), ('bf16', True)])
def test_video_angle_equals_video_map(precision, tc):
    if tc:
        _isolated(f'check_video_angle_equals_map({precision!r}, True)')
    else:
        check_video_angle_equals_map(precision, tc)


def check_full_size_launches():
    """the shipped size (6 layers, bf16, tensor cores): 55 launches per temporal video frame with a map or an angle"""
    cfg = fixtures.make_cfg('full', num_layers=6)
    eng = V._engine(cfg, 'bf16', True)
    frames = [[f[0].to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=300 + i)] for i in range(3)]
    angles, starts = [1.25, -2.5, 0.75], [True, False, False]
    maps = [torch.from_numpy(m).to(DEV) for m in _maps(cfg, angles)]
    want = ('flow', 'occ_cls_i64')
    eng.set_history(True)
    by_map, counts = [], []
    for fr, m, s in zip(frames, maps, starts):
        by_map.append(V._clone(eng.forward_video(fr, rotation=m, scene_start=s, want=want)))
        counts.append(eng.launches_per_frame)
    eng.set_history(True)
    by_angle = []
    for fr, a, s in zip(frames, angles, starts):
        by_angle.append(V._clone(eng.forward_video(fr, rotation=a, scene_start=s, want=want)))
        assert eng.launches_per_frame == counts[len(by_angle) - 1]
    assert counts[1:] == [55, 55], counts
    V.assert_frames_equal(by_angle, by_map, want)


def test_full_size_video_angle_launches():
    _isolated('check_full_size_launches()', timeout=1200)


# ------------------------------------------------------------------------------------------- 3. pipelined host path
def _host_angle_equals_device_map(eng, cfg, dev_frames, host_frames):
    maps = [torch.from_numpy(m).to(DEV) for m in _maps(cfg, ANGLES)]
    eng.set_history(True)
    dev = [(o['occ_cls_i64'].cpu(), o['flow'].cpu()) for o in
           (V._clone(eng.forward_video(fr, rotation=m, scene_start=s, want=('flow', 'occ_cls_i64')))
            for fr, m, s in zip(dev_frames, maps, STARTS))]
    items = list(zip(host_frames, ANGLES, STARTS))
    eng.set_history(True)
    got = [(o.clone(), f.clone()) for o, f in eng.stream_host_video(items)]
    eng.set_history(True)
    got_alt = V._host_stream_alternating(eng, items)                  # the caller's stream switching between submits
    for i in range(len(dev)):
        for g in (got, got_alt):
            assert torch.equal(g[i][0], dev[i][0]) and torch.equal(g[i][1], dev[i][1]), i


def check_host_features(precision, tc):
    cfg, eng, frames = V._small6(precision, tc, n=len(ANGLES))
    _host_angle_equals_device_map(eng, cfg, frames, [[f.cpu().contiguous().pin_memory() for f in fr] for fr in frames])


def check_host_camera_frames(precision):
    from occnet_b200.backbone import BackboneEngine
    cfg = fixtures.make_cfg('small6', num_layers=2, img_shape=(232, 400, 3), rotate_center=[20, 20])
    eng = V._engine(cfg, precision, precision == 'bf16')
    be = BackboneEngine(fixtures.init_backbone_params(seed=5), 6, (232, 400), precision=precision,
                        use_tensor_cores=precision == 'bf16', device=DEV)
    be.set_frame_format((220, 400), *V.NORMS_SHIPPED, False)
    eng.attach_backbone(be)
    eng.set_input_dtype(torch.uint8)
    host = [torch.from_numpy(np.random.default_rng(60 + i).integers(0, 256, size=(6, 220, 400, 3), dtype=np.uint8))
            for i in range(len(ANGLES))]
    _host_angle_equals_device_map(eng, cfg, [h.to(DEV) for h in host], [h.pin_memory() for h in host])
    eng.attach_backbone(None)


def test_host_video_angles_equal_device_maps():
    check_host_features('fp32', False)
    _isolated("check_host_features('bf16', True)")


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_host_video_angles_camera_frames(precision):
    _isolated(f'check_host_camera_frames({precision!r})')


# ---------------------------------------------------------------------------- 4. explicit prev_bev: set_prev_rotation
def check_prev_rotation_angle(precision, tc):
    cfg, eng, frames = V._small6(precision, tc, n=2)
    prev = V._clone(eng.forward(frames[0], want=WANT))['bev_embed']
    out = {}
    for name, rot in (('map', rotation_index_map(cfg['bev_h'], cfg['bev_w'], -7.75, cfg['rotate_center'])), ('angle', -7.75)):
        eng.set_prev_rotation(rot)
        out[name] = V._clone(eng.forward(frames[1], prev_bev=prev, want=WANT))
        n = eng.launches_per_frame
        out[name + '_n'] = n
    V.assert_frames_equal([out['angle']], [out['map']], WANT)
    assert out['angle_n'] == out['map_n']
    # the last call wins: an angle after a map, a map after an angle, None after an angle
    eng.set_prev_rotation(3.0)
    eng.set_prev_rotation(rotation_index_map(cfg['bev_h'], cfg['bev_w'], -7.75, cfg['rotate_center']))
    V.assert_frames_equal([V._clone(eng.forward(frames[1], prev_bev=prev, want=WANT))], [out['map']], WANT)
    eng.set_prev_rotation(rotation_index_map(cfg['bev_h'], cfg['bev_w'], 3.0, cfg['rotate_center']))
    eng.set_prev_rotation(-7.75)
    V.assert_frames_equal([V._clone(eng.forward(frames[1], prev_bev=prev, want=WANT))], [out['map']], WANT)
    eng.set_prev_rotation(None)
    plain = V._clone(eng.forward(frames[1], prev_bev=prev, want=WANT))
    assert not torch.equal(plain['bev_embed'], out['map']['bev_embed'])


@pytest.mark.parametrize('precision,tc', [('fp32', False), ('bf16', True)])
def test_prev_rotation_angle_equals_map(precision, tc):
    if tc:
        _isolated(f'check_prev_rotation_angle({precision!r}, True)')
    else:
        check_prev_rotation_angle(precision, tc)


# ------------------------------------------------------------------------------------------------------ 5. detector
SCENES = [('scene-a', 0.0), ('scene-a', 2.5), ('scene-a', -4.0), ('scene-a', 1.75), ('scene-b', -1.0), ('scene-b', 6.5),
          ('scene-b', -0.25)]


def _detectors(cfg, precision, frames):
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200.mmcv_shim import build_detector
    params = fixtures.init_params(cfg, seed=2)
    kw = dict(img_backbone=dict(type='ResNet', depth=50), img_neck=dict(type='FPN'), frame_pad=dict(size=(232, 400))) \
        if frames else {}
    dets = []
    for eh in (False, True):
        d = build_detector(dict(type='BEVFormerOcc', video_test_mode=True, temporal_test=True, engine_history=eh,
                                pts_bbox_head=dict(fixtures.head_cfg(cfg), precision=precision), **kw)).to(DEV).eval()
        d.pts_bbox_head.load_state_dict(params, strict=True)
        if frames:
            assert not d.load_state_dict(fixtures.init_backbone_params(seed=5), strict=False).unexpected_keys
        dets.append(d)
    return dets


def _metas(cfg, frames):
    out = []
    for tok, ang in SCENES:
        m = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=ang)
        m[0]['scene_token'] = tok
        if frames:
            m[0].pop('img_shape', None)
        out.append(m)
    return out


def check_detector(precision, frames):
    """temporal_test with engine_history against the prev_bev cache over two scenes: features handed over (img_feats), or
    uint8 camera frames through the native backbone"""
    if frames:
        cfg = fixtures.make_cfg('small6', num_layers=2, img_shape=(232, 400, 3), rotate_center=[20, 20])
        inputs = [dict(img=[torch.from_numpy(np.random.default_rng(90 + i).integers(0, 256, size=(1, 6, 220, 400, 3),
                                                                                    dtype=np.uint8)).to(DEV)])
                  for i in range(len(SCENES))]
    else:
        cfg = fixtures.make_cfg('small6', num_layers=2, rotate_center=[20, 20])
        inputs = [dict(img_feats=[f.to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=80 + i)]) for i in range(len(SCENES))]
    cache, hist = _detectors(cfg, precision, frames)
    metas = _metas(cfg, frames)
    want = [cache(return_loss=False, img_metas=[m], **x) for m, x in zip(metas, inputs)]
    got = [hist(return_loss=False, img_metas=[m], **x) for m, x in zip(metas, inputs)]
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g['occ_results'], w['occ_results']) and torch.equal(g['flow_results'], w['flow_results']), i
    assert hist.prev_frame_info['prev_bev'] is None and cache.prev_frame_info['prev_bev'] is not None
    # the history was used: a mid-scene frame differs from the same frame run as a scene start
    hist.prev_frame_info['scene_token'] = None
    fresh = hist(return_loss=False, img_metas=[metas[3]], **inputs[3])
    assert not torch.equal(fresh['flow_results'], got[3]['flow_results'])


def test_detector_engine_history_equals_prev_bev_cache():
    check_detector('fp32', False)
    _isolated("check_detector('bf16', False)")


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_detector_engine_history_camera_frames(precision):
    _isolated(f'check_detector({precision!r}, True)')
