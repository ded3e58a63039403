"""Temporal (video) inference with the BEV history kept inside the engine (occb200_engine_set_history, _forward_video,
_submit_host_video).  Every comparison is byte for byte (torch.equal) against the explicit path the caller would otherwise
run: occb200_engine_forward(prev_bev = the previous frame's bev_embed) with set_prev_rotation(map of the frame's angle)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occnet_b200 import fixtures

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'

# scene A: frames 0-4, scene B: frames 5-7 (can_bus[-1] angles in degrees)
ANGLES = [0.0, 2.0, -3.0, 1.5, 4.0, -1.0, 0.0, 2.5]
STARTS = [True, False, False, False, False, True, False, False]
WANT = ('bev_embed', 'occ', 'flow', 'occ_cls_i64')
NORMS_SHIPPED = ((103.530, 116.280, 123.675), (1.0, 1.0, 1.0))


def _isolated(call, timeout=900):
    """Tensor-core runs happen in a child process: a device fault there must not poison this session's context."""
    code = f"import sys; sys.path.insert(0, 'tests'); import test_video_engine_gpu as t; t.{call}; print('OK')"
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and 'OK' in r.stdout, f'child failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'


def _engine(cfg, precision, tc, seed=2):
    from occnet_b200.engine import OccEngine
    eng = OccEngine(cfg, fixtures.init_params(cfg, seed=seed), precision=precision, use_tensor_cores=tc, device=DEV)
    eng.set_cameras(fixtures.make_img_metas(cfg, bs=1))
    return eng


def _small6(precision, tc, n=8):
    cfg = fixtures.make_cfg('small6', num_layers=2, rotate_center=[20, 20])
    eng = _engine(cfg, precision, tc)
    frames = [[f[0].to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=200 + i)] for i in range(n)]
    return cfg, eng, frames


def _rot(cfg, angle):
    from occnet_b200.engine import rotation_index_map
    return rotation_index_map(cfg['bev_h'], cfg['bev_w'], angle, cfg.get('rotate_center', [100, 100]))


def _clone(out):
    return {k: v.clone() for k, v in out.items()}


def explicit_loop(eng, cfg, frames, angles, starts, want=WANT):
    """what a caller does without the history: bev_embed back in as prev_bev, the global rotation map set per frame"""
    outs, prev = [], None
    for fr, a, s in zip(frames, angles, starts):
        if s:
            prev = None
        eng.set_prev_rotation(_rot(cfg, a) if prev is not None else None)
        o = _clone(eng.forward(fr, prev_bev=prev, want=tuple(set(want) | {'bev_embed'})))
        outs.append(o)
        prev = o['bev_embed']
    eng.set_prev_rotation(None)
    return outs


def video_loop(eng, frames, angles, starts, want=WANT):
    eng.set_history(True)
    return [_clone(eng.forward_video(fr, rotation=a, scene_start=s, want=want)) for fr, a, s in zip(frames, angles, starts)]


def assert_frames_equal(got, want, keys):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        for k in keys:
            assert g[k].dtype == w[k].dtype and torch.equal(g[k], w[k]), (i, k, (g[k].double() - w[k].double()).abs().max().item())


# ---------------------------------------------------------------------------------------------- 1. device path, small6
def check_video_equals_explicit(precision, tc):
    cfg, eng, frames = _small6(precision, tc)
    ref = explicit_loop(eng, cfg, frames, ANGLES, STARTS)
    with_bev = video_loop(eng, frames, ANGLES, STARTS)
    n_video = eng.launches_per_frame
    assert_frames_equal(with_bev, ref, WANT)
    no_bev = video_loop(eng, frames, ANGLES, STARTS, want=('occ', 'flow', 'occ_cls_i64'))     # lift_from_t32 on the fused path
    assert 'bev_embed' not in no_bev[0]
    assert_frames_equal(no_bev, ref, ('occ', 'flow', 'occ_cls_i64'))
    assert eng.launches_per_frame <= n_video
    # the history matters: a temporal frame differs from the same frame in self mode
    self_mode = eng.forward(frames[3], want=('flow',))['flow']
    assert not torch.equal(self_mode, ref[3]['flow'])


@pytest.mark.parametrize('precision,tc', [('fp32', False), ('fp32', True), ('bf16', True)])
def test_video_equals_explicit_prev_bev(precision, tc):
    if tc:
        _isolated(f'check_video_equals_explicit({precision!r}, True)')
    else:
        check_video_equals_explicit(precision, tc)


# ------------------------------------------------------------------------------------------ 2. full size, six layers
def check_full_size():
    cfg = fixtures.make_cfg('full', num_layers=6)
    eng = _engine(cfg, 'bf16', True)
    frames = [[f[0].to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=300 + i)] for i in range(4)]
    angles, starts = [0.0, 3.0, -2.0, 1.0], [True, False, False, True]          # three frames, then a reset
    ref = explicit_loop(eng, cfg, frames, angles, starts)
    assert_frames_equal(video_loop(eng, frames, angles, starts), ref, WANT)
    assert_frames_equal(video_loop(eng, frames, angles, starts, want=('occ', 'flow', 'occ_cls_i64')), ref,
                        ('occ', 'flow', 'occ_cls_i64'))


def test_full_size_six_layers_bf16_video():
    _isolated('check_full_size()', timeout=1200)


# ---------------------------------------------------------------------------------------------- 3. pipelined host path
def _host_stream_alternating(eng, items):
    """two frames in flight, the caller's stream switching between submits"""
    streams = [torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)]
    X, Y, Z = eng.vox_shape
    outs = [(torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(), torch.empty((X, Y, Z, 2)).pin_memory()) for _ in range(2)]
    got, pending = [], []
    for i, (fr, a, s) in enumerate(items):
        if len(pending) == 2:
            j = pending.pop(0)
            eng.wait_host(j & 1)
            got.append((outs[j & 1][0].clone(), outs[j & 1][1].clone()))
        with torch.cuda.stream(streams[i % 2]):
            eng.submit_host_video(i & 1, fr, *outs[i & 1], rotation=a, scene_start=s)
        pending.append(i)
    for j in pending:
        eng.wait_host(j & 1)
        got.append((outs[j & 1][0].clone(), outs[j & 1][1].clone()))
    return got


def _check_host_paths(eng, dev_frames, host_frames):
    dev = [(o['occ_cls_i64'].cpu(), o['flow'].cpu())
           for o in video_loop(eng, dev_frames, ANGLES, STARTS, want=('flow', 'occ_cls_i64'))]
    items = list(zip(host_frames, ANGLES, STARTS))
    eng.set_history(True)
    got = [(o.clone(), f.clone()) for o, f in eng.stream_host_video(items)]
    eng.set_history(True)
    got_alt = _host_stream_alternating(eng, items)
    for i in range(len(dev)):
        for g in (got, got_alt):
            assert torch.equal(g[i][0], dev[i][0]) and torch.equal(g[i][1], dev[i][1]), i


def check_host_fp32_features(precision, tc):
    cfg, eng, frames = _small6(precision, tc)
    host = [[f.cpu().contiguous().pin_memory() for f in fr] for fr in frames]
    _check_host_paths(eng, frames, host)


@pytest.mark.parametrize('precision,tc', [('fp32', False), ('bf16', True)])
def test_host_video_pipeline_equals_device_video(precision, tc):
    if tc:
        _isolated(f'check_host_fp32_features({precision!r}, True)')
    else:
        check_host_fp32_features(precision, tc)


def check_host_camera_frames(precision):
    """input dtype 3: uint8 frames through the attached backbone, on the device and from pinned host buffers"""
    from occnet_b200.backbone import BackboneEngine
    cfg = fixtures.make_cfg('small6', num_layers=2, img_shape=(232, 400, 3), rotate_center=[20, 20])
    eng = _engine(cfg, precision, precision == 'bf16')
    be = BackboneEngine(fixtures.init_backbone_params(seed=5), 6, (232, 400), precision=precision,
                        use_tensor_cores=precision == 'bf16', device=DEV)
    be.set_frame_format((220, 400), *NORMS_SHIPPED, False)
    eng.attach_backbone(be)
    eng.set_input_dtype(torch.uint8)
    host = [torch.from_numpy(np.random.default_rng(40 + i).integers(0, 256, size=(6, 220, 400, 3), dtype=np.uint8))
            for i in range(len(ANGLES))]
    _check_host_paths(eng, [h.to(DEV) for h in host], [h.pin_memory() for h in host])
    eng.attach_backbone(None)


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_host_video_camera_frames(precision):
    _isolated(f'check_host_camera_frames({precision!r})')


# ------------------------------------------------------------------------------------ 4./5. self mode and isolation
def test_self_mode_frames_and_isolation_from_the_other_calls():
    """a scene-start frame and the first frame after set_history(1) equal forward(prev_bev=None), launch count included; a
    plain forward between video frames and the global set_prev_rotation map leave the video frames alone"""
    cfg, eng, frames = _small6('fp32', False, n=4)
    plain = [_clone(eng.forward(fr, want=WANT)) for fr in frames]
    n_plain = eng.launches_per_frame
    eng.set_history(True)
    v0 = _clone(eng.forward_video(frames[0], rotation=5.0, want=WANT))      # first frame: self mode, the angle is unused
    assert_frames_equal([v0], plain[:1], WANT)
    assert eng.launches_per_frame == n_plain
    # plain forwards (one with a prev_bev and a global map) between video frames
    eng.set_prev_rotation(_rot(cfg, 7.0))
    eng.forward(frames[3], prev_bev=torch.randn(eng.Nq, 256, device=DEV))
    eng.forward(frames[2])
    v1 = _clone(eng.forward_video(frames[1], rotation=2.0, want=WANT))
    v2 = _clone(eng.forward_video(frames[2], want=WANT))                     # no rotation; the global map must not apply
    v3 = _clone(eng.forward_video(frames[3], rotation=-1.0, scene_start=True, want=WANT))
    eng.set_prev_rotation(_rot(cfg, 2.0))
    r1 = _clone(eng.forward(frames[1], prev_bev=plain[0]['bev_embed'], want=WANT))
    eng.set_prev_rotation(None)
    r2 = _clone(eng.forward(frames[2], prev_bev=r1['bev_embed'], want=WANT))
    assert_frames_equal([v1, v2, v3], [r1, r2, plain[3]], WANT)
    # set_history(1) mid-stream starts a new scene
    eng.set_history(True)
    assert_frames_equal([_clone(eng.forward_video(frames[1], rotation=2.0, want=WANT))], plain[1:2], WANT)


# ------------------------------------------------------------------------------------------------ 6. rejected calls
def test_rejected_calls_leave_the_history_unchanged():
    from occnet_b200 import _lib
    cfg, eng, frames = _small6('fp32', False, n=5)
    angles, starts = [0.0, 2.0, -3.0, 1.5, 4.0], [True, False, False, False, False]
    ref = explicit_loop(eng, cfg, frames, angles, starts)
    with pytest.raises(_lib.OccB200Error, match='history not enabled'):
        eng.forward_video(frames[0])
    host = [[f.cpu().contiguous().pin_memory() for f in fr] for fr in frames]
    X, Y, Z = eng.vox_shape
    outs = [(torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(), torch.empty((X, Y, Z, 2)).pin_memory()) for _ in range(2)]
    with pytest.raises(_lib.OccB200Error, match='history not enabled'):
        eng.submit_host_video(0, host[0], *outs[0])
    eng.set_history(True)
    o = eng.forward_video(frames[0], want=WANT)
    assert_frames_equal([_clone(o)], ref[:1], WANT)
    bad = _rot(cfg, angles[1]).copy()
    bad[17] = eng.Nq
    with pytest.raises(_lib.OccB200Error, match='out of range'):
        eng.submit_host_video(0, host[1], *outs[0], rotation=bad)
    eng.submit_host_video(0, host[1], *outs[0], rotation=angles[1])
    with pytest.raises(_lib.OccB200Error, match='in flight'):
        eng.submit_host_video(0, host[2], *outs[0], rotation=angles[2])          # busy slot
    eng.wait_host(0)
    assert torch.equal(outs[0][0], ref[1]['occ_cls_i64'].cpu()) and torch.equal(outs[0][1], ref[1]['flow'].cpu())
    with pytest.raises(ValueError, match='range'):
        eng.forward_video(frames[2], rotation=bad, want=WANT)                # a host map on the device path
    # after every rejection the next valid frames still continue the sequence
    eng.submit_host_video(1, host[2], *outs[1], rotation=angles[2])
    eng.wait_host(1)
    assert torch.equal(outs[1][0], ref[2]['occ_cls_i64'].cpu()) and torch.equal(outs[1][1], ref[2]['flow'].cpu())
    assert_frames_equal([_clone(eng.forward_video(frames[3], rotation=angles[3], want=WANT))], ref[3:4], WANT)
    eng.set_history(False)
    with pytest.raises(_lib.OccB200Error, match='history not enabled'):
        eng.forward_video(frames[2])
    # device maps with entries outside [-1, Nq) read those rows as zeros: equal to the map with -1 there
    good = _rot(cfg, angles[2])
    wild, clean = good.copy(), good.copy()
    idx = np.arange(0, eng.Nq, 7)
    wild[idx] = np.where(idx % 2 == 0, eng.Nq + 5, -9)
    wild[3] = np.iinfo(np.int32).max
    clean[idx] = -1
    clean[3] = -1
    runs = []
    for m in (wild, clean):
        eng.set_history(True)
        eng.forward_video(frames[0])
        eng.forward_video(frames[1], rotation=angles[1])
        runs.append(_clone(eng.forward_video(frames[2], rotation=torch.from_numpy(m).to(DEV), want=WANT)))
    assert_frames_equal(runs[:1], runs[1:], WANT)
    assert not torch.equal(runs[0]['bev_embed'], ref[2]['bev_embed'])         # the zeroed rows changed the frame


# ------------------------------------------------------------------------------------ 7. hoisted queue-1 value maps
def check_temporal_digests(names):
    """The explicit temporal path's outputs equal, bit for bit, those of the engine that recomputed TSA's queue-1
    value_proj(bev_queries) in every layer of every frame (tests/golden/gen_temporal_digests.py wrote the digests); and the
    video path gives the same bits."""
    import json
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import gen_temporal_digests as G
    want = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'temporal_digests.json')))
    for name, kw, p, tc, angles in G.CASES:
        if name in names:
            assert G.run_case(kw, p, tc, angles) == want[name], name


def test_hoisted_query_values_keep_every_output_bit():
    check_temporal_digests(['small6_fp32'])
    _isolated("check_temporal_digests(['small6_fp32_tc', 'small6_bf16_tc', 'full6_bf16_tc'])", timeout=1200)
