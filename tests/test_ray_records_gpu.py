"""Ray records cast inside the frame engine (ray_records_kernel; occb200_ray_records, occb200_engine_set_rays, _request_rays).
Every comparison is byte for byte: against `RayMetric.add_frame(..., return_pcd=True)`'s prediction rows narrowed by numpy
(what `format_results` writes today), against the oracle's C DDA, and between the engine's paths."""
import gzip
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from occnet_b200 import fixtures

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
KEYS = ('ray_cls', 'ray_dist', 'ray_flow')
NORMS_SHIPPED = ((103.530, 116.280, 123.675), (1.0, 1.0, 1.0))


def _isolated(call, timeout=900):
    """Tensor-core runs happen in a child process: a device fault there must not poison this session's context."""
    code = f"import sys; sys.path.insert(0, 'tests'); import test_ray_records_gpu as t; t.{call}; print('OK')"
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and 'OK' in r.stdout, f'child failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'


def bits(t):
    """the bytes of a tensor / array, so that NaN payloads and signed zeros count"""
    a = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.ascontiguousarray(a).view(np.uint8 if a.dtype.itemsize == 1 else np.uint16)


def narrow(pcd):
    """process_one_sample's rows as format_results narrows them"""
    return {'ray_cls': pcd[:, 0].astype(np.int8), 'ray_dist': pcd[:, 1].astype(np.float16),
            'ray_flow': np.ascontiguousarray(pcd[:, 2:4].astype(np.float16))}


def assert_records(got, want, what=''):
    for k in KEYS:
        g, w = bits(got[k]), bits(want[k])
        assert g.shape == w.shape and np.array_equal(g, w), (what, k, int((g != w).sum()))


def origins(T, dtype=np.float32, seed=0):
    """T origins inside the grid, off the voxel lattice"""
    rng = np.random.default_rng(seed)
    o = fixtures.make_ray_origins(T=T)[0].astype(np.float64)
    o += rng.uniform(-0.37, 0.37, o.shape)
    return np.ascontiguousarray(o[None], dtype)


# ----------------------------------------------------------------------------------------------------------- 1. operator
def scene(seed):
    sem, flow = fixtures.make_occ_scene(seed=seed)
    # 7e4 overflows fp16, 1.00048828125 = 1 + 2^-11 is halfway between two halves (rounds to the even 1.0), 65519.9 is the
    # largest neighbourhood that still rounds to 65504
    flow[sem < 8] += np.float32(1.00048828125)
    x, y, z = np.nonzero(sem != 16)
    pick = np.random.default_rng(seed).permutation(len(x))[:4000]
    special = np.array([7e4, -7e4, np.nan, 1.00048828125, 65519.9, 65520.0, 1e-8, -0.0], np.float32)
    flow[x[pick], y[pick], z[pick], 0] = special[np.arange(len(pick)) % len(special)]
    flow[x[pick], y[pick], z[pick], 1] = special[(np.arange(len(pick)) + 3) % len(special)]
    return sem, flow


def metric_rows(sem, flow, org):
    from occnet_b200.metric import RayMetric
    s, f = torch.from_numpy(sem), torch.from_numpy(flow)
    pp, _ = RayMetric(DEV).add_frame(s, f, s, f, torch.as_tensor(org), return_pcd=True)
    return pp.cpu().numpy()


def records(sem, flow, org):
    from occnet_b200 import ops
    c, d, f = ops.ray_records(torch.from_numpy(sem).to(DEV), torch.from_numpy(flow).to(DEV), org)
    return dict(zip(KEYS, (c, d, f)))


@pytest.mark.parametrize('T', [1, 3, 8])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_operator_equals_the_metric_kernel_rows_narrowed_by_numpy(T, dtype):
    sem, flow = scene(seed=30 + T)
    org = origins(T, dtype, seed=T)
    got = records(sem, flow, org)
    assert got['ray_cls'].dtype == torch.int8 and got['ray_dist'].dtype == torch.float16 and got['ray_flow'].shape == (T * 14040, 2)
    assert_records(got, narrow(metric_rows(sem, flow, org)), (T, dtype))
    assert np.isnan(got['ray_flow'].float().cpu().numpy()).any() and np.isinf(got['ray_flow'].float().cpu().numpy()).any()
    if dtype == np.float32:
        from oracle import ray_metrics as ORM
        assert_records(got, narrow(ORM.process_one_sample(sem, ORM.generate_lidar_rays(), org, flow)), ('oracle', T))


def test_operator_degenerate_volumes_and_origins():
    sem, flow = scene(seed=41)
    sem[0, 0, 0] = 9
    flow[0, 0, 0] = [2.5, -3.25]
    # one origin inside, one far outside the grid: none of its rays enters -> voxel (0,0,0)'s class and flow, distance -0.4
    org = np.array([[[0.3, -0.2, 1.8], [500.0, 500.0, 50.0]]], np.float32)
    got = records(sem, flow, org)
    assert_records(got, narrow(metric_rows(sem, flow, org)))
    out = {k: v[14040:].float().cpu().numpy() for k, v in got.items()}
    assert (out['ray_cls'] == 9).all() and (out['ray_dist'] == np.float32(np.float16(-0.4))).all()
    assert (out['ray_flow'] == np.array([2.5, -3.25], np.float32)).all()
    # an all-free volume: every ray leaves the grid, the record is the exit voxel's
    free = np.full_like(sem, 16)
    got = records(free, flow, org)
    assert_records(got, narrow(metric_rows(free, flow, org)))
    assert (got['ray_cls'].cpu().numpy() == 16).all() and (got['ray_dist'][:14040].float() > 0).all()


def test_operator_rejects_bad_tensors():
    from occnet_b200 import ops
    sem, flow = torch.zeros(200, 200, 16, dtype=torch.uint8, device=DEV), torch.zeros(200, 200, 16, 2, device=DEV)
    with pytest.raises(ValueError, match='1..8'):
        ops.ray_records(sem, flow, np.zeros((9, 3), np.float32))
    with pytest.raises(ValueError, match='200,200,16'):
        ops.ray_records(sem[:100].contiguous(), flow, np.zeros((1, 3), np.float32))
    with pytest.raises(RuntimeError, match='uint8'):
        ops.ray_records(sem.long(), flow, np.zeros((1, 3), np.float32))


# ------------------------------------------------------------------------------------------------------------- 2. engine
def grid_cfg(**kw):
    """the metric's 200 x 200 x 16 grid over the small six-camera feature levels"""
    return fixtures.make_cfg('small6', bev_h=200, bev_w=200, num_layers=1, **kw)


def _engine(cfg, precision):
    from occnet_b200.engine import OccEngine
    eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS), precision=precision,
                    use_tensor_cores=precision == 'bf16', device=DEV)
    eng.set_cameras(fixtures.make_img_metas(cfg, bs=1))
    return eng


def _frames(cfg, n, seed=500):
    return [[f[0].to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=seed + i)] for i in range(n)]


def op_records(out, org):
    from occnet_b200 import ops
    return dict(zip(KEYS, ops.ray_records(out['occ_cls'], out['flow'], org)))


def check_engine_forward(precision):
    from occnet_b200 import _lib
    cfg = grid_cfg()
    eng = _engine(cfg, precision)
    fr = _frames(cfg, 2)
    want = ('bev_embed', 'occ', 'flow', 'occ_cls', 'occ_cls_i64')
    plain = {k: v.clone() for k, v in eng.forward(fr[0], want=want).items()}
    n_plain = eng.launches_per_frame
    org = origins(3, np.float64, seed=7)
    out = eng.forward(fr[0], want=want, ray_origins=org)
    assert eng.launches_per_frame == n_plain + 1
    for k in want:                                                     # the caller's outputs keep every byte
        assert torch.equal(out[k], plain[k]), k
    assert_records(out, op_records(out, org), 'armed forward')
    # no volume requested at all: the engine's own u8 / flow buffers feed the ray cast
    only = eng.forward(fr[0], want=('bev_embed',), ray_origins=org)
    assert_records(only, out, 'no volumes')
    # one-shot: the next frame leaves sentinel-filled record buffers alone
    bufs = eng.ray_buffers(3)
    for v in bufs.values():
        v.fill_(77)
    with eng._ray_request(org, bufs):
        eng.forward(fr[1], want=('flow',))
    n_armed = eng.launches_per_frame
    first = {k: v.clone() for k, v in bufs.items()}
    for v in bufs.values():
        v.fill_(77)
    eng.forward(fr[0], want=('flow',))
    torch.cuda.synchronize()
    assert all((v == 77).all() for v in bufs.values()) and not (first['ray_cls'] == 77).all()
    assert eng.launches_per_frame == n_armed - 1
    # rejections leave nothing armed
    for bad, msg in ((np.zeros((9, 3), np.float32), None), (np.array([[0, np.nan, 0]], np.float32), 'finite')):
        with pytest.raises((ValueError, _lib.OccB200Error), match=msg):
            eng.forward(fr[0], want=('flow',), ray_origins=bad)
    o = np.ascontiguousarray(org.reshape(-1, 3))
    rc = eng.lib.occb200_engine_request_rays(eng._h, _lib.ptr(o), 1, 3, _lib.ptr(bufs['ray_cls']), None, _lib.ptr(bufs['ray_flow']))
    assert rc == 1 and 'null pointer' in eng.lib.occb200_last_error().decode()
    eng.forward(fr[0], want=('flow',))
    torch.cuda.synchronize()
    assert all((v == 77).all() for v in bufs.values())
    # host calls without a request still need both volumes
    host = [f.cpu().contiguous().pin_memory() for f in fr[0]]
    with pytest.raises(_lib.OccB200Error, match='null pointer'):
        eng.submit_host(0, host, None, None)
    occ, flow, rec = eng.forward_host(host, ray_origins=org)
    assert torch.equal(occ, plain['occ_cls_i64'].cpu()) and torch.equal(flow, plain['flow'].cpu())
    assert_records(rec, out, 'forward_host')
    occ, flow, rec = eng.forward_host(host, ray_origins=org, volumes=False)
    assert occ is None and flow is None
    assert_records(rec, out, 'forward_host, no volumes')


def test_engine_forward_fp32():
    check_engine_forward('fp32')


def test_engine_forward_bf16():
    _isolated("check_engine_forward('bf16')")


def test_request_needs_a_ray_bundle_and_the_metric_grid():
    from occnet_b200 import _lib
    eng = _engine(grid_cfg(), 'fp32')
    o = np.ascontiguousarray(origins(2)[0])
    buf = torch.empty(2 * 14040 * 2, dtype=torch.float16, device=DEV)
    rc = eng.lib.occb200_engine_request_rays(eng._h, _lib.ptr(o), 0, 2, _lib.ptr(buf), _lib.ptr(buf), _lib.ptr(buf))
    assert rc == 1 and 'set_rays' in eng.lib.occb200_last_error().decode()
    small = _engine(fixtures.make_cfg('small6', num_layers=1), 'fp32')
    with pytest.raises(_lib.OccB200Error, match='200 x 200 x 16'):
        small.forward(_frames(small.cfg, 1)[0], want=('flow',), ray_origins=o)


# ------------------------------------------------------------------------------------------- 3. video and the host pipeline
ANGLES = [0.0, 2.0, -3.0, 1.5, 4.0, -1.0]
STARTS = [True, False, False, False, True, False]
TS = [8, 1, 3, 8, 2, 5]                                                # consecutive slots carry different T and origins


def _check_paths(eng, dev_frames, host_frames):
    orgs = [origins(T, np.float64 if i % 2 else np.float32, seed=60 + i) for i, T in enumerate(TS)]
    eng.set_history(True)
    want = []
    for fr, a, s, o in zip(dev_frames, ANGLES, STARTS, orgs):
        out = eng.forward_video(fr, rotation=a, scene_start=s, want=('flow', 'occ_cls', 'occ_cls_i64'), ray_origins=o)
        assert_records(out, op_records(out, o), 'forward_video (angle)')
        want.append({k: v.cpu().clone() for k, v in out.items()})
    eng.set_history(True)
    for i, (fr, a, s, o) in enumerate(zip(dev_frames, ANGLES, STARTS, orgs)):
        out = eng.forward_video(fr, rotation=eng.rotation_map(a), scene_start=s, want=('flow',), ray_origins=o)
        assert_records(out, want[i], ('forward_video (map)', i))
    for volumes in (True, False):
        eng.set_history(True)
        items = list(zip(host_frames, ANGLES, STARTS, orgs))
        for i, (occ, flow, rec) in enumerate(eng.stream_host_video(items, volumes=volumes)):
            assert_records(rec, want[i], ('stream_host_video', volumes, i))
            if volumes:
                assert torch.equal(occ, want[i]['occ_cls_i64']) and torch.equal(flow, want[i]['flow']), i
            else:
                assert occ is None and flow is None
    # the plain pipeline against the plain device call
    plain = [eng.forward(fr, want=('flow', 'occ_cls_i64'), ray_origins=o) for fr, o in zip(dev_frames[:4], orgs)]
    plain = [{k: v.cpu() for k, v in p.items()} for p in plain]
    for volumes in (True, False):
        for i, (occ, flow, rec) in enumerate(eng.stream_host(host_frames[:4], ray_origins=orgs[:4], volumes=volumes)):
            assert_records(rec, plain[i], ('stream_host', volumes, i))
            if volumes:
                assert torch.equal(occ, plain[i]['occ_cls_i64']) and torch.equal(flow, plain[i]['flow']), i
    # and without origins the generators yield what they always did
    occ, flow = next(iter(eng.stream_host(host_frames[:1])))
    assert torch.equal(occ, plain[0]['occ_cls_i64']) and torch.equal(flow, plain[0]['flow'])


def check_paths_features(precision):
    cfg = grid_cfg()
    eng = _engine(cfg, precision)
    frames = _frames(cfg, len(TS))
    _check_paths(eng, frames, [[f.cpu().contiguous().pin_memory() for f in fr] for fr in frames])


def check_paths_camera_frames(precision):
    from occnet_b200.backbone import BackboneEngine
    cfg = grid_cfg(img_shape=(232, 400, 3))
    eng = _engine(cfg, precision)
    be = BackboneEngine(fixtures.init_backbone_params(seed=5), 6, (232, 400), precision=precision,
                        use_tensor_cores=precision == 'bf16', device=DEV)
    be.set_frame_format((220, 400), *NORMS_SHIPPED, False)
    eng.attach_backbone(be)
    eng.set_input_dtype(torch.uint8)
    host = [torch.from_numpy(np.random.default_rng(40 + i).integers(0, 256, size=(6, 220, 400, 3), dtype=np.uint8))
            for i in range(len(TS))]
    _check_paths(eng, [h.to(DEV) for h in host], [h.pin_memory() for h in host])
    eng.attach_backbone(None)


def test_video_and_host_pipeline_fp32_features():
    check_paths_features('fp32')


def test_video_and_host_pipeline_bf16_features():
    _isolated("check_paths_features('bf16')")


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_video_and_host_pipeline_camera_frames(precision):
    _isolated(f'check_paths_camera_frames({precision!r})')


# ----------------------------------------------------------------------------------------------------------- 4. detector
SCENES = [('scene-a', 0.0), ('scene-a', 2.5), ('scene-b', -1.0), ('scene-b', 6.5)]


def _detector(cfg, precision, **kw):
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200.mmcv_shim import build_detector
    d = build_detector(dict(type='BEVFormerOcc', pts_bbox_head=dict(fixtures.head_cfg(cfg), precision=precision), **kw)).to(DEV).eval()
    d.pts_bbox_head.load_state_dict(fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS), strict=True)
    return d


def check_detector(precision, tmp):
    from projects.mmdet3d_plugin.datasets.submission import format_results
    cfg = grid_cfg()
    inputs = [[f.to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=80 + i)] for i in range(len(SCENES))]
    metas = []
    for tok, ang in SCENES:
        m = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=ang)
        m[0]['scene_token'] = tok
        metas.append(m)
    orgs = [origins(T, np.float64, seed=90 + i) for i, T in enumerate((8, 2, 5, 8))]
    tokens = [f'tok{i}' for i in range(len(SCENES))]
    modes = {'plain': {}, 'cache': dict(video_test_mode=True, temporal_test=True),
             'history': dict(video_test_mode=True, temporal_test=True, engine_history=True)}
    files = {}
    for name, kw in modes.items():
        det = _detector(cfg, precision, **kw)
        vol = [det(return_loss=False, img_metas=[m], img_feats=x) for m, x in zip(metas, inputs)]
        assert all(set(v) == {'occ_results', 'flow_results'} for v in vol)            # without origins: the result as it was
        det.prev_frame_info['scene_token'] = None
        got = [det(return_loss=False, img_metas=[m], img_feats=x, lidar_origins=o) for m, x, o in zip(metas, inputs, orgs)]
        today = format_results(vol, tokens, orgs, submission_prefix=os.path.join(tmp, name, 'volumes'), device=DEV)
        for i, (g, v) in enumerate(zip(got, vol)):
            assert torch.equal(g['occ_results'], v['occ_results']) and torch.equal(g['flow_results'], v['flow_results']), (name, i)
            r = g['ray_results']
            assert not r['pcd_cls'].is_cuda and r['pcd_cls'].shape == (orgs[i].shape[1] * 14040,)
            for k in ('pcd_cls', 'pcd_dist', 'pcd_flow'):
                assert np.array_equal(bits(r[k]), bits(today['results'][tokens[i]][k])), (name, i, k)
        format_results(got, tokens, [None] * 4, submission_prefix=os.path.join(tmp, name, 'records'))
        # the choice is made per result: a list mixing results with and without records
        format_results([got[0], vol[1], got[2], vol[3]], tokens, [None, orgs[1], None, orgs[3]],
                       submission_prefix=os.path.join(tmp, name, 'mixed'), device=DEV)
        files[name] = [open(os.path.join(tmp, name, d, 'submission.gz'), 'rb').read() for d in ('volumes', 'records', 'mixed')]
        assert files[name][0] == files[name][1] == files[name][2], name
        assert len(pickle.loads(gzip.decompress(files[name][1]))['results']) == 4
        # ray_only: records only, no volumes
        only = _detector(cfg, precision, ray_only=True, **kw)
        res = [only(return_loss=False, img_metas=[m], img_feats=x, lidar_origins=o) for m, x, o in zip(metas, inputs, orgs)]
        assert all(r['occ_results'] is None and r['flow_results'] is None for r in res)
        format_results(res, tokens, [None] * 4, submission_prefix=os.path.join(tmp, name, 'only'))
        assert open(os.path.join(tmp, name, 'only', 'submission.gz'), 'rb').read() == files[name][0], name
        with pytest.raises(ValueError, match='lidar_origins'):
            only(return_loss=False, img_metas=[metas[0]], img_feats=inputs[0])
    assert files['cache'][0] == files['history'][0] and files['cache'][0] != files['plain'][0]   # the history was used


def check_detector_camera_frames(precision):
    """uint8 frames and float images through the native backbone, records against the operator on the returned volumes"""
    from occnet_b200 import ops
    cfg = grid_cfg(img_shape=(232, 400, 3))
    det = _detector(cfg, precision, img_backbone=dict(type='ResNet', depth=50), img_neck=dict(type='FPN'),
                    frame_pad=dict(size=(232, 400)))
    assert not det.load_state_dict(fixtures.init_backbone_params(seed=5), strict=False).unexpected_keys
    org = origins(4, np.float64, seed=3)
    frames = torch.from_numpy(np.random.default_rng(90).integers(0, 256, size=(1, 6, 220, 400, 3), dtype=np.uint8)).to(DEV)
    m = fixtures.make_img_metas(cfg, bs=1)
    m[0].pop('img_shape', None)
    imgs = torch.randn(1, 6, 3, 232, 400, generator=torch.Generator().manual_seed(4)).to(DEV)
    for kw in (dict(img=[frames], img_metas=[m]), dict(img=[imgs], img_metas=[fixtures.make_img_metas(cfg, bs=1)])):
        res = det(return_loss=False, lidar_origins=org, **kw)
        want = ops.ray_records(res['occ_results'][0].to(DEV, torch.uint8), res['flow_results'][0].to(DEV), org)
        for k, w in zip(('pcd_cls', 'pcd_dist', 'pcd_flow'), want):
            assert np.array_equal(bits(res['ray_results'][k]), bits(w)), k


def test_detector_ray_results_fp32(tmp_path):
    check_detector('fp32', str(tmp_path))


def test_detector_ray_results_bf16(tmp_path):
    _isolated(f"check_detector('bf16', {str(tmp_path)!r})", timeout=1200)


def test_detector_ray_results_camera_frames():
    _isolated("check_detector_camera_frames('bf16')")
