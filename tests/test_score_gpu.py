"""A frame scored inside the frame engine (ray_score_kernel; occb200_engine_request_score, occb200_ray_score).  The reference
is `RayMetric.add_frame` (ray_metric_kernel) on the frame's own 'occ_cls' and 'flow' outputs with the same ground truth and
origins: the 136 integer counters must match bit for bit, the 51 `ave` sums to 1e-12 (the order of the fp64 atomics)."""
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
N = 17
KEYS = ('ray_cls', 'ray_dist', 'ray_flow')


def _isolated(call, timeout=1200):
    """Tensor-core runs happen in a child process: a device fault there must not poison this session's context."""
    code = f"import sys; sys.path.insert(0, 'tests'); import test_score_gpu as t; t.{call}; print('OK')"
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and 'OK' in r.stdout, f'child failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'


def origins(T, dtype=np.float32, seed=0):
    """T origins inside the grid, off the voxel lattice"""
    rng = np.random.default_rng(seed)
    o = fixtures.make_ray_origins(T=T)[0].astype(np.float64)
    o += rng.uniform(-0.37, 0.37, o.shape)
    return np.ascontiguousarray(o[None], dtype)


def metric_fixture():
    """the repository's metric fixture: a synthetic scene and a shifted, noisy prediction of it"""
    sem_gt, flow_gt = fixtures.make_occ_scene(seed=4)
    rng = np.random.RandomState(5)
    sem_pred = np.roll(sem_gt, 1, axis=0).copy()
    flip = rng.rand(*sem_pred.shape) < 0.03
    sem_pred[flip] = rng.randint(0, 17, int(flip.sum())).astype(np.uint8)
    flow_pred = (np.roll(flow_gt, 1, axis=0) + rng.normal(0, 0.5, flow_gt.shape)).astype(np.float32)
    return sem_pred, flow_pred, sem_gt, flow_gt


def gt_like(sem, flow, seed):
    """a ground truth close to a predicted frame (CUDA tensors in, CUDA tensors out): shifted by one cell, 3 % of the classes
    redrawn, noisy flow, so that every kind of counter receives something"""
    g = torch.Generator().manual_seed(seed)
    s = torch.roll(sem.cpu(), 1, 0)
    flip = torch.rand(s.shape, generator=g) < 0.03
    s[flip] = torch.randint(0, 17, (int(flip.sum()),), generator=g).to(torch.uint8)
    f = torch.roll(flow.cpu(), 1, 0) + 0.5 * torch.randn(flow.shape, generator=g)
    return s.to(DEV).contiguous(), f.to(DEV).contiguous()


def reference(sem, flow, gt, org):
    """ray_metric_kernel's counters for one frame"""
    from occnet_b200.metric import RayMetric
    rm = RayMetric(DEV)
    rm.add_frame(sem.to(DEV, torch.uint8), flow.to(DEV), gt[0], gt[1], torch.as_tensor(org))
    return rm.counters.cpu().numpy()


def assert_counters(got, want, what=''):
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    assert np.array_equal(got[:5 * N], want[:5 * N]), (what, 'gt_cnt / pred_cnt / tp')
    assert np.array_equal(got[8 * N:], want[8 * N:]), (what, 'ave_count')
    np.testing.assert_allclose(got[5 * N:8 * N], want[5 * N:8 * N], rtol=1e-12, atol=0, err_msg=str(what))


# ------------------------------------------------------------------------------------------------------------ 1. operator
@pytest.mark.parametrize('T', [1, 3, 8])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_score_kernel_equals_the_metric_kernel(T, dtype):
    from occnet_b200 import ops
    sem_pred, flow_pred, sem_gt, flow_gt = [torch.from_numpy(a).to(DEV) for a in metric_fixture()]
    org = origins(T, dtype, seed=T)
    cnt = torch.zeros(187, dtype=torch.float64, device=DEV)
    ops.ray_score(sem_pred, flow_pred, sem_gt, flow_gt, org, cnt)
    want = reference(sem_pred, flow_pred, (sem_gt, flow_gt), org)
    assert_counters(cnt, want, (T, dtype))
    assert want[2 * N:5 * N].sum() > 0 and want[5 * N:8 * N].sum() > 0
    ops.ray_score(sem_pred, flow_pred, sem_gt, flow_gt, org, cnt)                 # accumulated in place
    assert np.array_equal(cnt.cpu().numpy()[:5 * N], 2 * want[:5 * N])


def test_score_on_the_metric_fixture_matches_the_oracle():
    from occnet_b200 import metric, ops
    from oracle import ray_metrics as ORM
    fx = metric_fixture()
    org = fixtures.make_ray_origins(T=2)
    cnt = torch.zeros(187, dtype=torch.float64, device=DEV)
    ops.ray_score(*[torch.from_numpy(a).to(DEV) for a in fx], org, cnt)
    rays = ORM.generate_lidar_rays()
    rows_p = ORM.process_one_sample(fx[0], rays, org, fx[1])
    rows_g = ORM.process_one_sample(fx[2], rays, org, fx[3])
    valid = rows_g[:, 0].astype(np.int32) != 16
    oc = ORM.accumulate(ORM.new_counters(), rows_p[valid], rows_g[valid])
    vec, got = ORM.counters_to_vector(oc), cnt.cpu().numpy()
    np.testing.assert_array_equal(got[:5 * N], vec[:5 * N])
    np.testing.assert_array_equal(got[8 * N:], vec[8 * N:])
    np.testing.assert_allclose(got[5 * N:8 * N], vec[5 * N:8 * N], rtol=1e-5)
    fin, want = metric.finalize_counters(got), ORM.finalize(oc)
    assert abs(fin['miou'] - want['miou']) < 1e-12 and abs(fin['mave'] - want['mave']) < 1e-5
    assert abs(fin['score'] - want['score']) < 1e-5


def test_operator_edge_cases_and_bad_tensors():
    from occnet_b200 import ops
    sem_pred, flow_pred, sem_gt, flow_gt = [torch.from_numpy(a).to(DEV) for a in metric_fixture()]
    org = np.array([[[0.3, -0.2, 1.8], [500.0, 500.0, 50.0]]], np.float32)        # the second origin's rays never enter the grid
    cnt = torch.zeros(187, dtype=torch.float64, device=DEV)
    ops.ray_score(sem_pred, flow_pred, torch.full_like(sem_gt, 16), flow_gt, org, cnt)
    assert not cnt.any()                                                           # an all-free ground truth adds nothing
    sem_gt[0, 0, 0] = 3                                                            # what a ray that never enters reports
    ops.ray_score(sem_pred, flow_pred, sem_gt, flow_gt, org, cnt)
    assert_counters(cnt, reference(sem_pred, flow_pred, (sem_gt, flow_gt), org))
    with pytest.raises(ValueError, match='1..8'):
        ops.ray_score(sem_pred, flow_pred, sem_gt, flow_gt, np.zeros((9, 3), np.float32), cnt)
    with pytest.raises(ValueError, match='shape'):
        ops.ray_score(sem_pred, flow_pred, sem_gt[:100].contiguous(), flow_gt, org, cnt)
    with pytest.raises(RuntimeError, match='float64'):
        ops.ray_score(sem_pred, flow_pred, sem_gt, flow_gt, org, cnt.float())


# -------------------------------------------------------------------------------------------------------------- 2. engine
def grid_cfg(full=False):
    """the metric's 200 x 200 x 16 grid: over the small six-camera feature levels, or the shipped size with 6 layers"""
    if full:
        return fixtures.make_cfg('full', num_layers=6)
    return fixtures.make_cfg('small6', bev_h=200, bev_w=200, num_layers=1)


def _engine(cfg, precision):
    from occnet_b200.engine import OccEngine
    eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS), precision=precision,
                    use_tensor_cores=precision == 'bf16', device=DEV)
    eng.set_cameras(fixtures.make_img_metas(cfg, bs=1))
    return eng


def _frames(cfg, n, seed=500):
    return [[f[0].to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=seed + i)] for i in range(n)]


ANGLES = [0.0, 2.0, -3.0]
STARTS = [True, False, False]
TS = [8, 1, 3]                                                         # consecutive slots carry different T, dtype, ground truth
WANT = ('bev_embed', 'occ', 'flow', 'occ_cls', 'occ_cls_i64')


def check_frame_kinds(precision, full=False):
    """every kind of frame call, scored, against ray_metric_kernel on the frame's own outputs"""
    from occnet_b200 import _lib
    from occnet_b200.metric import RayMetric
    cfg = grid_cfg(full)
    eng = _engine(cfg, precision)
    dev_frames = _frames(cfg, 3)
    host_frames = [[f.cpu().contiguous().pin_memory() for f in fr] for fr in dev_frames]
    orgs = [origins(T, np.float64 if i % 2 else np.float32, seed=60 + i) for i, T in enumerate(TS)]
    rm = RayMetric(DEV)

    # _forward: the caller's outputs keep every byte, one kernel more, the counters of the frame's own volumes
    plain = [{k: v.clone() for k, v in eng.forward(fr, want=WANT).items()} for fr in dev_frames]
    n_plain = eng.launches_per_frame
    gts = [gt_like(p['occ_cls'], p['flow'], seed=70 + i) for i, p in enumerate(plain)]
    host_gts = [(s.cpu().pin_memory(), f.cpu().pin_memory()) for s, f in gts]
    want = [reference(p['occ_cls'], p['flow'], gt, o) for p, gt, o in zip(plain, gts, orgs)]
    assert all(w[2 * N:5 * N].sum() > 0 for w in want)
    out = eng.forward(dev_frames[0], want=WANT, score=(*gts[0], orgs[0]), metric=rm)
    assert eng.launches_per_frame == n_plain + 1
    for k in WANT:
        assert torch.equal(out[k], plain[0][k]), k
    assert_counters(rm.counters, want[0], '_forward')
    # a frame without a request leaves the counters alone: the request was consumed
    eng.forward(dev_frames[1], want=WANT)
    assert eng.launches_per_frame == n_plain
    assert_counters(rm.counters, want[0], 'one-shot')
    # no volume requested at all: the engine's own u8 / flow buffers feed the kernel
    rm.reset()
    eng.forward(dev_frames[1], want=('bev_embed',), score=(*gts[1], orgs[1]), metric=rm)
    assert_counters(rm.counters, want[1], '_forward, no volumes')
    # a ray request on the same frame: both kernels, and neither changes the other's result or the caller's outputs
    rec = eng.forward(dev_frames[2], want=WANT, ray_origins=orgs[2])
    rm.reset()
    both = eng.forward(dev_frames[2], want=WANT, ray_origins=orgs[2], score=(*gts[2], orgs[2]), metric=rm)
    assert eng.launches_per_frame == n_plain + 2
    for k in WANT + KEYS:
        assert torch.equal(both[k].view(torch.uint8), rec[k].view(torch.uint8)), k
        assert k in KEYS or torch.equal(both[k], plain[2][k]), k
    assert_counters(rm.counters, want[2], 'with a ray request')

    # ground-truth edge cases
    rm.reset()
    eng.forward(dev_frames[0], want=('flow',), score=(torch.full_like(gts[0][0], 16), gts[0][1], orgs[0]), metric=rm)
    assert not rm.counters.any()
    eng.forward(dev_frames[0], want=('flow',), score=(plain[0]['occ_cls'], plain[0]['flow'], orgs[0]), metric=rm)
    c = rm.counters.cpu().numpy()
    assert c[:N].sum() > 0 and np.array_equal(c[:N], c[N:2 * N]) and not c[5 * N:8 * N].any()
    for j in range(3):
        assert np.array_equal(c[(2 + j) * N:(3 + j) * N], c[:N]), j

    # _forward_host, with and without the volumes
    for volumes in (True, False):
        rm.reset()
        occ, flow = eng.forward_host(host_frames[1], score=(*host_gts[1], orgs[1]), metric=rm, volumes=volumes)
        assert_counters(rm.counters, want[1], ('_forward_host', volumes))
        if volumes:
            assert torch.equal(occ, plain[1]['occ_cls_i64'].cpu()) and torch.equal(flow, plain[1]['flow'].cpu())
        else:
            assert occ is None and flow is None
    with pytest.raises(_lib.OccB200Error, match='null pointer'):                  # nothing is armed any more
        eng.submit_host(0, host_frames[0], None, None)

    # _submit_host: three frames with three ground truths, two slots in flight, accumulate to the sum of the three
    total = want[0] + want[1] + want[2]
    scores = [(s, f, o) for (s, f), o in zip(host_gts, orgs)]
    for volumes in (True, False):
        rm.reset()
        for i, (occ, flow) in enumerate(eng.stream_host(host_frames, score=scores, metric=rm, volumes=volumes)):
            if volumes:
                assert torch.equal(occ, plain[i]['occ_cls_i64'].cpu()) and torch.equal(flow, plain[i]['flow'].cpu()), i
        assert_counters(rm.counters, total, ('stream_host', volumes))
    rm.reset()
    for i, (occ, flow, r) in enumerate(eng.stream_host(host_frames, ray_origins=orgs, score=[scores[0], None, scores[2]], metric=rm)):
        assert torch.equal(occ, plain[i]['occ_cls_i64'].cpu()), i
    assert_counters(rm.counters, want[0] + want[2], 'stream_host, the middle frame not scored')
    assert torch.equal(r['ray_cls'], rec['ray_cls'].cpu())

    # video: _forward_video (map), _forward_video_angle, _submit_host_video (map), _submit_host_video_angle
    eng.set_history(True)
    vplain = [{k: v.clone() for k, v in eng.forward_video(fr, rotation=a, scene_start=s, want=WANT).items()}
              for fr, a, s in zip(dev_frames, ANGLES, STARTS)]
    vwant = [reference(p['occ_cls'], p['flow'], gt, o) for p, gt, o in zip(vplain, gts, orgs)]
    vtotal = vwant[0] + vwant[1] + vwant[2]
    for as_map in (False, True):
        eng.set_history(True)
        rm.reset()
        for i, (fr, a, s) in enumerate(zip(dev_frames, ANGLES, STARTS)):
            out = eng.forward_video(fr, rotation=eng.rotation_map(a) if as_map else a, scene_start=s, want=WANT,
                                    score=(*gts[i], orgs[i]), metric=rm)
            for k in WANT:                                                       # outputs and, through them, the history
                assert torch.equal(out[k], vplain[i][k]), (as_map, i, k)
        assert_counters(rm.counters, vtotal, ('forward_video', as_map))
        eng.set_history(True)
        rm.reset()
        items = [(fr, eng.rotation_map(a).cpu().numpy() if as_map else a, s) for fr, a, s in zip(host_frames, ANGLES, STARTS)]
        for i, (occ, flow) in enumerate(eng.stream_host_video(items, score=scores, metric=rm, volumes=not as_map)):
            if not as_map:
                assert torch.equal(occ, vplain[i]['occ_cls_i64'].cpu()) and torch.equal(flow, vplain[i]['flow'].cpu()), i
        assert_counters(rm.counters, vtotal, ('stream_host_video', as_map))


def test_frame_kinds_fp32():
    check_frame_kinds('fp32')


def test_frame_kinds_bf16():
    _isolated("check_frame_kinds('bf16')")


def test_frame_kinds_full_size_bf16_tensor_cores():
    _isolated("check_frame_kinds('bf16', full=True)", timeout=2400)


def test_rejections_leave_the_counters_alone_and_nothing_armed():
    from occnet_b200 import _lib
    from occnet_b200.metric import RayMetric
    cfg = grid_cfg()
    eng = _engine(cfg, 'fp32')
    fr = _frames(cfg, 1)[0]
    host = [f.cpu().contiguous().pin_memory() for f in fr]
    rm = RayMetric(DEV)
    sem, flow = torch.zeros(200, 200, 16, dtype=torch.uint8, device=DEV), torch.zeros(200, 200, 16, 2, device=DEV)
    o = np.ascontiguousarray(origins(2)[0])
    request = eng.lib.occb200_engine_request_score

    def rejected(msg, *args):
        rc = request(eng._h, *args)
        assert rc == 1 and msg in eng.lib.occb200_last_error().decode(), (msg, rc)
        with pytest.raises(_lib.OccB200Error, match='null pointer'):             # nothing armed: the volumes are still required
            eng.submit_host(0, host, None, None)
        eng.forward(fr, want=('flow',))
        assert not rm.counters.any()

    p = _lib.ptr
    rejected('set_rays', p(sem), p(flow), p(o), 0, 2, p(rm.counters))             # no ray bundle yet
    eng.set_rays()
    bad = o.copy()
    bad[1, 2] = np.inf
    for msg, args in (('null pointer', (None, p(flow), p(o), 0, 2, p(rm.counters))),
                      ('null pointer', (p(sem), None, p(o), 0, 2, p(rm.counters))),
                      ('null pointer', (p(sem), p(flow), p(o), 0, 2, None)),
                      ('0..8', (p(sem), p(flow), p(o), 0, 9, p(rm.counters))),
                      ('finite', (p(sem), p(flow), p(bad), 0, 2, p(rm.counters)))):
        assert request(eng._h, p(sem), p(flow), p(o), 0, 2, p(rm.counters)) == 0  # armed: the rejection must disarm it
        rejected(msg, *args)
    # T = 0 and NULL origins disarm and return 0
    for args in ((p(sem), p(flow), p(o), 0, 0, p(rm.counters)), (p(sem), p(flow), None, 0, 2, p(rm.counters))):
        assert request(eng._h, p(sem), p(flow), p(o), 0, 2, p(rm.counters)) == 0
        assert request(eng._h, *args) == 0
        eng.forward(fr, want=('flow',))
        assert not rm.counters.any()
    # a frame call that is itself rejected leaves the request armed for the next one
    assert request(eng._h, p(sem), p(flow), p(o), 0, 2, p(rm.counters)) == 0
    with pytest.raises(_lib.OccB200Error, match='slot'):
        eng.submit_host(2, host, None, None)
    eng.forward(fr, want=('flow',))
    assert rm.counters.any()
    # the Python layer: score without metric, and the wrong grid
    with pytest.raises(ValueError, match='metric'):
        eng.forward(fr, want=('flow',), score=(sem, flow, o))
    with pytest.raises(ValueError, match='volumes=False'):
        eng.forward_host(host, volumes=False)
    small = _engine(fixtures.make_cfg('small6', num_layers=1), 'fp32')
    with pytest.raises(_lib.OccB200Error, match='200 x 200 x 16'):
        small.forward(_frames(small.cfg, 1)[0], want=('flow',), score=(sem, flow, o), metric=rm)


def test_host_calls_reject_a_null_feature_level_and_keep_the_requests():
    """_forward_host and _submit_host reject a NULL host feature level with error 1 before any CUDA call (through the C ABI:
    the Python wrapper never passes one): the slot stays free, and the armed ray and score requests are consumed by the next
    valid call, which returns what it returns on a fresh engine."""
    from occnet_b200 import _lib
    from occnet_b200.metric import RayMetric
    cfg = grid_cfg()
    host = [f.cpu().contiguous().pin_memory() for f in _frames(cfg, 1)[0]]
    _, _, sem_gt, flow_gt = metric_fixture()
    sem_gt = torch.from_numpy(np.ascontiguousarray(sem_gt, np.uint8)).pin_memory()
    flow_gt = torch.from_numpy(np.ascontiguousarray(flow_gt, np.float32)).pin_memory()
    o = np.ascontiguousarray(origins(3)[0])
    p = _lib.ptr

    def valid_frame(reject_first):
        eng = _engine(cfg, 'fp32')
        rm, rec = RayMetric(DEV), eng.ray_buffers(3, host=True)
        X, Y, Z = eng.vox_shape
        occ, flow = torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(), torch.empty((X, Y, Z, 2)).pin_memory()
        st = _lib.stream_ptr()
        assert eng.lib.occb200_engine_request_rays(eng._h, p(o), 0, 3, p(rec['ray_cls']), p(rec['ray_dist']),
                                                   p(rec['ray_flow'])) == 0
        assert eng.lib.occb200_engine_request_score(eng._h, p(sem_gt), p(flow_gt), p(o), 0, 3, p(rm.counters)) == 0
        if reject_first:
            for missing in range(4):
                feats = eng._feat_ptrs(host)
                feats[missing] = None
                for rc in (eng.lib.occb200_engine_forward_host(eng._h, feats, p(occ), p(flow), st),
                           eng.lib.occb200_engine_submit_host(eng._h, 0, feats, p(occ), p(flow), st)):
                    assert rc == 1 and 'null feature level' in eng.lib.occb200_last_error().decode(), (missing, rc)
        # slot 0 is free (a busy slot is rejected), and the frame consumes both requests
        assert eng.lib.occb200_engine_submit_host(eng._h, 0, eng._feat_ptrs(host), p(occ), p(flow), st) == 0
        eng.wait_host(0)
        with pytest.raises(_lib.OccB200Error, match='null pointer'):             # nothing is armed any more
            eng.submit_host(1, host, None, None)
        return occ, flow, rec, rm.counters.cpu().numpy()

    got, want = valid_frame(True), valid_frame(False)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    for k in KEYS:
        assert torch.equal(got[2][k].view(torch.uint8), want[2][k].view(torch.uint8)), k
    assert want[3][:N].sum() > 0                                                   # the frame was scored: gt_cnt
    assert_counters(got[3], want[3], 'after the rejected calls')


# ------------------------------------------------------------------------------------------------------------ 3. detector
SCENES = [('scene-a', 0.0), ('scene-a', 2.5), ('scene-b', -1.0)]


def _detector(cfg, precision, **kw):
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200.mmcv_shim import build_detector
    d = build_detector(dict(type='BEVFormerOcc', pts_bbox_head=dict(fixtures.head_cfg(cfg), precision=precision), **kw)).to(DEV).eval()
    d.pts_bbox_head.load_state_dict(fixtures.init_params(cfg, seed=2, free_bias=fixtures.FREE_BIAS), strict=True)
    return d


def check_detector(precision):
    from occnet_b200.metric import RayMetric
    cfg = grid_cfg()
    inputs = [[f.to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=80 + i)] for i in range(len(SCENES))]
    metas = []
    for tok, ang in SCENES:
        m = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=ang)
        m[0]['scene_token'] = tok
        metas.append(m)
    orgs = [origins(T, np.float64, seed=90 + i) for i, T in enumerate((8, 2, 5))]
    modes = {'plain': {}, 'history': dict(video_test_mode=True, temporal_test=True, engine_history=True)}
    totals = {}
    for name, kw in modes.items():
        det = _detector(cfg, precision, **kw)
        vol = [det(return_loss=False, img_metas=[m], img_feats=x) for m, x in zip(metas, inputs)]
        gts = [gt_like(v['occ_results'][0].to(torch.uint8), v['flow_results'][0], seed=40 + i) for i, v in enumerate(vol)]
        want = sum(reference(v['occ_results'][0], v['flow_results'][0], gt, o) for v, gt, o in zip(vol, gts, orgs))
        for score_only in (False, True):
            det = _detector(cfg, precision, score_only=score_only, **kw)
            rm = RayMetric(DEV)
            for i, (m, x, o) in enumerate(zip(metas, inputs, orgs)):
                res = det(return_loss=False, img_metas=[m], img_feats=x, lidar_origins=o, gt_semantics=gts[i][0][None],
                          gt_flow=gts[i][1][None], ray_metric=rm)
                assert set(res) == {'occ_results', 'flow_results'}
                if score_only:
                    assert res['occ_results'] is None and res['flow_results'] is None
                else:
                    assert torch.equal(res['occ_results'], vol[i]['occ_results']), (name, i)
                    assert torch.equal(res['flow_results'], vol[i]['flow_results']), (name, i)
            assert_counters(rm.counters, want, (name, score_only))
        totals[name] = want
        with pytest.raises(ValueError, match='score_only'):
            det(return_loss=False, img_metas=[metas[0]], img_feats=inputs[0])
    assert not np.array_equal(totals['plain'], totals['history'])                 # the history was used


def test_detector_scores_its_frames_fp32():
    check_detector('fp32')


def test_detector_scores_its_frames_bf16():
    _isolated("check_detector('bf16')")
