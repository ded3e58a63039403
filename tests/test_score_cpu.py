"""In-engine scoring (occb200_engine_request_score, occb200_ray_score) without a GPU: the argument rejections of the C ABI,
which happen before any CUDA call (return code 1, an argument check, not 2, a CUDA error), the skip rule and the counter
update of ray_score_kernel restated in numpy against the oracle's counters, and the Python argument checks.  The rejections
that need a live engine (no ray bundle, the grid, the one-shot request) are in test_score_gpu.py."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from occnet_b200 import fixtures
from oracle import ray_metrics as ORM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 12                       # never dereferenced: every call below is rejected before it reads a buffer
M = 14040
N = 17


def _call(name, *args):
    from occnet_b200 import _lib
    lib = _lib.load()
    rc = getattr(lib, 'occb200_' + name)(*args)
    return rc, lib.occb200_last_error().decode()


def _origins(T, dtype=np.float32, bad=None):
    o = np.ascontiguousarray(fixtures.make_ray_origins(T=max(T, 1))[0], dtype)
    if bad is not None:
        o[-1, 1] = bad
    return o


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


# ------------------------------------------------------------------------------------------------------------ the C ABI
def test_request_score_rejects_a_null_engine(lib_built):
    rc, err = _call('engine_request_score', None, FAKE, FAKE, _p(_origins(2)), 0, 2, FAKE)
    assert rc == 1 and 'null engine' in err
    rc, err = _call('engine_request_score', None, None, None, None, 0, 0, None)                 # even the disarming form
    assert rc == 1 and 'null engine' in err


@pytest.mark.parametrize('T', [-1, 9, 1000])
def test_request_score_rejects_T_outside_0_to_8(T, lib_built):
    rc, err = _call('engine_request_score', None, FAKE, FAKE, _p(_origins(8)), 0, T, FAKE)
    assert rc == 1 and '0..8' in err


@pytest.mark.parametrize('T', [0, -1, 9, 64])
def test_operator_rejects_T_outside_1_to_8(T, lib_built):
    rc, err = _call('ray_score', FAKE, FAKE, FAKE, FAKE, _p(_origins(8)), 0, T, FAKE, M, FAKE, None)
    assert rc == 1 and '1..8' in err


@pytest.mark.parametrize('missing', range(7))
def test_operator_rejects_null_pointers(missing, lib_built):
    o = _origins(2)
    ptrs = [FAKE, FAKE, FAKE, FAKE, _p(o), FAKE, FAKE]            # sem_pred, flow_pred, sem_gt, flow_gt, origins, rays, counters
    ptrs[missing] = None
    rc, err = _call('ray_score', ptrs[0], ptrs[1], ptrs[2], ptrs[3], ptrs[4], 0, 2, ptrs[5], M, ptrs[6], None)
    assert rc == 1 and 'null pointer' in err


@pytest.mark.parametrize('bad', [math.nan, math.inf, -math.inf])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_operator_rejects_non_finite_origins(bad, dtype, lib_built):
    o = _origins(3, dtype, bad)
    rc, err = _call('ray_score', FAKE, FAKE, FAKE, FAKE, _p(o), int(dtype == np.float64), 3, FAKE, M, FAKE, None)
    assert rc == 1 and 'finite' in err


def test_operator_rejects_an_empty_ray_bundle(lib_built):
    rc, err = _call('ray_score', FAKE, FAKE, FAKE, FAKE, _p(_origins(1)), 0, 1, FAKE, 0, FAKE, None)
    assert rc == 1 and 'positive' in err


def test_new_symbols_are_declared_and_exported(lib_built):
    from occnet_b200 import _lib
    header = open(os.path.join(ROOT, 'include', 'occ_b200.h')).read()
    lib = _lib.load()
    for name in ('occb200_engine_request_score', 'occb200_ray_score'):
        assert re.search(r'\bint ' + name + r'\(', header), name
        assert name in _lib.SIGNATURES and getattr(lib, name) is not None


# ------------------------------------------------------------------------------------- the kernel's arithmetic, in numpy
def kernel_mirror(rows_pred, rows_gt):
    """ray_score_kernel ray by ray from the rows of the two walks: a ray whose ground-truth class is free is skipped before
    its prediction row is looked at (the kernel does not walk it); every other ray updates the 187 counters."""
    cnt = np.zeros(11 * N)
    walked = 0
    for gt, pred in zip(rows_gt, rows_pred):
        cg = int(gt[0])
        if cg == 16:
            continue
        walked += 1
        cp = int(pred[0])
        cnt[cg] += 1
        cnt[N + cp] += 1
        if cg == cp:
            l1 = abs(np.float32(pred[1]) - np.float32(gt[1]))
            err = np.sqrt(np.float32((gt[2] - pred[2]) ** 2 + (gt[3] - pred[3]) ** 2), dtype=np.float32)
            for j, thr in enumerate((1.0, 2.0, 4.0)):
                if l1 < thr:
                    cnt[2 * N + j * N + cg] += 1
                    if cg < 8:
                        cnt[5 * N + j * N + cg] += float(err)
                        cnt[8 * N + j * N + cg] += 1
    return cnt, walked


def small_pair():
    """a ground truth with few occupied voxels (most rays end free) and a prediction that is a shifted, noisy copy"""
    rng = np.random.RandomState(11)
    sem_gt = np.full((200, 200, 16), 16, np.uint8)
    flow_gt = np.zeros((200, 200, 16, 2), np.float32)
    sem_gt[60:140, 60:140, 0] = 10
    for c in range(12):
        x, y = rng.randint(70, 130, 2)
        sem_gt[x:x + 4, y:y + 3, 1:5] = c
        flow_gt[x:x + 4, y:y + 3, 1:5] = rng.normal(0, 2, 2)
    sem_pred = np.roll(sem_gt, 1, axis=1).copy()
    flip = rng.rand(*sem_pred.shape) < 0.01
    sem_pred[flip] = rng.randint(0, 17, int(flip.sum())).astype(np.uint8)
    flow_pred = (np.roll(flow_gt, 1, axis=1) + rng.normal(0, 0.3, flow_gt.shape)).astype(np.float32)
    return sem_pred, flow_pred, sem_gt, flow_gt


def test_skip_rule_and_counter_update_equal_the_oracle():
    sem_pred, flow_pred, sem_gt, flow_gt = small_pair()
    rays = ORM.generate_lidar_rays()
    org = fixtures.make_ray_origins(T=2) * np.float32(0.4)                       # both origins above the occupied patch
    rows_p = ORM.process_one_sample(sem_pred, rays, org, flow_pred)
    rows_g = ORM.process_one_sample(sem_gt, rays, org, flow_gt)
    got, walked = kernel_mirror(rows_p, rows_g)
    valid = rows_g[:, 0].astype(np.int32) != 16
    want = ORM.counters_to_vector(ORM.accumulate(ORM.new_counters(), rows_p[valid], rows_g[valid]))
    assert 0 < walked < len(rows_g) // 2 and walked == int(valid.sum())          # most prediction walks are skipped
    np.testing.assert_array_equal(got[:5 * N], want[:5 * N])
    np.testing.assert_array_equal(got[8 * N:], want[8 * N:])
    np.testing.assert_allclose(got[5 * N:8 * N], want[5 * N:8 * N], rtol=1e-6)
    assert got[2 * N:5 * N].sum() > 0 and got[8 * N:].sum() > 0                  # true positives and flow errors were counted


# ------------------------------------------------------------------------------------------------- Python argument checks
class _Metric:
    def __init__(self, device):
        self.counters = torch.zeros(187, dtype=torch.float64, device=device)


def test_score_needs_a_metric_on_the_engines_device():
    from occnet_b200.engine import score_args
    sem, flow = torch.zeros(200, 200, 16, dtype=torch.uint8), torch.zeros(200, 200, 16, 2)
    org = fixtures.make_ray_origins(T=2)
    with pytest.raises(ValueError, match='metric'):
        score_args((sem, flow, org), None, torch.device('cpu'), host=True)
    with pytest.raises(ValueError, match="engine's device"):
        score_args((sem, flow, org), _Metric('cpu'), torch.device('cuda:0'), host=True)
    with pytest.raises(ValueError, match='ground truth'):
        score_args((sem[:100], flow, org), _Metric('cpu'), torch.device('cpu'), host=True)
    with pytest.raises(ValueError, match='1..8'):
        score_args((sem, flow, np.zeros((9, 3), np.float32)), _Metric('cpu'), torch.device('cpu'), host=True)
    s, f, o, is64 = score_args((sem.numpy().astype(np.int64), flow, org.astype(np.float64)), _Metric('cpu'), torch.device('cpu'),
                               host=True)
    assert s.dtype == torch.uint8 and f.dtype == torch.float32 and o.shape == (2, 3) and is64


def test_forward_test_checks_its_scoring_arguments_before_any_device_work():
    from occnet_b200.plugin import modules
    cfg = fixtures.make_cfg('toy')
    feats = fixtures.make_feats(cfg, bs=1, seed=1)
    metas = fixtures.make_img_metas(cfg, bs=1)
    sem, flow = torch.zeros(200, 200, 16, dtype=torch.uint8), torch.zeros(200, 200, 16, 2)
    det = modules.BEVFormerOcc(pts_bbox_head=fixtures.head_cfg(cfg), score_only=True)
    with pytest.raises(ValueError, match='score_only'):
        det.forward_test(metas, img_feats=feats)
    with pytest.raises(ValueError, match='score_only'):
        det.forward_test(metas, img_feats=feats, lidar_origins=fixtures.make_ray_origins(T=2))
    det = modules.BEVFormerOcc(pts_bbox_head=fixtures.head_cfg(cfg))
    for kw in (dict(gt_semantics=sem), dict(gt_semantics=sem, gt_flow=flow, lidar_origins=fixtures.make_ray_origins(T=2)),
               dict(gt_semantics=sem, gt_flow=flow, ray_metric=_Metric('cpu'))):
        with pytest.raises(ValueError, match='together'):
            det.forward_test(metas, img_feats=feats, **kw)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):                                       # complete arguments: no CPU fallback
            det.forward_test(metas, img_feats=feats, gt_semantics=sem, gt_flow=flow, ray_metric=_Metric('cpu'),
                             lidar_origins=fixtures.make_ray_origins(T=2))
        from occnet_b200 import ops
        with pytest.raises(RuntimeError):
            ops.ray_score(sem, flow, sem, flow, fixtures.make_ray_origins(T=1), torch.zeros(187, dtype=torch.float64))
