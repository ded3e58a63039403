"""Ray records (occb200_ray_records, occb200_engine_set_rays, _request_rays) without a GPU: the argument rejections of the C
ABI, which happen before any CUDA call (return code 1, an argument check, not 2, a CUDA error), and the submission writer fed
with a frame's records instead of its volumes.  The rejections that need a live engine (no ray bundle set, the one-shot
request) are in test_ray_records_gpu.py."""
import ctypes
import gzip
import math
import os
import pickle

import numpy as np
import pytest
import torch

from occnet_b200 import fixtures
from oracle import ray_metrics as ORM
from projects.mmdet3d_plugin.datasets import submission

FAKE = 1 << 12                       # never dereferenced: every call below is rejected before it reads a buffer
M = 14040


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


# ------------------------------------------------------------------------------------------------- the operator on its own
@pytest.mark.parametrize('T', [0, -1, 9, 64])
def test_operator_rejects_T_outside_1_to_8(T, lib_built):
    rc, err = _call('ray_records', FAKE, FAKE, _p(_origins(8)), 0, T, FAKE, M, FAKE, FAKE, FAKE, None)
    assert rc == 1 and '1..8' in err


@pytest.mark.parametrize('missing', range(7))
def test_operator_rejects_null_pointers(missing, lib_built):
    o = _origins(2)
    ptrs = [FAKE, FAKE, _p(o), FAKE, FAKE, FAKE, FAKE]          # sem, flow, origins, rays, cls, dist, flow16
    ptrs[missing] = None
    rc, err = _call('ray_records', ptrs[0], ptrs[1], ptrs[2], 0, 2, ptrs[3], M, ptrs[4], ptrs[5], ptrs[6], None)
    assert rc == 1 and 'null pointer' in err


@pytest.mark.parametrize('bad', [math.nan, math.inf, -math.inf])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_operator_rejects_non_finite_origins(bad, dtype, lib_built):
    o = _origins(3, dtype, bad)
    rc, err = _call('ray_records', FAKE, FAKE, _p(o), int(dtype == np.float64), 3, FAKE, M, FAKE, FAKE, FAKE, None)
    assert rc == 1 and 'finite' in err


def test_operator_rejects_an_empty_ray_bundle(lib_built):
    rc, err = _call('ray_records', FAKE, FAKE, _p(_origins(1)), 0, 1, FAKE, 0, FAKE, FAKE, FAKE, None)
    assert rc == 1 and 'positive' in err


# ------------------------------------------------------------------------------------------------------- the engine calls
def test_engine_calls_reject_a_null_engine(lib_built):
    rays = ORM.generate_lidar_rays()
    rc, err = _call('engine_set_rays', None, _p(rays), M)
    assert rc == 1 and 'null engine' in err
    rc, err = _call('engine_request_rays', None, _p(_origins(2)), 0, 2, FAKE, FAKE, FAKE)
    assert rc == 1 and 'null engine' in err
    rc, err = _call('engine_request_rays', None, None, 0, 0, None, None, None)          # even the disarming form
    assert rc == 1 and 'null engine' in err


@pytest.mark.parametrize('T', [-1, 9, 1000])
def test_request_rejects_T_outside_0_to_8(T, lib_built):
    rc, err = _call('engine_request_rays', None, _p(_origins(8)), 0, T, FAKE, FAKE, FAKE)
    assert rc == 1 and '0..8' in err


def test_host_calls_still_reject_null_volumes_without_a_request(lib_built):
    """NULL volume pointers are accepted only by a frame that has a ray request armed; no engine, no request"""
    feats = (ctypes.c_void_p * 4)(*([FAKE] * 4))
    for occ, flow in ((None, FAKE), (FAKE, None), (None, None)):
        for name, args in (('engine_forward_host', (None, feats, occ, flow, None)),
                           ('engine_submit_host', (None, 0, feats, occ, flow, None)),
                           ('engine_submit_host_video', (None, 0, feats, None, 0, occ, flow, None)),
                           ('engine_submit_host_video_angle', (None, 0, feats, 1.0, 0, occ, flow, None))):
            rc, err = _call(name, *args)
            assert rc == 1 and 'null pointer' in err, (name, occ, flow, err)


# --------------------------------------------------------------------------------------------------- the submission writer
def reference_writer(rows_per_token, meta):
    """numpy restatement of the reference writer (datasets/nuscenes_occ.py:230-255) from process_one_sample's rows"""
    results = {}
    for token, pcd in rows_per_token:
        results[token] = {'pcd_cls': pcd[:, 0].astype(np.int8), 'pcd_dist': pcd[:, 1].astype(np.float16),
                          'pcd_flow': pcd[:, 2:4].astype(np.float16)}
    final = dict(meta)
    final['results'] = results
    return gzip.compress(pickle.dumps(final), mtime=0)


def narrow(pcd, as_torch):
    rec = {'pcd_cls': pcd[:, 0].astype(np.int8), 'pcd_dist': pcd[:, 1].astype(np.float16),
           'pcd_flow': np.ascontiguousarray(pcd[:, 2:4].astype(np.float16))}
    return {k: torch.from_numpy(v) for k, v in rec.items()} if as_torch else rec


def test_format_results_writes_ray_results_byte_identically(tmp_path):
    rays = ORM.generate_lidar_rays()
    rows, results = [], []
    for i, T in enumerate((1, 3)):
        sem, flow = fixtures.make_occ_scene(seed=20 + i)
        flow[5:9, 7, 3] = [[7e4, -7e4], [np.nan, 1.00048828125], [1e-8, -1e-8], [65519.9, 65520.0]]
        pcd = ORM.process_one_sample(sem, rays, fixtures.make_ray_origins(T=T), flow)
        rows.append((f'token{i}', pcd))
        results.append({'occ_results': None, 'flow_results': None, 'ray_results': narrow(pcd, as_torch=i == 0)})
    meta = dict(submission.SUBMISSION_META, method='ray records')
    final = submission.format_results(results, [t for t, _ in rows], [None, None], submission_prefix=str(tmp_path), meta=meta)
    got = open(os.path.join(str(tmp_path), 'submission.gz'), 'rb').read()
    assert got == reference_writer(rows, meta)
    assert final['results']['token1']['pcd_flow'].dtype == np.float16 and final['results']['token0']['pcd_cls'].shape == (M,)


def test_format_results_rejects_records_that_would_need_a_conversion():
    pcd = np.zeros((M, 4), np.float32)
    rec = narrow(pcd, as_torch=False)
    for key, bad in (('pcd_cls', rec['pcd_cls'].astype(np.int64)), ('pcd_dist', rec['pcd_dist'].astype(np.float32)),
                     ('pcd_flow', rec['pcd_flow'][:, :1]), ('pcd_dist', rec['pcd_dist'][:-1])):
        with pytest.raises(ValueError, match=key):
            submission.format_results([{'ray_results': dict(rec, **{key: bad})}], ['t'], [None])


def test_forward_test_with_lidar_origins_fails_loudly_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from occnet_b200.plugin import modules
    cfg = fixtures.make_cfg('toy')
    det = modules.BEVFormerOcc(pts_bbox_head=fixtures.head_cfg(cfg))
    feats = fixtures.make_feats(cfg, bs=1, seed=1)
    with pytest.raises(RuntimeError):
        det.forward_test(fixtures.make_img_metas(cfg, bs=1), img_feats=feats, lidar_origins=fixtures.make_ray_origins(T=2))
    from occnet_b200 import ops
    with pytest.raises(RuntimeError):
        ops.ray_records(torch.zeros(200, 200, 16, dtype=torch.uint8), torch.zeros(200, 200, 16, 2), fixtures.make_ray_origins(T=1))
