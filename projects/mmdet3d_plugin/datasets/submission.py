"""Occupancy-and-flow challenge submission writer: the prediction half of the reference's
`NuSceneOcc.format_results` (`datasets/nuscenes_occ.py:188-257`).

The reference walks an `EgoPoseDataset` loader for (token, lidar origins), ray-casts every predicted volume with
`process_one_sample` and pickles {token: {pcd_cls int8, pcd_dist fp16, pcd_flow fp16}} into `submission.gz`.  The dataset plumbing
(nuScenes infos, ego poses) is outside this repository's scope; this function takes what that loader yields -- sample tokens and
per-sample lidar origins -- and does the rest with the CUDA ray caster of libocc_b200 (one launch per sample).  A result that
already carries the frame's ray records (`BEVFormerOcc.forward_test(lidar_origins=...)` -> 'ray_results', cast inside the frame
engine) is written from them with no ray cast at all.  Byte-for-byte deterministic like the reference
(`gzip.compress(..., mtime=0)`), and the same bytes on either path."""
import gzip
import os
import pickle

import numpy as np

from .ray_metrics import generate_lidar_rays, process_one_sample

# header fields of the challenge file (same keys as the reference writer; the values are for the submitter to fill in)
SUBMISSION_META = {'method': '', 'team': '', 'authors': '', 'e-mail': '', 'institution / company': '', 'country / region': ''}


_RECORD_DTYPES = (('pcd_cls', np.int8, 1), ('pcd_dist', np.float16, 1), ('pcd_flow', np.float16, 2))


def _records(ray_results):
    """a frame's ray records as the arrays the challenge file holds; a dtype or shape that would need a conversion is an error"""
    out = {}
    for key, dtype, ndim in _RECORD_DTYPES:
        a = ray_results[key]
        a = a.cpu().numpy() if hasattr(a, 'cpu') else np.asarray(a)
        if a.dtype != dtype or a.ndim != ndim or (ndim == 2 and a.shape[1] != 2) or a.shape[0] != ray_results['pcd_cls'].shape[0]:
            raise ValueError(f"ray_results[{key!r}]: expected {np.dtype(dtype).name} with {ndim} dim(s), got {a.dtype} {a.shape}")
        out[key] = np.ascontiguousarray(a)
    return out


def format_results(occ_results, sample_tokens, lidar_origins, submission_prefix=None, meta=None, device='cuda:0'):
    """occ_results: the detector's per-sample dicts {'occ_results', 'flow_results'} (tensors or arrays, any shape that reshapes
    to (200,200,16) / (200,200,16,2)); sample_tokens: one token per result; lidar_origins: per sample (1,T,3) or (T,3).
    A result with 'ray_results' {'pcd_cls' int8 (R,), 'pcd_dist' fp16 (R,), 'pcd_flow' fp16 (R,2)} is written from them: its
    volumes and its entry of lidar_origins are not read (both may be None).  The choice is made per result.
    Returns the submission dict; writes `<submission_prefix>/submission.gz` when a prefix is given."""
    assert len(occ_results) == len(sample_tokens) == len(lidar_origins), 'one token and one origin set per result'
    lidar_rays = None
    result_dict = {}
    for res, token, origin in zip(occ_results, sample_tokens, lidar_origins):
        if res.get('ray_results') is not None:
            result_dict[token] = _records(res['ray_results'])
            continue
        if lidar_rays is None:
            lidar_rays = generate_lidar_rays()
        sem = res['occ_results']; flow = res['flow_results']
        sem = sem.cpu().numpy() if hasattr(sem, 'cpu') else np.asarray(sem)
        flow = flow.cpu().numpy() if hasattr(flow, 'cpu') else np.asarray(flow)
        sem = np.reshape(sem, [200, 200, 16]); flow = np.reshape(flow, [200, 200, 16, 2])
        pcd = process_one_sample(sem, lidar_rays, origin, flow, device=device)
        result_dict[token] = {'pcd_cls': pcd[:, 0].astype(np.int8), 'pcd_dist': pcd[:, 1].astype(np.float16),
                              'pcd_flow': pcd[:, 2:4].astype(np.float16)}
    final = dict(SUBMISSION_META if meta is None else meta)
    final['results'] = result_dict
    if submission_prefix is not None:
        os.makedirs(submission_prefix, exist_ok=True)
        with open(os.path.join(submission_prefix, 'submission.gz'), 'wb') as f:
            f.write(gzip.compress(pickle.dumps(final), mtime=0))
    return final
