"""Golden of the reference's own ray-casting kernel (tools/ray_iou/lib/dvr/dvr.cu, built into oracle/_ref by
oracle/build_ref.py) on the edge families of tests/golden/dvr_edges.py: for every case the outputs pred_dist, gt_dist and
coord_index as the kernel wrote them (NaN payloads included).  The inputs are not stored: dvr_edges.cases() regenerates them
from closed forms and fixed seeds.  No case passes the kernel a tindex at or past sigma's T when T > 1 (it device-asserts
t < T) or past origin's To.  Needs a GPU.

    python tests/golden/gen_dvr_edges.py
"""
import glob
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
OUT = os.path.join(HERE, 'ref_dvr_edges.npz')


def main():
    import dvr_edges as E
    so = glob.glob(os.path.join(ROOT, 'oracle', '_ref', 'dvr_ref*.so'))
    spec = importlib.util.spec_from_file_location('dvr_ref', so[0])
    dvr = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dvr)
    out = {}
    for c in E.cases():
        T, Z, Y, X = c['sigma'].shape[1:]
        ti = c['tindex'][c['tindex'] >= 0].astype(np.int64)
        assert (ti < c['origin'].shape[1]).all() and (T == 1 or (ti < T).all())
        args = [torch.from_numpy(c[k]).cuda() for k in ('sigma', 'origin', 'points', 'tindex')]
        pd, gd, ci = dvr.render_forward(*args, [T, Z, Y, X], 'test')
        torch.cuda.synchronize()
        for k, v in (('pred_dist', pd), ('gt_dist', gd), ('coord_index', ci)):
            assert v.dtype == torch.float32
            out[f"{c['name']}/{k}"] = v.cpu().numpy()
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes,', len(out) // 3, 'cases')


if __name__ == '__main__':
    main()
