"""Golden of the reference's own ray-casting kernel (tools/ray_iou/lib/dvr/dvr.cu, built into oracle/_ref by
oracle/build_ref.py): render_forward outputs for the scene and origins of
tests/test_gpu_parity.py::test_render_forward_vs_reference_kernel_if_built.  Needs a GPU.

    python tests/golden/gen_dvr_ref.py
"""
import glob
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
OUT = os.path.join(ROOT, 'tests', 'golden', 'ref_dvr.npz')


def main():
    import test_gpu_parity as t
    so = glob.glob(os.path.join(ROOT, 'oracle', '_ref', 'dvr_ref*.so'))
    spec = importlib.util.spec_from_file_location('dvr_ref', so[0])
    dvr = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dvr)
    out = {}
    for i, (occ, o, p, ti) in enumerate(t.dvr_cases()):
        pd, gd, ci = dvr.render_forward(occ, o, p, ti, [1, 16, 200, 200], 'test')
        out[f'pred_dist_{i}'] = pd[0].cpu().numpy().astype(np.float32)
        out[f'gt_dist_{i}'] = gd[0].cpu().numpy().astype(np.float32)
        out[f'coord_{i}'] = ci[0].cpu().numpy().astype(np.int16)
        assert np.array_equal(out[f'coord_{i}'].astype(np.float32), ci[0].cpu().numpy())
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
