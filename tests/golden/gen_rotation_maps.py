"""Writes tests/golden/rotation_maps.npz: SHA-256 digests of torchvision's prev_bev rotation maps (`rotation_index_map`: the
source cell of every BEV cell, int32, -1 = outside) for a seeded angle set on the grids of tests/test_rotation_cpu.py.  The
digests pin the definition across hosts: test_rotation_cpu.py checks this host's torchvision and the device formula's mirror
against them, test_rotation_gpu.py the engine's device maps.

    python tests/golden/gen_rotation_maps.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from occnet_b200.engine import rotation_index_map          # noqa: E402
from test_rotation_cpu import GRIDS, SPECIAL, map_digest    # noqa: E402


def main():
    out = {'grids': np.array([(h, w, c[0], c[1]) for h, w, c in GRIDS], np.int32)}      # bev_h, bev_w, center x, center y
    for k, (h, w, c) in enumerate(GRIDS):
        rng = np.random.default_rng(1234 + k)
        angles = np.concatenate([SPECIAL, rng.uniform(-180, 180, 48), rng.uniform(-5, 5, 24)])
        out[f'angles_{k}'] = angles
        out[f'sha256_{k}'] = np.array([map_digest(rotation_index_map(h, w, float(a), c)) for a in angles], 'S64')
    path = os.path.join(ROOT, 'tests', 'golden', 'rotation_maps.npz')
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
