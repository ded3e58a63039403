"""The prev_bev rotation computed from an angle (occb200_rotation_coeffs, the gathers' rotation_source in elementwise.cu) against
its definition, `rotation_index_map`: torchvision's rotate of an index image.  No GPU: the coefficients come from the C ABI's
host-only entry, and a numpy mirror of the device formula (same operations, same order, same roundings) stands in for the
kernel, which test_rotation_gpu.py compares with the same maps on the device.  Also the argument rejections of the angle
entries, which happen before any CUDA call."""
import ctypes
import hashlib
import math
import os

import numpy as np
import pytest
import torch

from occnet_b200.engine import rotation_index_map

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'rotation_maps.npz')
FAKE = 1 << 12                       # never dereferenced: every call below is rejected before it reads a buffer
SPECIAL = [0.0, -0.0, 90.0, -90.0, 180.0, -180.0, 1e-3, -1e-3, 179.999, -179.999, 45.0, 0.5, -0.5, 360.0]
# (bev_h, bev_w, rotate_center): the shipped grid, the tests' small grid, and a non-square one with an off-grid centre
GRIDS = [(200, 200, (100, 100)), (50, 50, (20, 20)), (30, 44, (7, 31))]


def angle_set(seed, n_uniform, n_small):
    """every 0.5 degree step, the special angles, and seeded random angles in [-180, 180] and [-5, 5]"""
    rng = np.random.default_rng(seed)
    return np.concatenate([np.arange(-180.0, 180.0 + 0.25, 0.5), SPECIAL, rng.uniform(-180, 180, n_uniform),
                           rng.uniform(-5, 5, n_small)])


def coeffs(lib, angle, h, w, center):
    out = np.zeros(6, np.float32)
    rc = lib.occb200_rotation_coeffs(float(angle), h, w, int(center[0]), int(center[1]), out.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0, lib.occb200_last_error().decode()
    return out


def torchvision_coeffs(angle, h, w, center):
    """the first lines of torchvision's rotate + _gen_affine_grid: theta in double -> fp32, divided in fp32 by [W/2, H/2]"""
    from torchvision.transforms.functional import _get_inverse_affine_matrix
    center_f = [1.0 * (c - s * 0.5) for c, s in zip(center, [w, h])]
    m = _get_inverse_affine_matrix(center_f, -float(angle), [0.0, 0.0], 1.0, [0.0, 0.0])
    theta = torch.tensor(m, dtype=torch.float32).reshape(1, 2, 3)
    r = theta.transpose(1, 2) / torch.tensor([0.5 * w, 0.5 * h], dtype=torch.float32)      # (1, 3, 2)
    return r[0].t().contiguous().reshape(-1).numpy()                                        # rows g_x, g_y


def _fma32(a, b, c):
    """fp32 a * b + c with ONE rounding (the device's __fmaf_rn): the product is exact in double; the double sum is
    corrected with its TwoSum error when it lands exactly halfway between two floats (the only case where rounding the
    double sum to fp32 differs from rounding the exact sum)."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    f = s.astype(np.float32)
    d = s - f.astype(np.float64)
    toward = np.nextafter(f, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    half = np.abs(toward.astype(np.float64) - f.astype(np.float64)) * 0.5
    fix = (d != 0) & (np.abs(d) == half) & (err != 0) & (np.sign(err) == np.sign(d))
    return np.where(fix, toward, f)


def mirror_map(r, h, w):
    """numpy restatement of rotation_source (elementwise.cu), operation for operation"""
    r = r.astype(np.float32)
    i, j = np.divmod(np.arange(h * w), w)
    x = (np.float32(0.5) * (2 * j - w + 1).astype(np.float32)).astype(np.float32)
    y = (np.float32(0.5) * (2 * i - h + 1).astype(np.float32)).astype(np.float32)
    gx = _fma32(y, np.full_like(y, r[1]), x * r[0]) + r[2]
    gy = _fma32(y, np.full_like(y, r[4]), x * r[3]) + r[5]
    ix = np.rint(((gx + np.float32(1)) * np.float32(w) - np.float32(1)) / np.float32(2))
    iy = np.rint(((gy + np.float32(1)) * np.float32(h) - np.float32(1)) / np.float32(2))
    ok = (ix >= 0) & (ix < w) & (iy >= 0) & (iy < h)
    return np.where(ok, iy.astype(np.int64) * w + ix.astype(np.int64), -1).astype(np.int32)


def _mismatch(got, want, w):
    bad = np.flatnonzero(got != want)
    return f'{bad.size} cells differ, first (row, col, got, want): ' + \
        str([(int(q // w), int(q % w), int(got[q]), int(want[q])) for q in bad[:5]])


def test_fma32_mirror_rounds_once():
    a = np.array([1 + 2.0 ** -12, 3.0, 1.0], np.float32)
    b = np.array([1 + 2.0 ** -12, 1 / 3, 2.0 ** -30], np.float32)
    c = np.array([-(1 + 2.0 ** -11), -1.0, 1.0], np.float32)
    exact = [float(x) * float(y) + float(z) for x, y, z in zip(a, b, c)]
    want = np.array(exact, np.float64).astype(np.float32)          # each exact value is representable in double here
    assert np.array_equal(_fma32(a, b, c), want)
    # (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 lies halfway between two floats; a tiny c that the double sum drops decides the
    # rounding (plain double arithmetic would round both to the even neighbour 1 + 2^-11)
    ab = np.array([1 + 2.0 ** -12] * 2, np.float32)
    got = _fma32(ab, ab, np.array([2.0 ** -100, -2.0 ** -100], np.float32))
    assert got[0] == np.float32(1 + 2.0 ** -11 + 2.0 ** -23) and got[1] == np.float32(1 + 2.0 ** -11)


def test_rotation_coeffs_equal_torchvision(lib_built):
    from occnet_b200 import _lib
    lib = _lib.load()
    n = 0
    for h, w, center in GRIDS:
        for a in angle_set(7 + h, 3000, 1000):
            got, want = coeffs(lib, a, h, w, center), torchvision_coeffs(a, h, w, center)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (a, h, w, center, got, want)
            n += 1
    assert n >= 10000


def test_device_formula_mirror_equals_rotation_index_map(lib_built):
    from occnet_b200 import _lib
    lib = _lib.load()
    h, w, center = GRIDS[0]
    angles = angle_set(11, 2000, 1000)
    assert len(angles) >= 3000 and all(a in angles for a in (0.0, 90.0, -90.0, 180.0, 1e-3, -1e-3, 179.999, -179.999))
    for a in angles:
        got, want = mirror_map(coeffs(lib, a, h, w, center), h, w), rotation_index_map(h, w, float(a), center)
        assert np.array_equal(got, want), (a, _mismatch(got, want, w))
    for h, w, center in GRIDS[1:]:
        for a in angle_set(13 + w, 300, 200):
            got, want = mirror_map(coeffs(lib, a, h, w, center), h, w), rotation_index_map(h, w, float(a), center)
            assert np.array_equal(got, want), (a, h, w, center, _mismatch(got, want, w))


def map_digest(m):
    return hashlib.sha256(np.ascontiguousarray(m, np.int32).tobytes()).hexdigest().encode()


def test_golden_rotation_maps_pin_the_definition(lib_built):
    """tests/golden/rotation_maps.npz: SHA-256 of torchvision's maps for a seeded angle set, written by
    tests/golden/gen_rotation_maps.py.  Both this host's torchvision and the device formula's mirror must reproduce them."""
    from occnet_b200 import _lib
    lib = _lib.load()
    for h, w, center, angles, digests in golden_cases():
        for a, dig in zip(angles, digests):
            want = rotation_index_map(h, w, float(a), center)
            assert map_digest(want) == dig, ('torchvision', float(a), h, w, center)
            assert map_digest(mirror_map(coeffs(lib, a, h, w, center), h, w)) == dig, (float(a), h, w, center)


def golden_cases():
    """-> [(bev_h, bev_w, center, angles, sha256 digests)] of tests/golden/rotation_maps.npz"""
    g = np.load(GOLDEN)
    return [(int(h), int(w), (int(cx), int(cy)), g[f'angles_{k}'], list(g[f'sha256_{k}']))
            for k, (h, w, cx, cy) in enumerate(g['grids'])]


# ------------------------------------------------------------------------------------------------- argument rejections
def _call(name, *args):
    from occnet_b200 import _lib
    lib = _lib.load()
    rc = getattr(lib, 'occb200_' + name)(*args)
    return rc, lib.occb200_last_error().decode()


def _feats():
    return (ctypes.c_void_p * 4)(*([FAKE] * 4))


NON_FINITE = [math.nan, math.inf, -math.inf]


@pytest.mark.parametrize('angle', NON_FINITE)
def test_non_finite_angles_are_rejected(angle, lib_built):
    calls = [('engine_forward_video_angle', None, _feats(), angle, 0, None, None, FAKE, None, None, None),
             ('engine_submit_host_video_angle', None, 0, _feats(), angle, 0, FAKE, FAKE, None),
             ('engine_set_prev_rotation_angle', None, angle),
             ('engine_rotation_map', None, angle, FAKE, None),
             ('rotation_coeffs', angle, 200, 200, 100, 100, FAKE)]
    for name, *args in calls:
        rc, err = _call(name, *args)
        assert rc == 1 and 'finite' in err, (name, rc, err)


def test_null_engine_and_pointers_are_rejected(lib_built):
    for name, *args in [('engine_forward_video_angle', None, _feats(), 3.0, 0, None, None, FAKE, None, None, None),
                        ('engine_submit_host_video_angle', None, 0, _feats(), 3.0, 0, FAKE, FAKE, None),
                        ('engine_set_prev_rotation_angle', None, 3.0),
                        ('engine_rotation_map', None, 3.0, FAKE, None)]:
        rc, err = _call(name, *args)
        assert rc == 1 and 'null engine' in err, (name, err)
    rc, err = _call('engine_forward_video_angle', None, None, 3.0, 0, None, None, FAKE, None, None, None)
    assert rc == 1 and 'null pointer' in err
    for feats, occ, flow in ((None, FAKE, FAKE), (_feats(), None, FAKE), (_feats(), FAKE, None)):
        rc, err = _call('engine_submit_host_video_angle', None, 1, feats, 3.0, 0, occ, flow, None)
        assert rc == 1 and 'null pointer' in err, (feats, occ, flow)
    rc, err = _call('engine_rotation_map', None, 3.0, None, None)
    assert rc == 1 and 'null pointer' in err
    rc, err = _call('rotation_coeffs', 3.0, 200, 200, 100, 100, None)
    assert rc == 1 and 'null pointer' in err
    for h, w in ((0, 200), (200, 0), (-1, 5)):
        rc, err = _call('rotation_coeffs', 3.0, h, w, 100, 100, FAKE)
        assert rc == 1 and 'positive' in err


@pytest.mark.parametrize('slot', [-1, 2, 7])
def test_bad_slot_is_rejected(slot, lib_built):
    rc, err = _call('engine_submit_host_video_angle', None, slot, _feats(), 3.0, 0, FAKE, FAKE, None)
    assert rc == 1 and 'slot' in err
