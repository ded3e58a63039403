"""The ray caster's edge families (tests/golden/dvr_edges.py) without a GPU: every family produces the geometry it claims,
checked on a Python restatement of the walk that logs every branch; the C oracle (oracle/ray_dda.c) equals that restatement
on every ray of every family; and occb200_render_forward refuses bad arguments before any CUDA call (return code 1, an
argument check, not 2, a CUDA error)."""
import os
import sys

import numpy as np
import pytest

from oracle import ray_metrics as ORM

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import dvr_edges as E  # noqa: E402

CASES = E.cases()
NAMES = [c['name'] for c in CASES]
FAKE = 1 << 12                       # never dereferenced: every call below is rejected before it reads a buffer


def _case(name):
    return CASES[NAMES.index(name)]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_every_family_is_present():
    tags = {}
    for c in CASES:
        for tg in c['claims'].values():
            for t in tg:
                tags[t] = tags.get(t, 0) + 1
    for want in ('tie:xy', 'tie:xz', 'tie:yz', 'tie:xyz', 'zero:1', 'zero:2', 'zero:len', 'face', 'lattice', 'band',
                 'outside:x-', 'outside:x+', 'outside:y-', 'outside:y+', 'outside:z-', 'outside:z+', 'entry:999', 'entry:1000',
                 'entry:never', 'cut', 'hit:first', 'hit:last', 'miss:0.5', 'miss:nan', 'miss:-1', 'padded'):
        assert tags.get(want, 0) > 0, want
    shapes = {c['sigma'].shape[2:] for c in CASES}
    for zyx in ((16, 200, 200), (200, 13, 7), (13, 7, 200), (7, 200, 13), (1, 1, 1), (1, 9, 1), (2, 3, 1200)):
        assert zyx in shapes, zyx
    batch = {(c['sigma'].shape[1], c['origin'].shape[1]) for c in CASES if c['sigma'].shape[0] == 3}
    assert batch == {(1, 1), (1, 3), (3, 1), (3, 3)}


@pytest.mark.parametrize('name', NAMES)
def test_family_claims_hold(name):
    """ties are exact ties inside the grid in every octant, the entry happens at step 999 / 1000 (and never after 1001
    steps), the truncation band starts inside, the cut-off happens inside, sigma 0.5 / NaN / -1 miss and the others hit
    at the first or the last in-grid voxel"""
    c = _case(name)
    counts = E.check_claims(c)
    assert sum(counts.values()) == sum(len(t) for t in c['claims'].values())
    if name.startswith('tie_'):
        kind = name.split('_')[1]
        octants = set()
        for (n, m), tags in c['claims'].items():
            d = c['points'][n, m, :3] - c['origin'][0, int(c['tindex'][n, m])]
            octants.add(tuple(np.sign(d) >= 0))
        assert len(octants) == 8 and counts['tie:' + kind] >= 24, (octants, counts)


@pytest.mark.parametrize('name', NAMES)
def test_c_oracle_equals_the_logged_walk(name):
    """oracle/ray_dda.c and the Python restatement agree bit for bit on every ray (NaN for NaN)"""
    c = _case(name)
    pd, gd, ci = ORM.render_forward(c['sigma'], c['origin'], c['points'], c['tindex'])
    walks = E.walk_case(c)
    for (n, m), (outp, _) in walks.items():
        want = (np.float32(-1), np.float32(-1), np.zeros(3, np.float32)) if outp is None else outp
        for what, g, w in (('pred_dist', pd[n, m], want[0]), ('gt_dist', gd[n, m], want[1]), ('coord_index', ci[n, m], want[2])):
            g, w = np.atleast_1d(np.float32(g)), np.atleast_1d(np.float32(w))
            same = (_bits(g) == _bits(w)) | (np.isnan(g) & np.isnan(w))
            assert same.all(), f'{name}: ray (n={n}, m={m}) {what}: oracle {g} walk {w}'


def test_batch_cases_index_origin_through_its_own_To():
    """the oracle reads origin[n][t] through origin's own To: in the T = 1, To = 3 batch the rows n >= 1 would walk from
    another item's origin with sigma's T as the stride, and the outputs differ"""
    c = _case('batch_T1_To3')
    pd = ORM.render_forward(c['sigma'], c['origin'], c['points'], c['tindex'])[0]
    N, To = c['origin'].shape[:2]
    flat = c['origin'].reshape(-1, 3)
    wrong = np.stack([[flat[n * 1 + t] for t in range(To)] for n in range(N)])      # origin + (n * T + t) * 3 with T = 1
    pw = ORM.render_forward(c['sigma'], wrong, c['points'], c['tindex'])[0]
    assert np.array_equal(pd[0], pw[0]) and not np.array_equal(pd[1:], pw[1:])


def test_lidar_fixture_has_no_exact_ties():
    """the lidar-bundle scene the older render_forward tests use never reaches a tie: from its first origin not one of
    the in-grid decisions of a sample of its rays compares two equal tMax values (over the whole bundle, from both
    in-grid origins, none of 2.8 million), which is why the edge families above exist"""
    rays = ORM.generate_lidar_rays()[::20]
    o = ((np.float32([0.98, 0.0, 1.84]) - np.float32([-40, -40, -1])) / np.float32(0.4)).astype(np.float32)
    p = ((rays + np.float32([0.98, 0.0, 1.84]) - np.float32([-40, -40, -1])) / np.float32(0.4)).astype(np.float32)
    ties = decisions = 0
    for e in p:
        _, log = E.walk(o, e, (200, 200, 16), lambda x, y, z: False)
        decisions += len(log['ties'])
        ties += sum(1 for s in log['ties'] if s)
    assert decisions > 50000 and ties == 0, (ties, decisions)


# ------------------------------------------------------------------------------------------------------ C-ABI rejections
_RF = dict(sigma=1, origin=1, points=1, tindex=1, N=2, T=1, To=3, Z=4, Y=5, X=6, M=7, K=3, pred=1, gt=1, coord=1)
_REJECT = [
    (dict(sigma=None), 'null'), (dict(origin=None), 'null'), (dict(points=None), 'null'), (dict(tindex=None), 'null'),
    (dict(pred=None), 'null'), (dict(gt=None), 'null'), (dict(coord=None), 'null'),
    (dict(N=-1), '65535'), (dict(N=65536), '65535'), (dict(M=-1), 'M >= 0'),
    (dict(T=0), 'positive'), (dict(To=0), 'positive'), (dict(Z=0), 'positive'), (dict(Y=-2), 'positive'), (dict(X=0), 'positive'),
    (dict(K=2), 'K >= 3'), (dict(K=0), 'K >= 3'),
]


@pytest.mark.parametrize('case', range(len(_REJECT)))
def test_render_forward_entry_rejects_bad_arguments_before_any_cuda_call(case, lib_built):
    import ctypes
    from occnet_b200 import _lib
    lib = _lib.load()
    over, msg = _REJECT[case]
    a = dict(_RF, **over)
    p = {k: (None if a[k] is None else ctypes.c_void_p(FAKE)) for k in ('sigma', 'origin', 'points', 'tindex', 'pred', 'gt', 'coord')}
    rc = lib.occb200_render_forward(p['sigma'], p['origin'], p['points'], p['tindex'], a['N'], a['T'], a['To'], a['Z'], a['Y'],
                                    a['X'], a['M'], a['K'], p['pred'], p['gt'], p['coord'], None)
    err = lib.occb200_last_error().decode()
    assert rc == 1, (over, rc, err)
    assert msg in err, (over, err)
