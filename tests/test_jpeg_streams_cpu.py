"""CPU side of the hand-built baseline streams (tests/golden/jpeg_streams.py): the writer is pinned by the oracle's entropy
decoder, the oracle (oracle/jpeg_decode.py) is byte-identical to cv2.imdecode on every case, the library's header parser
accepts every case, every family holds what it claims on the bytes, and fill bytes before RSTn / EOI decode while FF FF 00
stays corrupt."""
import ctypes
import functools
import hashlib
import json
import os
import re
import sys

import numpy as np
import pytest

from oracle import jpeg_decode as J

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import jpeg_streams as S  # noqa: E402

FAMILIES = ['header', 'codes', 'coef', 'stuffing', 'restart', 'worst']
THREADS = 1024                                          # jpeg_entropy_kernel's block: step 1 gives each thread one chunk


@functools.lru_cache(maxsize=None)
def _cases():
    return tuple(S.cases())


def _family(f):
    return [c for c in _cases() if c['family'] == f]


def _scan(c):
    """the entropy-coded segment as the device sees it: from the end of the SOS header to the EOI marker"""
    return c['data'][c['info']['scan_off']:len(c['data']) - 2]


def _log(c):
    """per interval, the (kind, symbol, value) the writer emitted"""
    log = []
    S.interval_bits(c['spec'], log)
    return log


# ------------------------------------------------------------------------------------------------------- every case
@pytest.mark.parametrize('family', FAMILIES)
def test_writer_is_pinned_and_the_oracle_equals_cv2(family, lib_built):
    from occnet_b200 import _lib
    lib = _lib.load()
    for c in _family(family):
        hdr = J.parse(c['data'])
        planes = J.entropy_decode(hdr)
        for got, want in zip(planes, c['spec']['planes']):
            assert np.array_equal(got, want), c['name']
        want = J.cv2_decode(c['data'])
        assert want is not None and np.array_equal(J.decode(c['data']), want), c['name']
        h, w = ctypes.c_int(), ctypes.c_int()
        rc = lib.occb200_jpeg_info(c['data'], len(c['data']), ctypes.byref(h), ctypes.byref(w))
        assert rc == 0 and (h.value, w.value) == (c['spec']['h'], c['spec']['w']), (c['name'], lib.occb200_last_error())


def test_digests_pin_cv2_and_the_oracle(golden_dir):
    sums = json.load(open(os.path.join(golden_dir, 'jpeg_streams_sha256.json')))
    assert sorted(sums) == sorted(c['name'] for c in _cases())
    for c in _cases():
        assert hashlib.sha256(J.cv2_decode(c['data']).tobytes()).hexdigest() == sums[c['name']], ('cv2', c['name'])
        assert hashlib.sha256(J.decode(c['data']).tobytes()).hexdigest() == sums[c['name']], ('oracle', c['name'])


def test_every_family_in_both_samplings():
    for f in FAMILIES:
        assert {c['spec']['sub'] for c in _family(f)} == {1, 2}, f


# ------------------------------------------------------------------------------------------------------- family claims
def test_header_family():
    a420, b420, a444, b444 = (c for c in _family('header'))
    for c in (a420, a444):
        hdr = J.parse(c['data'])
        assert [x[0] for x in hdr['comps']] == [0, 1, 2] and [x[3] for x in hdr['comps']] == [0, 2, 3]
        assert [x[2:] for x in c['spec']['comps']] == [(1, 1), (0, 0), (2, 2)]
        assert c['data'].count(b'\xff\xc4') == 1 and c['data'].count(b'\xff\xdb') == 1       # all tables in one segment
        assert c['data'][2:4] == b'\xff\xff' and hdr['restart'] == 4
    for c in (b420, b444):
        d = c['data']
        hdr = J.parse(d)
        assert [x[0] for x in hdr['comps']] == [7, 200, 42] and [x[3] for x in hdr['comps']] == [3, 2, 0]
        assert c['spec']['comps'][2][2:] == (3, 3)
        assert d.index(b'\xff\xc1') < d.index(b'\xff\xdb') < d.index(b'\xff\xc4')            # SOF1, tables after it
        assert d.count(b'\xff\xdd') == 2 and hdr['restart'] == 0                              # DRI 5, then DRI 0
        # AC table 1 defined twice, the decoy first; quantisation table 2 too: the last definitions are the ones written
        dht = [m.start() for m in re.finditer(b'\xff\xc4', d)]
        assert sum(d[p + 4] == 0x11 for p in dht) == 2
        assert d.count(b'\xff\xfe') == 1 and d.count(b'\xff\xef') == 1 and b'\xff\xff\xff\xff\xff\xc4' in d


def test_codes_family():
    every = [c for c in _family('codes') if 'every-length' in c['name']]
    for c in every:
        used = {}                                        # code length -> codes emitted, over all four tables
        for tc, th in c['spec']['ht']:
            t = c['spec']['ht'][(tc, th)]
            emitted = {sym for kind, sym, _ in _log(c) if kind == ('dc' if tc == 0 else 'ac')}
            for ln, code, sym in t.codes:
                if sym in emitted:
                    used.setdefault(ln, set()).add(code)
        assert set(used) == set(range(1, 17)), (c['name'], sorted(used))
        assert 0xFFFE in used[16]                        # one below the reserved all-ones code
        comps = c['spec']['comps']
        assert any(td != ta for _, _, td, ta in comps)   # crossed DC / AC tables
    full = [c for c in _family('codes') if 'full-ac' in c['name']]
    for c in full:
        t = c['spec']['ht'][(1, 0)]
        assert sorted(t.vals) == sorted(S.AC_SYMBOLS) and {13, 14} <= t.lengths()
    for c in [c for c in _family('codes') if 'single' in c['name']]:
        scan = _scan(c)
        per = 1 if c['spec']['sub'] == 1 else 2          # 3 or 6 two-bit blocks per MCU and interval
        n_iv = np.prod(S.geometry(c['spec']['h'], c['spec']['w'], c['spec']['sub']))
        assert c['info']['iv_bits'] == [2 * len(S.mcu_layout(c['spec']['sub']))] * n_iv
        assert len(scan) == n_iv * per + (n_iv - 1) * 2


def test_coef_family():
    for c in _family('coef'):
        log = _log(c)
        dc = {s for kind, s, _ in log if kind == 'dc'}
        assert dc == set(range(12)), sorted(dc)
        ac = [(s >> 4, s & 15, v) for kind, s, v in log if kind == 'ac' and s not in (S.EOB, S.ZRL)]
        assert {r for r, _, _ in ac} == set(range(16))
        mags = {}
        for _, s, v in ac:
            mags.setdefault(s, set()).add(abs(v))
        for s in range(1, 11):                          # size 10's 1023 is beyond the FDCT: its bound at (0, 1) instead
            tops = {(1 << s) - 1} if s < 10 else {int(S.FDCT_MAX[1]), int(-S.FDCT_MIN[1])}
            assert {1 << (s - 1)} | tops <= mags[s], (s, sorted(mags[s]))
        # blocks as symbol sequences
        blocks, cur = [], None
        for kind, s, v in log:
            if kind == 'dc':
                cur = []
                blocks.append(cur)
            cur.append((kind, s, v))
        assert any(len(b) == 2 and b[1][1] == S.EOB for b in blocks)                         # EOB right after DC
        assert any(not p.reshape(-1, 64)[i].any() for p in c['spec']['planes'] for i in range(p.shape[0] * p.shape[1]))
        ends63 = [b for b in blocks if b[-1][1] != S.EOB]
        assert any(len(b) == 64 for b in ends63)                                             # 63 coefficients
        chains = set()                                                                       # ZRL chains before 63
        for b in ends63:
            k = 0
            while b[-2 - k][1] == S.ZRL:
                k += 1
            chains.add(k)
        assert {1, 2, 3} <= chains, chains
        assert len(c['info']['iv_bits']) >= 8


def _chunk_splits(scan, second):
    """byte offsets i with scan[i] = FF and scan[i + 1] matching `second`, where step 1 puts i and i + 1 in different chunks"""
    chunk = -(-len(scan) // THREADS)
    return [i for i in range(chunk - 1, len(scan) - 1, chunk) if scan[i] == 0xFF and second(scan[i + 1])]


def test_stuffing_family():
    for c in _family('stuffing'):
        scan = _scan(c)
        pairs = scan.count(b'\xff\x00')
        assert 2 * pairs >= 0.3 * len(scan), (c['name'], 2 * pairs / len(scan))
        assert _chunk_splits(scan, lambda b: b == 0), c['name']
        assert _chunk_splits(scan, lambda b: 0xD0 <= b <= 0xD7), c['name']


def _fill_runs(scan):
    """(start, length, marker byte) of every run of FF fill bytes before a marker in the scan, EOI included"""
    out = []
    for m in re.finditer(rb'\xff+(?=[\xd0-\xd7]|$)', scan):
        if m.end() - m.start() > 1 or m.end() == len(scan):
            out.append((m.start(), m.end() - m.start() - (m.end() < len(scan)), scan[m.end()] if m.end() < len(scan) else 0xD9))
    return out


def test_restart_family():
    byname = {c['name']: c for c in _family('restart')}
    for tag, sub in (('420', 2), ('444', 1)):
        c = byname[f'restart-dri-beyond-{tag}']
        assert c['spec']['restart'] > np.prod(S.geometry(c['spec']['h'], c['spec']['w'], sub))
        assert len(c['info']['iv_bits']) == 1
        c = byname[f'restart-dri-off-row-{tag}']
        assert S.geometry(c['spec']['h'], c['spec']['w'], sub)[1] % c['spec']['restart'] != 0
        c = byname[f'restart-1x1-{tag}']
        assert (c['spec']['h'], c['spec']['w'], c['spec']['restart']) == (1, 1, 1)
        c = byname[f'restart-dri1-1600x900-fill-{tag}']
        assert c['spec']['restart'] == 1 and len(c['info']['iv_bits']) > THREADS
        for name in (f'restart-exact1024-{tag}', f'restart-exact1024-fill-{tag}'):
            assert all(b % 1024 == 0 for b in byname[name]['info']['iv_bits']) and set(byname[name]['info']['pad']) == {0}
        for name in (f'restart-pad7-{tag}', f'restart-pad7-fill-{tag}'):
            assert set(byname[name]['info']['pad']) == {7}
    crossing = 0
    for c in _family('restart'):
        if not S.has_fill(c):
            assert not _fill_runs(_scan(c)), c['name']
            continue
        scan = _scan(c)
        runs = _fill_runs(scan)
        # 1-3 fill bytes before every RSTn and before EOI
        assert len(runs) == len(c['info']['iv_bits']) and all(1 <= n <= 3 for _, n, _ in runs), c['name']
        assert runs[-1][2] == 0xD9
        chunk = -(-len(scan) // THREADS)
        crossing += sum((s + n) // chunk != s // chunk for s, n, _ in runs)         # the run and its marker's FF
    assert crossing > 0


def test_worst_family_tables_never_meet_the_true_phase():
    """every table symbol has a code + extra bits of even total length but DC category 1, whose code is 1110"""
    dc, ac = S.worst_tables()
    for ln, code, sym in dc.codes:
        assert (ln + sym) % 2 == 0 or (sym == 1 and format(code, f'0{ln}b') == '1110'), (ln, code, sym)
    for ln, code, sym in ac.codes:
        assert (ln + (sym & 15)) % 2 == 0, (ln, code, sym)
    for t in (dc, ac):                                  # complete but for the all-ones prefix: a decoder never errs
        assert sum(1 << (16 - ln) for ln, _, _ in t.codes) == (1 << 16) - 1


def test_worst_family_streams():
    for c in _family('worst'):
        ivs = S.interval_bits(c['spec'])
        for bits in ivs:
            assert bits[:4] == '1110' and '111' not in bits[5:], c['name']
        n_sub = [-(-len(b) // 1024) for b in ivs]
        if len(ivs) == 1:
            assert n_sub[0] >= 2 * THREADS, (c['name'], n_sub)
        else:
            assert min(n_sub) >= 4, (c['name'], n_sub)
        # the unstuffed scan is the writer's bit string and its padding
        data, starts = J.unstuff(_scan(c))
        assert len(starts) == len(ivs) and len(data) == sum(-(-len(b) // 8) for b in ivs)


@pytest.mark.parametrize('sub', [1, 2])
def test_worst_family_reduced_instance_needs_one_pass_per_subsequence(sub):
    """the same construction at a size the Python model can run: every serial boundary after the first symbol at an odd bit
    offset, and the Jacobi model with 64-bit subsequences needs at least (subsequences - 2) passes and ends exact"""
    c = S.worst_case(sub, 16, 48, seed=1)
    hdr = J.parse(c['data'])
    bounds = J.true_boundaries(hdr)
    assert all(pos % 2 == 1 for pos, _, _ in bounds if pos >= 5)
    _, iv = J.intervals(hdr)
    n_sub = -(-(iv[0][1] - iv[0][0]) // 64)
    starts, passes = J.sync_model(hdr, 64)
    assert n_sub >= 20 and passes >= n_sub - 2, (n_sub, passes)
    assert set(starts) <= bounds


# ------------------------------------------------------------------------------------------------------- fill bytes
def _with_fill(data, k):
    """`data` (one scan) with k FF fill bytes before every RSTn marker and before EOI"""
    sos = data.index(b'\xff\xda')
    head, scan = data[:sos], data[sos:]
    scan = re.sub(rb'\xff([\xd0-\xd7\xd9])', lambda m: b'\xff' * (k + 1) + m.group(1), scan)
    return head + scan


@pytest.mark.parametrize('k', [1, 2, 3])
def test_oracle_decodes_fill_bytes_before_rst_and_eoi_as_cv2(k, lib_built):
    from occnet_b200 import _lib
    lib = _lib.load()
    for i, (h, w, s, r) in enumerate([(48, 64, '420', 1), (33, 47, '444', 7), (64, 512, '420', 'row'), (17, 9, '420', 0)]):
        base = J.encode(J.make_image('camera' if i % 2 else 'noise', h, w, seed=i), 90, s, r)
        data = _with_fill(base, k)
        assert len(data) > len(base)
        assert np.array_equal(J.cv2_decode(data), J.cv2_decode(base))
        assert np.array_equal(J.decode(data), J.cv2_decode(data)), (h, w, s, r)
        hh, ww = ctypes.c_int(), ctypes.c_int()
        assert lib.occb200_jpeg_info(data, len(data), ctypes.byref(hh), ctypes.byref(ww)) == 0


def test_ff_ff_00_stays_corrupt_in_the_oracle():
    """only a run of FF bytes that ends in RSTn or at the end of the scan is fill: FF FF 00 is no stuffed FF"""
    c = _family('stuffing')[0]
    data = bytearray(c['data'])
    p = data.index(b'\xff\x00', c['info']['scan_off'] + 40)
    data[p:p + 2] = b'\xff\xff\x00'
    with pytest.raises(ValueError, match='marker inside the scan'):
        J.decode(bytes(data))
    with pytest.raises(ValueError, match='marker inside the scan'):
        J.unstuff(b'\x12\xff\xff\x00\x34')
    assert J.unstuff(b'\x12\xff\x00\xff\xff\xd0\x34\xff\xff') == (b'\x12\xff\x34', [0, 2])
