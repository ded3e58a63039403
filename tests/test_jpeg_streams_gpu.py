"""The GPU JPEG decoder (occnet_b200/csrc/jpeg.cu) on the hand-built baseline streams of tests/golden/jpeg_streams.py, against
cv2.imdecode(IMREAD_UNCHANGED) byte for byte: header syntax libjpeg's writer never produces, every code length, every
coefficient category, FF-dense scans, restart geometry with fill bytes before RSTn and EOI, and scans that synchronise only
through their predecessors.  Each test runs in a child process."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
pytestmark = pytest.mark.gpu


def _run_isolated(code, timeout=1800):
    r = subprocess.run([sys.executable, '-c', 'import sys; sys.path.insert(0, "tests"); sys.path.insert(0, "tests/golden"); '
                        + code], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-20000:])
    assert r.returncode == 0, f'child failed ({r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'
    assert 'OK' in r.stdout
    return r.stdout


def _child(fn):
    return _run_isolated(f'import test_jpeg_streams_gpu as t; t.{fn}(); print("OK")')


def _mixed(cases):
    """round-robin over the families, so that every decode of six mixes them (and their subsequence counts)"""
    fams = {}
    for c in cases:
        fams.setdefault(c['family'], []).append(c)
    out = []
    while any(fams.values()):
        for f in list(fams):
            if fams[f]:
                out.append(fams[f].pop(0))
    return out


def _decode(dec, bufs):
    import torch
    got = dec.decode(bufs)
    torch.cuda.synchronize()
    return [g.cpu().numpy() for g in got], dec.status()


def streams_match_cv2():
    import jpeg_streams as S
    from occnet_b200.jpeg import JpegDecoder
    from oracle import jpeg_decode as J
    dec = JpegDecoder(DEV)
    cases = _mixed(S.cases())
    bad = []
    for k in range(0, len(cases), 6):
        batch = cases[k:k + 6]
        got, status = _decode(dec, [c['data'] for c in batch])
        for i, (c, g) in enumerate(zip(batch, got)):
            want = J.cv2_decode(c['data'])
            if status >> i & 1 or not np.array_equal(g, want):
                bad.append((c['name'], bool(status >> i & 1),
                            int(np.abs(g.astype(int) - want).max()) if g.shape == want.shape else 'shape'))
    print('cases', len(cases), 'failed (name, status bit, max |diff|):', bad)
    assert not bad, bad


def worst_case_alone_and_among_camera_files():
    """the single-interval worst cases alone, then each next to five cv2-encoded camera-like files; the decode time of the
    4:4:4 one, alone, from CUDA events"""
    import torch
    import jpeg_streams as S
    from occnet_b200.jpeg import JpegDecoder
    from oracle import jpeg_decode as J
    dec = JpegDecoder(DEV)
    worst = [S.worst_case(1, 900, 1600), S.worst_case(2, 900, 1600, n_ac=(10, 30))]
    natural = [J.encode(J.make_image('camera' if i % 2 else 'noise', 900, 1600, seed=i), 90, '420', [0, 'row', 7][i % 3],
                        bool(i % 2)) for i in range(5)]
    for c in worst:
        want = J.cv2_decode(c['data'])
        got, status = _decode(dec, [c['data']])
        assert status == 0 and np.array_equal(got[0], want), c['name']
        got, status = _decode(dec, natural[:2] + [c['data']] + natural[2:])
        assert status == 0, (c['name'], status)
        assert np.array_equal(got[2], want), c['name']
        for g, b in zip(got[:2] + got[3:], natural):
            assert np.array_equal(g, J.cv2_decode(b)), c['name']
    c = worst[0]
    bits = c['info']['iv_bits'][0]
    dec.decode([c['data']])
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = []
    for _ in range(3):
        ev[0].record()
        dec.decode([c['data']])
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    print(f'{c["name"]}: one interval of {bits} bits = {-(-bits // 1024)} subsequences of 1024 bits; '
          f'decode (upload + 3 kernels, one CUDA-event interval each) {ms} ms on {torch.cuda.get_device_name()}')


def ff_ff_00_stays_corrupt():
    """FF FF 00 inside the scan is not a stuffed FF: status bit set, the other images of the decode unaffected"""
    import jpeg_streams as S
    from occnet_b200.jpeg import JpegDecoder
    from oracle import jpeg_decode as J
    dec = JpegDecoder(DEV)
    good = [c for c in S.stuffing_cases()]
    data = bytearray(good[0]['data'])
    p = data.index(b'\xff\x00', good[0]['info']['scan_off'] + 40)
    data[p:p + 2] = b'\xff\xff\x00'
    got, status = _decode(dec, [good[1]['data'], bytes(data), good[1]['data']])
    assert status == 0b010, status
    assert np.array_equal(got[0], J.cv2_decode(good[1]['data'])) and np.array_equal(got[2], got[0])


def fill_files(n=6, h=220, w=400):
    """six camera files of natural content with 1-3 fill bytes before every RSTn and before EOI, DRI 1 / 7 / a row"""
    import jpeg_streams as S
    out = []
    for i in range(n):
        rng = np.random.default_rng([7, i])
        sub = 2 if i % 3 else 1
        qt = {0: S._qt(rng, 1, 16), 1: S._qt(rng, 1, 24)}
        ht = {(0, 0): S.full_dc(rng), (1, 0): S.full_ac(rng), (0, 1): S.full_dc(rng), (1, 1): S.full_ac(rng)}
        comps = [(1, 0, 0, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
        my, mx = S.geometry(h, w, sub)
        ri = [1, 7, mx][i % 3]
        planes = S.natural_planes(rng, h, w, sub, [qt[c[1]] for c in comps])
        out.append(S.write(dict(h=h, w=w, sub=sub, planes=planes, qt=qt, ht=ht, comps=comps, restart=ri,
                                fill_rst=S._fills(rng, -(-my * mx // ri)), fill_eoi=1 + i % 3))[0])
    return out


def engine_on_fill_files():
    """one frame-engine call with JPEG input (code 4) on six fill-byte files equals the call fed cv2's uint8 frames (code 3)"""
    import torch
    import test_jpeg_gpu as T
    from oracle import jpeg_decode as J
    files = fill_files()
    frames = torch.from_numpy(np.stack([J.cv2_decode(b) for b in files]))
    eng = T._engine('fp32')
    eng.set_input_dtype(torch.uint8)
    want = {k: v.clone() for k, v in eng.forward(frames.to(DEV), want=T.WANT).items()}
    eng.set_input_dtype('jpeg')
    got = eng.forward(files, want=T.WANT)
    torch.cuda.synchronize()
    assert eng.jpeg_status() == 0
    for k in want:
        assert torch.equal(want[k], got[k]), k


def test_streams_match_cv2():
    """every case of every family, in decodes of six that mix the families"""
    _child('streams_match_cv2')


def test_worst_case_alone_and_among_camera_files():
    _child('worst_case_alone_and_among_camera_files')


def test_ff_ff_00_stays_corrupt():
    _child('ff_ff_00_stays_corrupt')


def test_engine_on_fill_byte_files():
    _child('engine_on_fill_files')
