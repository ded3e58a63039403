"""CPU side of the JPEG input: the numpy oracle (oracle/jpeg_decode.py) byte-identical to cv2.imdecode(IMREAD_UNCHANGED),
the library's header parser accepting exactly the supported files and rejecting the rest before any CUDA call, and a CPU model
of the device decoder's self-synchronising Huffman phase landing on the true codeword boundaries."""
import ctypes
import hashlib
import itertools
import json
import os

import numpy as np
import pytest

from oracle import jpeg_decode as J

SIZES = [(48, 64), (17, 9), (9, 17), (8, 8), (1, 1)]
QUALITIES = [5, 50, 75, 95, 100]
SAMPLINGS = ['420', '444']
RESTARTS = [0, 1, 7, 'row']
OPTIMIZE = [False, True]


def _cases(h, w):
    for i, (q, s, r, o, c) in enumerate(itertools.product(QUALITIES, SAMPLINGS, RESTARTS, OPTIMIZE, J.CONTENTS)):
        yield (q, s, r, o, c), J.encode(J.make_image(c, h, w, seed=i + h), q, s, r, o)


@pytest.mark.parametrize('size', SIZES, ids=lambda s: f'{s[1]}x{s[0]}')
def test_oracle_is_byte_identical_to_cv2(size):
    for case, buf in _cases(*size):
        assert np.array_equal(J.decode(buf), J.cv2_decode(buf)), case


def test_oracle_is_byte_identical_to_cv2_at_256():
    for c in J.CONTENTS:
        buf = J.encode(J.make_image(c, 256, 256, seed=3), 90, '420', 0, False)
        assert np.array_equal(J.decode(buf), J.cv2_decode(buf)), c


def test_golden_files_pin_cv2_and_the_oracle(golden_dir):
    sums = json.load(open(os.path.join(golden_dir, 'jpeg_sha256.json')))
    assert len(sums) == 5
    for name, digest in sums.items():
        data = open(os.path.join(golden_dir, 'jpeg', name + '.jpg'), 'rb').read()
        assert hashlib.sha256(J.cv2_decode(data).tobytes()).hexdigest() == digest, name
        assert hashlib.sha256(J.decode(data).tobytes()).hexdigest() == digest, name


# ---------------------------------------------------------------------------------------------------------------- parser
def _info(lib, data):
    h, w = ctypes.c_int(), ctypes.c_int()
    rc = lib.occb200_jpeg_info(data, len(data), ctypes.byref(h), ctypes.byref(w))
    return rc, (h.value, w.value), lib.occb200_last_error().decode()


def _patch_sof(data, off, value):
    b = bytearray(data)
    p = b.index(b'\xff\xc0')
    b[p + 4 + off] = value
    return bytes(b)


def _unsupported():
    img = J.make_image('camera', 40, 56, seed=1)
    base = J.encode(img, 90)
    import cv2
    gray = cv2.imencode('.jpg', img[..., 0])[1].tobytes()
    adobe = base[:2] + b'\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00' + base[2:]
    dqt = bytearray(base)
    dqt[dqt.index(b'\xff\xdb') + 4] |= 0x10
    sos = bytearray(base)
    sos[sos.index(b'\xff\xda') + 4] = 1
    arith = bytearray(base)
    arith[arith.index(b'\xff\xc0') + 1] = 0xC9
    return {
        'progressive': (J.encode(img, 90, progressive=True), 'progressive'),
        '4:2:2': (J.encode(img, 90, '422'), 'sampling'),
        '4:1:1': (J.encode(img, 90, '411'), 'sampling'),
        '4:4:0': (J.encode(img, 90, '440'), 'sampling'),
        'grayscale': (gray, 'grayscale'),
        'cmyk': (_patch_sof(base, 5, 4), 'CMYK'),
        '12-bit': (_patch_sof(base, 0, 12), '12-bit'),
        '16-bit tables': (bytes(dqt), '16-bit quantisation'),
        'arithmetic': (bytes(arith), 'arithmetic'),
        'adobe': (adobe, 'Adobe'),
        'several scans': (bytes(sos), 'several scans'),
        'truncated': (base[:len(base) // 2], 'truncated'),
        'truncated header': (base[:100], 'truncated'),
        'over-subscribed table, 200 codes of 1 bit': (_dht(base, [200] + [0] * 15), 'over-subscribed'),
        'over-subscribed table, 2 + 1 codes': (_dht(base, [2, 1] + [0] * 14), 'over-subscribed'),
        'all-ones code used': (_dht(base, [1, 2] + [0] * 14), 'over-subscribed'),
    }


def _dht(data, bits):
    """`data` with DC table 0 redefined by one more DHT segment (the given code-length counts) just before the scan"""
    vals = bytes(range(sum(bits) % 256)) + bytes(max(0, sum(bits) - 256))
    seg = bytes([0x00]) + bytes(bits) + vals
    p = data.index(b'\xff\xda')
    return data[:p] + b'\xff\xc4' + (len(seg) + 2).to_bytes(2, 'big') + seg + data[p:]


def test_parser_accepts_the_scope(lib_built):
    from occnet_b200 import _lib
    lib = _lib.load()
    for (h, w), s, r, o in itertools.product([(900, 1600), (901, 1599), (1, 1)], SAMPLINGS, RESTARTS, OPTIMIZE):
        rc, hw, err = _info(lib, J.encode(J.make_image('flat', h, w), 75, s, r, o))
        assert rc == 0 and hw == (h, w), err


def test_parser_ignores_bytes_after_eoi(lib_built):
    """cv2 decodes a file with a trailer after its EOI marker; so does the oracle, and the parser accepts it"""
    from occnet_b200 import _lib
    data = J.encode(J.make_image('camera', 24, 40, seed=2), 90, '420', 1) + b'trailer \x00\xff\x00 bytes'
    rc, hw, err = _info(_lib.load(), data)
    assert rc == 0 and hw == (24, 40), err
    assert np.array_equal(J.decode(data), J.cv2_decode(data))


@pytest.mark.parametrize('name', list(_unsupported()))
def test_parser_rejects_the_rest_naming_the_feature(lib_built, name):
    """error 1 from a host-only entry (this machine has no GPU, so nothing can have reached CUDA); the oracle agrees"""
    from occnet_b200 import _lib
    data, word = _unsupported()[name]
    rc, _, err = _info(_lib.load(), data)
    assert rc == 1 and word.lower() in err.lower(), (name, err)
    with pytest.raises(J.JpegUnsupported, match=f'(?i){word}'):
        J.parse(data)


# ---------------------------------------------------------------------------------------------------- synchronisation
@pytest.mark.parametrize('sub_bits', [64, 256])
def test_sync_model_finds_the_true_boundaries(sub_bits):
    for (h, w) in [(48, 64), (17, 9)]:
        for case, buf in _cases(h, w):
            hdr = J.parse(buf)
            starts, _ = J.sync_model(hdr, sub_bits)
            assert set(starts) <= J.true_boundaries(hdr), case


def test_sync_model_worst_case_degrades_to_serial_and_stays_exact():
    """A stream built so that a decoder started off its true phase never meets the true path: both tables hold the two 1-bit
    codes, DC category 0 and EOB, so every block is two bits.  A decoder started one bit late reads the same stream one
    symbol out of phase forever, so no subsequence can synchronise except through its predecessor: the iteration count is
    the number of subsequences in the interval (serial decoding), and the result is still exact."""
    dc = ac = {(1, 0): 0, (1, 1): 0}                        # both 1-bit codes used: a table no encoder writes
    n_blocks = 3 * 400
    hdr = dict(sub=1, dc=[dc] * 3, ac=[ac] * 3, h=8, w=8 * 400, restart=0)
    data = np.random.default_rng(0).integers(0, 256, n_blocks * 2 // 8, dtype=np.uint8).tobytes()
    iv = [(0, 8 * len(data))]
    starts, iters = J.sync_model(hdr, 64, data=data, iv=iv)
    n_sub = -(-8 * len(data) // 64)
    assert len(starts) == n_sub and iters >= n_sub - 2
    # the true decoder is at block (pos // 2) % 3, before its DC code at even bits and before its EOB at odd ones
    assert all((blk, zz) == ((pos // 2) % 3, pos % 2) for pos, blk, zz in starts)
