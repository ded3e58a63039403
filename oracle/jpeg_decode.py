"""numpy restatement of the JPEG decode the test pipeline runs: `mmcv.imread(name, 'unchanged')` =
`cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)` on a baseline YCbCr file, i.e. libjpeg-turbo's default decompression path.

Settings assumed (libjpeg-turbo's defaults, which OpenCV does not change):
  * dct_method = JDCT_ISLOW: jidctint.c's integer IDCT (CONST_BITS 13, PASS1_BITS 2), dequantisation as int products, and the
    output range limited through libjpeg's post-IDCT table (index x & 1023 of the table prepare_range_limit_table builds);
  * do_fancy_upsampling = TRUE: h2v2 triangle filter (nearer row x 3 + farther row, then nearer column x 3 + neighbour,
    biases 8 and 7 alternating), edge rows duplicated, edge columns weighted x 4; components at most 2 samples wide are
    replicated instead (jinit_upsampler's downsampled_width > 2 condition);
  * out_color_space = BGR from YCbCr through jdcolor.c's integer tables (SCALEBITS 16, ONE_HALF rounding);
  * EXIF orientation is ignored (IMREAD_UNCHANGED).

Only what the frame engine decodes is covered: SOF0 / SOF1, 8-bit samples and quantisation tables, three components in one
interleaved scan, 4:2:0 or 4:4:4, any restart interval.  `parse` rejects everything else with JpegUnsupported.

`sync_model` restates the device decoder's self-synchronising Huffman phase (Weissenberger & Schmidt) on the CPU.
"""
import numpy as np


class JpegUnsupported(ValueError):
    pass


ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


def _huff_table(bits, vals):
    """canonical code -> symbol dict {(length, code): symbol}"""
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        if code + bits[length - 1] >= 1 << length:          # jdhuff.c: the all-ones code of every length is reserved
            raise JpegUnsupported('corrupt Huffman table (over-subscribed code lengths)')
        for _ in range(bits[length - 1]):
            table[(length, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return table


def parse(data):
    """Header of a baseline YCbCr JPEG -> dict; raises JpegUnsupported naming what is outside the scope."""
    d = bytes(data)
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise JpegUnsupported('not a JPEG file (no SOI marker)')
    qt, dc, ac, restart, sof, p = {}, {}, {}, 0, None, 2
    while True:
        while p < len(d) and d[p] == 0xFF and p + 1 < len(d) and d[p + 1] == 0xFF:
            p += 1
        if p + 4 > len(d):
            raise JpegUnsupported('truncated file (header)')
        if d[p] != 0xFF:
            raise JpegUnsupported('corrupt header (marker expected)')
        m = d[p + 1]
        ln = (d[p + 2] << 8) | d[p + 3]
        seg = d[p + 4:p + 2 + ln]
        if ln < 2 or p + 2 + ln > len(d):
            raise JpegUnsupported('truncated file (header)')
        if m in (0xC2, 0xC6, 0xCA, 0xCE):
            raise JpegUnsupported('progressive JPEG is not supported')
        if m in (0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF) or m == 0xCC:
            raise JpegUnsupported('arithmetic coding is not supported')
        if m in (0xC3, 0xC5, 0xC7):
            raise JpegUnsupported('lossless / hierarchical JPEG is not supported')
        if m == 0xEE and seg[:5] == b'Adobe':
            raise JpegUnsupported('Adobe-transform (APP14) files are not supported')
        if m in (0xC0, 0xC1):
            if seg[0] != 8:
                raise JpegUnsupported(f'{seg[0]}-bit samples are not supported')
            h, w, nc = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if nc == 1:
                raise JpegUnsupported('grayscale JPEG is not supported')
            if nc != 3:
                raise JpegUnsupported(f'{nc}-component (CMYK) JPEG is not supported')
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(3)]
            if bytes(c[0] for c in comps) == b'RGB':
                raise JpegUnsupported('RGB (untransformed) JPEG is not supported')
            samp = tuple((c[1], c[2]) for c in comps)
            if samp == ((2, 2), (1, 1), (1, 1)):
                sub = 2
            elif samp == ((1, 1), (1, 1), (1, 1)):
                sub = 1
            else:
                raise JpegUnsupported(f'chroma sampling {samp} is not supported (only 4:2:0 and 4:4:4)')
            if h == 0 or w == 0:
                raise JpegUnsupported('empty image')
            sof = dict(h=h, w=w, comps=comps, sub=sub)
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                if pq != 0:
                    raise JpegUnsupported('16-bit quantisation tables are not supported')
                qt[tq] = np.zeros(64, np.int64)                  # stored in zig-zag order
                qt[tq][ZIGZAG] = np.frombuffer(seg[q + 1:q + 65], np.uint8)
                q += 65
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                tc, th = seg[q] >> 4, seg[q] & 15
                bits = list(seg[q + 1:q + 17])
                vals = list(seg[q + 17:q + 17 + sum(bits)])
                (dc if tc == 0 else ac)[th] = _huff_table(bits, vals)
                q += 17 + sum(bits)
        elif m == 0xDD:
            restart = (seg[0] << 8) | seg[1]
        elif m == 0xDA:
            if sof is None:
                raise JpegUnsupported('scan before frame header')
            ns = seg[0]
            if ns != 3:
                raise JpegUnsupported('several scans (non-interleaved components) are not supported')
            sel = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(3)]
            ss, se, ahl = seg[7], seg[8], seg[9]
            if (ss, se, ahl) != (0, 63, 0):
                raise JpegUnsupported('progressive scan parameters are not supported')
            start = p + 2 + ln
            eoi = d.rfind(b'\xff\xd9', start)                  # bytes after the last EOI marker are ignored
            if eoi < 0:
                raise JpegUnsupported('truncated file (no EOI marker after the scan)')
            d = d[:eoi + 2]
            ids = [c[0] for c in sof['comps']]
            if [s[0] for s in sel] != ids:
                raise JpegUnsupported('scan components differ from the frame components')
            sof.update(qt=[qt[c[3]] for c in sof['comps']], dc=[dc[s[1]] for s in sel], ac=[ac[s[2]] for s in sel],
                       restart=restart, scan=d[start:len(d) - 2])
            return sof
        elif m in (0xD9,):
            raise JpegUnsupported('no scan in the file')
        p += 2 + ln


def unstuff(scan):
    """entropy-coded segment -> (bytes without FF00 stuffing / RSTn markers, byte offset of every interval start).
    A marker may be preceded by any number of FF fill bytes (T.81 B.1.1.2): a run of FF bytes that ends in an RSTn byte, or
    at the end of the segment (the EOI marker follows), is fill plus that marker.  Every other FF not followed by 00, and
    FF FF 00 in particular, is corrupt (libjpeg-turbo's two bit readers disagree on what FF FF 00 means)."""
    out, starts, i, n = bytearray(), [0], 0, len(scan)
    while i < n:
        b = scan[i]
        if b == 0xFF:
            k = i + 1
            while k < n and scan[k] == 0xFF:
                k += 1
            if k == n:                                       # fill bytes before the EOI marker
                break
            if 0xD0 <= scan[k] <= 0xD7:
                starts.append(len(out))
            elif scan[k] == 0 and k == i + 1:
                out.append(0xFF)
            else:
                raise ValueError('marker inside the scan')
            i = k + 1
        else:
            out.append(b)
            i += 1
    return bytes(out), starts


class _Bits:
    def __init__(self, data):
        self.d = bytes(data) + b'\xff' * 12

    def get(self, pos, k):
        """k <= 16 bits from bit `pos` (the stream continues with 1-bits past its end)"""
        if not k:
            return 0
        v = int.from_bytes(self.d[pos >> 3:(pos >> 3) + 4], 'big')
        return (v >> (32 - (pos & 7) - k)) & ((1 << k) - 1)


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def mcu_layout(hdr):
    """blocks of one MCU as (component, block row, block column) offsets"""
    if hdr['sub'] == 2:
        return [(0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (2, 0, 0)]
    return [(0, 0, 0), (1, 0, 0), (2, 0, 0)]


def decode_symbol(bits, hdr, pos, blk, zz, block=None):
    """one Huffman code + its extra bits from decoder state (pos, blk, zz) -> (pos, blk, zz, ok); `block` (64 zig-zag
    coefficients, DC as the difference) receives the value."""
    comp = mcu_layout(hdr)[blk][0]
    table = hdr['dc'][comp] if zz == 0 else hdr['ac'][comp]
    for length in range(1, 17):
        sym = table.get((length, bits.get(pos, length)))
        if sym is not None:
            break
    else:
        return pos + 1, blk, zz, False
    pos += length
    if zz == 0:
        s = sym
        if block is not None:
            block[0] = _extend(bits.get(pos, s), s)
        pos += s
        zz = 1
    else:
        r, s = sym >> 4, sym & 15
        if s == 0:
            zz = zz + 16 if r == 15 else 64
        else:
            zz += r
            if zz > 63:                                      # corrupt: the block ends here (the device does the same)
                return pos + s, (blk + 1) % len(mcu_layout(hdr)), 0, False
            if block is not None:
                block[zz] = _extend(bits.get(pos, s), s)
            pos += s
            zz += 1
    if zz >= 64:
        ok = zz == 64
        zz, blk = 0, (blk + 1) % len(mcu_layout(hdr))
        return pos, blk, zz, ok
    return pos, blk, zz, True


def entropy_decode(hdr):
    """-> list of 3 int arrays (block rows, block cols, 64) of quantised coefficients in natural order (DC predicted)"""
    h, w, sub = hdr['h'], hdr['w'], hdr['sub']
    mh, mw = 8 * sub, 8 * sub
    my, mx = -(-h // mh), -(-w // mw)
    planes = [np.zeros((my * sub, mx * sub, 64), np.int64)] + [np.zeros((my, mx, 64), np.int64) for _ in range(2)]
    data, starts = unstuff(hdr['scan'])
    bits = _Bits(data)
    lay = mcu_layout(hdr)
    ri = hdr['restart'] or my * mx
    for m in range(my * mx):
        if m % ri == 0:
            pos = 8 * starts[m // ri]
            pred = [0, 0, 0]
        for b, (c, dy, dx) in enumerate(lay):
            blk = np.zeros(64, np.int64)
            zz = 0
            while True:
                pos, nb, zz, ok = decode_symbol(bits, hdr, pos, b, zz, blk)
                if not ok:
                    raise ValueError('corrupt scan')
                if nb != b:
                    break
            pred[c] += blk[0]
            blk[0] = pred[c]
            nat = np.zeros(64, np.int64)
            nat[ZIGZAG] = blk
            s = sub if c == 0 else 1
            planes[c][(m // mx) * s + dy, (m % mx) * s + dx] = nat
    return planes


# ---- jidctint.c (ISLOW)
def _range_limit_table():
    t = np.zeros(1024, np.int64)
    for i in range(1024):
        if i < 128:
            t[i] = i + 128
        elif i < 512:
            t[i] = 255
        elif i < 896:
            t[i] = 0
        else:
            t[i] = i - 896
    return t


_RL = _range_limit_table()


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(d0, d1, d2, d3, d4, d5, d6, d7):
    z1 = (d2 + d6) * 4433
    tmp2 = z1 + d6 * -15137
    tmp3 = z1 + d2 * 6270
    tmp0 = (d0 + d4) << 13
    tmp1 = (d0 - d4) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = d7, d5, d3, d1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * 9633
    t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069, z4 * -3196
    z3 = z3 + z5
    z4 = z4 + z5
    t0 = t0 + z1 + z3
    t1 = t1 + z2 + z4
    t2 = t2 + z2 + z3
    t3 = t3 + z1 + z4
    return (tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3)


def idct_islow(coef, q):
    """coef (..., 64) natural-order quantised coefficients, q (64,) natural order -> (..., 8, 8) uint8 samples"""
    x = (coef * q).reshape(coef.shape[:-1] + (8, 8))
    cols = [x[..., r, :] for r in range(8)]                # pass 1 over columns: rows 0..7 of every column at once
    out = _idct_1d(*cols)
    ws = np.stack([_descale(v, 11) for v in out], axis=-2)  # CONST_BITS - PASS1_BITS
    ac_zero = np.all(x[..., 1:, :] == 0, axis=-2, keepdims=True)
    ws = np.where(ac_zero, x[..., 0:1, :] << 2, ws)
    rows = [ws[..., :, c] for c in range(8)]
    out = _idct_1d(*rows)
    px = np.stack([_descale(v, 18) for v in out], axis=-1)  # CONST_BITS + PASS1_BITS + 3
    rz = np.all(ws[..., :, 1:] == 0, axis=-1, keepdims=True)
    px = np.where(rz, _descale(ws[..., :, 0:1], 5), px)
    return _RL[px & 1023].astype(np.uint8)


def _plane(blocks, q):
    by, bx = blocks.shape[:2]
    px = idct_islow(blocks, q)                               # (by, bx, 8, 8)
    return px.transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)


def upsample_h2v2_fancy(c, h, w):
    """chroma plane c (>= ceil(h/2) x ceil(w/2) real samples) -> (h, w) int, jdsample.c h2v2_fancy_upsample"""
    dh, dw = -(-h // 2), -(-w // 2)
    c = c[:dh, :dw].astype(np.int64)
    if dw <= 2:                                              # h2v2_upsample: replication
        return np.repeat(np.repeat(c, 2, 0), 2, 1)[:h, :w]
    up = np.concatenate([c[:1], c[:-1]], 0)
    dn = np.concatenate([c[1:], c[-1:]], 0)
    rows = np.empty((2 * dh, dw), np.int64)
    rows[0::2] = 3 * c + up
    rows[1::2] = 3 * c + dn
    left = np.concatenate([rows[:, :1], rows[:, :-1]], 1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], 1)
    out = np.empty((2 * dh, 2 * dw), np.int64)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    return out[:h, :w]


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc_to_bgr(y, cb, cr):
    x = np.arange(256) - 128
    cr_r = (_fix(1.40200) * x + 32768) >> 16
    cb_b = (_fix(1.77200) * x + 32768) >> 16
    cr_g = -_fix(0.71414) * x
    cb_g = -_fix(0.34414) * x + 32768
    r = np.clip(y + cr_r[cr], 0, 255)
    g = np.clip(y + ((cb_g[cb] + cr_g[cr]) >> 16), 0, 255)
    b = np.clip(y + cb_b[cb], 0, 255)
    return np.stack([b, g, r], -1).astype(np.uint8)


def decode(data):
    """encoded bytes -> (h, w, 3) uint8 BGR, byte-identical to cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)"""
    hdr = parse(data)
    h, w = hdr['h'], hdr['w']
    planes = entropy_decode(hdr)
    y, cb, cr = (_plane(p, q) for p, q in zip(planes, hdr['qt']))
    y = y[:h, :w].astype(np.int64)
    if hdr['sub'] == 2:
        cb, cr = upsample_h2v2_fancy(cb, h, w), upsample_h2v2_fancy(cr, h, w)
    else:
        cb, cr = cb[:h, :w].astype(np.int64), cr[:h, :w].astype(np.int64)
    return ycc_to_bgr(y, cb, cr)


# ---- the device decoder's synchronisation phase
def intervals(hdr):
    """unstuffed stream and the bit range [start, end) of every restart interval"""
    data, starts = unstuff(hdr['scan'])
    ends = starts[1:] + [len(data)]
    return data, [(8 * s, 8 * e) for s, e in zip(starts, ends)]


def _run(bits, hdr, state, end):
    """decode from `state` until the first codeword boundary at or after bit `end` -> (exit state, blocks started)"""
    pos, blk, zz = state
    n = 0
    while pos < end:
        if zz == 0:
            n += 1
        pos, blk, zz, _ = decode_symbol(bits, hdr, pos, blk, zz)
    return (pos, blk, zz), n


def sync_model(hdr, sub_bits=256, data=None, iv=None):
    """Jacobi form of self-synchronising decoding, as the device runs it: every interval is cut into `sub_bits`-bit
    subsequences; subsequence j first decodes from a guess (its own start, block 0, zig-zag 0; the interval's first from the
    true start) to its exit state, then takes its predecessor's exit state as its start and decodes again, until no start
    changes.  -> (start states, iterations).  At convergence every start is a true codeword boundary."""
    if data is None:
        data, iv = intervals(hdr)
    bits = _Bits(data)
    subs = []                                                # (start bit, end bit, first of its interval)
    for s, e in iv:
        k = max(1, -(-(e - s) // sub_bits))
        subs += [(s + i * sub_bits, min(e, s + (i + 1) * sub_bits), i == 0) for i in range(k)]
    start = [(s, 0, 0) for s, _, _ in subs]
    exit_ = [_run(bits, hdr, st, e)[0] for st, (_, e, _) in zip(start, subs)]
    it = 0
    while True:
        new = [start[j] if subs[j][2] else exit_[j - 1] for j in range(len(subs))]
        changed = [j for j in range(len(subs)) if new[j] != start[j]]
        if not changed:
            return start, it
        it += 1
        start = new
        for j in changed:
            exit_[j] = _run(bits, hdr, start[j], subs[j][1])[0]


def true_boundaries(hdr):
    """every codeword boundary state (pos, blk, zz) of the serial decode, per interval"""
    data, iv = intervals(hdr)
    bits = _Bits(data)
    n_blk = len(mcu_layout(hdr))
    my, mx = -(-hdr['h'] // (8 * hdr['sub'])), -(-hdr['w'] // (8 * hdr['sub']))
    ri = hdr['restart'] or my * mx
    out = set()
    for r, (s, _) in enumerate(iv):
        need = min(ri, my * mx - r * ri) * n_blk
        st = (s, 0, 0)
        for _ in range(need):
            while True:
                out.add(st)
                st = decode_symbol(bits, hdr, *st)[:3]
                if st[2] == 0:
                    break
        out.add(st)                                          # the end of the interval's data
    return out


# ---- test fixtures: the content kinds the decoder is tested on, encoded by OpenCV's writer
CONTENTS = ('noise', 'flat', 'bars', 'camera')


def make_image(kind, h, w, seed=0):
    """(h, w, 3) uint8 BGR: seeded noise; flat grey (no AC coefficients); saturated colour bars (range limiting); a smooth
    camera-like gradient with texture"""
    rng = np.random.default_rng(seed)
    if kind == 'noise':
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == 'flat':
        return np.full((h, w, 3), 128, np.uint8)
    if kind == 'bars':
        cols = np.array([[255, 255, 255], [0, 255, 255], [255, 255, 0], [0, 255, 0], [255, 0, 255], [0, 0, 255],
                         [255, 0, 0], [0, 0, 0]], np.uint8)
        return np.ascontiguousarray(np.broadcast_to(cols[np.arange(w) * 8 // w][None], (h, w, 3)))
    y, x = np.mgrid[:h, :w]
    g = np.stack([x * 255 // max(w - 1, 1), y * 255 // max(h - 1, 1), (x + y) * 127 // max(h + w - 2, 1)], -1)
    return np.clip(g + rng.integers(-6, 7, (h, w, 3)), 0, 255).astype(np.uint8)


def encode(img, quality=95, sampling='420', restart=0, optimize=False, progressive=False):
    """cv2.imencode('.jpg') with the given quality, chroma sampling ('420', '422', '411', '444', '440'), restart interval
    (MCUs, 0 = none; 'row' = one MCU row) and optimised Huffman tables -> bytes"""
    import cv2
    samp = {'420': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, '422': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            '411': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411, '444': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444,
            '440': cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440}[sampling]
    if restart == 'row':
        restart = -(-img.shape[1] // (16 if sampling == '420' else 8))
    ok, buf = cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp,
                                         cv2.IMWRITE_JPEG_RST_INTERVAL, restart, cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize),
                                         cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)])
    assert ok
    return buf.tobytes()


def cv2_decode(data):
    import cv2
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)
