"""Baseline JPEG streams written from quantised coefficients, for the decoders of tests/test_jpeg_streams_*.py.

OpenCV's writer (libjpeg's) only ever produces a few forms of file: component ids 1, 2, 3; Y on Huffman / quantisation slot 0
and both chromas on slot 1; one table per DHT / DQT segment; standard or optimised code lengths; no fill bytes.  `write()`
takes the coefficient blocks themselves and every choice libjpeg makes for us: Huffman tables as (bits, vals), per-component
table selectors and ids, the order and grouping of the header segments, APPn / COM segments, fill bytes before header markers,
SOF0 / SOF1, DRI, fill bytes before every RSTn and before EOI, and the padding bit.  `cases()` builds the families the tests
run, seeded, in 4:2:0 and 4:4:4:

  header     ids 0/1/2 and arbitrary ones, Y on DC/AC slot 1, Cb on 0, Cr on 2 or 3, quantisation tables 2 and 3, all tables in
             one DHT / DQT, tables after SOF, a table redefined before SOS (the last definition wins), APPn / COM, fill bytes
             before header markers, SOF1, DRI 0 after a non-zero DRI
  codes      every code length 1-16 (the 9 -> 10 boundary of the device's lookup, 13- and 14-bit codes, a 16-bit code one
             below all-ones), single-code 1-bit tables, a full 162-symbol AC table, crossed DC / AC tables
  coef       every DC category 0-11, every AC size 1-10 at both ends of its range, runs 0-15, ZRL chains before a
             coefficient at 63, blocks ending at 63 without EOB, EOB right after DC, all-zero blocks, many intervals
  stuffing   FF-dense scans (>= 30 % of the scan bytes in FF 00 pairs) with many short restart intervals
  restart    DRI beyond the MCU count, DRI not dividing a row, DRI 1 on 1x1 and on 1600x900, intervals of exactly 1024 k bits
             and of 8 k + 1 bits (7 padding bits), 1-3 fill bytes before every RSTn and before EOI
  worst      intervals that synchronise only through their predecessors (`worst_tables`)

Every DC value lies in [-1024, 1016] and every dequantised coefficient within what round(FDCT) of 8-bit samples can produce
(`FDCT_MIN` / `FDCT_MAX`): outside that, libjpeg-turbo's SIMD and C IDCTs need not agree and cv2 stops being a reference.
The extreme blocks are the rounded DCTs of 0 / 255 checkerboards, stripes and single-pixel spikes at q = 1.

    python tests/golden/gen_jpeg_streams.py    # digests of cv2's decode of every case -> jpeg_streams_sha256.json
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
EOB, ZRL = 0x00, 0xF0
AC_SYMBOLS = [EOB, ZRL] + [r << 4 | s for r in range(16) for s in range(1, 11)]      # the 162 baseline AC symbols
DC_MIN, DC_MAX = -1024, 1016

# orthonormal 8-point DCT-II: JPEG's FDCT is C X C^T of the level-shifted samples
_C = np.array([[np.sqrt((1 if u else 0.5) / 4) * np.cos((2 * x + 1) * u * np.pi / 16) for x in range(8)] for u in range(8)])
_W = np.einsum('ux,vy->uvxy', _C, _C).reshape(64, 64)
FDCT_MAX = np.round(np.where(_W > 0, 127 * _W, -128 * _W).sum(1)).astype(np.int64)    # per natural position
FDCT_MIN = np.round(np.where(_W > 0, -128 * _W, 127 * _W).sum(1)).astype(np.int64)


def fdct_q(px, q):
    """(..., 8, 8) samples 0..255 -> (..., 64) natural-order coefficients round(FDCT / q)"""
    x = px.reshape(px.shape[:-2] + (64,)).astype(np.float64) - 128
    return np.round(x @ _W.T / q).astype(np.int64)


def category(v):
    return int(abs(int(v))).bit_length()


# ------------------------------------------------------------------------------------------------------------- Huffman
class Huff:
    """a canonical Huffman table: bits[l - 1] codes of length l, vals in code order; `enc[sym]` = (length, code) of the
    first code carrying sym (what the writer emits)"""

    def __init__(self, bits, vals):
        self.bits, self.vals = list(bits), list(vals)
        assert len(self.bits) == 16 and sum(self.bits) == len(self.vals) <= 256
        self.enc, self.codes = {}, []
        code, k = 0, 0
        for length in range(1, 17):
            assert code + self.bits[length - 1] < 1 << length, 'over-subscribed (the all-ones code is reserved)'
            for _ in range(self.bits[length - 1]):
                self.codes.append((length, code, self.vals[k]))
                self.enc.setdefault(self.vals[k], (length, code))
                code += 1
                k += 1
            code <<= 1

    def lengths(self):
        return {ln for ln, _, _ in self.codes}

    def segment(self, tc, th):
        return bytes([tc << 4 | th]) + bytes(self.bits) + bytes(self.vals)


def huff(lengths):
    """[(symbol, code length), ...] -> Huff (symbols of one length keep their order)"""
    bits = [0] * 16
    for _, ln in lengths:
        bits[ln - 1] += 1
    return Huff(bits, [s for s, _ in sorted(lengths, key=lambda t: t[1])])


def full_dc(rng, bits=(0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0)):
    """all 12 DC categories in a seeded order on the given code-length counts"""
    return Huff(bits, list(rng.permutation(12)))


def full_ac(rng, bits=(0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D)):
    """all 162 AC symbols in a seeded order (EOB and ZRL kept short) on the given code-length counts"""
    rest = [s for s in AC_SYMBOLS if s not in (EOB, ZRL)]
    vals = [EOB] + list(rng.permutation(rest))
    vals.insert(3, ZRL)
    return Huff(bits, vals)


def every_length_ac(rng):
    """16 AC symbols on codes of every length 1..16; the 16-bit code is 1111111111111110, one below all-ones"""
    syms = [EOB, ZRL] + list(rng.choice([s for s in AC_SYMBOLS[2:]], 14, replace=False))
    rng.shuffle(syms)
    return huff([(s, ln) for s, ln in zip(syms, range(1, 17))])


def every_length_dc(rng):
    """12 DC categories on lengths 1..10 and 13, 14 (9 -> 10 and the long tail)"""
    cats = list(rng.permutation(12))
    return huff([(c, ln) for c, ln in zip(cats, list(range(1, 11)) + [13, 14])])


# ------------------------------------------------------------------------------------------------------------- writer
def _seg(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, 'big') + payload


def _default_header(spec):
    ht = spec['ht']
    hdr = [('app', 0, b'JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00'), ('dqt', sorted(spec['qt'])), ('sof', 0xC0),
           ('dht', sorted(ht))]
    if spec.get('restart'):
        hdr.append(('dri', spec['restart']))
    return hdr


def mcu_layout(sub):
    return [(0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (2, 0, 0)] if sub == 2 else [(0, 0, 0), (1, 0, 0), (2, 0, 0)]


def geometry(h, w, sub):
    """(MCU rows, MCU columns)"""
    return -(-h // (8 * sub)), -(-w // (8 * sub))


def decode_order(h, w, sub):
    """[(mcu, component, block row, block column)] in scan order"""
    my, mx = geometry(h, w, sub)
    out = []
    for m in range(my * mx):
        for c, dy, dx in mcu_layout(sub):
            s = sub if c == 0 else 1
            out.append((m, c, (m // mx) * s + dy, (m % mx) * s + dx))
    return out


class BitWriter:
    def __init__(self):
        self.parts, self.n = [], 0

    def put(self, length, value):
        if length:
            self.parts.append(format(value, f'0{length}b'))
            self.n += length

    def bits(self):
        return ''.join(self.parts)


def encode_block(bw, zz, diff, dc, ac, log=None):
    """one block: zz the 64 zig-zag coefficients, diff the DC difference; `log` collects (kind, symbol, value)"""
    s = category(diff)
    bw.put(*dc.enc[s])
    bw.put(s, diff if diff >= 0 else diff + (1 << s) - 1)
    if log is not None:
        log.append(('dc', s, diff))
    run = 0
    for k in range(1, 64):
        v = int(zz[k])
        if v == 0:
            run += 1
            continue
        while run > 15:
            bw.put(*ac.enc[ZRL])
            if log is not None:
                log.append(('ac', ZRL, 0))
            run -= 16
        s = category(v)
        assert 1 <= s <= 10, v
        bw.put(*ac.enc[run << 4 | s])
        bw.put(s, v if v >= 0 else v + (1 << s) - 1)
        if log is not None:
            log.append(('ac', run << 4 | s, v))
        run = 0
    if run:
        bw.put(*ac.enc[EOB])
        if log is not None:
            log.append(('ac', EOB, 0))


def check_planes(spec):
    """DC in [-1024, 1016]; dequantised coefficients within round(FDCT) of 8-bit samples"""
    for c, p in enumerate(spec['planes']):
        q = spec['qt'][spec['comps'][c][1]]
        assert p[..., 0].min() >= DC_MIN and p[..., 0].max() <= DC_MAX, c
        d = p * q
        assert (d >= FDCT_MIN).all() and (d <= FDCT_MAX).all(), c


def interval_bits(spec, log=None):
    """the bit string of every restart interval (before padding)"""
    h, w, sub = spec['h'], spec['w'], spec['sub']
    my, mx = geometry(h, w, sub)
    ri = spec.get('restart') or my * mx
    ri = min(ri, my * mx)
    tabs = [(spec['ht'][(0, td)], spec['ht'][(1, ta)]) for _, _, td, ta in spec['comps']]
    out, cur = [], -1
    for m, c, by, bx in decode_order(h, w, sub):
        if m // ri != cur:
            cur, bw, pred = m // ri, BitWriter(), [0, 0, 0]
            out.append(bw)
        nat = spec['planes'][c][by, bx]
        encode_block(bw, nat[ZIGZAG], int(nat[0]) - pred[c], *tabs[c], log=log)
        pred[c] = int(nat[0])
    return [b.bits() for b in out]


def _stuff(bits, pad_bit):
    n = -len(bits) % 8
    bits += str(pad_bit) * n
    data = int(bits, 2).to_bytes(len(bits) // 8, 'big') if bits else b''
    return data.replace(b'\xff', b'\xff\x00'), n


def write(spec):
    """spec -> (file bytes, info).  spec: h, w, sub (2 = 4:2:0, 1 = 4:4:4); planes: 3 int arrays (block rows, block cols, 64)
    of quantised coefficients in natural order, DC as values, at the full MCU size; qt {slot: 64 natural-order values}; ht
    {(class, slot): Huff}; comps [(id, quant slot, DC slot, AC slot)] * 3; restart (the DRI in force at SOS, 0 = none);
    optional: header (a list of ('app', n, payload), ('com', payload), ('dqt', [slots]), ('dht', [(class, slot)]),
    ('dqt_def', slot, table), ('dht_def', class, slot, Huff), ('sof', 0xC0 / 0xC1), ('dri', n), ('fill', k): k FF bytes
    before the next marker); fill_rst (a list: FF fill bytes before RSTn number i); fill_eoi; pad_bit.
    info: the intervals' unstuffed bit lengths and padding, the scan's offset in the file."""
    check_planes(spec)
    h, w, sub = spec['h'], spec['w'], spec['sub']
    out = bytearray(b'\xff\xd8')
    fill = 0
    for item in spec.get('header') or _default_header(spec):
        kind = item[0]
        if kind == 'fill':
            fill += item[1]
            continue
        out += b'\xff' * fill
        fill = 0
        if kind == 'app':
            out += _seg(0xE0 + item[1], item[2])
        elif kind == 'com':
            out += _seg(0xFE, item[1])
        elif kind in ('dqt', 'dqt_def'):
            tabs = [(t, spec['qt'][t]) for t in item[1]] if kind == 'dqt' else [(item[1], item[2])]
            out += _seg(0xDB, b''.join(bytes([t]) + bytes(np.asarray(q)[ZIGZAG].astype(np.uint8)) for t, q in tabs))
        elif kind in ('dht', 'dht_def'):
            tabs = [(tc, th, spec['ht'][(tc, th)]) for tc, th in item[1]] if kind == 'dht' else [item[1:]]
            out += _seg(0xC4, b''.join(t.segment(tc, th) for tc, th, t in tabs))
        elif kind == 'sof':
            p = bytes([8]) + h.to_bytes(2, 'big') + w.to_bytes(2, 'big') + bytes([3])
            for c, (cid, tq, _, _) in enumerate(spec['comps']):
                p += bytes([cid, 0x22 if (sub == 2 and c == 0) else 0x11, tq])
            out += _seg(item[1], p)
        elif kind == 'dri':
            out += _seg(0xDD, item[1].to_bytes(2, 'big'))
        else:
            raise ValueError(kind)
    out += b'\xff' * fill
    out += _seg(0xDA, bytes([3]) + b''.join(bytes([cid, td << 4 | ta]) for cid, _, td, ta in spec['comps']) + b'\x00\x3f\x00')
    scan_off = len(out)
    ivs = interval_bits(spec)
    fills = spec.get('fill_rst') or [0] * len(ivs)
    pad = []
    for i, bits in enumerate(ivs):
        data, n = _stuff(bits, spec.get('pad_bit', 1))
        pad.append(n)
        out += data
        if i + 1 < len(ivs):
            out += b'\xff' * fills[i] + bytes([0xFF, 0xD0 + i % 8])
    out += b'\xff' * spec.get('fill_eoi', 0) + b'\xff\xd9'
    return bytes(out), dict(iv_bits=[len(b) for b in ivs], pad=pad, scan_off=scan_off)


# ------------------------------------------------------------------------------------------------------------- content
def blank_planes(h, w, sub):
    my, mx = geometry(h, w, sub)
    return [np.zeros((my * sub, mx * sub, 64), np.int64)] + [np.zeros((my, mx, 64), np.int64) for _ in range(2)]


def natural_planes(rng, h, w, sub, qs, kinds=('smooth', 'noise', 'edge', 'flat')):
    """the quantised FDCT of seeded 8x8 sample blocks (smooth ramps with texture, noise, edges, flat)"""
    planes = blank_planes(h, w, sub)
    for c, p in enumerate(planes):
        n = p.shape[0] * p.shape[1]
        kind = rng.integers(0, len(kinds), n)
        y, x = np.mgrid[:8, :8]
        base = rng.uniform(16, 240, (n, 1, 1)) + rng.uniform(-6, 6, (n, 1, 1)) * y + rng.uniform(-6, 6, (n, 1, 1)) * x
        px = np.where(np.array(kinds)[kind][:, None, None] == 'noise', rng.uniform(0, 255, (n, 8, 8)),
                      base + rng.normal(0, 3, (n, 8, 8)))
        edge = np.array(kinds)[kind] == 'edge'
        px[edge] = np.where(x[None] * rng.uniform(-1, 1, (edge.sum(), 1, 1)) + y[None] > 4, 230, 25)
        flat = np.array(kinds)[kind] == 'flat'
        px[flat] = np.round(px[flat][:, :1, :1])
        p[:] = fdct_q(np.clip(px, 0, 255), qs[c]).reshape(p.shape)
    return planes


def extreme_blocks():
    """rounded DCTs (q = 1) of 0 / 255 checkerboards, stripes of every period and phase and single-pixel spikes"""
    y, x = np.mgrid[:8, :8]
    pats = [((x + y) % 2) * 255, (1 - (x + y) % 2) * 255]
    for per in (1, 2, 4):
        for ph in range(2):
            pats += [((x // per + ph) % 2) * 255, ((y // per + ph) % 2) * 255]
    for v in (0, 255):
        for yy, xx in ((0, 0), (7, 7), (3, 4), (0, 7)):
            p = np.full((8, 8), 255 - v)
            p[yy, xx] = v
            pats.append(p)
    return fdct_q(np.array(pats), 1)


def fill_decode_order(planes, h, w, sub, blocks):
    """blocks (n, 64 natural) into the planes in scan order, cycling"""
    for i, (_, c, by, bx) in enumerate(decode_order(h, w, sub)):
        planes[c][by, bx] = blocks[i % len(blocks)]


def dc_walk(rng, cats, lo=DC_MIN, hi=DC_MAX, start=0):
    """DC values whose successive differences have the given categories, inside [lo, hi]"""
    out, pred = [], start
    for s in cats:
        if s == 0:
            out.append(pred)
            continue
        opts = []
        for sign in (1, -1):
            a, b = 1 << (s - 1), (1 << s) - 1
            # pred + sign * m in [lo, hi]
            mlo, mhi = (lo - pred, hi - pred) if sign > 0 else (pred - hi, pred - lo)
            a2, b2 = max(a, mlo), min(b, mhi)
            if a2 <= b2:
                opts.append((sign, a2, b2))
        assert opts, (s, pred)
        sign, a2, b2 = opts[rng.integers(len(opts))]
        m = int(rng.choice([a2, b2, rng.integers(a2, b2 + 1)]))
        pred += sign * m
        out.append(pred)
    return out


def fit_tail(costs, total):
    """choose one option per position so that the costs sum to `total`: costs[i] = {option: cost} -> [option]"""
    reach = [{0: None}]
    for cs in costs:
        nxt = {}
        for t in reach[-1]:
            for o, c in cs.items():
                if t + c <= total and t + c not in nxt:
                    nxt[t + c] = (t, o)
        reach.append(nxt)
    assert total in reach[-1], 'no choice reaches the target length'
    pick, t = [], total
    for i in range(len(costs), 0, -1):
        t, o = reach[i][t]
        pick.append(o)
    return pick[::-1]


def _idct_ok(nat, q):
    """the float IDCT of the dequantised block stays within +-384 of the sample range (the range-limit table's unambiguous
    part), so that no decoder's intermediate precision matters"""
    x = (nat * q) @ _W
    return x.min() >= -128 - 384 and x.max() <= 127 + 384


def build_planes(h, w, sub, ri, block_fn):
    """planes filled in scan order by block_fn(component, DC predictor, first block of its interval) -> natural block"""
    planes = blank_planes(h, w, sub)
    my, mx = geometry(h, w, sub)
    ri = min(ri or my * mx, my * mx)
    cur, pred = -1, None
    for m, c, by, bx in decode_order(h, w, sub):
        first = m // ri != cur
        if first:
            cur, pred = m // ri, [0, 0, 0]
        b = block_fn(c, pred[c], m % ri == 0 and first)
        planes[c][by, bx] = b
        pred[c] = int(b[0])
    return planes


def symbol_block(rng, pred, dc, ac, q, p_eob=0.25, lo=DC_MIN, hi=DC_MAX):
    """a block drawn from the symbols of its tables: a DC category the DC table holds, then AC symbols of the AC table
    (ZRL chains and runs included) until EOB or coefficient 63, values anywhere in their size's range within the FDCT bound"""
    dc_cats = sorted({v for v in dc.vals if category((1 << v) - 1) == v and v <= 11})
    ac_syms = sorted(set(ac.vals))
    while True:
        nat = np.zeros(64, np.int64)
        lo_, hi_ = max(lo, -(1024 // q[0])), min(hi, 1016 // q[0])
        cats = [s for s in dc_cats if s == 0 or min(hi_ - pred, pred - lo_) >= 1 << (s - 1) or
                max(hi_ - pred, pred - lo_) >= 1 << (s - 1)]
        nat[0] = dc_walk(rng, [int(rng.choice(cats))], lo_, hi_, pred)[0]
        k = 1
        while k < 64:
            sym = int(rng.choice(ac_syms))
            if sym == EOB:
                if rng.random() < p_eob or len(ac_syms) == 1:
                    break
                continue
            r, s = (16, 0) if sym == ZRL else (sym >> 4, sym & 15)
            if sym == ZRL:
                k += 16
                continue
            if k + r > 63:
                break
            pos = ZIGZAG[k + r]
            top = min((1 << s) - 1, FDCT_MAX[pos] // q[pos], -FDCT_MIN[pos] // q[pos])
            if top < 1 << (s - 1):
                continue
            m = int(rng.choice([1 << (s - 1), top, rng.integers(1 << (s - 1), top + 1)]))
            nat[pos] = m if rng.random() < 0.5 else -m
            k += r + 1
        if _idct_ok(nat, q) and (EOB in ac.enc or nat[ZIGZAG[63]] != 0):
            return nat


def worst_tables():
    """Tables on which a decoder started off its true phase never meets it.  Every DC category and every AC symbol has a code
    and extra bits of even total length, except DC category 1, whose code 1110 only the first block of an interval uses.  The
    codes and extra-bit patterns used after it are made of the 2-bit units 00, 01 and 10, so the scan holds no 111 between
    that first symbol and the padding: every true boundary after it lies at an odd bit offset, a decoder started at an even
    one stays at even ones (both tables are complete but for the all-ones prefix, which it can never read), and only its
    predecessor can synchronise a subsequence."""
    ev = [0, 2, 4, 6, 8, 10]
    dc = Huff([0, 3, 0, 3, 0, 3, 0, 3, 0, 3, 0, 3, 0, 3, 0, 3], [0, 2, 4, 6, 8, 1] + [ev[i % 6] for i in range(18)])
    fill = [r << 4 | s for s in (2, 4, 6, 8, 10) for r in range(16) if (r, s) not in ((0, 2), (0, 4), (1, 2), (2, 2))]
    ac = Huff([0, 2, 0, 6, 0, 7, 0, 3, 0, 3, 0, 3, 0, 3, 0, 3], [EOB, 0x02, 0x04, 0x12, 0x22] + fill[:25])
    return dc, ac


WORST_AC = [0x02, 0x04, 0x12, 0x22]                 # with EOB, the AC symbols whose codes are made of 00 / 01 / 10
_UNIT_VALUES = {2: [-3, -2, 2], 4: [-15, -14, -13, -11, -10, -9, 8, 9, 10]}  # extra bits made of 00 / 01 / 10


def worst_block(rng, pred, first, n_ac):
    """DC category 1 on the first block of an interval, else 0 / 2 / 4 towards the middle of the range; n_ac AC symbols"""
    nat = np.zeros(64, np.int64)
    if first:
        nat[0] = pred + int(rng.choice([-1, 1]))
    else:
        opts = [0] + _UNIT_VALUES[2] + _UNIT_VALUES[4]
        d = int(rng.choice([v for v in opts if abs(pred + v) < 400 or (pred + v) * pred < pred * pred]))
        nat[0] = pred + d
    k = 1
    for _ in range(n_ac):
        sym = WORST_AC[rng.integers(4)]
        k += sym >> 4
        if k > 63:
            break
        nat[ZIGZAG[k]] = int(rng.choice(_UNIT_VALUES[sym & 15]))
        k += 1
    return nat


# ------------------------------------------------------------------------------------------------------------- families
def _qt(rng, lo=1, hi=24):
    q = rng.integers(lo, hi + 1, 64)
    q[0] = rng.integers(1, 9)
    return q


def _case(name, family, h, w, sub, planes, qt, ht, comps, restart=0, **kw):
    spec = dict(h=h, w=w, sub=sub, planes=planes, qt=qt, ht=ht, comps=comps, restart=restart, **kw)
    data, info = write(spec)
    return dict(name=name, family=family, data=data, spec=spec, info=info)


def _subs():
    return (('420', 2), ('444', 1))


def header_cases():
    out = []
    for tag, sub in _subs():
        for v in 'ab':
            rng = np.random.default_rng([1, sub, ord(v)])
            h, w = (40, 56) if sub == 2 else (24, 40)
            qt = {0: _qt(rng), 2: _qt(rng), 3: _qt(rng)}
            ht = {(tc, th): (full_dc if tc == 0 else full_ac)(rng) for tc in (0, 1) for th in range(4)}
            if v == 'a':    # ids 0/1/2; Y on slots 1, Cb on 0, Cr on 2; quant Y 0, Cb 2, Cr 3; one DHT, one DQT
                comps = [(0, 0, 1, 1), (1, 2, 0, 0), (2, 3, 2, 2)]
                header = [('fill', 2), ('app', 0, b'JFIF\x00\x01\x02\x00\x00\x01\x00\x01\x00\x00'), ('com', b'comment'),
                          ('dqt', [0, 2, 3]), ('fill', 1), ('sof', 0xC0), ('dht', sorted(ht)), ('dri', 4), ('fill', 3)]
                restart = 4
            else:           # arbitrary ids, Cr on 3, quant Y 3 / Cb 2 / Cr 0, tables after SOF1, a table redefined, DRI 0
                comps = [(7, 3, 1, 1), (200, 2, 0, 0), (42, 0, 3, 3)]
                decoy = full_ac(np.random.default_rng(99))
                header = [('app', 1, b'Exif\x00\x00'), ('sof', 0xC1), ('fill', 1), ('dqt', [3]), ('com', b'x' * 40),
                          ('dqt_def', 2, np.ones(64, np.int64) * 50), ('dri', 5),
                          ('dht_def', 1, 1, decoy), ('dqt', [0, 2]), ('app', 15, b'\x00' * 10),
                          ('dht', [k for k in sorted(ht) if k != (1, 1)]), ('fill', 4), ('dht', [(1, 1)]), ('dri', 0)]
                restart = 0
            planes = natural_planes(rng, h, w, sub, [qt[c[1]] for c in comps])
            out.append(_case(f'header-{v}-{tag}', 'header', h, w, sub, planes, qt, ht, comps, restart, header=header))
    return out


def code_cases():
    out = []
    for tag, sub in _subs():
        rng = np.random.default_rng([2, sub])
        h, w = (48, 64) if sub == 2 else (32, 40)
        qt = {0: np.ones(64, np.int64), 1: _qt(rng, 1, 4)}
        # every length 1..16 (AC) and 1..10, 13, 14 (DC), crossed: Y DC 0 / AC 1, Cb DC 1 / AC 0, Cr DC 0 / AC 0
        ht = {(0, 0): every_length_dc(rng), (0, 1): every_length_dc(rng), (1, 0): every_length_ac(rng),
              (1, 1): every_length_ac(rng)}
        comps = [(1, 0, 0, 1), (2, 1, 1, 0), (3, 1, 0, 0)]
        qs = [qt[c[1]] for c in comps]
        planes = build_planes(h, w, sub, 0, lambda c, pred, first: symbol_block(
            rng, pred, ht[(0, comps[c][2])], ht[(1, comps[c][3])], qs[c], p_eob=0.15))
        out.append(_case(f'codes-every-length-{tag}', 'codes', h, w, sub, planes, qt, ht, comps))
        # a full 162-symbol AC table with 13- and 14-bit codes, on natural content
        bits = (0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 3, 3, 2, 2, 1, 123)
        ht = {(0, 0): full_dc(rng), (1, 0): full_ac(rng, bits), (0, 1): full_dc(rng, (0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0,
                                                                                        0, 0, 0)),
              (1, 1): full_ac(rng)}
        comps = [(1, 0, 1, 0), (2, 1, 0, 1), (3, 1, 1, 0)]
        qs = [qt[c[1]] for c in comps]
        planes = natural_planes(rng, h, w, sub, qs)
        out.append(_case(f'codes-full-ac-{tag}', 'codes', h, w, sub, planes, qt, ht, comps, 3))
        # single-code 1-bit tables: 2-bit blocks, restart intervals of one (4:4:4) or two (4:2:0) bytes
        one_dc, one_ac = Huff([1] + [0] * 15, [0]), Huff([1] + [0] * 15, [EOB])
        ht = {(0, 0): one_dc, (1, 0): one_ac}
        comps = [(1, 0, 0, 0), (2, 0, 0, 0), (3, 0, 0, 0)]
        out.append(_case(f'codes-single-{tag}', 'codes', 24, 40, sub, blank_planes(24, 40, sub), {0: _qt(rng)}, ht, comps,
                         1))
    return out


def coef_blocks(rng):
    """the special blocks of the coefficient family, DC 0 (set later): every AC size at both ends of its range, runs 0-15,
    ZRL chains before coefficient 63, a block of 63 coefficients, DC-only and all-zero blocks, the extreme blocks"""
    out = []
    k = 1
    for s in range(1, 11):
        for v in (1 << (s - 1), (1 << s) - 1):
            for sign in (1, -1):
                b = np.zeros(64, np.int64)
                pos = ZIGZAG[k] if s < 10 else 1  # size 10's top end, 1023, is beyond any 8-bit block's FDCT: the
                top = FDCT_MAX[pos] if sign > 0 else -FDCT_MIN[pos]      # bound at (0, 1), the largest, stands for it
                b[pos] = sign * min(v, top)
                out.append(b)
                k = k % 20 + 1
    for r in range(16):
        b = np.zeros(64, np.int64)
        b[ZIGZAG[1]], b[ZIGZAG[2 + r]] = 3, -2
        out.append(b)
    for k0 in (1, 14, 30, 40):                  # 3, 3, 2 and 1 ZRLs, then the coefficient at 63: no EOB
        b = np.zeros(64, np.int64)
        b[ZIGZAG[k0]], b[63] = -5, 7
        out.append(b)
    b = rng.choice([-2, -1, 1, 2], 64)
    out.append(b)
    out += [np.zeros(64, np.int64)] * 6                                        # DC-only blocks
    return [(b, False) for b in out] + [(b, True) for b in list(extreme_blocks()) + [np.zeros(64, np.int64)] * 4]


def coef_cases():
    out = []
    for tag, sub in _subs():
        rng = np.random.default_rng([3, sub])
        h, w = (64, 96) if sub == 2 else (48, 64)
        qt = {0: np.ones(64, np.int64)}
        ht = {(0, 0): full_dc(rng), (1, 0): full_ac(rng), (0, 1): full_dc(rng), (1, 1): full_ac(rng)}
        comps = [(1, 0, 0, 0), (2, 0, 1, 1), (3, 0, 1, 1)]
        specials = coef_blocks(rng)
        order = list(rng.permutation(len(specials)))
        it = iter(order)
        cats = iter(list(range(12)) * 40)
        nat = natural_planes(rng, h, w, sub, [qt[0]] * 3)
        state = dict(i=0)

        def block(c, pred, first):
            state['i'] += 1
            j = next(it, None)
            if j is None:
                b = nat[c].reshape(-1, 64)[state['i'] % nat[c].reshape(-1, 64).shape[0]].copy()
                return b
            b, fixed = specials[j]
            b = b.copy()
            if not fixed:
                s = next(cats)
                if s == 11 and -8 < pred < 0:
                    s = 10
                b[0] = dc_walk(rng, [s], start=pred)[0]
            return b

        planes = build_planes(h, w, sub, 3, block)
        out.append(_case(f'coef-{tag}', 'coef', h, w, sub, planes, qt, ht, comps, 3))
    return out


def ff_dense_tables():
    """the frequent symbols (DC category 1, AC 0/1 and EOB) on the 16-bit codes just below all-ones, every other symbol on
    shorter codes that fill the rest of the code space: blocks of these symbols with +1 values are nearly all 1-bits"""
    def table(others, frequent):
        budget, terms = (65536 - 8) // 2, []
        for k in range(15, -1, -1):                        # binary decomposition in units of 2^-15, then split to fit
            if budget >> k & 1:
                terms.append(k)
        while len(terms) < len(others):
            terms.sort()
            k = terms.pop()
            terms += [k - 1, k - 1]
        assert len(terms) == len(others)
        lengths = [(s, 15 - k) for s, k in zip(others, sorted(terms, reverse=True))]
        lengths += [(s, 16) for s in frequent]
        return huff(lengths)
    dc = table([c for c in range(12) if c != 1] + [9, 10, 11, 0], [2, 3, 4, 5, 6, 0, 1])    # repeated values are legal
    rest = [s for s in AC_SYMBOLS if s not in (EOB, 0x01, 0x02, 0x11, 0x03, 0x21, 0x12)]
    ac = table(rest, [0x03, 0x21, 0x12, 0x11, 0x02, EOB, 0x01])
    return dc, ac


def stuffing_cases():
    out = []
    dc, ac = ff_dense_tables()
    for tag, sub in _subs():
        rng = np.random.default_rng([4, sub])
        h, w = (96, 192) if sub == 2 else (64, 96)
        qt = {0: np.ones(64, np.int64)}

        def block(c, pred, first):
            b = np.zeros(64, np.int64)
            b[0] = pred + (1 if pred < 900 else -1)
            n = rng.integers(0, 6)
            b[ZIGZAG[1:1 + n]] = 1
            return b

        planes = build_planes(h, w, sub, 1, block)
        out.append(_case(f'stuffing-{tag}', 'stuffing', h, w, sub, planes, qt, {(0, 0): dc, (1, 0): ac},
                         [(1, 0, 0, 0), (2, 0, 0, 0), (3, 0, 0, 0)], 1))
    return out


def _fills(rng, n):
    return [int(v) for v in rng.integers(1, 4, n)]


def _exact_planes(rng, h, w, sub, ri, ht, qs, target_mod, target_rem):
    """natural first MCU in every interval, then DC-only blocks whose categories make the interval's bit length
    = target_rem (mod target_mod)"""
    dc, ac = ht[(0, 0)], ht[(1, 0)]
    nat = natural_planes(rng, h, w, sub, qs)
    planes = blank_planes(h, w, sub)
    order = decode_order(h, w, sub)
    bpm = len(mcu_layout(sub))
    for i0 in range(0, len(order), ri * bpm):
        blocks = order[i0:i0 + ri * bpm]
        bw, pred = BitWriter(), [0, 0, 0]
        for m, c, by, bx in blocks[:bpm]:
            b = nat[c][by, bx]
            planes[c][by, bx] = b
            encode_block(bw, b[ZIGZAG], int(b[0]) - pred[c], dc, ac)
            pred[c] = int(b[0])
        tail = blocks[bpm:]
        costs = [{s: dc.enc[s][0] + s + ac.enc[EOB][0] for s in range(11)} for _ in tail]
        lo = bw.n + sum(min(cs.values()) for cs in costs)
        total = lo + (target_rem - lo) % target_mod
        cats = fit_tail(costs, total - bw.n)
        for (m, c, by, bx), s in zip(tail, cats):
            planes[c][by, bx, 0] = dc_walk(rng, [s], max(DC_MIN, -(1024 // qs[c][0])), min(DC_MAX, 1016 // qs[c][0]),
                                           pred[c])[0]
            pred[c] = int(planes[c][by, bx, 0])
    return planes


def restart_cases():
    out = []
    for tag, sub in _subs():
        rng = np.random.default_rng([5, sub])
        qt = {0: _qt(rng, 1, 12)}
        ht = {(0, 0): full_dc(rng), (1, 0): full_ac(rng)}
        comps = [(1, 0, 0, 0), (2, 0, 0, 0), (3, 0, 0, 0)]
        qs = [qt[0]] * 3

        def nat(h, w):
            return natural_planes(rng, h, w, sub, qs)

        h, w = (24, 40) if sub == 1 else (32, 48)
        out.append(_case(f'restart-dri-beyond-{tag}', 'restart', h, w, sub, nat(h, w), qt, ht, comps, 40))
        h, w = (48, 208) if sub == 2 else (40, 56)        # 13 or 7 MCUs per row
        out.append(_case(f'restart-dri-off-row-{tag}', 'restart', h, w, sub, nat(h, w), qt, ht, comps, 5))
        n_iv = -(-geometry(h, w, sub)[0] * geometry(h, w, sub)[1] // 5)
        out.append(_case(f'restart-dri-off-row-fill-{tag}', 'restart', h, w, sub, nat(h, w), qt, ht, comps, 5,
                         fill_rst=_fills(rng, n_iv), fill_eoi=2))
        out.append(_case(f'restart-1x1-{tag}', 'restart', 1, 1, sub, nat(1, 1), qt, ht, comps, 1))
        out.append(_case(f'restart-1x1-fill-{tag}', 'restart', 1, 1, sub, nat(1, 1), qt, ht, comps, 1, fill_eoi=3))
        # DRI 1 on 1600x900: 5700 / 22600 intervals, light content
        h, w = 900, 1600
        my, mx = geometry(h, w, sub)
        light = build_planes(h, w, sub, 1, lambda c, pred, first: symbol_block(
            rng, pred, ht[(0, 0)], Huff([0, 1] + [0] * 14, [EOB]) if rng.random() < 0.8 else ht[(1, 0)], qs[c], 0.8,
            -100, 100))
        out.append(_case(f'restart-dri1-1600x900-fill-{tag}', 'restart', h, w, sub, light, qt, ht, comps, 1,
                         fill_rst=_fills(rng, my * mx - 1), fill_eoi=1))
        # intervals of exactly 1024 k bits (no padding), and of 8 k + 1 bits (7 padding bits)
        h, w = (64, 256) if sub == 2 else (64, 128)
        ri = 32 if sub == 2 else 64
        for mod, rem, name in ((1024, 0, 'exact1024'), (8, 1, 'pad7')):
            planes = _exact_planes(rng, h, w, sub, ri, ht, qs, mod, rem)
            n_iv = geometry(h, w, sub)[0] * geometry(h, w, sub)[1] // ri
            out.append(_case(f'restart-{name}-{tag}', 'restart', h, w, sub, planes, qt, ht, comps, ri))
            out.append(_case(f'restart-{name}-fill-{tag}', 'restart', h, w, sub, planes, qt, ht, comps, ri,
                             fill_rst=_fills(rng, n_iv), fill_eoi=3))
    return out


def worst_case(sub, h, w, restart=0, seed=0, n_ac=(6, 24)):
    rng = np.random.default_rng([6, sub, seed])
    dc, ac = worst_tables()
    qt = {0: np.ones(64, np.int64)}
    planes = build_planes(h, w, sub, restart, lambda c, pred, first: worst_block(rng, pred, first,
                                                                               int(rng.integers(*n_ac))))
    tag = '420' if sub == 2 else '444'
    name = f'worst-{w}x{h}-{tag}' + (f'-dri{restart}' if restart else '')
    return _case(name, 'worst', h, w, sub, planes, qt, {(0, 0): dc, (1, 0): ac}, [(1, 0, 0, 0), (2, 0, 0, 0), (3, 0, 0, 0)],
                 restart)


def worst_cases():
    return [worst_case(1, 900, 1600), worst_case(2, 900, 1600, n_ac=(10, 30)), worst_case(2, 220, 400, restart=50),
            worst_case(1, 120, 200, restart=40)]


def cases():
    """every case: dict(name, family, data (file bytes), spec (the writer's input, planes included), info)"""
    return header_cases() + code_cases() + coef_cases() + stuffing_cases() + restart_cases() + worst_cases()


def has_fill(case):
    return bool(case['spec'].get('fill_eoi') or any(case['spec'].get('fill_rst') or []))
