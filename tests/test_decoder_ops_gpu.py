"""Operator tests of the voxel decoder (decoder_simt.cu: bev_to_voxel, t32_to_voxel, conv3d_simt, occ_head; conv3d_tc.cu;
head_tc.cu) through the C-ABI entries `occb200_decoder_lift`, `_conv3d` and `_head`, which build their weights with the
engine's own helpers and run the engine's own decoder steps on the route make_frame_plan picks for (precision,
use_tensor_cores, num_classes).  Routes: fp32 on CUDA cores; fp32 on tensor cores (conv3d_tc in three passes on bf16 hi / lo
splits, CUDA-core head); bf16 on CUDA cores; bf16 on tensor cores (conv3d_tc, and head_tc for at most 17 classes, else the
CUDA-core head).

(a) Route table: the path and launch count every entry reports in each configuration with 17 and 18 classes, and their sum
    equals what a frame adds to launches_per_frame when it asks for the volumes as well as bev_embed.
(b) Lift, bit-exact: vox[x][y][z][cm] = stored(bev[y*W + x][cm*16 + z]) on non-square grids, for both lift kernels; the T32
    input's pad rows hold NaN, which must not reach the output.
(c) Conv3d, bit-exact on integer operands: inputs and weights in [-3, 3], so |S| <= 27 * 32 * 9 = 7776 and every partial sum
    is exact in fp32 in any order; BatchNorm chosen so the fold is exact (fl(var + 1e-5) in {1, 4}, gamma = 2^k * root, mean
    and beta small integers).  The output must equal, bit for bit, the storage rounding of relu(S + b): bf16 round-to-nearest
    -even in bf16 storage (tensor cores and CUDA cores alike), fp32 in fp32 storage.  One-hot weights (one tap x one input
    channel per output channel) make the output a shifted copy of the input, so a failure names the tap.
(d) The BatchNorm fold, pinned: on the fp32 CUDA-core route with one-hot weights the accumulator starts at the folded bias
    b_f and takes one FMA with a nonzero weight (the zero weights add exactly nothing), so each output is the single fp32
    rounding of relu(b_f + x w_f): bit-exact against oracle.backbone.fold_conv3d_bn (correctly rounded root) with random BN.
(e) Conv3d against fp64 at production size (200 x 200 x 16, cin 16 and 32), real operands, every path.  Reference: the
    convolution in fp64 on the stored input with the mirrored fold; weights rounded to bf16 on the tensor cores, fp32 on the
    CUDA cores (also in bf16 storage) and on the split path.  With S = conv(|x|, |w|), K = 27 cin, u = 2^-23 (twice fp32's
    unit roundoff, which also covers the tensor cores' truncating accumulation), per element:
        CUDA cores     e = K u (S + |b|)                  the bias is the initial accumulator: K FMAs, each rounding a partial
                                                          sum bounded by S + |b|
        tensor cores   e = K u S + u (S + |b|)            the K-term accumulation, then the epilogue's bias add
        split          e = K u S (1 + 2^-7) + 2 u (S + |b|) + 2^-16 S
                                                          three passes (the lo passes sum to <= 2^-8 S each), two fp32 adds of
                                                          a pass into the output, and the split's own term: the dropped lo.lo
                                                          product (2^-18 S) and the bf16 rounding of the lo halves (2^-18 S for
                                                          the input, 2^-18 S for the weights), below 2^-16 S, the bar of
                                                          gemm_tc_split3
        bf16 storage   e += 2^-8 (|F64| + e)              one bf16 rounding of the output
    ReLU is 1-Lipschitz, so the bounds hold after it.  Every bound carries a factor 1.001.
(f) Heads against fp64, every path, num_classes in {1, 2, 16, 17, 18, 32}.  Reference: fp64 on the route's stored operands
    (bf16 voxels and weights on head_tc, fp32 weights on the CUDA cores).  Per element, with u = 2^-23:
        CUDA cores  hidden  e_a = 32 u (|v| |W1| + |b1|)      FMA chain from the bias
                            softplus log1pf(expf(x)) (x <= 20) or x: e_h = e_a + 8 u sp(a) + 2^-28
                                                          (expf within 2 ulp moves log1p by at most 2^-22 sp / ln 2,
                                                          log1pf within 2 ulp; e^-20 < 2^-28 past the cut)
                            ReLU: e_h = e_a
                    output  e = 64 u (|h| |W2| + |b2|) + |W2| e_h
        head_tc     hidden  e_a = 32 u S1 + u (S1 + |b1|)      K = 32 on the tensor cores, then the bias add
                            softplus: e_h = e_a + (1.2e-5 + |a| 2^-24) sp(a) (the degree-5 polynomial, 7.2e-6 relative
                                                          to t, i.e. 1.04e-5 relative to log1p(t) >= t ln 2; MUFU ex2 2^-22
                                                          relative; the fp32 rounding of its argument |a| log2(e); the final
                                                          FMA), ReLU: e_h = e_a; then e_h += 2^-8 (|h| + e_h) for the
                                                          bf16 rounding of the hidden activation
                    output  e = 64 u S2 + u (S2 + |b2|) + |W2| e_h   (the block-diagonal zeros add exactly nothing)
    Exact subcases: integer operands whose softplus pre-activations are integers in [21, 255] or <= -200 (both softplus
    forms return exactly x or exactly 0) and whose ReLU pre-activations are integers with |h| <= 256, so every hidden value
    is exact in bf16 and logits and flow are bit-exact.  Argmax, bit-exact on every path: cls is the first argmax of the
    kernel's own logits, cls_u8 == cls_i64; ties from duplicated predicter.2 rows with equal biases (inside one lane, across
    the lanes of a quad, at class 0 and at the last class) must resolve to the lower class, as torch.argmax does; and cls
    equals the fp64 argmax wherever the fp64 top-2 gap exceeds twice the bound.  Output subsets: all 16 NULL / non-NULL
    combinations, each requested output bit-identical to the all-outputs call.
(g) Argument rejections, before any CUDA call (CPU suite).
Every output is surrounded by guard elements pre-filled with a NaN bit pattern, which must survive the launch.  A conv3d
mismatch names the voxel (x, y, z, c), its 8-row y tile and the segment of the CTA that computed it on conv3d_tc.

GPU cases run in a child process per test function, so that a device fault cannot poison this session.

Known difference, not tested: both head kernels skip a NaN logit in the argmax, where torch.argmax reports the NaN's index.
"""
import ctypes
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NAN16 = 0x7FA5
NAN32 = 0x7FA5A5A5
GUARD = 4096
U23 = 2.0 ** -23
U8 = 2.0 ** -8
Z = 16
OD = 32

CUDA_CORES, TC, SPLIT = 0, 1, 2
PATH_NAME = {0: 'CUDA cores', 1: 'tensor cores', 2: 'split tensor cores (3 passes)'}
HEAD_NAME = {0: 'CUDA-core head', 1: 'head_tc'}
CONFIGS = [('fp32', 0, 0), ('fp32 tensor cores', 0, 1), ('bf16 CUDA cores', 1, 0), ('bf16 tensor cores', 1, 1)]
CLASSES = (1, 2, 16, 17, 18, 32)


def expected_route(precision, tc, nc):
    """{'lift': launches, 'conv': (path, launches), 'head': (path, launches)} of make_frame_plan's route"""
    conv = SPLIT if (precision == 0 and tc) else TC if (precision == 1 and tc) else CUDA_CORES
    head = 1 if conv == TC and nc + 2 <= 19 else 0
    return {'lift': 1, 'conv': (conv, 4 if conv == SPLIT else 1), 'head': (head, 1)}


# ------------------------------------------------------------------------------------------------ fold and reference (CPU)
def exact_bn(g, od=OD):
    """BatchNorm parameters [4][32] = gamma | beta | mean | var whose fold is exact: fl(var + 1e-5f) is 1 or 4, gamma =
    2^k * sqrt of it (so the scale is 2^k, k in {-1, 0, 1}), mean and beta small integers"""
    eps = np.float32(1e-5)
    var = np.empty(od, np.float32)
    gamma = np.empty(od, np.float32)
    for c in range(od):
        root = 1.0 if c % 2 == 0 else 2.0
        v = np.float32(root * root) - eps
        while np.float32(v + eps) != np.float32(root * root):          # the fp32 value whose sum with eps rounds to root^2
            v = np.nextafter(v, np.float32(root * root), dtype=np.float32)
        var[c] = v
        gamma[c] = np.float32(root * 2.0 ** int(torch.randint(-1, 2, (1,), generator=g)))
    mean = torch.randint(-3, 4, (od,), generator=g).numpy().astype(np.float32)
    beta = torch.randint(-3, 4, (od,), generator=g).numpy().astype(np.float32)
    return np.stack([gamma, beta, mean, var])


def fold(w, bn):
    """the engine's fold (oracle mirror): w [32, cin, 3, 3, 3] fp32, bn [4][32] -> (wf [32, cin, 3, 3, 3], bf [32]) fp32"""
    from oracle.backbone import fold_conv3d_bn
    t = torch.as_tensor
    return fold_conv3d_bn(t(w), t(bn[0]), t(bn[1]), t(bn[2]), t(bn[3]))


def conv3d_64(x, wf, bf=None):
    """fp64 3x3x3 convolution, pad 1, of channels-last x [X, Y, Z, cin] with torch-layout wf [32, cin, kz, ky, kx] (+ bf):
    the sum over the 27 taps of shifted [X*Y*Z, cin] x [cin, 32] products, [X, Y, Z, 32]"""
    X, Y, Zd, cin = x.shape
    xp = F.pad(x.double(), (0, 0, 1, 1, 1, 1, 1, 1))
    w = wf.double().to(x.device)
    out = torch.zeros(X * Y * Zd, w.shape[0], dtype=torch.float64, device=x.device)
    for dz, dy, dx in itertools.product(range(3), range(3), range(3)):
        out += xp[dx:dx + X, dy:dy + Y, dz:dz + Zd].reshape(-1, cin) @ w[:, :, dz, dy, dx].t()
    if bf is not None:
        out += bf.double().to(x.device)
    return out.view(X, Y, Zd, -1)


def test_fp64_reference_convolution_is_torch_conv3d_on_the_reference_layout():
    """conv3d_64 on channels-last [X][Y][Z][C] is F.conv3d on the reference's (1, C, Z, Y, X) volume (transformer_occ.py
    reshapes the BEV to (bs, C, Z, H, W)); a non-cubic shape and asymmetric weights pin every axis"""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 4, 3, 16, generator=g, dtype=torch.float64)
    w = torch.randn(32, 16, 3, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(32, generator=g, dtype=torch.float64)
    want = F.conv3d(x.permute(3, 2, 1, 0)[None], w, b, padding=1)[0].permute(3, 2, 1, 0)
    assert torch.allclose(conv3d_64(x, w, b), want, rtol=1e-12, atol=1e-12)


def test_exact_batchnorm_folds_exactly():
    """the (c) BatchNorm: fl(var + 1e-5) is 1 or 4, the scale a power of two, and the fold equals the exact fold"""
    g = torch.Generator().manual_seed(3)
    bn = exact_bn(g)
    s2 = bn[3] + np.float32(1e-5)
    assert s2.dtype == np.float32 and set(s2.tolist()) == {1.0, 4.0}
    w = torch.randint(-3, 4, (32, 16, 3, 3, 3), generator=g).float().numpy()
    wf, bf = fold(w, bn)
    scale = bn[0].astype(np.float64) / np.sqrt(s2.astype(np.float64))
    assert set(np.log2(scale).tolist()) <= {-1.0, 0.0, 1.0}
    assert np.array_equal(wf.numpy().astype(np.float64), w.astype(np.float64) * scale[:, None, None, None, None])
    assert np.array_equal(bf.numpy().astype(np.float64), bn[1].astype(np.float64) - bn[2].astype(np.float64) * scale)


def test_fold_mirror_against_numpy_restatement_and_the_bf16_model():
    """oracle.backbone.fold_conv3d_bn is engine.cu's fold_conv3d_bn (sqrtf of fl(var + 1e-5f), scale and shift in fp32) bit
    for bit, over random BatchNorm statistics; oracle/bf16_model.py folds with torch's fp32 sqrt, which the goldens were
    made with, and is reported, not changed"""
    g = torch.Generator().manual_seed(11)
    w = torch.randn(32, 32, 3, 3, 3, generator=g).numpy()
    differ = 0
    for _ in range(50):
        bn = np.stack([torch.rand(32, generator=g).numpy() * 2 + 0.1, torch.randn(32, generator=g).numpy(),
                       torch.randn(32, generator=g).numpy(), torch.rand(32, generator=g).numpy() * 3 + 1e-3]).astype(np.float32)
        wf, bf = fold(w, bn)
        s = bn[0] / np.sqrt(bn[3] + np.float32(1e-5))
        assert s.dtype == np.float32
        assert np.array_equal(wf.numpy(), w * s[:, None, None, None, None])
        assert np.array_equal(bf.numpy(), bn[1] - bn[2] * s)
        st = torch.as_tensor(bn[0]) / torch.sqrt(torch.as_tensor(bn[3]) + 1e-5)
        differ += int((st.numpy() != s).sum())
    print(f'bf16_model fold scale differs from the engine fold in {differ} of {50 * 32} channels')


# ------------------------------------------------------------------------------------------------ (g) rejections (CPU)
_LIFT = dict(precision=1, tc=1, t32=0, bev=1, H=8, W=8, vox=1, launches=1)
_CONV = dict(precision=1, tc=1, x=1, X=4, Y=8, cin=16, w=1, bn=1, out=1, path=1, launches=1)
_HEAD = dict(precision=1, tc=1, nc=17, vox=1, nvox=128, w=1, out=1, path=1, launches=1)
_REJECT = [
    ('lift', dict(bev=None), 'null'), ('lift', dict(vox=None), 'null'), ('lift', dict(launches=None), 'null'),
    ('lift', dict(precision=2), 'precision'), ('lift', dict(tc=2), 'use_tensor_cores'), ('lift', dict(precision=-1), 'precision'),
    ('lift', dict(t32=1, precision=0, tc=0), 'from_t32'), ('lift', dict(t32=1, precision=0, tc=1), 'from_t32'),
    ('lift', dict(t32=1, precision=1, tc=0), 'from_t32'), ('lift', dict(t32=2), 'from_t32'),
    ('lift', dict(H=0), 'BEV grid'), ('lift', dict(W=-1), 'BEV grid'), ('lift', dict(H=4097, W=4097), 'BEV grid'),
    ('conv', dict(x=None), 'null'), ('conv', dict(w=None), 'null'), ('conv', dict(bn=None), 'null'),
    ('conv', dict(out=None), 'null'), ('conv', dict(path=None), 'null'), ('conv', dict(launches=None), 'null'),
    ('conv', dict(precision=3), 'precision'), ('conv', dict(tc=-1), 'use_tensor_cores'),
    ('conv', dict(X=0), 'X and Y'), ('conv', dict(Y=0), 'X and Y'), ('conv', dict(X=4097), 'X and Y'),
    ('conv', dict(cin=8), 'cin'), ('conv', dict(cin=64), 'cin'), ('conv', dict(cin=24), 'cin'),
    ('head', dict(vox=None), 'null'), ('head', dict(w=None), 'null'), ('head', dict(path=None), 'null'),
    ('head', dict(launches=None), 'null'), ('head', dict(precision=2), 'precision'), ('head', dict(tc=2), 'use_tensor_cores'),
    ('head', dict(nc=0), 'num_classes'), ('head', dict(nc=33), 'num_classes'),
    ('head', dict(nvox=0), 'nvox'), ('head', dict(nvox=1 << 31), 'nvox'),
]


@pytest.mark.parametrize('case', range(len(_REJECT)))
def test_entry_point_rejects_bad_arguments_before_any_cuda_call(case, lib_built):
    """Return code 1 (an argument check, not 2, a CUDA error) and a message.  Device pointers are a real buffer when a GPU is
    present, a dummy otherwise (a CUDA call would then fail with 2)."""
    from occnet_b200 import _lib
    lib = _lib.load()
    name, over, msg = _REJECT[case]
    buf = torch.zeros(1 << 20, device='cuda') if torch.cuda.is_available() else None
    dev = ctypes.c_void_p(buf.data_ptr()) if buf is not None else ctypes.c_void_p(1 << 12)
    host = np.ones(1 << 16, np.float32)
    hp = ctypes.c_void_p(host.ctypes.data)
    ints = [ctypes.c_int() for _ in range(2)]
    if name == 'lift':
        a = dict(_LIFT, **over)
        rc = lib.occb200_decoder_lift(a['precision'], a['tc'], a['t32'], dev if a['bev'] else None, a['H'], a['W'],
                                      dev if a['vox'] else None, ctypes.byref(ints[0]) if a['launches'] else None, None)
    elif name == 'conv':
        a = dict(_CONV, **over)
        rc = lib.occb200_decoder_conv3d(a['precision'], a['tc'], dev if a['x'] else None, a['X'], a['Y'], a['cin'],
                                        hp if a['w'] else None, hp if a['bn'] else None, dev if a['out'] else None,
                                        ctypes.byref(ints[0]) if a['path'] else None,
                                        ctypes.byref(ints[1]) if a['launches'] else None, None)
    else:
        a = dict(_HEAD, **over)
        ws = [hp if a['w'] else None] + [hp] * 7
        rc = lib.occb200_decoder_head(a['precision'], a['tc'], a['nc'], dev if a['vox'] else None, a['nvox'], *ws,
                                      dev if a['out'] else None, None, None, None,
                                      ctypes.byref(ints[0]) if a['path'] else None,
                                      ctypes.byref(ints[1]) if a['launches'] else None, None)
    err = lib.occb200_last_error().decode()
    assert rc == 1, (name, over, rc, err)
    assert msg in err, (name, over, err)


# ------------------------------------------------------------------------------------------------ GPU: child processes
def _run_isolated(code, timeout=1800):
    r = subprocess.run([sys.executable, '-c', 'import sys; sys.path.insert(0, "tests"); ' + code], cwd=ROOT, capture_output=True,
                       text=True, timeout=timeout)
    print(r.stdout[-20000:])
    assert r.returncode == 0, f'child failed ({r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'
    assert 'OK' in r.stdout
    return r.stdout


def _child(fn):
    return _run_isolated(f'import test_decoder_ops_gpu as t; t.{fn}(); print("OK")')


DEV = 'cuda:0'
_DT = {0: torch.float32, 1: torch.bfloat16}


def _lib():
    from occnet_b200 import _lib as L
    return L, L.load()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _h(a):
    return ctypes.c_void_p(a.ctypes.data)


class Out:
    """an output of `shape` with GUARD guard elements on each side, all pre-filled with NaN bits (integer outputs: 0x5A)"""

    def __init__(self, shape, dtype):
        self.shape, self.dtype = tuple(shape), dtype
        self.n = int(np.prod(self.shape))
        self.fill = {torch.float32: NAN32, torch.bfloat16: NAN16, torch.uint8: 0x5A, torch.int64: 0x5A5A5A5A5A5A5A5A}[dtype]
        it = {torch.float32: torch.int32, torch.bfloat16: torch.int16}.get(dtype, dtype)
        self.bits = torch.full((self.n + 2 * GUARD,), self.fill, dtype=it, device=DEV)
        self.buf = self.bits.view(dtype)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + GUARD * self.buf.element_size())

    def value(self):
        return self.buf[GUARD:GUARD + self.n].view(self.shape)

    def untouched(self):
        return bool((self.bits == self.fill).all())

    def check_guards(self, what):
        for name, p in (('leading guard', self.bits[:GUARD]), ('trailing guard', self.bits[GUARD + self.n:])):
            bad = (p != self.fill).nonzero()
            assert bad.numel() == 0, f'{what}: {bad.numel()} elements of the {name} were written (first at {int(bad[0])})'


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16) if t.dtype == torch.bfloat16 else t


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def segment_of(X, Y, x, y, sms):
    """conv3d_tc's CTA and segment for output (x, y): tiles t = y_tile * X + x are cut into min(tiles, SMs) contiguous CTA
    ranges, each cut into segments of constant y_tile"""
    yt = y // 8
    total = X * ((Y + 7) // 8)
    grid = min(total, sms)
    t = yt * X + x
    cta = next(b for b in range(grid) if total * b // grid <= t < total * (b + 1) // grid)
    t0, t1 = total * cta // grid, total * (cta + 1) // grid
    xa, xb = max(t0, yt * X) - yt * X, min(t1, (yt + 1) * X) - yt * X
    return f'CTA {cta} of {grid}, segment x in [{xa}, {xb}) of y tile {yt}'


def _where_vox(bad, what, got=None, want=None, extra=None):
    """AssertionError text naming the first bad voxel (x, y, z, c), its 8-row y tile and its conv3d_tc segment"""
    idx = bad.nonzero()
    x, y, z, c = (int(v) for v in idx[0])
    X, Y = bad.shape[0], bad.shape[1]
    s = (f'{what}: {idx.shape[0]} mismatches; first at (x, y, z, c) = ({x}, {y}, {z}, {c}): y tile {y // 8}, '
         f'{segment_of(X, Y, x, y, _sms())}; bad x planes {sorted(set(idx[:, 0].tolist()))[:12]}, '
         f'bad y {sorted(set(idx[:, 1].tolist()))[:12]}, bad z {sorted(set(idx[:, 2].tolist()))[:16]}')
    if got is not None:
        s += f'; got {got[x, y, z, c].item()!r} want {want[x, y, z, c].item()!r}'
    if extra is not None:
        s += extra(x, y, z, c)
    return s


# ---- the entries
def lift(precision, tc, from_t32, bev, H, W, tag):
    L, lib = _lib()
    o = Out((W, H, Z, 256 // Z), _DT[precision])
    n = ctypes.c_int()
    L.check(lib.occb200_decoder_lift(precision, tc, from_t32, _p(bev), H, W, o.ptr(), ctypes.byref(n), L.stream_ptr()))
    o.check_guards(tag)
    return o.value(), n.value


def conv3d(precision, tc, x, w, bn, tag):
    """x [X, Y, 16, cin] device (storage type), w fp32 numpy [32, cin, 3, 3, 3] (torch layout), bn [4, 32]"""
    L, lib = _lib()
    X, Y, _, cin = x.shape
    o = Out((X, Y, Z, OD), _DT[precision])
    wh, bh = np.ascontiguousarray(w, np.float32), np.ascontiguousarray(bn, np.float32)
    path, n = ctypes.c_int(), ctypes.c_int()
    L.check(lib.occb200_decoder_conv3d(precision, tc, _p(x), X, Y, cin, _h(wh), _h(bh), o.ptr(), ctypes.byref(path),
                                       ctypes.byref(n), L.stream_ptr()))
    o.check_guards(tag)
    return o.value(), path.value, n.value


OUTS = ('occ', 'flow', 'u8', 'i64')


def head(precision, tc, nc, vox, hw, want=OUTS, tag=''):
    """vox [nvox, 32] device; hw: the eight torch-layout fp32 numpy arrays.  -> ({output: tensor}, path, launches, outs)"""
    L, lib = _lib()
    nvox = vox.shape[0]
    outs = {'occ': Out((nvox, nc), torch.float32), 'flow': Out((nvox, 2), torch.float32),
            'u8': Out((nvox,), torch.uint8), 'i64': Out((nvox,), torch.int64)}
    hs = [np.ascontiguousarray(a, np.float32) for a in hw]
    path, n = ctypes.c_int(), ctypes.c_int()
    L.check(lib.occb200_decoder_head(precision, tc, nc, _p(vox), nvox, *[_h(a) for a in hs],
                                     *[outs[k].ptr() if k in want else None for k in OUTS], ctypes.byref(path),
                                     ctypes.byref(n), L.stream_ptr()))
    for k in OUTS:
        if k in want:
            outs[k].check_guards(f'{tag} {k}')
        else:
            assert outs[k].untouched(), f'{tag}: the NULL output {k} was written'
    return {k: outs[k].value() for k in want}, path.value, n.value


# ---- (a) the route table
def check_route_table():
    from occnet_b200 import fixtures
    from occnet_b200.engine import OccEngine
    g = torch.Generator().manual_seed(0)
    rows = []
    for cfg_name, precision, tc in CONFIGS:
        dt = _DT[precision]
        for nc in (17, 18):
            want = expected_route(precision, tc, nc)
            bev = torch.randn(6 * 5, 256, device=DEV)
            _, n_lift = lift(precision, tc, 0, bev, 6, 5, 'route lift')
            counts = {'lift': n_lift}
            for cin in (16, 32):
                x = torch.zeros(5, 6, Z, cin, device=DEV).to(dt)
                _, path, n = conv3d(precision, tc, x, np.zeros((OD, cin, 3, 3, 3), np.float32), exact_bn(g), 'route conv')
                assert (path, n) == want['conv'], (cfg_name, nc, cin, path, n, want)
                counts[f'conv{cin}'] = n
            hw = head_weights(torch.Generator().manual_seed(1), nc, 'real')
            _, path, n = head(precision, tc, nc, torch.zeros(300, OD, device=DEV).to(dt), hw, tag='route head')
            assert (path, n) == want['head'], (cfg_name, nc, path, n, want)
            counts['head'] = n
            # the engine: a frame that asks for the volumes too launches exactly these kernels more than a bev_embed-only frame
            cfg = fixtures.make_cfg('small6', num_layers=1, num_classes=nc)
            eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2), precision='bf16' if precision else 'fp32',
                            use_tensor_cores=bool(tc), device=DEV)
            eng.set_cameras(fixtures.make_img_metas(cfg, bs=1))
            feats = [f[0].to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=3)]
            eng.forward(feats, want=('bev_embed',))
            n_bev = eng.launches_per_frame
            eng.forward(feats, want=('bev_embed', 'occ', 'flow', 'occ_cls', 'occ_cls_i64'))
            n_all = eng.launches_per_frame
            assert n_all - n_bev == sum(counts.values()), (cfg_name, nc, n_all, n_bev, counts)
            del eng
            rows.append(f'{cfg_name:18s} {nc:2d} classes: lift 1, conv {PATH_NAME[want["conv"][0]]} x {want["conv"][1]} '
                        f'launches per layer, {HEAD_NAME[want["head"][0]]} 1; frame adds {n_all - n_bev} '
                        f'({n_bev} -> {n_all})')
    print('route table:\n  ' + '\n  '.join(rows))


# ---- (b) the lift
def check_lift():
    from test_gemm_tc_gpu import t32_pack
    for i, (H, W) in enumerate([(1, 1), (1, 45), (45, 1), (7, 5), (5, 7), (13, 9), (30, 44), (200, 200)]):
        g = torch.Generator(device=DEV).manual_seed(100 + i)
        bev = torch.randn(H * W, 256, device=DEV, generator=g)
        for precision, tc, t32 in [(0, 0, 0), (0, 1, 0), (1, 0, 0), (1, 1, 0), (1, 1, 1)]:
            dt = _DT[precision]
            inp = t32_pack(bev, fill=float('nan')) if t32 else bev
            tag = f'lift {H}x{W} {dt} {"t32_to_voxel" if t32 else "bev_to_voxel"}'
            got, n = lift(precision, tc, t32, inp, H, W, tag)
            assert n == 1, tag
            want = bev.view(H, W, 16, Z).permute(1, 0, 3, 2).to(dt)     # [x][y][z][cm] = bev[y*W + x][cm*16 + z]
            bad = _bits(got) != _bits(want)
            if bool(bad.any()):
                raise AssertionError(_where_vox(bad, tag + ' (c = cm)', got, want))
        print(f'lift {H}x{W} (Nq % 8 = {H * W % 8}, Nq % 32 = {H * W % 32}): bit-exact, both kernels')


# ---- (c) conv3d on integer operands
def conv_shapes():
    sms = _sms()
    shapes = [(x, y) for x in (1, 2, 3) for y in (1, 8, 9, 10, 11, 12, 13, 14, 15)]
    shapes += [(200, y) for y in (1, 5, 16)]
    shapes += [(sms - 1, 8), (sms, 8), (sms + 1, 8), (sms + 1, 3), ((sms + 1) // 2, 16)]    # tiles below / at / above the SMs
    shapes += [(37, 61), (3, 200), (1, 203), (200, 47)]               # several tiles per CTA: segments cross y tiles, ring wraps
    return shapes


def check_exact_case(X, Y, cin, onehot, seed, configs=CONFIGS, production=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-3, 4, (X, Y, Z, cin), generator=g).float().to(DEV)
    taps = None
    if onehot:
        taps = (torch.randint(0, 27, (OD,), generator=g), torch.randint(0, cin, (OD,), generator=g))
        w = torch.zeros(OD, cin, 27)
        w[torch.arange(OD), taps[1], taps[0]] = torch.randint(1, 4, (OD,), generator=g).float() * \
            (torch.randint(0, 2, (OD,), generator=g).float() * 2 - 1)
        w = w.view(OD, cin, 3, 3, 3)
    else:
        w = torch.randint(-3, 4, (OD, cin, 3, 3, 3), generator=g).float()
    bn = exact_bn(g)
    wf, bf = fold(w.numpy(), bn)
    ref = conv3d_64(x, wf, bf).clamp_min(0)
    for cfg, precision, tc in configs:
        dt = _DT[precision]
        tag = f'{"one-hot" if onehot else "integer"} conv3d {X}x{Y}x16 cin {cin} {cfg}'
        got, path, n = conv3d(precision, tc, x.to(dt), w.numpy(), bn, tag)
        assert (path, n) == expected_route(precision, tc, 17)['conv'], (tag, path, n)
        want = ref.float().to(dt)
        bad = _bits(got) != _bits(want)
        if bool(bad.any()):
            extra = None
            if taps is not None:
                extra = lambda x_, y_, z_, c: (f'; one-hot weight of c {c}: tap (dz, dy, dx) = '
                                               f'{np.unravel_index(int(taps[0][c]), (3, 3, 3))}, ci {int(taps[1][c])}')
            raise AssertionError(_where_vox(bad, f'{tag} [{PATH_NAME[path]}]', got, want, extra))


def check_conv_exact():
    shapes = conv_shapes()
    for i, (X, Y) in enumerate(shapes):
        for cin in (16, 32):
            check_exact_case(X, Y, cin, False, 1000 + 10 * i + cin)
            check_exact_case(X, Y, cin, True, 2000 + 10 * i + cin)
    print(f'conv3d: {len(shapes)} shapes x cin 16 / 32 bit-exact on integer and one-hot weights, every route')
    for cin in (16, 32):
        check_exact_case(200, 200, cin, False, 3000 + cin)
        check_exact_case(200, 200, cin, True, 3100 + cin)
    print('conv3d: production 200x200x16, cin 16 and 32: bit-exact on integer and one-hot weights, every route')


# ---- (d) the fold, pinned on the fp32 CUDA-core route
def check_fold_pinned():
    for i, (X, Y, cin) in enumerate([(3, 9, 16), (5, 17, 32), (40, 40, 32)]):
        g = torch.Generator().manual_seed(4000 + i)
        x = torch.randint(-3, 4, (X, Y, Z, cin), generator=g).float().to(DEV)
        taps = torch.randint(0, 27, (OD,), generator=g), torch.randint(0, cin, (OD,), generator=g)
        w = torch.zeros(OD, cin, 27)
        w[torch.arange(OD), taps[1], taps[0]] = torch.randint(1, 4, (OD,), generator=g).float()
        w = w.view(OD, cin, 3, 3, 3)
        bn = np.stack([torch.rand(OD, generator=g).numpy() * 2 + 0.1, torch.randn(OD, generator=g).numpy(),
                       torch.randn(OD, generator=g).numpy(), torch.rand(OD, generator=g).numpy() * 3 + 1e-3]).astype(np.float32)
        wf, bf = fold(w.numpy(), bn)
        # x w_f (at most 26 significant bits) + b_f is exact in fp64, so rounding it to fp32 is the FMA's single rounding
        want = conv3d_64(x, wf, bf).clamp_min(0).float()
        got, path, _ = conv3d(0, 0, x, w.numpy(), bn, f'fold {X}x{Y} cin {cin}')
        assert path == CUDA_CORES
        bad = _bits(got) != _bits(want)
        if bool(bad.any()):
            raise AssertionError(_where_vox(bad, f'BN fold {X}x{Y} cin {cin}', got, want))
    print('BN fold: bit-exact against the oracle mirror on the fp32 CUDA-core route')


# ---- (e) conv3d against fp64
def conv_bound(path, out16, K, S, b, F64):
    b = b.double().to(S.device).abs()
    if path == CUDA_CORES:
        e = K * U23 * (S + b)
    elif path == TC:
        e = K * U23 * S + U23 * (S + b)
    else:
        e = K * U23 * S * (1 + 2.0 ** -7) + 2 * U23 * (S + b) + 2.0 ** -16 * S
    if out16:
        e = e + U8 * (F64.abs() + e)
    return e * 1.001


def check_conv_fp64():
    worst = {}
    for cin in (16, 32):
        X = Y = 200
        g = torch.Generator(device=DEV).manual_seed(5000 + cin)
        gc = torch.Generator().manual_seed(5100 + cin)
        # mixed magnitudes: per-channel scales 2^-4 .. 2^4, non-negative like the ReLU outputs the second layer reads
        x32 = (torch.randn(X, Y, Z, cin, device=DEV, generator=g) * 2.0 ** torch.randint(-4, 5, (cin,), device=DEV, generator=g))
        if cin == 32:
            x32 = x32.abs()
        w = (torch.randn(OD, cin, 3, 3, 3, generator=gc) * (2.0 / (27 * cin)) ** 0.5).numpy()
        bn = np.stack([torch.rand(OD, generator=gc).numpy() + 0.5, torch.randn(OD, generator=gc).numpy(),
                       torch.randn(OD, generator=gc).numpy() * 0.1, torch.rand(OD, generator=gc).numpy() + 0.5]).astype(np.float32)
        wf, bf = fold(w, bn)
        K = 27 * cin
        for cfg, precision, tc in CONFIGS:
            dt = _DT[precision]
            xs = x32.to(dt)
            got, path, _ = conv3d(precision, tc, xs, w, bn, f'fp64 cin {cin} {cfg}')
            wr = wf.bfloat16().float() if path == TC else wf
            F64 = conv3d_64(xs, wr, bf).clamp_min(0)
            S = conv3d_64(xs.abs(), wr.abs())
            bound = conv_bound(path, precision == 1, K, S, bf, F64)
            del S
            err = (got.double() - F64).abs()
            ratio = (err / bound).max().item()
            worst[cfg] = max(worst.get(cfg, 0.0), ratio)
            print(f'fp64 conv3d 200x200x16 cin {cin} {cfg} [{PATH_NAME[path]}]: max err/bound {ratio:.3f}')
            bad = ~(err <= bound)
            if bool(bad.any()):
                raise AssertionError(_where_vox(bad, f'fp64 cin {cin} {cfg} (got = error, want = bound)', err, bound))
            del F64, err, bound, got
    print('fp64 conv3d largest err/bound per route: ' + ', '.join(f'{c} {v:.3f}' for c, v in worst.items()))


# ---- (f) the heads
def head_weights(g, nc, kind, ties=()):
    """(w1, b1, w2, b2, f1, g1, f2, g2) fp32 numpy, torch layout.  kind 'real': random; 'exact': integer weights with the
    softplus pre-activations in [21, 255] or <= -200 and the ReLU ones in [-256, 256] for voxels in [0, 3].  ties: groups of
    classes whose predicter.2 rows and biases are copies of the group's first, lifted above every other class."""
    H = 2 * OD
    if kind == 'real':
        w1 = torch.randn(H, OD, generator=g) * OD ** -0.5
        b1 = torch.randn(H, generator=g)
        w2 = torch.randn(nc, H, generator=g) * H ** -0.5
        b2 = torch.randn(nc, generator=g)
        f1 = torch.randn(H, OD, generator=g) * OD ** -0.5
        g1 = torch.randn(H, generator=g)
        f2 = torch.randn(2, H, generator=g) * H ** -0.5
        g2 = torch.randn(2, generator=g)
        lift_by = 8.0
    else:
        pos = torch.randint(0, 2, (H,), generator=g).bool()                       # softplus unit on its identity branch
        w1 = torch.where(pos[:, None], torch.randint(0, 3, (H, OD), generator=g), -torch.randint(0, 3, (H, OD), generator=g))
        b1 = torch.where(pos, torch.randint(21, 40, (H,), generator=g), -torch.randint(200, 300, (H,), generator=g))
        w2 = torch.randint(-3, 4, (nc, H), generator=g)
        b2 = torch.randint(-50, 51, (nc,), generator=g)
        f1 = torch.randint(-1, 2, (H, OD), generator=g)                            # |v . f1| <= 96
        g1 = torch.randint(-100, 101, (H,), generator=g)
        f2 = torch.randint(-3, 4, (2, H), generator=g)
        g2 = torch.randint(-50, 51, (2,), generator=g)
        lift_by = 200000.0
    w2, b2 = w2.clone().float(), b2.clone().float()
    for grp in ties:
        for c in grp[1:]:
            w2[c], b2[c] = w2[grp[0]], b2[grp[0]]
        for c in grp:
            b2[c] = b2[c] + lift_by
    return tuple(t.float().numpy() for t in (w1, b1, w2, b2, f1, g1, f2, g2))


def head_ref(vox, hw, path, exact=False):
    """fp64 logits, flow and their bounds over the route's stored operands (exact: the pre-activations of head_weights'
    'exact' kind, whose softplus both kernels compute as exactly max(a, 0))"""
    w1, b1, w2, b2, f1, g1, f2, g2 = (torch.as_tensor(a, device=DEV).double() for a in hw)
    if path == 1:
        w1, w2, f1, f2 = (t.bfloat16().double() for t in (w1, w2, f1, f2))
    v = vox.double()
    a, s1 = v @ w1.t() + b1, v.abs() @ w1.abs().t()
    af, sf = v @ f1.t() + g1, v.abs() @ f1.abs().t()
    sp = F.softplus(a, threshold=1e4)
    if exact:
        assert bool(((a >= 21) & (a <= 255) | (a <= -200)).all()) and bool((af.abs() <= 256).all())
        sp = a.clamp_min(0)
    hf = af.clamp_min(0)
    if path == 1:
        ea, eaf = 32 * U23 * s1 + U23 * (s1 + b1.abs()), 32 * U23 * sf + U23 * (sf + g1.abs())
        eh = ea + (1.2e-5 + a.abs() * 2.0 ** -24) * sp
        eh = eh + U8 * (sp + eh)
        ehf = eaf + U8 * (hf + eaf)
    else:
        ea, eaf = 32 * U23 * (s1 + b1.abs()), 32 * U23 * (sf + g1.abs())
        eh, ehf = ea + 8 * U23 * sp + 2.0 ** -28, eaf
    logits, flow = sp @ w2.t() + b2, hf @ f2.t() + g2
    s2, s2f = sp @ w2.abs().t(), hf @ f2.abs().t()
    if path == 1:
        el = 64 * U23 * s2 + U23 * (s2 + b2.abs()) + eh @ w2.abs().t()
        ef = 64 * U23 * s2f + U23 * (s2f + g2.abs()) + ehf @ f2.abs().t()
    else:
        el = 64 * U23 * (s2 + b2.abs()) + eh @ w2.abs().t()
        ef = 64 * U23 * (s2f + g2.abs()) + ehf @ f2.abs().t()
    return logits, flow, el * 1.001 + 1e-30, ef * 1.001 + 1e-30


def tie_sets(nc):
    """sets of disjoint tie groups: inside one lane of head_tc's quad (classes 0, 1 and 8, 9), across the lanes of a quad
    (1, 2 and 3, 6), at class 0 and at the last class, and a three-way tie across lanes and column blocks"""
    out = []
    for cands in ([(0, 1), (3, 6), (8, 9)], [(1, 2), (0, nc - 1)], [(nc - 2, nc - 1), (2, 5, 12)]):
        groups, used = [], set()
        for grp in cands:
            if len(set(grp)) == len(grp) and max(grp) < nc and min(grp) >= 0 and not used & set(grp):
                groups.append(grp)
                used |= set(grp)
        if groups and groups not in out:
            out.append(groups)
    return out


def _head_fail(what, bad, got=None, want=None):
    idx = bad.nonzero()
    v = int(idx[0][0])
    s = f'{what}: {idx.shape[0]} mismatches; first at voxel {v} (128-voxel tile {v // 128}, row {v % 128})'
    if idx.shape[1] > 1:
        c = int(idx[0][1])
        s += f', column {c}'
        if got is not None:
            s += f'; got {got[v, c].item()!r} want {want[v, c].item()!r}'
    elif got is not None:
        s += f'; got {got[v].item()!r} want {want[v].item()!r}'
    return s


def check_argmax(outs, tag):
    lg, u8, i64 = outs['occ'], outs['u8'], outs['i64']
    assert torch.equal(u8.long(), i64), tag + ': cls_u8 != cls_i64'
    first = torch.argmax(lg, dim=1)                                     # the first maximum
    bad = i64 != first
    if bool(bad.any()):
        raise AssertionError(_head_fail(tag + ': cls is not the first argmax of the kernel logits', bad, i64, first))


def check_heads():
    sms = _sms()
    worst = {}
    nv_small = [1, 127, 129, 1000, 128 * (sms // 3) + 77]
    for nc in CLASSES:
        for cfg, precision, tc in CONFIGS:
            dt = _DT[precision]
            hp = expected_route(precision, tc, nc)['head'][0]
            name = f'{cfg} {nc} classes [{HEAD_NAME[hp]}]'
            for nvox in nv_small + [640000]:
                g = torch.Generator().manual_seed(nc * 1000 + nvox % 997)
                gd = torch.Generator(device=DEV).manual_seed(nc * 1000 + nvox % 991)
                # real operands: the ReLU outputs of the last conv layer, stored
                vox = (torch.randn(nvox, OD, device=DEV, generator=gd).clamp_min(0) * 2).to(dt)
                hw = head_weights(g, nc, 'real')
                outs, path, n = head(precision, tc, nc, vox, hw, tag=name)
                assert (path, n) == (hp, 1), (name, path, n)
                logits, flow, el, ef = head_ref(vox, hw, path)
                for key, got, want, bound in (('logits', outs['occ'], logits, el), ('flow', outs['flow'], flow, ef)):
                    err = (got.double() - want).abs()
                    r = (err / bound).max().item()
                    worst[(HEAD_NAME[hp], cfg, key)] = max(worst.get((HEAD_NAME[hp], cfg, key), 0.0), r)
                    bad = ~(err <= bound)
                    if bool(bad.any()):
                        raise AssertionError(_head_fail(f'fp64 {name} nvox {nvox} {key} (got = error, want = bound)', bad,
                                                        err, bound))
                check_argmax(outs, f'{name} nvox {nvox}')
                if nc > 1:                                              # the fp64 argmax where the top-2 gap is resolvable
                    top = torch.topk(logits, 2, dim=1)
                    sure = (top.values[:, 0] - top.values[:, 1]) > 2 * el.max(dim=1).values
                    bad = sure & (outs['i64'] != top.indices[:, 0])
                    assert sure.float().mean().item() > 0.5, name
                    if bool(bad.any()):
                        raise AssertionError(_head_fail(f'{name}: cls differs from the fp64 argmax', bad, outs['i64'],
                                                        top.indices[:, 0]))
                del vox, outs, logits, flow, el, ef
                # exact operands, with and without ties
                vox = torch.randint(0, 4, (min(nvox, 20000), OD), device=DEV, generator=gd).float().to(dt)
                for ties in [()] + tie_sets(nc):
                    hw = head_weights(g, nc, 'exact', ties=ties)
                    tag = f'exact {name} nvox {vox.shape[0]} ties {ties}'
                    outs, _, _ = head(precision, tc, nc, vox, hw, tag=tag)
                    logits, flow, _, _ = head_ref(vox, hw, path, exact=True)
                    for key, got, want in (('logits', outs['occ'], logits), ('flow', outs['flow'], flow)):
                        bad = _bits(got) != _bits(want.float())
                        if bool(bad.any()):
                            raise AssertionError(_head_fail(f'{tag} {key}', bad, got, want.float()))
                    check_argmax(outs, tag)
                    first = torch.argmax(logits, dim=1)                 # exact logits: torch's first maximum in fp64
                    bad = outs['i64'] != first
                    if bool(bad.any()):
                        raise AssertionError(_head_fail(f'{tag}: tie not resolved to the first class', bad, outs['i64'], first))
                    if ties:                                            # every voxel's maximum is a tie, won by its first class
                        assert set(first.unique().tolist()) <= {grp[0] for grp in ties}, tag
            # output subsets: every NULL / non-NULL combination is bit-identical to the all-outputs call
            gd = torch.Generator(device=DEV).manual_seed(7 + nc)
            vox = (torch.randn(1000, OD, device=DEV, generator=gd).clamp_min(0)).to(dt)
            hw = head_weights(torch.Generator().manual_seed(8 + nc), nc, 'real', ties=(tie_sets(nc) or [()])[0])
            full, _, _ = head(precision, tc, nc, vox, hw, tag=name + ' all outputs')
            for mask in range(16):
                want = tuple(k for i, k in enumerate(OUTS) if mask >> i & 1)
                sub, _, _ = head(precision, tc, nc, vox, hw, want=want, tag=f'{name} outputs {want}')
                for k in want:
                    assert torch.equal(_bits(sub[k]), _bits(full[k])), f'{name}: output {k} of subset {want} differs'
        print(f'heads {nc} classes: fp64 bound, exact operands, ties and output subsets hold on every route')
    print('heads largest err/bound: ' + ', '.join(f'{h} / {c} / {k} {v:.3f}' for (h, c, k), v in sorted(worst.items())))


# ---- the GPU tests
@pytest.mark.gpu
def test_route_table_and_launch_counts_match_the_engine():
    _child('check_route_table')


@pytest.mark.gpu
def test_voxel_lift_bit_exact_on_non_square_grids():
    _child('check_lift')


@pytest.mark.gpu
def test_conv3d_bit_exact_on_integer_operands_every_route():
    _child('check_conv_exact')


@pytest.mark.gpu
def test_conv3d_batchnorm_fold_matches_the_oracle_mirror_bit_for_bit():
    _child('check_fold_pinned')


@pytest.mark.gpu
def test_conv3d_matches_fp64_at_production_size_every_route():
    _child('check_conv_fp64')


@pytest.mark.gpu
def test_heads_match_fp64_exact_operands_ties_and_output_subsets():
    _child('check_heads')
