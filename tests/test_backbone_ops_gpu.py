"""Operator tests of the image backbone's convolutions (conv2d_tc.cu, im2col + gemm_tc / gemm_simt) and its two other layer
kernels (max-pool, top-down upsample-add in backbone_kernels.cu), through the C-ABI entries `occb200_backbone_conv`,
`_maxpool` and `_upsample_add`, which run the code the backbone runs (the convolution entry builds its weights with the
backbone's upload and routes through its conv() / residual step).

(a) Route table: every distinct convolution of ResNet-50 + FPN at the production size (six 928 x 1600 images) must take the
    expected path in each configuration (fp32; bf16 on CUDA cores; bf16 on tensor cores), with the expected number of
    launches; on the tensor cores nothing may fall back to the CUDA-core GEMM.
(b) Bit-exact on integer operands: inputs, weights, biases and residuals are integers in [-3, 3], so every product and
    partial sum is an integer below 2^24, exact in fp32 in any summation order.  The output must then equal, bit for bit,
    the route's roundings applied to the exact sum S (fp64): act(S + b) stored; a fused residual relu(S + b + r) stored
    once; a residual applied by add_relu relu(stored(S + b) + r) stored.  One-hot weights (one tap x one input channel per
    output channel) make the output a shifted copy of the input, so a failure names the tap.
(c) Real-valued operands against fp64 (F.conv2d in float64 on the GPU on the same stored operands), per element:
        |out - F64| <= e,  e = K u S + u (S + |b|) [+ u T with a residual]                      (u = 2^-23, K = k*k*cin,
                                                                                                  S = conv(|x|, |w|),
                                                                                                  T = S + |b| + |r|)
    the accumulation bound of the GEMM tests plus the fp32 bias / residual adds; for a 16-bit output add one bf16 rounding,
    e += 2^-8 (|F64| + e), and for a residual applied after storing the convolution first e += 2^-8 (|S + b| + e) + u T.
(d) Max-pool 3x3 / 2 / 1 and nearest upsample-add against torch, bit-exact (the add in fp32, then stored).
Every output is surrounded by guard elements pre-filled with a NaN bit pattern, which must survive the launch.  A mismatch
names the case, the first bad element (n, y, x, co), its 16 x 8 tile and its 64-column block.

GPU cases run in a child process per test function, so that a device fault cannot poison this session.  Argument
rejections and the nearest-index mirror need no GPU and run in the CPU suite.

Not reached by the backbone, hence not tested: im2col_nhwc_any_kernel and the VEC = 1 im2col (C % 8 != 0 together with a
staged span over 1024 elements, or more than 65535 images or output rows).
"""
import ctypes
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
GUARD = 4096                        # guard elements before and after every output
U23 = 2.0 ** -23
U8 = 2.0 ** -8

IMPLICIT_TC, IM2COL_TC, DIRECT_TC, IM2COL_SIMT, DIRECT_SIMT = 1, 2, 3, 4, 5
PATH_NAME = {1: 'implicit-GEMM tensor cores', 2: 'im2col + tensor-core GEMM', 3: 'tensor-core GEMM',
             4: 'im2col + CUDA-core GEMM', 5: 'CUDA-core GEMM'}
CONFIGS = [('fp32', 0, 0), ('bf16 CUDA cores', 1, 0), ('bf16 tensor cores', 1, 1)]


def out_size(n, k, s):
    return (n + 2 * ((k - 1) // 2) - k) // s + 1


# ------------------------------------------------------------------------------------------------ (a) the route table
def route_table(N=6, H=928, W=1600):
    """(name, N, H, W, cin, cout, k, stride, residual, tensor-core path, CUDA-core path) of every distinct convolution of the
    backbone at image size H x W, in forward order; H, W is each convolution's INPUT size."""
    h, w = out_size(H, 7, 2), out_size(W, 7, 2)
    rows = [('stem', N, H, W, 3, 64, 7, 2, False, IM2COL_TC, IM2COL_SIMT)]
    h, w = out_size(h, 3, 2), out_size(w, 3, 2)
    cin = 64
    for s, planes in enumerate((64, 128, 256, 512)):
        st = 1 if s == 0 else 2
        ho, wo = out_size(h, 3, st), out_size(w, 3, st)
        L = f'layer{s + 1}'
        rows += [(f'{L}.0.conv1', N, h, w, cin, planes, 1, 1, False, DIRECT_TC, DIRECT_SIMT),
                 (f'{L}.0.conv2', N, h, w, planes, planes, 3, st, False,
                  IMPLICIT_TC if st == 1 else IM2COL_TC, IM2COL_SIMT),
                 (f'{L}.0.downsample', N, h, w, cin, 4 * planes, 1, st, False,
                  DIRECT_TC if st == 1 else IM2COL_TC, DIRECT_SIMT if st == 1 else IM2COL_SIMT),
                 (f'{L}.conv3', N, ho, wo, planes, 4 * planes, 1, 1, True, IMPLICIT_TC, DIRECT_SIMT),
                 (f'{L}.1.conv1', N, ho, wo, 4 * planes, planes, 1, 1, False, DIRECT_TC, DIRECT_SIMT)]
        if st == 2:
            rows.append((f'{L}.1.conv2', N, ho, wo, planes, planes, 3, 1, False, IMPLICIT_TC, IM2COL_SIMT))
        h, w, cin = ho, wo, 4 * planes
        if s >= 1:
            rows.append((f'fpn.lateral{s - 1}', N, h, w, cin, 256, 1, 1, False, DIRECT_TC, DIRECT_SIMT))
            rows.append((f'fpn.output{s - 1}', N, h, w, 256, 256, 3, 1, False, IMPLICIT_TC, IM2COL_SIMT))
    rows.append(('fpn.extra', N, h, w, 256, 256, 3, 2, False, IM2COL_TC, IM2COL_SIMT))
    return rows


def expected_route(row, precision, tc):
    """(path, launches, residual fused) the entry must report for a route-table row"""
    path = row[9] if tc else row[10]
    launches = 2 if path in (IM2COL_TC, IM2COL_SIMT) else 1
    fused = bool(row[8]) and path == IMPLICIT_TC
    return path, launches + (1 if row[8] and not fused else 0), fused


def test_route_table_lists_every_distinct_convolution():
    rows = route_table()
    assert len(rows) == 31 and len({r[0] for r in rows}) == 31
    assert len({r[1:9] for r in rows}) == 28              # fpn.lateral0 / 1 and fpn.output1 share shapes with layer 3
    # output sizes of the chain: 464 x 800 stem, 232 x 400 layer 1, then 116 x 200, 58 x 100, 29 x 50, extra 15 x 25
    assert [r[2:4] for r in rows if r[0].startswith('fpn.lateral')] == [(116, 200), (58, 100), (29, 50)]
    assert rows[-1][2:4] == (29, 50)
    # K of the explicit tensor-core GEMMs: the stem's 147 (padded to 192) and the strided 3x3 ones
    assert sorted({r[6] * r[6] * r[4] for r in rows if r[9] == IM2COL_TC}) == [147, 256, 512, 1024, 1152, 2304, 4608]


# ------------------------------------------------------------------------------------------------ (d) nearest index (CPU)
def level_pairs(lo=64, hi=1600, step=8):
    """the (coarse, fine) sizes of the FPN's two top-down adds, per dimension, for every image size lo..hi"""
    pairs = set()
    for n in range(lo, hi + 1, step):
        s = out_size(out_size(n, 7, 2), 3, 2)
        l0 = out_size(s, 3, 2); l1 = out_size(l0, 3, 2); l2 = out_size(l1, 3, 2)
        pairs |= {(l1, l0), (l2, l1)}
    return sorted(pairs)


def kernel_nearest(cin, cout):
    """upsample_add_nhwc_kernel's source index: min(floor(dst * ((float)in / (float)out)), in - 1) in fp32"""
    sc = np.float32(cin) / np.float32(cout)
    return np.minimum(np.floor(np.arange(cout, dtype=np.float32) * sc).astype(np.int64), cin - 1)


def torch_nearest(cin, cout):
    x = torch.arange(cin, dtype=torch.float32).view(1, 1, cin, 1)
    return F.interpolate(x, size=(cout, 1), mode='nearest').view(-1).long().numpy()


def float_rule_pairs(limit=64):
    """small (in, out) pairs where the float-scale rule and exact division floor(dst * in / out) pick different sources"""
    out = []
    for o in range(2, limit):
        for i in range(1, limit):
            exact = np.minimum(np.arange(o) * i // o, i - 1)
            if not np.array_equal(kernel_nearest(i, o), exact):
                out.append((i, o))
    return out


def test_upsample_nearest_index_matches_torch_on_every_level_pair():
    pairs = level_pairs()
    assert (15, 29) in pairs and (8, 15) in pairs and len(pairs) > 100
    for cin, cout in pairs + float_rule_pairs():
        assert np.array_equal(kernel_nearest(cin, cout), torch_nearest(cin, cout)), (cin, cout)


# ------------------------------------------------------------------------------------------------ argument rejection (CPU)
_CONV = dict(precision=1, tc=1, x=1, N=1, H=8, W=16, cin=64, w=1, bias=None, res=None, cout=64, k=3, stride=1, pad=1, act=0,
             out=1, path=1, launches=1, fused=1)
_CONV_ORDER = ['precision', 'tc', 'x', 'N', 'H', 'W', 'cin', 'w', 'bias', 'res', 'cout', 'k', 'stride', 'pad', 'act', 'out',
               'path', 'launches', 'fused']
_CONV_PTRS = {'x', 'res', 'out'}            # device pointers; w, bias: host fp32; path / launches / fused: host int
_REJECT = [
    ('conv', dict(x=None), 'null'), ('conv', dict(w=None), 'null'), ('conv', dict(out=None), 'null'),
    ('conv', dict(path=None), 'null'), ('conv', dict(launches=None), 'null'), ('conv', dict(fused=None), 'null'),
    ('conv', dict(precision=2), 'precision'), ('conv', dict(precision=0, tc=1), 'use_tensor_cores'),
    ('conv', dict(N=0), 'positive'), ('conv', dict(H=-1), 'positive'), ('conv', dict(W=0), 'positive'),
    ('conv', dict(cin=0), 'positive'), ('conv', dict(cout=0), 'positive'),
    ('conv', dict(cin=12), 'cin'), ('conv', dict(cout=60), 'cout'),
    ('conv', dict(k=5, pad=2), 'k must'), ('conv', dict(stride=3), 'stride'), ('conv', dict(pad=0), 'pad'),
    ('conv', dict(k=1, pad=1), 'pad'), ('conv', dict(act=2), 'act'), ('conv', dict(act=-1), 'act'),
    ('conv', dict(res=1, stride=2, act=1), 'residual'), ('conv', dict(res=1, act=0), 'residual'),
    ('maxpool', dict(x=None), 'null'), ('maxpool', dict(out=None), 'null'), ('maxpool', dict(C=12), 'shape'),
    ('maxpool', dict(H=0), 'shape'), ('maxpool', dict(precision=3), 'precision'),
    ('upsample_add', dict(fine=None), 'null'), ('upsample_add', dict(coarse=None), 'null'),
    ('upsample_add', dict(Hc=0), 'shape'), ('upsample_add', dict(C=4), 'shape'), ('upsample_add', dict(precision=-1), 'precision'),
]
_POOL = dict(precision=1, x=1, N=1, H=8, W=8, C=64, out=1)
_UP = dict(precision=1, fine=1, coarse=1, N=1, Hf=8, Wf=8, Hc=4, Wc=4, C=64)


@pytest.mark.parametrize('case', range(len(_REJECT)))
def test_entry_point_rejects_bad_arguments_before_any_cuda_call(case, lib_built):
    """Return code 1 (an argument check, not 2, a CUDA error) and a message.  Device pointers are a real buffer when a GPU is
    present, a dummy otherwise (a CUDA call would then fail with 2)."""
    from occnet_b200 import _lib
    lib = _lib.load()
    name, over, msg = _REJECT[case]
    buf = torch.zeros(1 << 20, device='cuda') if torch.cuda.is_available() else None
    dev = ctypes.c_void_p(buf.data_ptr()) if buf is not None else ctypes.c_void_p(1 << 12)
    if name == 'conv':
        a = dict(_CONV, **over)
        host_w = np.ones(a['cout'] * a['k'] * a['k'] * max(a['cin'], 1) + 64, np.float32)
        ints = [ctypes.c_int() for _ in range(3)]
        call = []
        for key in _CONV_ORDER:
            v = a[key]
            if key in _CONV_PTRS:
                call.append(dev if v else None)
            elif key in ('w', 'bias'):
                call.append(ctypes.c_void_p(host_w.ctypes.data) if v else None)
            elif key in ('path', 'launches', 'fused'):
                call.append(ctypes.byref(ints[('path', 'launches', 'fused').index(key)]) if v else None)
            else:
                call.append(v)
        rc = lib.occb200_backbone_conv(*call, None)
    elif name == 'maxpool':
        a = dict(_POOL, **over)
        rc = lib.occb200_backbone_maxpool(a['precision'], dev if a['x'] else None, a['N'], a['H'], a['W'], a['C'],
                                          dev if a['out'] else None, None)
    else:
        a = dict(_UP, **over)
        rc = lib.occb200_backbone_upsample_add(a['precision'], dev if a['fine'] else None, dev if a['coarse'] else None, a['N'],
                                               a['Hf'], a['Wf'], a['Hc'], a['Wc'], a['C'], None)
    err = lib.occb200_last_error().decode()
    assert rc == 1, (name, over, rc, err)
    assert msg in err, (name, over, err)


# ------------------------------------------------------------------------------------------------ GPU: child processes
def _run_isolated(code, timeout=1200):
    r = subprocess.run([sys.executable, '-c', 'import sys; sys.path.insert(0, "tests"); ' + code], cwd=ROOT, capture_output=True,
                       text=True, timeout=timeout)
    print(r.stdout[-20000:])
    assert r.returncode == 0, f'child failed ({r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'
    assert 'OK' in r.stdout
    return r.stdout


def _child(fn):
    return _run_isolated(f'import test_backbone_ops_gpu as t; t.{fn}(); print("OK")')


DEV = 'cuda:0'
_DT = {0: torch.float32, 1: torch.bfloat16}


def _lib():
    from occnet_b200 import _lib as L
    return L, L.load()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Out:
    """an NHWC output [N, H, W, C] with GUARD guard elements on each side, all pre-filled with NaN bits"""

    def __init__(self, shape, dtype, init=None):
        self.shape, self.dtype = tuple(shape), dtype
        self.n = int(np.prod(self.shape))
        it = torch.int32 if dtype == torch.float32 else torch.int16
        self.bits = torch.full((self.n + 2 * GUARD,), NAN32 if it == torch.int32 else NAN16, dtype=it, device=DEV)
        self.buf = self.bits.view(dtype)
        if init is not None:
            self.value().copy_(init)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + GUARD * self.buf.element_size())

    def value(self):
        return self.buf[GUARD:GUARD + self.n].view(self.shape)

    def check_guards(self, what):
        fill = NAN32 if self.bits.dtype == torch.int32 else NAN16
        for name, p in (('leading guard', self.bits[:GUARD]), ('trailing guard', self.bits[GUARD + self.n:])):
            bad = (p != fill).nonzero()
            assert bad.numel() == 0, f'{what}: {bad.numel()} elements of the {name} were written (first at {int(bad[0])})'


def _where(bad, what, got=None, want=None, extra=None):
    """AssertionError text naming the first bad element (n, y, x, co), its 16 x 8 tile and its 64-column block"""
    idx = bad.nonzero()
    n, y, x, c = (int(v) for v in idx[0])
    s = (f'{what}: {idx.shape[0]} mismatches; first at (n, y, x, co) = ({n}, {y}, {x}, {c}): 16x8 tile (ty {y // 8}, '
         f'tx {x // 16}), 64-column block {c // 64}; bad 64-column blocks {sorted(set((idx[:, 3] // 64).tolist()))[:12]}')
    if got is not None:
        s += f'; got {got[n, y, x, c].item()!r} want {want[n, y, x, c].item()!r}'
    if extra is not None:
        s += extra(n, y, x, c)
    return s


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def conv(precision, tc, x, w, bias, residual, k, stride, act, expect=None, tag=''):
    """one occb200_backbone_conv into a guarded output: x NHWC device (storage type), w fp32 [cout, k, k, cin] (tap-major),
    bias fp32 [cout] or None, residual NHWC or None.  Returns (out, path, launches, fused)."""
    L, lib = _lib()
    N, H, W, cin = x.shape
    cout = w.shape[0]
    Ho, Wo = out_size(H, k, stride), out_size(W, k, stride)
    o = Out((N, Ho, Wo, cout), _DT[precision])
    wh = np.ascontiguousarray(w.reshape(cout, -1).float().cpu().numpy())
    bh = None if bias is None else np.ascontiguousarray(bias.float().cpu().numpy())
    path, launches, fused = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    L.check(lib.occb200_backbone_conv(precision, tc, _p(x), N, H, W, cin, ctypes.c_void_p(wh.ctypes.data),
                                      None if bh is None else ctypes.c_void_p(bh.ctypes.data), _p(residual), cout, k, stride,
                                      (k - 1) // 2, act, o.ptr(), ctypes.byref(path), ctypes.byref(launches),
                                      ctypes.byref(fused), L.stream_ptr()))
    o.check_guards(tag)
    got = (path.value, launches.value, bool(fused.value))
    if expect is not None:
        assert got == expect, (f'{tag}: path {PATH_NAME.get(got[0], got[0])}, {got[1]} launches, residual fused {got[2]}; '
                               f'expected {PATH_NAME[expect[0]]}, {expect[1]} launches, fused {expect[2]}')
    return o.value(), got


def conv64(x, w, bias, k, stride):
    """fp64 convolution of NHWC x with tap-major w [cout, k, k, cin] (+ bias), NHWC out"""
    y = F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None if bias is None else bias.double(),
                 stride=stride, padding=(k - 1) // 2)
    return y.permute(0, 2, 3, 1)


def stored(v, precision):
    """v (fp64, exactly representable in fp32) stored in the storage type, back as fp64"""
    return v.float().to(_DT[precision]).double()


def exact_expected(precision, fused, x, w, bias, residual, k, stride, act):
    S = conv64(x, w, bias, k, stride)
    if residual is None:
        return stored(S.clamp_min(0) if act else S, precision)
    r = residual.double()
    if fused:
        return stored((S + r).clamp_min(0), precision)
    return stored((stored(S, precision) + r).clamp_min(0), precision)


def _ints(shape, g, lo=-3, hi=3):
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float()


def check_exact(precision, tc, N, H, W, cin, cout, k, stride, bias, res, act, seed, expect=None, onehot=False, neg=False,
                tag=''):
    g = torch.Generator(device=DEV).manual_seed(seed)
    dt = _DT[precision]
    x = _ints((N, H, W, cin), g).to(dt)
    Ho, Wo = out_size(H, k, stride), out_size(W, k, stride)
    taps = None
    if onehot:
        taps = (torch.randint(0, k * k, (cout,), generator=g, device=DEV), torch.randint(0, cin, (cout,), generator=g, device=DEV))
        w = torch.zeros(cout, k * k, cin, device=DEV)
        w[torch.arange(cout, device=DEV), taps[0], taps[1]] = 1.0
        w = w.view(cout, k, k, cin)
    else:
        w = _ints((cout, k, k, cin), g)
    b = _ints((cout,), g) if bias else None
    r = None
    if res:
        r = _ints((N, Ho, Wo, cout), g, -3 - (40 if neg else 0), 3).to(dt)     # neg: sums driven below zero, ReLU bites
    out, (path, _, fused) = conv(precision, tc, x, w, b, r, k, stride, act if r is None else 1, expect, tag)
    want = exact_expected(precision, fused, x, w, b, r, k, stride, act if r is None else 1)
    bad = _bits(out) != _bits(want.float().to(dt))
    if bool(bad.any()):
        extra = None
        if taps is not None:
            extra = lambda n, y, xx, c: f'; one-hot weight of co {c}: tap (ky, kx) = {divmod(int(taps[0][c]), k)}, ci {int(taps[1][c])}'
        raise AssertionError(_where(bad, f'{tag} [{PATH_NAME[path]}]', out, want, extra))
    return path


# ---- (a) + (b): the route table at production size, and bit-exact on reduced shapes
def check_route_table():
    for row in route_table():
        name, N, H, W, cin, cout, k, st, res, _, _ = row
        for cfg, precision, tc in CONFIGS:
            g = torch.Generator(device=DEV).manual_seed(1)
            x = _ints((N, H, W, cin), g).to(_DT[precision])
            w = torch.zeros(cout, k, k, cin, device=DEV)
            r = torch.zeros(N, out_size(H, k, st), out_size(W, k, st), cout, device=DEV).to(_DT[precision]) if res else None
            conv(precision, tc, x, w, None, r, k, st, 1, expected_route(row, precision, tc), f'route {name} {cfg} {N}x{H}x{W}')
            del x, r
        print(f'route {name}: fp32 / bf16 CUDA cores {PATH_NAME[row[10]]}, tensor cores {PATH_NAME[row[9]]}')


def check_exact_route_shapes():
    for i, row in enumerate(route_table(N=2, H=232, W=400)):
        name, _, H, W, cin, cout, k, st, res, _, _ = row
        H, W = min(H, 19), min(W, 37)
        for cfg, precision, tc in CONFIGS:
            check_exact(precision, tc, 2, H, W, cin, cout, k, st, True, res, 1, 1000 + i, expect=expected_route(row, precision, tc),
                        tag=f'exact {name} {cfg} 2x{H}x{W}')
            check_exact(precision, tc, 2, H, W, cin, cout, k, st, True, res, 1, 2000 + i, onehot=True,
                        tag=f'one-hot {name} {cfg} 2x{H}x{W}')
        print(f'exact {name} (2x{H}x{W}, {cin}->{cout}, k{k} s{st}{" + residual" if res else ""}): bit-exact in every configuration')


def conv2d_tc_edges():
    """(N, H, W, cin, cout, k, bias, residual, act, negative residual) for the implicit-GEMM kernel"""
    cases = [(1, h, w, 64, 64, 3, True, False, 1, False) for h in (1, 7, 8, 9) for w in (1, 15, 16, 17, 33)]
    cases += [(n, 9, 17, 64, 128, 3, True, False, 0, False) for n in (1, 2, 7)]
    cases += [(2, 8, 17, 64 * c, 64, 3, True, False, 1, False) for c in (1, 2, 3, 8, 32)]
    # BN = 64 (n_tiles 3, 5, 133 > SM count), 128 (3, 5), 256 (3, 5)
    cases += [(1, 9, 17, 64, co, k, True, k == 1, 1, False) for co in (192, 320, 384, 640, 768, 1280) for k in (3, 1)]
    cases += [(1, 8, 16, 64, 64 * 133, 3, True, False, 1, False), (1, 8, 16, 64, 64 * 133, 1, True, True, 1, True)]
    # m-tiles: fewer than the SMs (5), and a count that no per_n divides evenly (7 x 4 x 5 = 140 > 132)
    cases += [(1, 8, 80, 64, 64, 3, True, False, 1, False), (7, 32, 80, 64, 64, 3, False, False, 1, False),
              (7, 32, 80, 128, 256, 1, False, True, 1, True)]
    # bias / residual / ReLU combinations, residuals that drive the sum negative
    for bias in (False, True):
        cases += [(2, 9, 33, 128, 256, 3, bias, False, act, False) for act in (0, 1)]
        cases += [(2, 9, 33, 128, 256, 1, bias, True, 1, neg) for neg in (False, True)]
        cases += [(2, 9, 33, 128, 256, 3, bias, True, 1, True)]
    return cases


def check_exact_conv2d_tc_edges():
    for i, (N, H, W, cin, cout, k, bias, res, act, neg) in enumerate(conv2d_tc_edges()):
        tag = f'conv2d_tc N={N} H={H} W={W} cin={cin} cout={cout} k={k} bias={bias} res={res} relu={act} neg={neg}'
        expect = (IMPLICIT_TC, 1, res)
        check_exact(1, 1, N, H, W, cin, cout, k, 1, bias, res, act, 3000 + i, expect=expect, neg=neg, tag=tag)
        check_exact(1, 1, N, H, W, cin, cout, k, 1, bias, res, act, 4000 + i, expect=expect, neg=neg, onehot=True,
                    tag='one-hot ' + tag)
    print(f'conv2d_tc edges: {len(conv2d_tc_edges())} cases bit-exact (integer and one-hot weights)')


# ---- (c) real-valued operands against fp64, production sizes
def fp64_bound(K, S, b, r, F64, P64, out16, fused):
    T = S + b.abs() + (0 if r is None else r.abs())
    e = K * U23 * S + U23 * (S + b.abs()) + (0 if r is None else U23 * T)
    if out16:
        if r is not None and not fused:
            e = e + U8 * (P64.abs() + e) + U23 * T
        e = e + U8 * (F64.abs() + e)
    return e * 1.001


def check_fp64():
    worst = {}
    for i, row in enumerate(route_table()):
        name, N, H, W, cin, cout, k, st, res, _, _ = row
        g = torch.Generator(device=DEV).manual_seed(5000 + i)
        # mixed magnitudes: per-channel scales 2^-4 .. 2^4; every operand a bf16 value, so the three configurations share them
        x = (torch.randn(N, H, W, cin, device=DEV, generator=g) *
             2.0 ** torch.randint(-4, 5, (cin,), device=DEV, generator=g)).bfloat16()
        w = (torch.randn(cout, k, k, cin, device=DEV, generator=g) * (2.0 / (k * k * cin)) ** 0.5 *
             2.0 ** torch.randint(-3, 4, (cout, 1, 1, 1), device=DEV, generator=g)).bfloat16().float()
        b = torch.randn(cout, device=DEV, generator=g)
        Ho, Wo = out_size(H, k, st), out_size(W, k, st)
        r = torch.randn(N, Ho, Wo, cout, device=DEV, generator=g).bfloat16() if res else None
        P64 = conv64(x, w, b, k, st)
        S = conv64(x.abs(), w.abs(), None, k, st)
        F64 = (P64 + r.double()).clamp_min(0) if res else P64
        for cfg, precision, tc in CONFIGS:
            xi = x.float() if precision == 0 else x
            ri = None if r is None else (r.float() if precision == 0 else r)
            out, (path, _, fused) = conv(precision, tc, xi, w, b, ri, k, st, 1 if res else 0,
                                         expected_route(row, precision, tc), f'fp64 {name} {cfg}')
            bound = fp64_bound(k * k * cin, S, b.double(), None if r is None else r.double(), F64, P64, precision == 1, fused)
            err = (out.double() - F64).abs()
            ratio = (err / bound).max().item()
            worst[cfg] = max(worst.get(cfg, 0.0), ratio)
            print(f'fp64 {name} {cfg} [{PATH_NAME[path]}] {N}x{H}x{W} {cin}->{cout} k{k} s{st}: max err/bound {ratio:.3f}')
            bad = ~(err <= bound)
            if bool(bad.any()):
                raise AssertionError(_where(bad, f'fp64 {name} {cfg} (got = error, want = bound)', err, bound))
            del out, err, bound
        del x, r, P64, S, F64
    print('fp64 largest err/bound per configuration: ' + ', '.join(f'{c} {v:.3f}' for c, v in worst.items()))


# ---- (d) max-pool and top-down add
def check_maxpool_upsample():
    L, lib = _lib()
    for precision, dt in _DT.items():
        for i, (N, H, W, C) in enumerate([(2, 1, 1, 64), (2, 7, 9, 64), (2, 8, 10, 64), (1, 2, 3, 8), (3, 33, 17, 72),
                                          (6, 464, 800, 64)]):
            g = torch.Generator(device=DEV).manual_seed(6000 + i)
            x = torch.randn(N, H, W, C, device=DEV, generator=g).to(dt)
            Ho, Wo = out_size(H, 3, 2), out_size(W, 3, 2)
            o = Out((N, Ho, Wo, C), dt)
            L.check(lib.occb200_backbone_maxpool(precision, _p(x), N, H, W, C, o.ptr(), L.stream_ptr()))
            tag = f'maxpool {dt} {N}x{H}x{W}x{C}'
            o.check_guards(tag)
            want = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).to(dt)
            bad = _bits(o.value()) != _bits(want)
            if bool(bad.any()):
                raise AssertionError(_where(bad, tag, o.value(), want))
        pairs = level_pairs()
        sub = sorted(set(pairs[::7] + [(15, 29), (8, 15), (4, 8), (25, 50)] + float_rule_pairs()[:8]))
        for i, ((hc, hf), (wc, wf)) in enumerate(zip(sub, sub[3:] + sub[:3])):
            N, C = 2, 256 if i % 3 else 64
            g = torch.Generator(device=DEV).manual_seed(7000 + i)
            fine = torch.randn(N, hf, wf, C, device=DEV, generator=g).to(dt)
            coarse = torch.randn(N, hc, wc, C, device=DEV, generator=g).to(dt)
            o = Out(fine.shape, dt, init=fine)
            L.check(lib.occb200_backbone_upsample_add(precision, o.ptr(), _p(coarse), N, hf, wf, hc, wc, C, L.stream_ptr()))
            tag = f'upsample_add {dt} {hc}x{wc} -> {hf}x{wf}'
            o.check_guards(tag)
            up = F.interpolate(coarse.float().permute(0, 3, 1, 2), size=(hf, wf), mode='nearest').permute(0, 2, 3, 1)
            want = (fine.float() + up).to(dt)
            bad = _bits(o.value()) != _bits(want)
            if bool(bad.any()):
                raise AssertionError(_where(bad, tag, o.value(), want))
        print(f'maxpool and upsample_add {dt}: bit-exact ({len(sub)} level pairs)')


# ---- the GPU tests
@pytest.mark.gpu
def test_route_table_paths_at_production_size():
    _child('check_route_table')


@pytest.mark.gpu
def test_route_table_shapes_bit_exact_on_integer_operands():
    _child('check_exact_route_shapes')


@pytest.mark.gpu
def test_conv2d_tc_edge_shapes_bit_exact_on_integer_operands():
    _child('check_exact_conv2d_tc_edges')


@pytest.mark.gpu
def test_convolutions_match_fp64_at_production_size():
    _child('check_fp64')


@pytest.mark.gpu
def test_maxpool_and_upsample_add_bit_exact_against_torch():
    _child('check_maxpool_upsample')
