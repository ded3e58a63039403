"""Operator tests of the encoder's unfused kernels (gemm_simt.cu; gemm_tc.cu on the routes the frame plan gives it;
elementwise.cu: layernorm256, pack_levels, pack_levels_nhwc, prepare_query, t32_convert) through the C-ABI entries
`occb200_encoder_dense`, `_layernorm`, `_pack`, `_prepare_query` and `occb200_t32_convert`.  The dense entry builds its weights
with the engine's own `upload_dense` and runs the engine's own `dense_gemm` on the plan make_frame_plan makes for (precision,
use_tensor_cores).  Routes: fp32 on CUDA cores; fp32 on tensor cores (gemm_tc_split3 on bf16 hi / lo splits); bf16 on CUDA
cores; bf16 on tensor cores (gemm_tc, fp16 sampling projections).  A shape the tensor-core GEMM does not take (N or K not a
multiple of 64, a split point K1 not a multiple of 64 on gemm_tc) runs on the CUDA cores in every configuration.

(a) Route table: the path and launch count of every dense layer a 200x200, 6-camera frame runs, in each configuration, and
    the CUDA-core fallback of N = 68 and K = 48.  For the three unfused configurations (fp32, fp32 tensor cores, bf16 CUDA
    cores) the launches of a small6 frame that asks for bev_embed only are
        1 (pack) + [split: 1 (the camera tokens' split)] + 1 (prepare_query)
        + L * (sum of the dense layers' launches - [split: 1] + 2 (gathers) + 3 (LayerNorms)) + [previous BEV: 1 (gather_rows)]
    (the split route's SCA value projection reads the tokens split once per frame: 1 launch, where the entry, which splits
    its operand itself, reports 2), with and without a previous BEV.
(b) Dense layers, bit-exact on integer operands, every route: operands, bias and residual integers in [-4, 4], weights
    integers with K <= 512, so every partial sum is exact in fp32 in any order and every hi / lo split has lo = 0.  The output
    must equal, bit for bit, relu(exact + b) + r rounded once to the output type (ReLU before the residual).  One-hot weights
    (output column n reads operand column perm(n), which alternates between the two sides of the [A | A2] split point, with
    weight +-2^j) name the k that went wrong; dense integer weights cover the accumulation.  M in {1, 127, 128, 129, 40000},
    N in {4, 60, 64, 68, 192, 256, 512, 768}, K in {16, 48, 256, 512}, K1 in {8, 16, K - 8, K / 2} and no split, bias and
    residual each NULL and present, ReLU on and off.
(c) Dense layers against fp64 at production shapes, every route, in the output type the frame uses.  Reference: fp64 on the
    stored operands; weights fp32 on the CUDA cores (also in bf16 storage: gemm_simt reads fp32 W), bf16 on the tensor cores,
    fp32 on the split route.  With S = sum_k |a_k w_k| and u = 2^-23, per element:
        CUDA cores     e = K u S + u (S + |b|)            an FMA chain from 0, then the bias add rounded once
        tensor cores   e = K u S + u (S + |b|)            the same (u covers the tensor cores' truncating accumulation)
        split          e = K u S (1 + 2^-7) + 2 u (S + |b|) + 2^-16 S    (the decoder's split bound: three passes, the
                                                          dropped lo.lo product and the bf16 rounding of the lo halves)
        residual       e += u (S + |b| + |r|)             the residual add rounded once
        16-bit output  e += 2^-8 (|F64| + e) (bf16) or 2^-11 (|F64| + e) (fp16)
    ReLU is 1-Lipschitz, so the bounds hold after it.  Every bound carries a factor 1.001.
(d) Standalone LayerNorm (layernorm256) against fp64, both precisions, rows in {1, 7, 8, 9, 33, 1600, 40000} (partial 8-row
    CTAs): rows whose mean is 0, 1, 4, 8, 16, 64 or 256 standard deviations, and constant rows on the 1/64 grid (the kinds of
    test_gemm_tc_gpu.ln_case), gamma in [0.5, 2]: |y_f32 - y64| <= 2e-4, the fused LayerNorm's bar; a constant row gives
    exactly beta; y_t = T(y_f32) and y_pos_t = T(y_f32 + pos) bit for bit (the add in fp32); all 8 NULL / non-NULL output
    subsets bit-identical to the all-outputs call.
(e) Packing, bit-exact: tokens = T((x + cams_embeds[cam]) + level_embeds[l]) in fp32, the kernels' order, for the three
    layouts (fp32 NCHW, bf16 NCHW, bf16 NHWC) in both storage types, cams_embeds NULL and present, 1, 6 and 8 cameras, levels
    that take every load branch (hw % 8 == 0; hw % 4 == 0 but not % 8; odd hw; hw in {1, 63, 64, 65}), up to eight levels,
    and the production levels 116x200, 58x100, 29x50 and 15x25 (1450 and 375 take the scalar tails).
(f) prepare_query and t32_convert, bit-exact: q_f32 (row-major and T32), q_t = T(q), q_pos_t = T(q + pos); t32_convert
    both ways for ncols in {32, 192, 256} against test_gemm_tc_gpu.t32_index; the pad rows of a T32 output stay untouched.
(g) Argument rejections, before any CUDA call (CPU suite).
Every output is surrounded by guard elements pre-filled with a NaN bit pattern, which must survive the launch.

GPU cases run in a child process per test function, so that a device fault cannot poison this session.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NAN16 = 0x7FA5                      # a NaN in both bf16 and fp16
NAN32 = 0x7FA5A5A5
GUARD = 4096
U23 = 2.0 ** -23

CUDA_CORES, TC, SPLIT = 0, 1, 2
PATH_NAME = {0: 'CUDA cores', 1: 'tensor cores', 2: 'split tensor cores'}
CONFIGS = [('fp32', 0, 0), ('fp32 tensor cores', 0, 1), ('bf16 CUDA cores', 1, 0), ('bf16 tensor cores', 1, 1)]
UNFUSED = CONFIGS[:3]
F32, BF16, F16 = 0, 1, 2
_DT = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}
STORAGE = {0: F32, 1: BF16}

NQ, NV, NCAM = 40000, 116 * 200 + 58 * 100 + 29 * 50 + 15 * 25, 6
PROD_LEVELS = [(116, 200), (58, 100), (29, 50), (15, 25)]


def dense_layers(precision, tc):
    """the dense layers of one encoder layer at 200x200 with 6 cameras: (name, M, N, K, K1 (0: no split), act, residual,
    out_dtype the frame asks for)"""
    st = STORAGE[precision]
    qproj = F16 if (precision, tc) == (1, 1) else F32
    return [('value_proj', NQ, 256, 256, 0, 0, False, st),
            ('TSA query projection [a | q+pos]', NQ, 192, 512, 256, 0, False, qproj),
            ('TSA output_proj', NQ, 256, 256, 0, 0, True, F32),
            ('SCA query projection', NQ, 768, 256, 0, 0, False, qproj),
            ('SCA value_proj', NCAM * NV, 256, 256, 0, 0, False, st),
            ('SCA output_proj', NQ, 256, 256, 0, 0, True, F32),
            ('FFN1', NQ, 512, 256, 0, 1, False, st),
            ('FFN2', NQ, 256, 512, 0, 0, True, F32)]


def expected_route(precision, tc, N, K, K1=0):
    """(path, launches) of make_frame_plan's route for a dense layer: the tensor-core GEMM where N and K (and a split point)
    are multiples of 64, otherwise the CUDA cores; the split route splits its operand first"""
    if tc and N % 64 == 0 and K % 64 == 0:
        if precision == 0:
            return SPLIT, 2
        if K1 % 64 == 0:
            return TC, 1
    return CUDA_CORES, 1


def frame_launches(split, layers, dense_sum, prev):
    """launches of an unfused frame that asks for bev_embed only (see the module docstring)"""
    return 1 + split + 1 + layers * (dense_sum - split + 2 + 3) + prev


def test_expected_routes_follow_the_tensor_core_gemm_shapes():
    """the table the GPU test holds the entry to: every production layer takes the configuration's tensor-core route, and
    the frame formula counts 2 launches per layer fewer than the entries on the split route (the tokens' split is shared)"""
    for _, precision, tc in CONFIGS:
        for name, M, N, K, K1, _, _, _ in dense_layers(precision, tc):
            want = {(0, 0): (CUDA_CORES, 1), (0, 1): (SPLIT, 2), (1, 0): (CUDA_CORES, 1), (1, 1): (TC, 1)}[(precision, tc)]
            assert expected_route(precision, tc, N, K, K1) == want, name
        assert expected_route(precision, tc, 68, 256) == (CUDA_CORES, 1)
        assert expected_route(precision, tc, 256, 48) == (CUDA_CORES, 1)
    assert expected_route(1, 1, 256, 512, 256) == (TC, 1) and expected_route(1, 1, 256, 512, 200) == (CUDA_CORES, 1)
    assert frame_launches(0, 2, 8, 0) == 1 + 1 + 2 * 13 and frame_launches(1, 2, 16, 1) == 1 + 1 + 1 + 2 * 20 + 1


# ------------------------------------------------------------------------------------------------ (g) rejections (CPU)
_DENSE = dict(precision=1, tc=1, A=1, A2=0, K1=0, w=1, bias=1, res=1, out=1, out_dtype=0, M=128, N=64, K=64, act=0, path=1,
              launches=1)
_LN = dict(precision=1, x=1, gamma=1, beta=1, pos=1, rows=8, y=1, yt=1, ypt=1)
_PACK = dict(precision=1, layout=0, feats=1, nl=2, hw=(4, 4, 2, 2), cams=6, ce=1, le=1, tokens=1)
_PQ = dict(precision=1, tiled=0, q=1, pos=1, n=256, qf=1, qt=1, qpt=1)
_T32 = dict(src=1, dst=1, rows=32, untile=0, ncols=256)
_REJECT = [
    ('dense', dict(A=None), 'null'), ('dense', dict(w=None), 'null'), ('dense', dict(out=None), 'null'),
    ('dense', dict(path=None), 'null'), ('dense', dict(launches=None), 'null'),
    ('dense', dict(precision=2), 'precision'), ('dense', dict(tc=2), 'use_tensor_cores'), ('dense', dict(act=2), 'act'),
    ('dense', dict(K=40), 'shape'), ('dense', dict(K=0), 'shape'), ('dense', dict(N=66), 'shape'), ('dense', dict(N=0), 'shape'),
    ('dense', dict(M=-1), 'shape'),
    ('dense', dict(A2=1, K1=12, K=64), 'split point'), ('dense', dict(A2=1, K1=0), 'split point'),
    ('dense', dict(A2=1, K1=64, K=64), 'split point'), ('dense', dict(A2=1, K1=72, K=64), 'split point'),
    ('dense', dict(A2=1, K1=-8), 'split point'), ('dense', dict(A2=0, K1=32), 'split point'),
    ('dense', dict(A='odd'), 'aligned'), ('dense', dict(A2='odd', K1=32), 'aligned'), ('dense', dict(res='odd'), 'aligned'),
    ('dense', dict(out='odd'), 'aligned'),
    ('dense', dict(out_dtype=3), 'out_dtype'), ('dense', dict(out_dtype=-1), 'out_dtype'),
    ('dense', dict(precision=0, out_dtype=1), 'out_dtype'),
    ('dense', dict(precision=0, tc=1, out_dtype=2), 'fp16'), ('dense', dict(precision=1, tc=0, out_dtype=2), 'fp16'),
    ('dense', dict(precision=0, tc=0, out_dtype=2), 'fp16'), ('dense', dict(N=68, out_dtype=2), 'fp16'),
    ('dense', dict(A2=1, K1=32, out_dtype=2), 'fp16'),
    ('ln', dict(x=None), 'null'), ('ln', dict(gamma=None), 'null'), ('ln', dict(beta=None), 'null'),
    ('ln', dict(precision=2), 'precision'), ('ln', dict(pos=None), 'pos'), ('ln', dict(rows=0), 'rows'),
    ('ln', dict(rows=-3), 'rows'), ('ln', dict(x='odd'), 'aligned'), ('ln', dict(yt='odd'), 'aligned'),
    ('ln', dict(ypt='odd'), 'aligned'), ('ln', dict(y='odd'), 'aligned'),
    ('pack', dict(feats=None), 'null'), ('pack', dict(hw=None), 'null'), ('pack', dict(le=None), 'null'),
    ('pack', dict(tokens=None), 'null'), ('pack', dict(precision=-1), 'precision'), ('pack', dict(layout=3), 'layout'),
    ('pack', dict(layout=4), 'layout'), ('pack', dict(layout=-1), 'layout'), ('pack', dict(nl=0), 'num_levels'),
    ('pack', dict(nl=9), 'num_levels'), ('pack', dict(cams=0), 'num_cams'), ('pack', dict(cams=9), 'num_cams'),
    ('pack', dict(hw=(4, 4, 0, 2)), 'level'), ('pack', dict(hw=(4, -1, 2, 2)), 'level'),
    ('pack', dict(hw=(4096, 4097, 2, 2)), 'level'), ('pack', dict(hw=(4096, 4096, 1, 1)), '2^24'),
    ('pack', dict(feats='null1'), 'null feature level'), ('pack', dict(feats='odd'), 'aligned'),
    ('pack', dict(ce='odd'), 'aligned'), ('pack', dict(tokens='odd'), 'aligned'),
    ('pq', dict(q=None), 'null'), ('pq', dict(pos=None), 'null'), ('pq', dict(precision=2), 'precision'),
    ('pq', dict(tiled=2), 'tiled'), ('pq', dict(n=0), 'multiple'), ('pq', dict(n=12), 'multiple'),
    ('pq', dict(n=-8), 'multiple'), ('pq', dict(tiled=1, n=264), 'multiple'), ('pq', dict(qf='odd'), 'aligned'),
    ('pq', dict(qpt='odd'), 'aligned'),
    ('t32', dict(src=None), 'null'), ('t32', dict(dst=None), 'null'), ('t32', dict(untile=2), 'untile'),
    ('t32', dict(rows=0), 'rows'), ('t32', dict(ncols=0), 'ncols'), ('t32', dict(ncols=48), 'ncols'),
    ('t32', dict(ncols=-32), 'ncols'), ('t32', dict(src='odd'), 'aligned'), ('t32', dict(dst='odd'), 'aligned'),
]


@pytest.mark.parametrize('case', range(len(_REJECT)))
def test_entry_point_rejects_bad_arguments_before_any_cuda_call(case, lib_built):
    """Return code 1 (an argument check, not 2, a CUDA error) and a message.  Device pointers are a real buffer when a GPU is
    present, a dummy otherwise (a CUDA call would then fail with 2)."""
    from occnet_b200 import _lib
    lib = _lib.load()
    name, over, msg = _REJECT[case]
    buf = torch.zeros(1 << 20, device='cuda') if torch.cuda.is_available() else None
    base = buf.data_ptr() if buf is not None else 1 << 12
    host = np.ones(1 << 16, np.float32)
    hp = ctypes.c_void_p(host.ctypes.data)

    def dev(v):
        return None if not v else ctypes.c_void_p(base + 4 if v == 'odd' else base)

    ints = [ctypes.c_int() for _ in range(2)]
    if name == 'dense':
        a = dict(_DENSE, **over)
        rc = lib.occb200_encoder_dense(a['precision'], a['tc'], dev(a['A']), dev(a['A2']), a['K1'], hp if a['w'] else None,
                                       hp if a['bias'] else None, dev(a['res']), dev(a['out']), a['out_dtype'], a['M'], a['N'],
                                       a['K'], a['act'], ctypes.byref(ints[0]) if a['path'] else None,
                                       ctypes.byref(ints[1]) if a['launches'] else None, None)
    elif name == 'ln':
        a = dict(_LN, **over)
        rc = lib.occb200_encoder_layernorm(a['precision'], dev(a['x']), dev(a['gamma']), dev(a['beta']), dev(a['pos']),
                                           a['rows'], dev(a['y']), dev(a['yt']), dev(a['ypt']), None)
    elif name == 'pack':
        a = dict(_PACK, **over)
        fv = a['feats']
        feats = None if fv is None else (ctypes.c_void_p * 8)(*[None if (fv == 'null1' and i == 1) else dev(fv if fv == 'odd' else 1)
                                                               for i in range(8)])
        hw = None if a['hw'] is None else (ctypes.c_int * 16)(*(list(a['hw']) + [1] * (16 - len(a['hw']))))
        rc = lib.occb200_encoder_pack(a['precision'], a['layout'], feats, a['nl'], hw, a['cams'], dev(a['ce']), dev(a['le']),
                                      dev(a['tokens']), None)
    elif name == 'pq':
        a = dict(_PQ, **over)
        rc = lib.occb200_encoder_prepare_query(a['precision'], a['tiled'], dev(a['q']), dev(a['pos']), a['n'], dev(a['qf']),
                                               dev(a['qt']), dev(a['qpt']), None)
    else:
        a = dict(_T32, **over)
        rc = lib.occb200_t32_convert(dev(a['src']), dev(a['dst']), a['rows'], a['untile'], a['ncols'], None)
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
    return _run_isolated(f'import test_encoder_ops_gpu as t; t.{fn}(); print("OK")')


DEV = 'cuda:0'


def _lib():
    from occnet_b200 import _lib as L
    return L, L.load()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _h(a):
    return ctypes.c_void_p(a.ctypes.data)


class Out:
    """an output of `shape` with GUARD guard elements on each side, all pre-filled with NaN bits"""

    def __init__(self, shape, dtype):
        self.shape, self.dtype = tuple(shape), dtype
        self.n = int(np.prod(self.shape))
        self.fill = NAN32 if dtype == torch.float32 else NAN16
        it = torch.int32 if dtype == torch.float32 else torch.int16
        self.bits = torch.full((self.n + 2 * GUARD,), self.fill, dtype=it, device=DEV)
        self.buf = self.bits.view(dtype)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + GUARD * self.buf.element_size())

    def value(self):
        return self.buf[GUARD:GUARD + self.n].view(self.shape)

    def body_bits(self):
        return self.bits[GUARD:GUARD + self.n]

    def untouched(self):
        return bool((self.bits == self.fill).all())

    def check_guards(self, what):
        for name, p in (('leading guard', self.bits[:GUARD]), ('trailing guard', self.bits[GUARD + self.n:])):
            bad = (p != self.fill).nonzero()
            assert bad.numel() == 0, f'{what}: {bad.numel()} elements of the {name} were written (first at {int(bad[0])})'


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _first_bad(bad, what, got=None, want=None, extra=None):
    """AssertionError text naming the first mismatch of a 2-D comparison: row, column, its 128-row tile and 64-column block"""
    idx = bad.nonzero()
    r, c = int(idx[0][0]), int(idx[0][1])
    s = (f'{what}: {idx.shape[0]} mismatches; first at row {r} (128-row tile {r // 128}), column {c} (64-column block '
         f'{c // 64}); bad rows {sorted(set(idx[:, 0].tolist()))[:8]}, bad columns {sorted(set(idx[:, 1].tolist()))[:12]}')
    if got is not None:
        s += f'; got {got[r, c].item()!r} want {want[r, c].item()!r}'
    if extra is not None:
        s += extra(r, c)
    return s


# ---- the entries
def dense(precision, tc, A, W, bias=None, residual=None, out_dtype=None, act=0, A2=None, K1=0, tag=''):
    """A (and A2) device, storage type; W fp32 [N, K] and bias fp32 [N] on the host (numpy); residual fp32 [M, N] device.
    -> (out [M, N], path, launches)"""
    L, lib = _lib()
    M = A.shape[0]
    K = A.shape[1] + (A2.shape[1] if A2 is not None else 0)
    N = W.shape[0]
    od = STORAGE[precision] if out_dtype is None else out_dtype
    o = Out((M, N), _DT[od])
    wh = np.ascontiguousarray(W, np.float32)
    bh = None if bias is None else np.ascontiguousarray(bias, np.float32)
    path, n = ctypes.c_int(), ctypes.c_int()
    L.check(lib.occb200_encoder_dense(precision, tc, _p(A), _p(A2), K1, _h(wh), None if bh is None else _h(bh), _p(residual),
                                      o.ptr(), od, M, N, K, act, ctypes.byref(path), ctypes.byref(n), L.stream_ptr()))
    o.check_guards(tag)
    return o.value(), path.value, n.value


# ---- (a) the route table
def check_route_table():
    from occnet_b200 import fixtures
    from occnet_b200.engine import OccEngine
    rows = []
    for cfg_name, precision, tc in CONFIGS:
        dt = _DT[precision]
        total = 0
        for name, M, N, K, K1, act, res, od in dense_layers(precision, tc) + [
                ('N = 68 (fallback)', 1000, 68, 256, 0, 0, False, STORAGE[precision]),
                ('K = 48 (fallback)', 1000, 256, 48, 0, 0, True, F32),
                ('K1 = 200 (fallback on gemm_tc)', 1000, 256, 512, 200, 0, False, F32)]:
            A = torch.zeros(M, K1 or K, device=DEV).to(dt)
            A2 = torch.zeros(M, K - K1, device=DEV).to(dt) if K1 else None
            R = torch.zeros(M, N, device=DEV) if res else None
            _, path, n = dense(precision, tc, A, np.zeros((N, K), np.float32), np.zeros(N, np.float32), R, od, act, A2, K1,
                               tag=f'route {cfg_name} {name}')
            want = expected_route(precision, tc, N, K, K1)
            assert (path, n) == want, (f'{cfg_name} {name} (N {N}, K {K}, K1 {K1}): {PATH_NAME[path]} x {n} launches, '
                                       f'expected {PATH_NAME[want[0]]} x {want[1]}')
            if 'fallback' not in name:
                total += n
            rows.append(f'{cfg_name:18s} {name:32s} M {M:6d} N {N:3d} K {K:3d}: {PATH_NAME[path]} x {n}')
            del A, A2, R
        if (precision, tc) == (1, 1):
            continue
        # an unfused frame: every launch but the dense layers' is a fixed count (the module docstring's formula)
        split = int(precision == 0 and tc == 1)
        cfg = fixtures.make_cfg('small6')
        eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2), precision='bf16' if precision else 'fp32',
                        use_tensor_cores=bool(tc), device=DEV)
        eng.set_cameras(fixtures.make_img_metas(cfg, bs=1))
        feats = [f[0].to(DEV) for f in fixtures.make_feats(cfg, bs=1, seed=3)]
        out = eng.forward(feats, want=('bev_embed',))
        n_self = eng.launches_per_frame
        eng.forward(feats, prev_bev=out['bev_embed'], want=('bev_embed',))
        n_prev = eng.launches_per_frame
        L = cfg['num_layers']
        want_self, want_prev = frame_launches(split, L, total, 0), frame_launches(split, L, total, 1)
        assert (n_self, n_prev) == (want_self, want_prev), (cfg_name, n_self, n_prev, want_self, want_prev, total)
        rows.append(f'{cfg_name:18s} frame ({L} layers, bev_embed only): {n_self} launches, {n_prev} with a previous BEV '
                    f'(dense layers {total} per layer)')
        del eng
    print('route table:\n  ' + '\n  '.join(rows))


# ---- (b) dense layers on integer operands
def perm_of(N, K, K1):
    """operand column of output column n: alternately just below and at / above the split point, moving outwards"""
    n = np.arange(N)
    return np.where(n % 2 == 0, K1 - 1 - n // 2, K1 + n // 2) % K


def exact_case(M, N, K, K1, onehot, seed):
    """integer operands: A [M, K] and R [M, N] on the device, W [N, K] and b [N] on the host, all fp64"""
    g = torch.Generator().manual_seed(seed)
    gd = torch.Generator(device=DEV).manual_seed(seed)
    A = torch.randint(-4, 5, (M, K), generator=gd, device=DEV).double()
    if onehot:
        perm = perm_of(N, K, K1 or K // 2)
        W = torch.zeros(N, K, dtype=torch.float64)
        mag = 2.0 ** torch.randint(0, 4, (N,), generator=g).double() * (torch.randint(0, 2, (N,), generator=g) * 2 - 1).double()
        W[torch.arange(N), torch.as_tensor(perm)] = mag
    else:
        perm = None
        W = torch.randint(-2, 3, (N, K), generator=g).double()
    b = torch.randint(-4, 5, (N,), generator=g).double()
    R = torch.randint(-4, 5, (M, N), generator=gd, device=DEV).double()
    return A, W, b, R, perm


def exact_shapes():
    """(M, N, K, K1, bias, residual, relu, one-hot, seed): every split point (and none) at the small M, one of them in turn
    at M = 40000; bias, residual, ReLU and the weight kind drawn at random per shape"""
    rng = np.random.default_rng(12345)
    out = []
    for N in (4, 60, 64, 68, 192, 256, 512, 768):
        for K in (16, 48, 256, 512):
            k1s = sorted({k for k in (8, 16, K - 8, K // 2) if 0 < k < K}) + [0]
            for M in (1, 127, 128, 129, 40000):
                for K1 in (k1s if M < 40000 else [k1s[len(out) % len(k1s)]]):
                    use_b, use_r, act, onehot = (int(v) for v in rng.integers(0, 2, 4))
                    out.append((M, N, K, K1, bool(use_b), bool(use_r), act, bool(onehot), len(out)))
    return out


def check_dense_exact():
    shapes = exact_shapes()
    seen = set()
    for M, N, K, K1, use_b, use_r, act, onehot, i in shapes:
        A, W, b, R, perm = exact_case(M, N, K, K1, onehot, 7000 + i)
        Rd = R.float() if use_r else None
        bh = b.float().numpy() if use_b else None
        exact = (A @ W.to(DEV).t()) + (b.to(DEV) if use_b else 0)
        if act:
            exact = exact.clamp_min(0)
        if use_r:
            exact = exact + R
        for cfg, precision, tc in CONFIGS:
            Ad = A.float().to(_DT[precision])
            A1, A2 = (Ad[:, :K1].contiguous(), Ad[:, K1:].contiguous()) if K1 else (Ad, None)
            route = expected_route(precision, tc, N, K, K1)
            ods = [STORAGE[precision], F32] if precision else [F32]
            if precision == 1 and route[0] == TC:
                ods.append(F16)
            for od in sorted(set(ods)):
                tag = (f'{"one-hot" if onehot else "integer"} {cfg} M {M} N {N} K {K} K1 {K1 or "-"} bias {use_b} residual '
                       f'{use_r} relu {act} -> {_DT[od]}')
                got, path, n = dense(precision, tc, A1, W.float().numpy(), bh, Rd, od, act, A2, K1, tag)
                assert (path, n) == route, (tag, path, n, route)
                seen.add((cfg, path))
                want = exact.float().to(_DT[od])
                bad = _bits(got) != _bits(want)
                if bool(bad.any()):
                    def extra(r, c, perm=perm, K1=K1, K=K):
                        if perm is None:
                            return ''
                        k = int(perm[c])
                        side = 'A' if (not K1 or k < K1) else f'A2 (column {k - K1})'
                        return f'; one-hot column {c} reads k = {k} of {side}'
                    raise AssertionError(_first_bad(bad, f'{tag} [{PATH_NAME[path]}]', got, want, extra))
    print(f'dense: {len(shapes)} shapes per configuration bit-exact on integer and one-hot operands, every output type; '
          f'routes exercised: {sorted(seen)}')


# ---- (c) dense layers against fp64
def dense_bound(path, K, S, b, r, F64, od):
    b = b.abs()
    if path == SPLIT:
        e = K * U23 * S * (1 + 2.0 ** -7) + 2 * U23 * (S + b) + 2.0 ** -16 * S
    else:
        e = K * U23 * S + U23 * (S + b)
    if r is not None:
        e = e + U23 * (S + b + r.abs())
    if od == BF16:
        e = e + 2.0 ** -8 * (F64.abs() + e)
    elif od == F16:
        e = e + 2.0 ** -11 * (F64.abs() + e)
    return e * 1.001


def check_dense_fp64():
    worst = {}
    for cfg, precision, tc in CONFIGS:
        dt = _DT[precision]
        for li, (name, M, N, K, K1, act, res, od) in enumerate(dense_layers(precision, tc)):
            g = torch.Generator(device=DEV).manual_seed(9000 + 10 * li + precision)
            gc = torch.Generator().manual_seed(9100 + 10 * li + precision)
            # mixed column magnitudes 2^-3 .. 2^3; FFN2 reads FFN1's ReLU outputs
            A = torch.randn(M, K, device=DEV, generator=g) * 2.0 ** torch.randint(-3, 4, (K,), device=DEV, generator=g)
            if name == 'FFN2':
                A = A.clamp_min(0)
            A = A.to(dt)
            W = (torch.randn(N, K, generator=gc) * K ** -0.5).numpy()
            b = torch.randn(N, generator=gc).numpy()
            R = torch.randn(M, N, device=DEV, generator=g) * 4 if res else None
            A1, A2 = (A[:, :K1].contiguous(), A[:, K1:].contiguous()) if K1 else (A, None)
            got, path, _ = dense(precision, tc, A1, W, b, R, od, act, A2, K1, f'fp64 {cfg} {name}')
            Wd = torch.as_tensor(W, device=DEV)
            if path == TC:
                Wd = Wd.bfloat16()
            Wd = Wd.double()
            Ad, bd = A.double(), torch.as_tensor(b, device=DEV).double()
            F64 = Ad @ Wd.t() + bd
            if act:
                F64 = F64.clamp_min(0)
            if res:
                F64 = F64 + R.double()
            S = Ad.abs() @ Wd.abs().t()
            bound = dense_bound(path, K, S, bd, None if R is None else R.double(), F64, od)
            del S, Ad
            err = (got.double() - F64).abs()
            ratio = (err / bound).max().item()
            key = (cfg, PATH_NAME[path])
            worst[key] = max(worst.get(key, 0.0), ratio)
            print(f'fp64 {cfg} {name} M {M} N {N} K {K} -> {_DT[od]} [{PATH_NAME[path]}]: max err/bound {ratio:.3f}')
            bad = ~(err <= bound)
            if bool(bad.any()):
                raise AssertionError(_first_bad(bad, f'fp64 {cfg} {name} (got = error, want = bound)', err, bound))
            del F64, err, bound, got, A, A1, A2, R
    print('dense fp64 largest err/bound per route: ' + ', '.join(f'{c} [{p}] {v:.3f}' for (c, p), v in worst.items()))


# ---- (d) the standalone LayerNorm
LN_ROWS = (1, 7, 8, 9, 33, 1600, 40000)


def ln_rows(M, seed):
    """rows with mean/std in LN_RATIOS (alternating signs) or constant on the 1/64 grid (kind CONST): the row kinds of
    test_gemm_tc_gpu.ln_case, changing every row in the first half and every 8 rows (one CTA) in the second"""
    from test_gemm_tc_gpu import CONST, LN_RATIOS
    g = torch.Generator(device=DEV).manual_seed(seed)
    i = torch.arange(M, device=DEV)
    kind = torch.where(i < M // 2, i, i // 8) % (CONST + 1)
    noise = torch.randn(M, 256, device=DEV, generator=g, dtype=torch.float64)
    sd = noise.std(1, unbiased=False, keepdim=True)
    ratio = torch.tensor(LN_RATIOS + (0,), device=DEV, dtype=torch.float64)[kind][:, None]
    sign = torch.where(i % 2 == 0, 1.0, -1.0).double()[:, None]
    x = (noise + sign * ratio * sd).float()
    cval = torch.tensor([0.0, 1.5, -3.25, 100.5], device=DEV)[i % 4]
    const = kind == CONST
    x[const] = cval[const][:, None].expand(-1, 256)
    gamma = 0.5 + 1.5 * torch.rand(256, device=DEV, generator=g)
    beta = torch.rand(256, device=DEV, generator=g) * 2 - 1
    pos = torch.randn(M, 256, device=DEV, generator=g)
    return x, gamma, beta, pos, kind


def layernorm(precision, x, gamma, beta, pos, outs=(1, 1, 1), tag=''):
    L, lib = _lib()
    M = x.shape[0]
    dt = _DT[precision]
    o = [Out((M, 256), torch.float32), Out((M, 256), dt), Out((M, 256), dt)]
    L.check(lib.occb200_encoder_layernorm(precision, _p(x), _p(gamma), _p(beta), _p(pos), M,
                                          *[o[k].ptr() if outs[k] else None for k in range(3)], L.stream_ptr()))
    for k, nm in enumerate(('y_f32', 'y_t', 'y_pos_t')):
        if outs[k]:
            o[k].check_guards(f'{tag} {nm}')
        else:
            assert o[k].untouched(), f'{tag}: the NULL output {nm} was written'
    return [o[k].value() if outs[k] else None for k in range(3)]


def check_layernorm():
    from test_gemm_tc_gpu import CONST, LN_RATIOS, LN_TOL
    worst = {}
    for precision in (0, 1):
        dt = _DT[precision]
        for M in LN_ROWS:
            x, gamma, beta, pos, kind = ln_rows(M, 600 + M + precision)
            tag = f'layernorm256 {dt} rows {M}'
            yf, yt, ypt = layernorm(precision, x, gamma, beta, pos, tag=tag)
            x64 = x.double()
            mu = x64.mean(1, keepdim=True)
            var = ((x64 - mu) ** 2).mean(1, keepdim=True)
            y64 = (x64 - mu) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double()
            err = (yf.double() - y64).abs()
            for k, r in enumerate(LN_RATIOS):
                if bool((kind == k).any()):
                    worst[r] = max(worst.get(r, 0.0), err[kind == k].max().item())
            bad = ~(err <= LN_TOL)
            if bool(bad.any()):
                def extra(r, c):
                    kd = int(kind[r])
                    return f'; row kind {"constant" if kd == CONST else "mean/std " + str(LN_RATIOS[kd])}'
                raise AssertionError(_first_bad(bad, f'{tag}: |y - y64| > {LN_TOL}', yf, y64, extra))
            const = kind == CONST
            if bool(const.any()):
                want = beta[None, :].expand(int(const.sum()), -1)
                bad = _bits(yf[const]) != _bits(want.contiguous())
                if bool(bad.any()):
                    raise AssertionError(_first_bad(bad, f'{tag}: constant rows (numbered among the constant rows) != beta',
                                                    yf[const], want))
            for got, want, nm in ((yt, yf.to(dt), 'y_t vs T(y_f32)'), (ypt, (yf + pos).to(dt), 'y_pos_t vs T(y_f32 + pos)')):
                bad = _bits(got) != _bits(want)
                if bool(bad.any()):
                    raise AssertionError(_first_bad(bad, f'{tag}: {nm}', got, want))
            if M in (9, 1600):
                for mask in range(8):
                    outs = tuple(mask >> k & 1 for k in range(3))
                    sub = layernorm(precision, x, gamma, beta, pos, outs, tag=f'{tag} outputs {outs}')
                    for k, full in enumerate((yf, yt, ypt)):
                        if outs[k]:
                            assert torch.equal(_bits(sub[k]), _bits(full)), f'{tag}: output {k} of subset {outs} differs'
    print('layernorm256 largest |y - y64| by mean/std: ' + ', '.join(f'{r}: {v:.2e}' for r, v in sorted(worst.items())) +
          f' (bar {LN_TOL}, largest ratio {max(worst.values()) / LN_TOL:.3f})')


# ---- (e) packing
LEVEL_SETS = [
    [(8, 8), (3, 4), (3, 5), (1, 1)],                                  # hw % 8 == 0, % 4 but not % 8, odd, 1
    [(7, 9), (8, 8), (5, 13), (2, 2)],                                 # 63, 64, 65, 4
    [(1, 1), (2, 2), (3, 5), (8, 8), (1, 63), (5, 13), (4, 6), (9, 9)],  # eight levels
    PROD_LEVELS,
]


def pack(precision, layout, feats, levels, num_cams, cams, lvl_emb, tag):
    L, lib = _lib()
    Nv = sum(h * w for h, w in levels)
    o = Out((num_cams, Nv, 256), _DT[precision])
    fp = (ctypes.c_void_p * 8)(*([_p(f) for f in feats] + [None] * (8 - len(feats))))
    hw = (ctypes.c_int * 16)(*([v for hw_ in levels for v in hw_] + [0] * (16 - 2 * len(levels))))
    L.check(lib.occb200_encoder_pack(precision, layout, fp, len(levels), hw, num_cams, _p(cams), _p(lvl_emb), o.ptr(),
                                     L.stream_ptr()))
    o.check_guards(tag)
    return o.value()


def check_pack():
    count = 0
    for si, levels in enumerate(LEVEL_SETS):
        for num_cams in (1, 6, 8):
            g = torch.Generator(device=DEV).manual_seed(300 + 10 * si + num_cams)
            nl = len(levels)
            lvl_emb = torch.randn(nl, 256, device=DEV, generator=g)
            cams = torch.randn(num_cams, 256, device=DEV, generator=g)
            x32 = [torch.randn(num_cams, h * w, 256, device=DEV, generator=g) * 4 for h, w in levels]   # [cam, pixel, C]
            for layout in (0, 1, 2):
                xs = [x if layout == 0 else x.bfloat16() for x in x32]
                if layout == 2:
                    feats = [x.contiguous() for x in xs]                                        # NHWC [cam, h*w, C]
                else:
                    feats = [x.transpose(1, 2).contiguous() for x in xs]                        # NCHW [cam, C, h*w]
                for with_cams in (False, True):
                    tok32 = torch.cat([(x.float() + cams[:, None, :] if with_cams else x.float()) + lvl_emb[l]
                                       for l, x in enumerate(xs)], dim=1)
                    for precision in (0, 1):
                        dt = _DT[precision]
                        tag = (f'pack layout {layout} -> {dt}, levels {levels}, {num_cams} cameras, cams_embeds '
                               f'{"present" if with_cams else "NULL"}')
                        got = pack(precision, layout, feats, levels, num_cams, cams if with_cams else None, lvl_emb, tag)
                        want = tok32.to(dt)
                        bad = _bits(got) != _bits(want)
                        if bool(bad.any()):
                            idx = bad.nonzero()
                            cam, tok, c = (int(v) for v in idx[0])
                            starts = np.cumsum([0] + [h * w for h, w in levels])
                            lv = int(np.searchsorted(starts, tok, side='right') - 1)
                            p = tok - int(starts[lv])
                            raise AssertionError(f'{tag}: {idx.shape[0]} mismatches; first at camera {cam}, level {lv} '
                                                 f'({levels[lv][0]}x{levels[lv][1]}, hw {levels[lv][0] * levels[lv][1]}), '
                                                 f'pixel {p} (64-pixel tile {p // 64}, {p % 64} in it), channel {c}; got '
                                                 f'{got[cam, tok, c].item()!r} want {want[cam, tok, c].item()!r}')
                        count += 1
            del x32, xs, feats
    print(f'pack: {count} cases bit-exact (3 layouts x 2 storage types x cams_embeds NULL / present x 1, 6, 8 cameras x '
          f'{len(LEVEL_SETS)} level sets)')


# ---- (f) prepare_query and t32_convert
def check_prepare_query_and_t32():
    from test_gemm_tc_gpu import pad32, t32_index
    L, lib = _lib()
    for precision in (0, 1):
        dt = _DT[precision]
        for rows, tiled in [(1, 0), (1, 1), (31, 1), (32, 1), (33, 1), (37, 0), (1600, 0), (1600, 1), (40000, 0), (40000, 1)]:
            for n in ([rows * 256] + ([8 * 37, 8] if rows == 37 else [])):
                g = torch.Generator(device=DEV).manual_seed(rows + n + precision)
                q = torch.randn(n, device=DEV, generator=g)
                pos = torch.randn(n, device=DEV, generator=g)
                tag = f'prepare_query {dt} n {n} {"T32" if tiled else "row-major"}'
                qf = Out((pad32(n // 256) * 256,) if tiled else (n,), torch.float32)
                qt, qpt = Out((n,), dt), Out((n,), dt)
                L.check(lib.occb200_encoder_prepare_query(precision, tiled, _p(q), _p(pos), n, qf.ptr(), qt.ptr(), qpt.ptr(),
                                                          L.stream_ptr()))
                for o, nm in ((qf, 'q_f32'), (qt, 'q_t'), (qpt, 'q_pos_t')):
                    o.check_guards(f'{tag} {nm}')
                if tiled:
                    r = n // 256
                    idx = t32_index(r, 256, DEV)
                    got = qf.value()[idx]
                    pad = t32_index(pad32(r), 256, DEV)[r:].reshape(-1)
                    assert bool((qf.body_bits()[pad] == NAN32).all()), f'{tag}: T32 pad rows were written'
                    want = q.view(r, 256)
                else:
                    got, want = qf.value(), q
                assert torch.equal(_bits(got), _bits(want)), f'{tag}: q_f32 != q'
                assert torch.equal(_bits(qt.value()), _bits(q.to(dt))), f'{tag}: q_t != T(q)'
                assert torch.equal(_bits(qpt.value()), _bits((q + pos).to(dt))), f'{tag}: q_pos_t != T(q + pos)'
                # outputs may be NULL
                qt2 = Out((n,), dt)
                L.check(lib.occb200_encoder_prepare_query(precision, tiled, _p(q), _p(pos), n, None, None, qt2.ptr(),
                                                          L.stream_ptr()))
                assert torch.equal(_bits(qt2.value()), _bits(qpt.value())), f'{tag}: q_pos_t alone differs'
    print('prepare_query: q_f32 (row-major and T32), q_t and q_pos_t bit-exact, T32 pad rows untouched')
    for ncols in (32, 192, 256):
        for rows in (1, 31, 32, 33, 1000, 40000):
            g = torch.Generator(device=DEV).manual_seed(ncols + rows)
            x = torch.randn(rows, ncols, device=DEV, generator=g)
            tag = f't32_convert {rows} x {ncols}'
            tiled = Out((pad32(rows) * ncols,), torch.float32)
            L.check(lib.occb200_t32_convert(_p(x), tiled.ptr(), rows, 0, ncols, L.stream_ptr()))
            tiled.check_guards(tag + ' tile')
            idx = t32_index(rows, ncols, DEV)
            assert torch.equal(_bits(tiled.value()[idx]), _bits(x)), f'{tag}: tile differs from t32_index'
            pad = t32_index(pad32(rows), ncols, DEV)[rows:].reshape(-1)
            assert bool((tiled.body_bits()[pad] == NAN32).all()), f'{tag}: T32 pad rows were written'
            back = Out((rows, ncols), torch.float32)
            src = tiled.value().clone()
            L.check(lib.occb200_t32_convert(_p(src), back.ptr(), rows, 1, ncols, L.stream_ptr()))
            back.check_guards(tag + ' untile')
            bad = _bits(back.value()) != _bits(x)
            if bool(bad.any()):
                raise AssertionError(_first_bad(bad, f'{tag}: untile(tile(x)) != x', back.value(), x))
    print('t32_convert: both directions bit-exact for ncols 32, 192, 256, pad rows neither read nor written')


# ---- the GPU tests
@pytest.mark.gpu
def test_route_table_and_launch_counts_match_the_engine():
    _child('check_route_table')


@pytest.mark.gpu
def test_dense_layers_bit_exact_on_integer_operands_every_route():
    _child('check_dense_exact')


@pytest.mark.gpu
def test_dense_layers_match_fp64_at_production_shapes_every_route():
    _child('check_dense_fp64')


@pytest.mark.gpu
def test_standalone_layernorm_matches_fp64_and_its_copies_are_exact():
    _child('check_layernorm')


@pytest.mark.gpu
def test_pack_levels_bit_exact_every_layout_and_load_branch():
    _child('check_pack')


@pytest.mark.gpu
def test_prepare_query_and_t32_convert_bit_exact():
    _child('check_prepare_query_and_t32')
