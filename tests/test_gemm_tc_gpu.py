"""Operator tests of the dense-layer tensor-core GEMM (gemm_tc.cu) through its C-ABI test entries, one variant at a time.

(a) Mainloop: the fp32-output GEMM F = A.W^T + bias against fp64 on the same bf16 operands, element by element, with the
    bound |F - F64| <= K 2^-23 sum_k |a_k w_k| (+ the final fp32 rounding of the bias add).  A dropped, repeated or misplaced
    16-deep k-slice breaks it by orders of magnitude.
(b) Epilogues and partitions, bit-exact against F of the same shape (same plan, same k order, so the same accumulators):
    16-bit roundings, ReLU, residual, the K-split A operand, row independence, the n-blocked output, the merged TSA-input
    launch and the split-bf16 fp32-grade GEMM.
(c) Fused LayerNorm against LN in fp64 of F + residual, on rows whose mean is up to 256 standard deviations.
Every output buffer is surrounded by guard rows pre-filled with a NaN bit pattern (and T32 outputs keep their pad rows), which
must survive the launch.  A mismatch names the variant, the first bad element, its 128-row tile, its 32-row block and the
64-column blocks that differ.

The tensor-core cases of one test function run in one child process, so that a device fault cannot poison this session.
The argument rejections need no GPU and run in the CPU suite."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

NAN16 = 0x7FA5                      # a NaN in both bf16 and fp16
NAN32 = 0x7FA5A5A5
GUARD = 64                          # guard rows before and after every output
U23 = 2.0 ** -23


# ------------------------------------------------------------------------------------------------ helpers (no GPU needed)
def t32_index(rows, ncols, device=None):
    """tc::t32_index (tc_common.cuh) for every element of a [rows, ncols] matrix: int64 [rows, ncols] float offsets into
    the T32 block layout (32 x 32 blocks; inside a block, float4 piece (col % 32) / 4 of row r at piece * 32 + r)."""
    r = torch.arange(rows, dtype=torch.int64, device=device)[:, None]
    c = torch.arange(ncols, dtype=torch.int64, device=device)[None, :]
    return ((((r >> 5) * (ncols >> 5) + (c >> 5)) * 256 + ((c & 31) >> 2) * 32 + (r & 31)) << 2) + (c & 3)


def pad32(m):
    return (m + 31) // 32 * 32


def t32_pack(x, fill=0.0):
    """row-major fp32 [M, n] -> T32 buffer of pad32(M) * n floats; pad rows hold `fill`."""
    m, n = x.shape
    out = torch.full((pad32(m) * n,), fill, dtype=torch.float32, device=x.device)
    out[t32_index(m, n, x.device).reshape(-1)] = x.reshape(-1)
    return out


def t32_unpack(buf, m, n):
    return buf[t32_index(m, n, buf.device)]


def test_t32_helper_matches_the_host_logic_mirror():
    """The vectorised restatement used below agrees with the element-wise mirror of elementwise.cu, and is a permutation."""
    sys.path.insert(0, HERE)
    from test_host_logic_cpu import _t32_index
    for rows, ncols in [(96, 256), (64, 192), (33, 320)]:
        got = t32_index(rows, ncols)
        want = torch.tensor([[_t32_index(r, c, ncols) for c in range(ncols)] for r in range(rows)])
        assert torch.equal(got, want)
        x = torch.randn(rows, ncols)
        buf = t32_pack(x, fill=float('nan'))
        assert torch.equal(t32_unpack(buf, rows, ncols), x)
        assert int(torch.isnan(buf).sum()) == (pad32(rows) - rows) * ncols


# ------------------------------------------------------------------------------------------------ argument rejection (CPU)
def _rejections():
    """(entry point, argument dict overrides, expected message fragment).  Base shapes are valid; one argument is broken."""
    gemm = dict(A=1, A2=None, K1=0, W=1, bias=None, residual=None, C=1, out_dtype=0, M=128, N=256, K=256, act=0)
    cases = [
        ('gemm_tc', gemm, dict(N=100), 'shape'),
        ('gemm_tc', gemm, dict(N=32), 'shape'),
        ('gemm_tc', gemm, dict(K=96), 'shape'),
        ('gemm_tc', gemm, dict(K=0), 'shape'),
        ('gemm_tc', gemm, dict(A2=1, K1=96, K=256), 'shape'),
        ('gemm_tc', gemm, dict(A2=1, K1=320, K=256), 'shape'),
        ('gemm_tc', gemm, dict(A2=1, K1=256, K=256), 'shape'),
        ('gemm_tc', gemm, dict(A2=1, K1=0, K=256), 'shape'),
        ('gemm_tc', gemm, dict(M=0), 'shape'),
        ('gemm_tc', gemm, dict(M=-5), 'shape'),
        ('gemm_tc', gemm, dict(out_dtype=3), 'out_dtype'),
        ('gemm_tc', gemm, dict(act=2), 'act'),
        ('gemm_tc', gemm, dict(A=None), 'null'),
        ('gemm_tc', gemm, dict(W=None), 'null'),
        ('gemm_tc', gemm, dict(C=None), 'null'),
    ]
    ln = dict(A=1, W=1, bias=1, residual=1, gamma=1, beta=1, pos=None, y_f32=1, y_bf16=None, y_pos_bf16=None, M=128, K=256)
    cases += [
        ('gemm_tc_ln', ln, dict(K=200), 'shape'),
        ('gemm_tc_ln', ln, dict(M=0), 'shape'),
        ('gemm_tc_ln', ln, dict(residual=None), 'null'),
        ('gemm_tc_ln', ln, dict(gamma=None), 'null'),
        ('gemm_tc_ln', ln, dict(y_pos_bf16=1), 'pos'),
    ]
    blk = dict(A=1, W=1, bias=None, C=1, M=128, N=512, K=256)
    cases += [
        ('gemm_tc_blocked256', blk, dict(N=320), 'shape'),
        ('gemm_tc_blocked256', blk, dict(N=192), 'shape'),
        ('gemm_tc_blocked256', blk, dict(K=100), 'shape'),
        ('gemm_tc_blocked256', blk, dict(M=0), 'shape'),
        ('gemm_tc_blocked256', blk, dict(C=None), 'null'),
    ]
    tsa = dict(Av=[1], nv=1, Wv=1, bv=None, Cv=[1], Aq=1, Aq2=None, K1q=0, Wq=1, bq=None, rq=None, rq_t32=None, Cq=1,
               M=128, Nq=192, Kq=256)
    cases += [
        ('gemm_tc_tsa_inputs', tsa, dict(nv=3, Av=[1, 1, 1], Cv=[1, 1, 1]), 'nv'),
        ('gemm_tc_tsa_inputs', tsa, dict(nv=0), 'nv'),
        ('gemm_tc_tsa_inputs', tsa, dict(Nq=100), 'shape'),
        ('gemm_tc_tsa_inputs', tsa, dict(Kq=200), 'shape'),
        ('gemm_tc_tsa_inputs', tsa, dict(Aq2=1, K1q=320, Kq=256), 'shape'),
        ('gemm_tc_tsa_inputs', tsa, dict(Aq2=1, K1q=100, Kq=256), 'shape'),
        ('gemm_tc_tsa_inputs', tsa, dict(M=0), 'shape'),
        ('gemm_tc_tsa_inputs', tsa, dict(nv=2, Av=[1, None], Cv=[1, 1]), 'null'),
        ('gemm_tc_tsa_inputs', tsa, dict(Cq=None), 'null'),
        ('gemm_tc_tsa_inputs', tsa, dict(rq_t32=1), 'rq_t32'),
    ]
    s3 = dict(S=1, Ks=256, W3=1, bias=None, residual=None, C=1, M=128, N=256, act=0)
    cases += [
        ('gemm_tc_split3', s3, dict(Ks=96), 'shape'),
        ('gemm_tc_split3', s3, dict(N=96), 'shape'),
        ('gemm_tc_split3', s3, dict(M=0), 'shape'),
        ('gemm_tc_split3', s3, dict(W3=None), 'null'),
    ]
    sp = dict(a=1, Ka=256, b=None, Kb=0, rows=10, S=1)
    cases += [
        ('split_bf16', sp, dict(Ka=12), 'multiples of 8'),
        ('split_bf16', sp, dict(b=1, Kb=4), 'multiples of 8'),
        ('split_bf16', sp, dict(Kb=8), 'null'),
        ('split_bf16', sp, dict(S=None), 'null'),
    ]
    return cases


_ORDER = {
    'gemm_tc': ['A', 'A2', 'K1', 'W', 'bias', 'residual', 'C', 'out_dtype', 'M', 'N', 'K', 'act'],
    'gemm_tc_ln': ['A', 'W', 'bias', 'residual', 'gamma', 'beta', 'pos', 'y_f32', 'y_bf16', 'y_pos_bf16', 'M', 'K'],
    'gemm_tc_blocked256': ['A', 'W', 'bias', 'C', 'M', 'N', 'K'],
    'gemm_tc_tsa_inputs': ['Av', 'nv', 'Wv', 'bv', 'Cv', 'Aq', 'Aq2', 'K1q', 'Wq', 'bq', 'rq', 'rq_t32', 'Cq', 'M', 'Nq', 'Kq'],
    'gemm_tc_split3': ['S', 'Ks', 'W3', 'bias', 'residual', 'C', 'M', 'N', 'act'],
    'split_bf16': ['a', 'Ka', 'b', 'Kb', 'rows', 'S'],
}
_INTS = {'K1', 'out_dtype', 'M', 'N', 'K', 'act', 'nv', 'K1q', 'Nq', 'Kq', 'Ks', 'Ka', 'Kb', 'rows'}


@pytest.mark.parametrize('case', range(len(_rejections())))
def test_entry_point_rejects_bad_arguments_before_any_cuda_call(case, lib_built):
    """Return code 1 (an argument check, not 2, a CUDA error) and a message.  Pointer arguments are 1 (non-null) or None.
    Without a GPU a CUDA call would fail with code 2; with one, every non-null pointer is a real 16 MB device buffer."""
    from occnet_b200 import _lib
    lib = _lib.load()
    name, base, over, msg = _rejections()[case]
    args = dict(base, **over)
    buf = torch.zeros(1 << 22, device='cuda') if torch.cuda.is_available() else None
    dev = ctypes.c_void_p(buf.data_ptr()) if buf is not None else ctypes.c_void_p(1 << 12)
    keep = []
    call = []
    for k in _ORDER[name]:
        v = args[k]
        if k in _INTS:
            call.append(v)
        elif isinstance(v, list):
            arr = (ctypes.c_void_p * max(len(v), 2))(*[dev.value if p else None for p in v])
            keep.append(arr)
            call.append(ctypes.cast(arr, ctypes.c_void_p))
        else:
            call.append(dev if v else None)
    rc = getattr(lib, 'occb200_' + name)(*call, None)
    err = lib.occb200_last_error().decode()
    assert rc == 1, (name, over, rc, err)
    assert msg in err, (name, over, err)


# ------------------------------------------------------------------------------------------------ GPU: child processes
def _run_isolated(code, timeout=600):
    """Tensor-core runs happen in a child process: a device fault there must not poison this session's context."""
    r = subprocess.run([sys.executable, '-c', 'import sys; sys.path.insert(0, "tests"); ' + code], cwd=ROOT, capture_output=True,
                       text=True, timeout=timeout)
    print(r.stdout[-20000:])
    assert r.returncode == 0, f'child failed ({r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'
    assert 'OK' in r.stdout
    return r.stdout


def _child(fn):
    return _run_isolated(f'import test_gemm_tc_gpu as t; t.{fn}(); print("OK")')


# ---- device-side fixtures (run in the child)
DEV = 'cuda:0'


def _lib():
    from occnet_b200 import _lib as L
    return L, L.load()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Out:
    """An output of `rows` x `cols` elements (contiguous) with GUARD guard rows on each side, all pre-filled with NaN bits."""

    def __init__(self, rows, cols, dtype):
        self.rows, self.cols, self.dtype = rows, cols, dtype
        it = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}[dtype]
        self.bits = torch.full(((rows + 2 * GUARD) * cols,), NAN32 if it == torch.int32 else NAN16, dtype=it, device=DEV)
        self.buf = self.bits.view(dtype)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + GUARD * self.cols * self.buf.element_size())

    def body(self):
        return self.buf[GUARD * self.cols:(GUARD + self.rows) * self.cols]

    def value(self, rows=None, cols=None):
        return self.body().view(rows or self.rows, cols or self.cols)

    def check_guards(self, what):
        """the guard rows still hold the NaN pattern"""
        fill = NAN32 if self.bits.dtype == torch.int32 else NAN16
        g = GUARD * self.cols
        parts = [('leading guard', self.bits[:g]), ('trailing guard', self.bits[g + self.rows * self.cols:])]
        for name, p in parts:
            bad = (p != fill).nonzero()
            assert bad.numel() == 0, f'{what}: {bad.numel()} elements of the {name} were written (first at {int(bad[0])})'


def _where(bad, what, got=None, want=None, extra=''):
    """AssertionError text naming the first mismatching element, its tile / block and the differing 64-column blocks"""
    idx = bad.nonzero()
    r, c = int(idx[0, 0]), int(idx[0, 1])
    cblk = sorted(set((idx[:, 1] // 64).tolist()))[:16]
    rows = idx[:, 0]
    s = (f'{what}: {idx.shape[0]} mismatches; first at row {r} col {c} (128-row tile {r // 128}, 32-row block {r // 32}, '
         f'64-col block {c // 64}); bad rows {int(rows.min())}..{int(rows.max())}; bad 64-col blocks {cblk}')
    if got is not None:
        s += f'; got {got[r, c].item()!r} want {want[r, c].item()!r}'
    return s + extra


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _assert_bits(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bad = _bits(got) != _bits(want)
    if bool(bad.any()):
        raise AssertionError(_where(bad, what, got, want))


def _operands(M, N, K, seed, wscale=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    W = (torch.randn(N, K, device=DEV, generator=g) * (wscale or K ** -0.5)).bfloat16()
    b = torch.randn(N, device=DEV, generator=g)
    return A, W, b


_DT = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}


def gemm(A, W, bias=None, residual=None, out_dtype=0, act=0, A2=None, K1=0, M=None):
    """one occb200_gemm_tc launch into a guarded output; returns the [M, N] result (guards checked)"""
    L, lib = _lib()
    M = M or A.shape[0]
    N, K = W.shape
    o = Out(M, N, _DT[out_dtype])
    L.check(lib.occb200_gemm_tc(_p(A), _p(A2), K1, _p(W), _p(bias), _p(residual), o.ptr(), out_dtype, M, N, K, act,
                                L.stream_ptr()))
    torch.cuda.synchronize()
    o.check_guards(f'gemm_tc M={M} N={N} K={K} out={out_dtype} act={act} res={residual is not None} K1={K1 if A2 is not None else K}')
    return o.value()


# ---- (a) mainloop against fp64
PROD_M = [40000, 1600, 6 * 30825]
PROD_NK = [(256, 256), (192, 256), (192, 512), (768, 256), (512, 256), (256, 512)]
EDGE = ([(m, 256, 256) for m in (1, 31, 33, 127, 129, 1000, 2500)] +
        [(1000, 256, k) for k in (64, 768, 1536)] + [(2500, 192, 1536), (1000, 64, 256), (2500, 320, 256), (129, 320, 768)] +
        # the shapes of test_tcgen05_gemm_matches_fp32_matmul (test_gpu_parity.py)
        [(128, 256, 256), (1000, 192, 512), (4100, 768, 256), (333, 512, 256), (2000, 256, 768), (777, 192, 1536),
         (1000, 192, 256)])
MAINLOOP_SHAPES = [(m, n, k) for m in PROD_M for (n, k) in PROD_NK] + EDGE


def mainloop_err(A, W, b, F):
    """max |F - F64| / sum|aw| and whether every element meets K 2^-23 sum|aw| + 2^-23 |F64| (the bias add's rounding)"""
    K = A.shape[1]
    Ad, Wd = A.double(), W.double()
    F64 = Ad @ Wd.t() + b.double()
    S = Ad.abs() @ Wd.abs().t()
    err = (F.double() - F64).abs()
    bound = K * U23 * S + U23 * F64.abs()
    bad = ~(err <= bound)
    return (err / S.clamp_min(1e-30)).max().item(), bad, err, bound


def check_mainloop():
    torch.manual_seed(0)
    for i, (M, N, K) in enumerate(MAINLOOP_SHAPES):
        A, W, b = _operands(M, N, K, seed=100 + i)
        F = gemm(A, W, b)
        ratio, bad, err, bound = mainloop_err(A, W, b, F)
        print(f'mainloop M={M} N={N} K={K}: max |F - F64| / sum|aw| = {ratio:.3e} (bound {K * U23:.3e})')
        if bool(bad.any()):
            raise AssertionError(_where(bad, f'mainloop M={M} N={N} K={K}', err, bound, ' (got = error, want = bound)'))
        del A, W, F, bad, err, bound


# ---- (b) epilogues, bit-exact against F
EPI_SHAPES = ([(40000, n, k) for (n, k) in PROD_NK] + [(1600, 768, 256), (6 * 30825, 256, 256)] +
              [(m, 256, 256) for m in (1, 31, 33, 127, 129, 2500)] +
              [(1000, 256, 64), (1000, 192, 768), (1000, 256, 1536), (1000, 64, 256), (2500, 320, 256)])


def check_epilogues():
    for i, (M, N, K) in enumerate(EPI_SHAPES):
        A, W, b = _operands(M, N, K, seed=200 + i)
        R = torch.randn(M, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7 + i))
        F = gemm(A, W, b)
        tag = f'M={M} N={N} K={K}'
        _assert_bits(gemm(A, W, b, out_dtype=1), F.bfloat16(), f'bf16 output {tag}')
        _assert_bits(gemm(A, W, b, out_dtype=2), F.half(), f'fp16 output {tag}')
        relu = F.clamp_min(0)
        for od in (0, 1, 2):
            cast = (lambda x: x) if od == 0 else (lambda x, d=_DT[od]: x.to(d))
            _assert_bits(gemm(A, W, b, act=1, out_dtype=od), cast(relu), f'relu out={od} {tag}')
            _assert_bits(gemm(A, W, b, residual=R, out_dtype=od), cast(F + R), f'residual out={od} {tag}')
            _assert_bits(gemm(A, W, b, residual=R, act=1, out_dtype=od), cast(relu + R), f'relu + residual out={od} {tag}')
        _assert_bits(gemm(A, W, None), gemm(A, W, torch.zeros_like(b)), f'null bias {tag}')
        print(f'epilogues {tag}: bit-exact')


SPLITS = [(1000, 256, 512, 256), (1000, 256, 512, 64), (2500, 192, 512, 448), (40000, 192, 512, 256), (129, 256, 256, 64),
          (1000, 320, 768, 192), (777, 192, 1536, 512), (33, 256, 1536, 1472)]


def check_split_operand():
    for i, (M, N, K, K1) in enumerate(SPLITS):
        A, W, b = _operands(M, N, K, seed=300 + i)
        A1, A2 = A[:, :K1].contiguous(), A[:, K1:].contiguous()
        R = torch.randn(M, N, device=DEV)
        for od, act, res in [(0, 0, None), (1, 1, R), (2, 0, R)]:
            _assert_bits(gemm(A1, W, b, res, od, act, A2=A2, K1=K1), gemm(A, W, b, res, od, act),
                         f'A | A2 split at K1={K1} (M={M} N={N} K={K} out={od} act={act} res={res is not None})')
        print(f'split operand M={M} N={N} K={K} K1={K1}: bit-exact')


def check_row_independence():
    for i, (M, N, K) in enumerate([(40000, 256, 256), (40000, 192, 512), (6 * 30825, 768, 256), (2500, 320, 1536)]):
        A, W, b = _operands(M, N, K, seed=400 + i)
        full = gemm(A, W, b, out_dtype=1)
        for M1 in (1, 33, 129, 1000, 2500 - 37):
            if M1 < M:
                _assert_bits(gemm(A, W, b, out_dtype=1, M=M1), full[:M1], f'first {M1} rows of M={M} (N={N} K={K})')
        print(f'row independence M={M} N={N} K={K}: bit-exact')


def check_blocked256():
    L, lib = _lib()
    for i, (M, N, K) in enumerate([(6 * 30825, 6 * 256, 256), (1000, 6 * 256, 256), (33, 512, 256), (129, 256, 128)]):
        A, W, b = _operands(M, N, K, seed=500 + i)
        F = gemm(A, W, b)
        o = Out(M * (N // 256), 256, torch.bfloat16)
        L.check(lib.occb200_gemm_tc_blocked256(_p(A), _p(W), _p(b), o.ptr(), M, N, K, L.stream_ptr()))
        torch.cuda.synchronize()
        o.check_guards(f'blocked256 M={M} N={N}')
        got = o.value().view(N // 256, M, 256)
        for blk in range(N // 256):
            _assert_bits(got[blk], F[:, 256 * blk:256 * blk + 256].bfloat16(), f'blocked256 block {blk} (M={M} N={N} K={K})')
        print(f'blocked256 M={M} N={N} K={K}: bit-exact')


def check_tsa_inputs():
    """value problems equal their single launches; the projection equals (F_q + constant).half(), where the constant comes
    from rq_t32 only when M % 32 == 0 (the other source is filled with NaN, so reading the wrong one cannot pass)"""
    L, lib = _lib()
    nan = float('nan')
    cases = []
    for M in (40000, 2500, 1000, 33):
        for nv in (1, 2):
            for aq2 in (False, True):
                for const in ('none', 'rq', 't32'):
                    cases.append((M, nv, aq2, const))
    cases = [c for c in cases if c[0] == 40000 or (c[1] == 2) == c[2]]   # the full cross product at M = 40000 only
    Nq = 192
    for i, (M, nv, aq2, const) in enumerate(cases):
        g = torch.Generator(device=DEV).manual_seed(600 + i)
        Kq = 512 if aq2 else 256
        Av = [torch.randn(M, 256, device=DEV, generator=g).bfloat16() for _ in range(nv)]
        Wv = (torch.randn(256, 256, device=DEV, generator=g) / 16).bfloat16()
        bv = torch.randn(256, device=DEV, generator=g)
        Aq = torch.randn(M, Kq, device=DEV, generator=g).bfloat16()
        Wq = (torch.randn(Nq, Kq, device=DEV, generator=g) / 16).bfloat16()
        bq = None if i % 2 else torch.randn(Nq, device=DEV, generator=g)
        Cn = torch.randn(M, Nq, device=DEV, generator=g) * 4
        rq = rq_t32 = None
        if const == 'rq':
            rq = Cn
        elif const == 't32':
            rq_t32 = t32_pack(Cn, fill=nan) if M % 32 == 0 else torch.full((pad32(M) * Nq,), nan, device=DEV)
            rq = torch.full_like(Cn, nan) if M % 32 == 0 else Cn
        Aq1, Aq2 = (Aq[:, :256].contiguous(), Aq[:, 256:].contiguous()) if aq2 else (Aq, None)
        ov = [Out(M, 256, torch.bfloat16) for _ in range(nv)]
        oq = Out(M, Nq, torch.float16)
        av = (ctypes.c_void_p * 2)(*[a.data_ptr() for a in Av])
        cv = (ctypes.c_void_p * 2)(*[o.ptr().value for o in ov])
        L.check(lib.occb200_gemm_tc_tsa_inputs(ctypes.cast(av, ctypes.c_void_p), nv, _p(Wv), _p(bv), ctypes.cast(cv, ctypes.c_void_p),
                                               _p(Aq1), _p(Aq2), 256 if aq2 else 0, _p(Wq), _p(bq), _p(rq), _p(rq_t32), oq.ptr(),
                                               M, Nq, Kq, L.stream_ptr()))
        torch.cuda.synchronize()
        tag = f'tsa_inputs M={M} nv={nv} Aq2={aq2} bq={bq is not None} constant={const}'
        for k in range(nv):
            ov[k].check_guards(f'{tag} value {k}')
            _assert_bits(ov[k].value(), gemm(Av[k], Wv, bv, out_dtype=1), f'{tag}: value problem {k}')
        oq.check_guards(f'{tag} projection')
        Fq = gemm(Aq1, Wq, bq, A2=Aq2, K1=256 if aq2 else 0)
        _assert_bits(oq.value(), (Fq + Cn).half() if const != 'none' else Fq.half(), f'{tag}: projection')
        print(f'{tag}: bit-exact')


def check_split3():
    """split_bf16 against its definition; split3 against the plain GEMM on the materialised operands (bit-exact) and against
    fp64 on the fp32 operands (2^-16 sum|aw| for the dropped lo.lo term plus the accumulation bound)"""
    L, lib = _lib()
    for i, (M, N, Ks, Kb) in enumerate([(40000, 256, 256, 0), (2500, 192, 512, 256), (33, 320, 64, 0), (1000, 256, 512, 0),
                                        (129, 64, 768, 0)]):
        g = torch.Generator(device=DEV).manual_seed(700 + i)
        Ka = Ks - Kb
        a = torch.randn(M, Ka, device=DEV, generator=g) * 3
        bb = torch.randn(M, Kb, device=DEV, generator=g) if Kb else None
        x = torch.cat([a, bb], 1) if Kb else a
        S = Out(M, 2 * Ks, torch.bfloat16)
        L.check(lib.occb200_split_bf16(_p(a), Ka, _p(bb), Kb, M, S.ptr(), L.stream_ptr()))
        torch.cuda.synchronize()
        S.check_guards(f'split_bf16 M={M} Ka={Ka} Kb={Kb}')
        hi = x.bfloat16()
        lo = (x - hi.float()).bfloat16()
        _assert_bits(S.value(), torch.cat([hi, lo], 1), f'split_bf16 M={M} Ka={Ka} Kb={Kb}')
        Wf = torch.randn(N, Ks, device=DEV, generator=g) * Ks ** -0.5
        whi = Wf.bfloat16()
        wlo = (Wf - whi.float()).bfloat16()
        W3 = torch.cat([whi, whi, wlo], 1).contiguous()
        bias = torch.randn(N, device=DEV, generator=g)
        R = torch.randn(M, N, device=DEV, generator=g)
        Sv = S.value().contiguous()
        for act, res in [(0, None), (1, R)]:
            o = Out(M, N, torch.float32)
            L.check(lib.occb200_gemm_tc_split3(_p(Sv), Ks, _p(W3), _p(bias), _p(res), o.ptr(), M, N, act, L.stream_ptr()))
            torch.cuda.synchronize()
            tag = f'split3 M={M} N={N} Ks={Ks} act={act} res={res is not None}'
            o.check_guards(tag)
            mat = torch.cat([hi, lo, hi], 1).contiguous()
            _assert_bits(o.value(), gemm(mat, W3, bias, res, act=act), tag)
            if act == 0:
                F64 = x.double() @ Wf.double().t() + bias.double()
                Sabs = x.double().abs() @ Wf.double().abs().t()
                err = (o.value().double() - F64).abs()
                bound = 2.0 ** -16 * Sabs + 3 * Ks * U23 * Sabs * 1.01 + U23 * F64.abs()
                bad = ~(err <= bound)
                print(f'{tag}: max |C - C64| / sum|aw| = {(err / Sabs).max().item():.3e}')
                if bool(bad.any()):
                    raise AssertionError(_where(bad, tag + ' vs fp64', err, bound, ' (got = error, want = bound)'))


# ---- (c) fused LayerNorm
LN_RATIOS = (0, 1, 4, 8, 16, 64, 256)
CONST = len(LN_RATIOS)              # row kind of the constant rows
LN_TOL = 2e-4


def ln_case(M, K, seed):
    """operands whose rows x = F + residual have mean/std in LN_RATIOS (alternating signs) or are constant: a constant row
    has a zero A row and residual = c - bias, exact on the 1/64 grid of the bias.  The kernel picks the one- or two-pass
    variance per row but runs the second pass per warp (16 rows): in the first half the kind changes every 16 rows (warps of
    one kind), in the second half every row (mixed warps)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    A, W, _ = _operands(M, 256, K, seed, wscale=0.5 * K ** -0.5)
    b = torch.round((torch.rand(256, device=DEV, generator=g) * 2 - 1) * 64) / 64
    i = torch.arange(M, device=DEV)
    kind = torch.where(i < M // 2, i // 16, i) % (CONST + 1)
    const = kind == CONST
    A[const] = 0
    F = gemm(A, W, b)
    noise = torch.randn(M, 256, device=DEV, generator=g)
    x0 = F.double() + noise.double()
    sd = x0.std(1, unbiased=False, keepdim=True)
    ratio = torch.tensor(LN_RATIOS + (0,), device=DEV, dtype=torch.float64)[kind][:, None]
    sign = torch.where(torch.arange(M, device=DEV) % 2 == 0, 1.0, -1.0).double()[:, None]
    R = (noise.double() + sign * ratio * sd).float()
    cval = torch.tensor([0.0, 1.5, -3.25, 100.5], device=DEV)[torch.arange(M, device=DEV) % 4]
    R[const] = (cval[:, None] - b[None, :])[const]
    gamma = 0.5 + 1.5 * torch.rand(256, device=DEV, generator=g)
    beta = torch.rand(256, device=DEV, generator=g) * 2 - 1
    pos = torch.randn(M, 256, device=DEV, generator=g)
    return A, W, b, R, gamma, beta, pos, F, kind


def check_layernorm():
    L, lib = _lib()
    for i, (M, K) in enumerate([(40000, 256), (40000, 512), (1600, 256), (1600, 512), (2500, 256), (33, 256), (129, 512),
                                (1, 256)]):
        A, W, b, R, gamma, beta, pos, F, kind = ln_case(M, K, 800 + i)
        Mp = pad32(M)
        Rt = t32_pack(R, fill=float('nan'))
        Pt = t32_pack(pos, fill=float('nan'))
        y = Out(Mp, 256, torch.float32)
        yb = Out(M, 256, torch.bfloat16)
        yp = Out(M, 256, torch.bfloat16)
        L.check(lib.occb200_gemm_tc_ln(_p(A), _p(W), _p(b), _p(Rt), _p(gamma), _p(beta), _p(Pt), y.ptr(), yb.ptr(), yp.ptr(),
                                       M, K, L.stream_ptr()))
        torch.cuda.synchronize()
        tag = f'gemm_tc_ln M={M} K={K}'
        # pad rows of the T32 output: the elements of rows >= M
        pad = t32_index(Mp, 256, DEV)[M:].reshape(-1)
        assert bool((y.body().view(torch.int32)[pad] == NAN32).all()), f'{tag}: T32 pad rows were written'
        y.check_guards(tag)
        yb.check_guards(tag + ' y_bf16')
        yp.check_guards(tag + ' y_pos_bf16')
        yf = t32_unpack(y.body(), M, 256)
        x64 = F.double() + R.double()
        mu = x64.mean(1, keepdim=True)
        var = ((x64 - mu) ** 2).mean(1, keepdim=True)
        y64 = (x64 - mu) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double()
        err = (yf.double() - y64).abs()
        per = ', '.join(f'{r}: {err[kind == k].max().item():.2e}' for k, r in enumerate(LN_RATIOS) if bool((kind == k).any()))
        print(f'{tag}: max |y - y64| by mean/std {{{per}}}, constant rows {err[kind == CONST].max().item() if bool((kind == CONST).any()) else 0:.2e}')
        bad = ~(err <= LN_TOL)
        if bool(bad.any()):
            r = int(bad.nonzero()[0, 0])
            raise AssertionError(_where(bad, f'{tag}: |y - y64| > {LN_TOL}', yf, y64,
                                        f'; row kind {"constant" if int(kind[r]) == CONST else "mean/std " + str(LN_RATIOS[int(kind[r])])}'))
        _assert_bits(yb.value(), yf.bfloat16(), f'{tag}: y_bf16 vs y_f32')
        _assert_bits(yp.value(), (yf + pos).bfloat16(), f'{tag}: y_pos_bf16 vs y_f32 + pos')


# ---- the GPU tests
@pytest.mark.gpu
def test_mainloop_matches_fp64():
    _child('check_mainloop')


@pytest.mark.gpu
def test_16bit_relu_and_residual_epilogues_are_bit_exact():
    _child('check_epilogues')


@pytest.mark.gpu
def test_split_a_operand_equals_concatenated_operand():
    _child('check_split_operand')


@pytest.mark.gpu
def test_rows_are_independent_of_the_launch_size():
    _child('check_row_independence')


@pytest.mark.gpu
def test_blocked256_blocks_equal_the_column_slices():
    _child('check_blocked256')


@pytest.mark.gpu
def test_tsa_inputs_equal_single_problem_launches():
    _child('check_tsa_inputs')


@pytest.mark.gpu
def test_split_bf16_and_split3_gemm():
    _child('check_split3')


@pytest.mark.gpu
def test_fused_layernorm_matches_fp64():
    _child('check_layernorm')
