"""Operator tests of the mmcv `_ext` drop-ins in occnet_b200/ops.py: `ms_deform_attn_forward` (msda_forward_kernel<8> when
C % 8 == 0 and value and out are 16-byte aligned, <1> otherwise), `ms_deform_attn_backward` (msda_backward_kernel, fp32
atomicAdd into grad_value), `MultiScaleDeformableAttnFunction_fp32`, and `linear` / `layer_norm` (gemm_simt<float, float>,
layernorm256), through the C-ABI entries and the Python wrappers.

Reference: oracle.msda.msda_reference, mmcv's rule in float64 on the stored fp32 operands (pinned on the CPU in
tests/test_oracle_cpu.py against the kernel loops, float64 autograd through grid_sample, finite differences, and the h = -1
rule where it departs from grid_sample).  It addresses levels through level_start_index and returns, per output element, the
sum of the absolute values of its terms S, the number n of atomic adds into each grad_value element, and the sensitivity D
of each output to an error in the pixel coordinates.

(a) Bit-exact on dyadic operands, both forward kernels and the backward.  Locations are multiples of 1/32, values and
    grad_output integers in [-8, 8] (in [-2, 2] where many samples meet), weights multiples of 1/8.  The pixel coordinates
    x * W - 0.5 are then exact in fp32 and multiples of 2^-e (e <= 5 per axis), every corner weight a multiple of
    2^-(e_h + e_x), and every term of an output a multiple of a unit f: 2^-(3 + e_h + e_x) for out and grad_value,
    2^-(e_h + e_x) for grad_attn, 2^-(3 + e_h) and 2^-(3 + e_x) for grad_loc's x and y.  The test asserts S < 2^24 f for
    every element of every output (grad_loc after its factor W or H): every partial sum is then a multiple of f below 2^24 f,
    so exact in fp32 in any order, fused or not, atomics included, and each output must equal the fp64 reference bit for bit
    (the sign of a zero aside).  Cases: C in {1, 3, 12, 33} (<1>) and {8, 32, 40, 64, 96} (<8>), which gives the backward
    C < 32, C = 32 and C > 32 not a multiple of 32; M in {1, 3, 8}; L in {1, 2, 4, 5}; P in {1, 3, 4, 8}; levels 1x1, 1xW,
    Hx1, non-square and power-of-two; level_start_index with NaN gap rows between and after the levels (never read; their
    grad_value rows never written); B in {1, 2, 3} with Nq in {1, 7, 1000}, and B = 128 with im2col_step 64.  On power-of-two
    levels up to 16 an axis lands on -1 and on H exactly (skipped), inside (-1, 0), on integers (lh = 0), on H - 1, inside
    (H - 1, H), and far outside on both sides.  Two collision cases aim 4000 queries at one 2x2 pixel block.
(b) Against fp64 at the plugin's production shapes: TSA (B 2, Nv = Nq = 40000, 200x200, M 8, C 32, L 1, P 4), SCA (B 6 cameras,
    Nv 30825, Nq 40000, 116x200 / 58x100 / 29x50 / 15x25, M 8, C 32, L 4, P 8) and one C = 12 shape for the per-channel
    kernel.  With u = 2^-24, per element:
        out          e = (4 L P + 8) u S + D      <8>: each corner weight wt * (hh * hw) carries 4 roundings (1 - lh, 1 - lw,
                                                  the product, the weight) and the 4 L P fused multiply-adds 4 L P more; <1>
                                                  sums 4 corners first (4 + 3) and then L P samples: fewer
        grad_value   e = (n + 5) u S + D          t = go * w, 1 - lh, 1 - lw and the two products: 5; n atomic adds
        grad_attn    e = (13 + ceil(C/32)) u S + D    corner weights 3, the 4-term corner sum 4, go * (...) 1; the lane's
                                                  ceil(C/32) additions and 5 shuffle levels
        grad_loc     e = (13 + ceil(C/32)) u S + D    t 1, v2 - v1 1, 1 - lh 1, the product and the sum 2, t * (...) 1,
                                                  the lane chain, 5 shuffle levels, the factor W or H 1
    D: the kernel rounds loc * W - 0.5 in fp32, an error |dx| <= 2u(|loc W| + 1).  out, grad_attn and grad_value are
    continuous in the location and bilinear inside a pixel cell, so D = dh |d/dh| + dx |d/dx|, bounded with the absolute
    values of the corners; grad_loc's x part is linear in h inside a cell (D = W dh |w| sum_c |go_c| (|v1|+..+|v4|)), and so
    on.  grad_loc jumps across pixel lines, so every sample here is more than 10^-3 pixels from a pixel line, from -1 and from
    H; (a) covers the lines.  Every bound carries a factor 1.001; the largest err/bound per output is printed.
(c) Contracts: grad_value accumulates into its contents; grad_sampling_loc and grad_attn_weight are overwritten (they start
    as NaN); a sample outside the map gives exact zeros; im2col_step 64 refuses B = 96 and takes B = 128; B * Nq = 0 writes
    nothing; MultiScaleDeformableAttnFunction_fp32 on fp16 / bf16 inputs with a non-contiguous upstream gradient returns
    gradients of the input dtype equal to the fp32 op's cast to it; misaligned value and out (the per-channel kernel) give the
    aligned result exactly.
(d) ops.linear and ops.layer_norm at the plugin's shapes (M 40000; (N, K) = (256, 256), (512, 256) with ReLU, (256, 512)
    with a residual, (128, 512), (64, 512); LayerNorm C 256): linear within K u' S + u' (S + |b|) (+ u' (S + |b| + |r|) with
    a residual), u' = 2^-23, S = sum_k |x_k w_k| (test_encoder_ops_gpu (c)), LayerNorm within 2e-4 (its (d)); misaligned
    views give the bits of aligned copies.
(e) Argument checks: every shape, device, dtype and alignment error is refused before a kernel runs (the C-ABI rejections
    run in the CPU suite, the wrappers' on the GPU).
Every output lies between guard elements: NaN bits around out, grad_sampling_loc and grad_attn_weight, a non-zero pattern
around grad_value, which must all come back unchanged.  GPU cases run in a child process per test function, so that a device
fault cannot poison this session.
"""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
NAN32 = 0x7FA5A5A5
PAT32 = 0x3FB00001              # 1.375...: the pattern of grad_value's guards and gap rows
GUARD = 1024
U24 = 2.0 ** -24
U23 = 2.0 ** -23


# ------------------------------------------------------------------------------------------------ (e) rejections (CPU)
_LIN = dict(A=1, W=1, bias=1, res=1, C=1, M=128, N=64, K=64, act=0)
_LN = dict(x=1, gamma=1, beta=1, y=1, rows=8, C=256)
_FWD = dict(B=2, Nv=16, M=1, C=8, Nq=3, L=1, P=1, step=64, value=1, out=1)
_REJECT = [
    ('linear', dict(A=None), 'null'), ('linear', dict(W=None), 'null'), ('linear', dict(C=None), 'null'),
    ('linear', dict(A='odd'), 'aligned'), ('linear', dict(W='odd'), 'aligned'), ('linear', dict(bias='odd'), 'aligned'),
    ('linear', dict(res='odd'), 'aligned'), ('linear', dict(C='odd'), 'aligned'), ('linear', dict(act=2), 'act'),
    ('linear', dict(M=-1), 'sizes'), ('linear', dict(N=0), 'sizes'), ('linear', dict(K=40), 'multiple'),
    ('linear', dict(N=66), 'multiple'),
    ('ln', dict(x=None), 'null'), ('ln', dict(gamma=None), 'null'), ('ln', dict(beta=None), 'null'), ('ln', dict(y=None), 'null'),
    ('ln', dict(x='odd'), 'aligned'), ('ln', dict(gamma='odd'), 'aligned'), ('ln', dict(beta='odd'), 'aligned'),
    ('ln', dict(y='odd'), 'aligned'), ('ln', dict(rows=-1), 'rows'), ('ln', dict(C=128), '256'),
    ('fwd', dict(B=96, step=64), 'im2col_step'), ('fwd', dict(value=None), 'null'), ('fwd', dict(out=None), 'null'),
    ('fwd', dict(M=0), 'sizes'), ('fwd', dict(C=0), 'sizes'), ('fwd', dict(L=0), 'sizes'), ('fwd', dict(P=0), 'sizes'),
    ('fwd', dict(Nq=-1), 'sizes'),
    ('bwd', dict(B=96, step=64), 'im2col_step'), ('bwd', dict(value=None), 'null'), ('bwd', dict(out=None), 'null'),
    ('bwd', dict(M=0), 'sizes'),
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

    def dev(v):
        return None if not v else ctypes.c_void_p(base + 4 if v == 'odd' else base)

    if name == 'linear':
        a = dict(_LIN, **over)
        rc = lib.occb200_linear_f32(dev(a['A']), dev(a['W']), dev(a['bias']), dev(a['res']), dev(a['C']), a['M'], a['N'],
                                    a['K'], a['act'], None)
    elif name == 'ln':
        a = dict(_LN, **over)
        rc = lib.occb200_layernorm_f32(dev(a['x']), dev(a['gamma']), dev(a['beta']), dev(a['y']), a['rows'], a['C'], None)
    elif name == 'fwd':
        a = dict(_FWD, **over)
        rc = lib.occb200_ms_deform_attn_forward(dev(a['value']), dev(1), dev(1), dev(1), dev(1), a['B'], a['Nv'], a['M'],
                                                a['C'], a['Nq'], a['L'], a['P'], a['step'], dev(a['out']), None)
    else:
        a = dict(_FWD, **over)
        rc = lib.occb200_ms_deform_attn_backward(dev(a['value']), dev(1), dev(1), dev(1), dev(1), dev(1), a['B'], a['Nv'],
                                                 a['M'], a['C'], a['Nq'], a['L'], a['P'], a['step'], dev(1), dev(a['out']),
                                                 dev(1), None)
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
    return _run_isolated(f'import test_msda_op_gpu as t; t.{fn}(); print("OK")')


def _lib():
    from occnet_b200 import _lib as L
    return L, L.load()


def _p(t, off=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + off)


class Guarded:
    """an fp32 array of `shape` with GUARD elements on each side; body and guards pre-filled with the bits `fill` (the
    body with `body` when given), `offset` extra elements before the body (a misaligned pointer when not a multiple of 4)"""

    def __init__(self, shape, fill=NAN32, body=None, offset=0):
        self.shape = tuple(shape)
        self.n = int(np.prod(self.shape))
        self.fill, self.off = fill, GUARD + offset
        self.bits = torch.full((self.n + 2 * GUARD + offset,), fill, dtype=torch.int32, device=DEV)
        self.buf = self.bits.view(torch.float32)
        if body is not None:
            self.value().copy_(body)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + self.off * 4)

    def value(self):
        return self.buf[self.off:self.off + self.n].view(self.shape)

    def untouched(self):
        return bool((self.bits == self.fill).all())

    def check_guards(self, what):
        for name, p in (('leading guard', self.bits[:self.off]), ('trailing guard', self.bits[self.off + self.n:])):
            bad = (p != self.fill).nonzero()
            assert bad.numel() == 0, f'{what}: {bad.numel()} elements of the {name} were written (first at {int(bad[0])})'


def _where(idx, shape, names):
    return ', '.join(f'{n} {int(i)}' for n, i in zip(names, np.unravel_index(int(idx), shape)))


OUT_NAMES = ('b', 'q', 'channel m*C+c')
GV_NAMES = ('b', 'row', 'head', 'c')
GA_NAMES = ('b', 'q', 'head', 'level', 'point')
GL_NAMES = ('b', 'q', 'head', 'level', 'point', 'xy')


def _named(what, bad, names, got, want, extra=''):
    """AssertionError text naming the first bad element"""
    flat = bad.reshape(-1).nonzero()
    i = int(flat[0])
    return (f'{what}: {flat.numel()} bad elements; first at {_where(i, tuple(bad.shape), names)}: got '
            f'{got.reshape(-1)[i].item()!r} want {want.reshape(-1)[i].item()!r}{extra}')


# ---- the op through the C ABI, every output guarded
def forward(value, shapes, lsi, loc, w, step=64, out_offset=0, value_offset=0, tag=''):
    """-> out [B, Nq, M*C]; value_offset > 0 passes value from a copy that many floats into a buffer"""
    L, lib = _lib()
    B, Nv, M, C = value.shape
    _, Nq, _, Lv, P, _ = loc.shape
    o = Guarded((B, Nq, M * C), offset=out_offset)
    vbuf = None
    if value_offset:
        vbuf = torch.empty(value.numel() + value_offset, device=DEV)
        vbuf[value_offset:] = value.reshape(-1)
    L.check(lib.occb200_ms_deform_attn_forward(_p(value) if vbuf is None else _p(vbuf, 4 * value_offset), _p(shapes), _p(lsi),
                                               _p(loc), _p(w), B, Nv, M, C, Nq, Lv, P, step, o.ptr(), L.stream_ptr()))
    o.check_guards(f'{tag} out')
    return o.value()


def backward(value, shapes, lsi, loc, w, go, gv_init=None, step=64, tag=''):
    """-> (grad_value, grad_loc, grad_attn); grad_value starts as gv_init (zeros), the other two as NaN"""
    L, lib = _lib()
    B, Nv, M, C = value.shape
    _, Nq, _, Lv, P, _ = loc.shape
    gv = Guarded(value.shape, fill=PAT32, body=torch.zeros_like(value) if gv_init is None else gv_init)
    gl, ga = Guarded(loc.shape), Guarded(w.shape)
    L.check(lib.occb200_ms_deform_attn_backward(_p(value), _p(shapes), _p(lsi), _p(loc), _p(w), _p(go), B, Nv, M, C, Nq, Lv,
                                                P, step, gv.ptr(), gl.ptr(), ga.ptr(), L.stream_ptr()))
    for g, nm in ((gv, 'grad_value'), (gl, 'grad_sampling_loc'), (ga, 'grad_attn_weight')):
        g.check_guards(f'{tag} {nm}')
    return gv.value(), gl.value(), ga.value()


# ---- (a) dyadic operands
def dyadic_exponent(x):
    """smallest e with every x * 2^e an integer (x float64 on the device, e <= 30)"""
    for e in range(31):
        y = x * 2.0 ** e
        if bool((y == torch.round(y)).all()):
            return e
    raise AssertionError('not dyadic')


def special_coords(n, size, g):
    """pixel coordinates on one axis of a power-of-two level up to 16: -1 and size exactly (skipped), inside (-1, 0),
    integers (lh = 0) with 0 and size - 1, inside (size - 1, size), far outside on both sides"""
    table = torch.tensor([-1.0, -0.5, -0.75, 0.0, 1.0, size - 1.0, size - 0.5, size - 0.25, float(size), -9.0,
                          size + 7.0] + [float(j) for j in range(size)], dtype=torch.float64, device=DEV)
    return table[torch.randint(0, table.numel(), (n,), generator=g, device=DEV)]


def make_exact(B, Nq, M, C, levels, P, gaps=False, collide=False, seed=0):
    """dyadic operands on the device: value [B, Nv, M, C] (NaN gap rows when `gaps`), shapes, lsi, loc, w, go"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    L = len(levels)
    starts, pos = [], 0
    for i, (h, w_) in enumerate(levels):
        pos += (3 + i) if gaps else 0
        starts.append(pos)
        pos += h * w_
    Nv = pos + (5 if gaps else 0)
    big = 2 if (collide or Nq * P >= 4000) else 8
    value = torch.randint(-8, 9, (B, Nv, M, C), generator=g, device=DEV).float()
    gap_rows = torch.ones(Nv, dtype=torch.bool, device=DEV)
    for (h, w_), s in zip(levels, starts):
        gap_rows[s:s + h * w_] = False
    value[:, gap_rows] = float('nan')
    shapes = torch.tensor(levels, dtype=torch.int64, device=DEV)
    lsi = torch.tensor(starts, dtype=torch.int64, device=DEV)
    loc = torch.randint(-8, 41, (B, Nq, M, L, P, 2), generator=g, device=DEV).double() / 32
    for l, (h, w_) in enumerate(levels):
        for ax, size in ((0, w_), (1, h)):
            if collide:                                   # every sample on the 2x2 block at (1, 1): coordinates 1 or 1.5
                pix = 1.0 + 0.5 * torch.randint(0, 2, loc[..., l, :, ax].shape, generator=g, device=DEV).double()
                loc[..., l, :, ax] = (pix + 0.5) / size
            elif size <= 16 and (size & (size - 1)) == 0:  # half the samples on the special coordinates
                sel = torch.rand(loc[..., l, :, ax].shape, generator=g, device=DEV) < 0.5
                pix = special_coords(int(sel.sum()), size, g)
                sub = loc[..., l, :, ax]
                sub[sel] = (pix + 0.5) / size
                loc[..., l, :, ax] = sub
    loc = loc.float()
    w = torch.randint(-8, 9, (B, Nq, M, L, P), generator=g, device=DEV).float() / 8
    go = torch.randint(-big, big + 1, (B, Nq, M * C), generator=g, device=DEV).float()
    return value, shapes, lsi, loc, w, go


def exactness_units(value, shapes, loc):
    """the unit every term of each output is a multiple of (asserting first that the pixel coordinates are exact in fp32):
    with coordinates multiples of 2^-e_h and 2^-e_x, corner weights are multiples of 2^-(e_h + e_x) and weights of 2^-3, so
    out and grad_value terms of f = 2^-(3 + e_h + e_x), grad_attn terms (go * corner weight * v) of 2^-(e_h + e_x), and
    grad_loc's x terms (t * (hh (v2 - v1) + lh (v4 - v3)), times the integer W) of 2^-(3 + e_h), its y terms of 2^-(3 + e_x)"""
    eh = ex = 0
    for l, (h, w_) in enumerate(shapes.tolist()):
        x64 = loc[..., l, :, 0].double() * w_ - 0.5
        h64 = loc[..., l, :, 1].double() * h - 0.5
        assert torch.equal((loc[..., l, :, 0] * float(w_) - 0.5).double(), x64), 'x * W - 0.5 is not exact in fp32'
        assert torch.equal((loc[..., l, :, 1] * float(h) - 0.5).double(), h64), 'y * H - 0.5 is not exact in fp32'
        ex, eh = max(ex, dyadic_exponent(x64)), max(eh, dyadic_exponent(h64))
    gl = torch.tensor([2.0 ** -(3 + eh), 2.0 ** -(3 + ex)], dtype=torch.float64, device=loc.device)
    return {'out_abs': 2.0 ** -(3 + eh + ex), 'gv_abs': 2.0 ** -(3 + eh + ex), 'ga_abs': 2.0 ** -(eh + ex), 'gl_abs': gl}


EXACT_CASES = [
    # (B, Nq, M, C, levels, P, gaps, collide, im2col_step)
    (1, 1, 1, 1, [(1, 1)], 1, False, False, 64),
    (2, 7, 3, 3, [(1, 8), (4, 1)], 3, True, False, 64),
    (3, 1000, 8, 12, [(8, 16), (4, 8), (2, 4), (1, 2)], 4, False, False, 64),
    (2, 7, 3, 33, [(5, 7), (3, 9), (16, 16), (1, 6), (7, 1)], 8, True, False, 64),
    (1, 1000, 8, 8, [(5, 7), (3, 9), (16, 16), (1, 6), (7, 1)], 3, True, False, 64),
    (3, 1000, 8, 32, [(8, 16), (4, 8), (2, 4), (1, 2)], 8, True, False, 64),
    (2, 7, 1, 40, [(1, 8), (4, 1)], 4, False, False, 64),
    (1, 1000, 3, 64, [(16, 16)], 1, False, False, 64),
    (3, 7, 1, 96, [(6, 10), (3, 5), (2, 4), (1, 1), (4, 16)], 4, True, False, 64),
    (128, 3, 8, 32, [(1, 8), (4, 1)], 4, False, False, 64),
    (128, 2, 3, 12, [(8, 16), (4, 8), (2, 4), (1, 2)], 3, True, False, 64),
    (2, 4000, 8, 32, [(8, 8)], 4, False, True, 64),
    (1, 4000, 1, 12, [(4, 4), (8, 2)], 8, False, True, 64),
]


def _exact_bits(x):
    return (x + 0.0).view(torch.int32)            # +0.0 folds -0 into +0


def compare_exact(got, want, what, names, extra=''):
    want32 = want.float()
    assert torch.equal(want32.double(), want), f'{what}: the reference is not representable in fp32'
    bad = _exact_bits(got) != _exact_bits(want32)
    if bool(bad.any()):
        raise AssertionError(_named(what, bad, names, got, want32, extra))


def check_exact():
    from oracle.msda import msda_reference
    worst = 0.0
    for i, (B, Nq, M, C, levels, P, gaps, collide, step) in enumerate(EXACT_CASES):
        value, shapes, lsi, loc, w, go = make_exact(B, Nq, M, C, levels, P, gaps, collide, seed=100 + i)
        tag = (f'exact case {i}: B {B} Nq {Nq} M {M} C {C} levels {levels} P {P}{" gaps" if gaps else ""}'
               f'{" collisions" if collide else ""} [{"<8>" if C % 8 == 0 else "<1>"}]')
        gap = torch.isnan(value[0, :, 0, 0])
        ref = msda_reference(torch.nan_to_num(value), shapes, lsi, loc, w, go)
        units = exactness_units(value, shapes, loc)
        tops = {}
        for k, s in (('out', 'out_abs'), ('grad_value', 'gv_abs'), ('grad_attn', 'ga_abs'), ('grad_loc', 'gl_abs')):
            tops[k] = float((ref[s] / (2 ** 24 * units[s])).max())
            assert tops[k] < 1, f'{tag}: exactness precondition fails for {k}: max S = {tops[k]:.3f} * 2^24 f'
        worst = max(worst, max(tops.values()))
        out = forward(value, shapes, lsi, loc, w, step, tag=tag)
        compare_exact(out, ref['out'], f'{tag} out', OUT_NAMES)
        gv_init = torch.zeros_like(value)
        gv_init[:, gap] = torch.tensor(PAT32, dtype=torch.int32).view(torch.float32).item()
        gv, gl, ga = backward(value, shapes, lsi, loc, w, go, gv_init=gv_init, step=step, tag=tag)
        compare_exact(gv[:, ~gap], ref['grad_value'][:, ~gap], f'{tag} grad_value (rows numbered without the gaps)', GV_NAMES,
                      extra=f'; {int(ref["gv_count"].max())} atomic adds at most per element')
        if gaps:
            assert bool((gv[:, gap].view(torch.int32) == PAT32).all()), f'{tag}: grad_value gap rows were written'
        compare_exact(ga, ref['grad_attn'], f'{tag} grad_attn_weight', GA_NAMES)
        compare_exact(gl, ref['grad_loc'], f'{tag} grad_sampling_loc', GL_NAMES)
        print(f'{tag}: bit-exact; largest S / 2^24 f ' + ', '.join(f'{k} {v:.4f}' for k, v in tops.items()) +
              f'; most atomic adds into one element {int(ref["gv_count"].max())}')
        del value, loc, w, go, ref, out, gv, gl, ga
    print(f'{len(EXACT_CASES)} exact cases bit-exact (largest S / 2^24 f {worst:.4f})')


# ---- (b) production shapes against fp64
PROD_CASES = [
    # (name, B, Nv, Nq, levels, M, C, P)
    ('TSA', 2, 40000, 40000, [(200, 200)], 8, 32, 4),
    ('SCA', 6, 30825, 40000, [(116, 200), (58, 100), (29, 50), (15, 25)], 8, 32, 8),
    ('C = 12', 2, 2500 + 625, 5000, [(50, 50), (25, 25)], 8, 12, 4),
]


def make_real(B, Nv, Nq, levels, M, C, P, seed, margin=1e-3):
    """random fp32 operands; every sample more than `margin` pixels from a pixel line, from -1 and from H / W"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    L = len(levels)
    shapes = torch.tensor(levels, dtype=torch.int64, device=DEV)
    lsi = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
    assert int(shapes.prod(1).sum()) == Nv
    value = torch.randn(B, Nv, M, C, generator=g, device=DEV) * 2.0 ** torch.randint(-2, 3, (C,), generator=g, device=DEV)
    size = shapes.flip(1).double()[None, None, None, :, None, :]                                   # (W, H)
    pix = torch.floor(torch.rand(B, Nq, M, L, P, 2, generator=g, device=DEV, dtype=torch.float64) * (size + 3)) - 2
    frac = 2 * margin + (1 - 4 * margin) * torch.rand(B, Nq, M, L, P, 2, generator=g, device=DEV, dtype=torch.float64)
    loc = ((pix + frac + 0.5) / size).float()
    coord = loc.double() * size - 0.5                  # the stored location's exact pixel coordinate
    fr = coord - torch.floor(coord)
    assert bool(((fr > margin) & (fr < 1 - margin)).all()), 'a sample lies on a pixel line'
    w = torch.rand(B, Nq, M, L, P, generator=g, device=DEV) * 2 - 1
    go = torch.randn(B, Nq, M * C, generator=g, device=DEV)
    return value, shapes, lsi, loc, w, go


def check_bound(got, want, bound, what, names):
    err = (got.double() - want).abs()
    ratio = float((err / bound).nan_to_num(0.0).max())
    bad = ~(err <= bound)
    if bool(bad.any()):
        raise AssertionError(_named(what + ' (got = |error|, want = bound)', bad, names, err, bound))
    return ratio


def check_production():
    from oracle.msda import msda_reference
    summary = []
    for i, (name, B, Nv, Nq, levels, M, C, P) in enumerate(PROD_CASES):
        L = len(levels)
        value, shapes, lsi, loc, w, go = make_real(B, Nv, Nq, levels, M, C, P, seed=200 + i)
        tag = f'{name}: B {B} Nv {Nv} Nq {Nq} levels {levels} M {M} C {C} P {P} [{"<8>" if C % 8 == 0 else "<1>"}]'
        ref = msda_reference(value, shapes, lsi, loc, w, go)
        out = forward(value, shapes, lsi, loc, w, tag=tag)
        kb = 13 + math.ceil(C / 32)
        r = {'out': check_bound(out, ref['out'], 1.001 * ((4 * L * P + 8) * U24 * ref['out_abs'] + ref['out_dl']),
                                f'{tag} out', OUT_NAMES)}
        del out
        gv, gl, ga = backward(value, shapes, lsi, loc, w, go, tag=tag)
        r['grad_value'] = check_bound(gv, ref['grad_value'],
                                      1.001 * ((ref['gv_count'] + 5) * U24 * ref['gv_abs'] + ref['gv_dl']),
                                      f'{tag} grad_value', GV_NAMES)
        r['grad_attn'] = check_bound(ga, ref['grad_attn'], 1.001 * (kb * U24 * ref['ga_abs'] + ref['ga_dl']),
                                     f'{tag} grad_attn_weight', GA_NAMES)
        r['grad_loc'] = check_bound(gl, ref['grad_loc'], 1.001 * (kb * U24 * ref['gl_abs'] + ref['gl_dl']),
                                    f'{tag} grad_sampling_loc', GL_NAMES)
        line = f'{tag}: largest err/bound ' + ', '.join(f'{k} {v:.3f}' for k, v in r.items())
        print(line)
        summary.append(line)
        del value, loc, w, go, ref, gv, gl, ga
        torch.cuda.empty_cache()
    print('production shapes against fp64:\n  ' + '\n  '.join(summary))


# ---- (c) contracts
def check_contracts():
    from occnet_b200 import ops
    from occnet_b200 import _lib as L
    from oracle.msda import msda_reference
    # grad_value accumulates; the other two are overwritten (they start as NaN, and their guards stay NaN)
    value, shapes, lsi, loc, w, go = make_exact(2, 7, 3, 12, [(4, 8), (2, 2)], 4, seed=300)
    ref = msda_reference(value, shapes, lsi, loc, w, go)
    g = torch.Generator(device=DEV).manual_seed(301)
    init = torch.randint(-64, 65, value.shape, generator=g, device=DEV).float() / 4
    gv, gl, ga = backward(value, shapes, lsi, loc, w, go, gv_init=init, tag='accumulate')
    compare_exact(gv, ref['grad_value'] + init.double(), 'grad_value accumulated onto its contents', GV_NAMES)
    compare_exact(gl, ref['grad_loc'], 'grad_sampling_loc overwritten', GL_NAMES)
    compare_exact(ga, ref['grad_attn'], 'grad_attn_weight overwritten', GA_NAMES)
    # through the wrapper the same: grad_value += , the others =
    gv2, gl2, ga2 = init.clone(), torch.full_like(loc, 7.0), torch.full_like(w, -3.0)
    ops.ms_deform_attn_backward(value, shapes, lsi, loc, w, go, gv2, gl2, ga2, 64)
    assert torch.equal(gv2, gv) and torch.equal(gl2, gl) and torch.equal(ga2, ga), 'ops.ms_deform_attn_backward differs'
    print('contracts: grad_value accumulates, grad_sampling_loc and grad_attn_weight are overwritten')

    # samples outside the map (exactly -1, exactly H, far away): exact zeros, grad_value untouched
    value, shapes, lsi, loc, w, go = make_exact(2, 5, 2, 8, [(4, 8)], 4, seed=302)
    H, W = 4, 8
    choice = torch.tensor([[-0.5 / W, 0.3], [0.3, -0.5 / H], [(W + 0.5) / W, 0.3], [0.3, (H + 0.5) / H], [-3.0, 5.0],
                           [1e6, -1e6]], device=DEV)
    loc = choice[torch.arange(loc[..., 0].numel(), device=DEV) % choice.shape[0]].view(loc.shape)
    init = torch.randint(-8, 9, value.shape, generator=g, device=DEV).float()
    out = forward(value, shapes, lsi, loc, w, tag='outside')
    gv, gl, ga = backward(value, shapes, lsi, loc, w, go, gv_init=init, tag='outside')
    for t, nm in ((out, 'out'), (gl, 'grad_sampling_loc'), (ga, 'grad_attn_weight')):
        assert bool((t.view(torch.int32) == 0).all()), f'outside samples: {nm} is not exactly +0'
    assert torch.equal(gv, init), 'outside samples: grad_value changed'
    print('contracts: samples outside the map give exact zeros')

    # im2col_step: 96 is not a multiple of 64 (refused), 128 is (EXACT_CASES run it)
    value, shapes, lsi, loc, w, go = make_exact(96, 2, 1, 8, [(2, 2)], 1, seed=303)
    for call in (lambda: ops.ms_deform_attn_forward(value, shapes, lsi, loc, w, 64),
                 lambda: ops.ms_deform_attn_backward(value, shapes, lsi, loc, w, go, torch.zeros_like(value),
                                                     torch.zeros_like(loc), torch.zeros_like(w), 64)):
        try:
            call()
        except L.OccB200Error as e:
            assert 'im2col_step' in str(e), e
        else:
            raise AssertionError('B = 96 with im2col_step 64 was accepted')
    print('contracts: B = 96 refused with im2col_step 64')

    # B * Nq = 0: nothing written
    Lb, lib = _lib()
    for B, Nq in ((0, 5), (3, 0)):
        o, gv, gl, ga = Guarded((64,)), Guarded((64,), fill=PAT32), Guarded((64,)), Guarded((64,))
        v = torch.zeros(64, device=DEV)
        sh, ls = torch.tensor([[2, 2]], device=DEV), torch.tensor([0], device=DEV)
        Lb.check(lib.occb200_ms_deform_attn_forward(_p(v), _p(sh), _p(ls), _p(v), _p(v), B, 4, 1, 8, Nq, 1, 1, 64, o.ptr(),
                                                    Lb.stream_ptr()))
        Lb.check(lib.occb200_ms_deform_attn_backward(_p(v), _p(sh), _p(ls), _p(v), _p(v), _p(v), B, 4, 1, 8, Nq, 1, 1, 64,
                                                     gv.ptr(), gl.ptr(), ga.ptr(), Lb.stream_ptr()))
        torch.cuda.synchronize()
        assert o.untouched() and gv.untouched() and gl.untouched() and ga.untouched(), f'B {B} Nq {Nq}: something was written'
    print('contracts: B * Nq = 0 writes nothing')

    # misaligned value (ops and the C ABI) and misaligned out run the per-channel kernel: the aligned result exactly
    value, shapes, lsi, loc, w, go = make_exact(2, 300, 8, 32, [(8, 16), (4, 8)], 4, seed=304)
    ref = forward(value, shapes, lsi, loc, w, tag='aligned')
    for voff, ooff in ((1, 0), (0, 1), (2, 3), (0, 4)):
        got = forward(value, shapes, lsi, loc, w, value_offset=voff, out_offset=ooff, tag=f'value +{voff}, out +{ooff} floats')
        bad = _exact_bits(got) != _exact_bits(ref)
        if bool(bad.any()):
            raise AssertionError(_named(f'value offset {voff}, out offset {ooff} floats', bad, OUT_NAMES, got, ref))
    buf = torch.empty(value.numel() + 1, device=DEV)
    view = buf[1:].view(value.shape)
    view.copy_(value)
    assert view.data_ptr() % 16 != 0 and view.is_contiguous()
    got = ops.ms_deform_attn_forward(view, shapes, lsi, loc, w, 64)
    assert torch.equal(_exact_bits(got), _exact_bits(ref)), 'ops on a misaligned value view differs'
    print('contracts: misaligned value and out give the aligned result exactly')

    # the autograd Function on fp16 / bf16 inputs, non-contiguous upstream gradient
    value, shapes, lsi, loc, w, go = make_exact(2, 50, 4, 16, [(8, 8), (4, 4)], 4, seed=305)
    go_nc = torch.empty(2, 50, 128, device=DEV)[..., ::2]
    go_nc.copy_(go)
    assert not go_nc.is_contiguous()
    gv32, gl32, ga32 = torch.zeros_like(value), torch.zeros_like(loc), torch.zeros_like(w)
    ops.ms_deform_attn_backward(value, shapes, lsi, loc, w, go, gv32, gl32, ga32, 64)
    for dt in (torch.float16, torch.bfloat16):
        vd, ld, wd = (t.to(dt).requires_grad_(True) for t in (value, loc, w))
        out = ops.MultiScaleDeformableAttnFunction_fp32.apply(vd, shapes, lsi, ld, wd, 64)
        assert out.dtype == torch.float32
        # the dyadic operands survive the cast to fp16 / bf16 only where they fit; the fp32 op on the cast inputs is the want
        v32, l32, w32 = vd.detach().float(), ld.detach().float(), wd.detach().float()
        gv_w, gl_w, ga_w = torch.zeros_like(v32), torch.zeros_like(l32), torch.zeros_like(w32)
        ops.ms_deform_attn_backward(v32, shapes, lsi, l32, w32, go, gv_w, gl_w, ga_w, 64)
        out.backward(go_nc)
        for got, want, nm in ((vd.grad, gv_w, 'value'), (ld.grad, gl_w, 'sampling_locations'),
                              (wd.grad, ga_w, 'attention_weights')):
            assert got.dtype == dt, f'{dt}: grad of {nm} is {got.dtype}'
            assert torch.equal(got, want.to(dt)), f'{dt}: grad of {nm} differs from the fp32 op cast to {dt}'
    print('contracts: fp16 / bf16 inputs get gradients of their dtype, equal to the fp32 op cast')


# ---- (d) ops.linear and ops.layer_norm
LIN_SHAPES = [(256, 256, 0, False), (512, 256, 1, False), (256, 512, 0, True), (128, 512, 0, False), (64, 512, 0, False)]


def check_linear_layernorm():
    from occnet_b200 import ops
    from test_gemm_tc_gpu import LN_TOL
    M = 40000
    worst = {}
    for i, (N, K, act, res) in enumerate(LIN_SHAPES):
        g = torch.Generator(device=DEV).manual_seed(400 + i)
        x = torch.randn(M, K, device=DEV, generator=g) * 2.0 ** torch.randint(-3, 4, (K,), device=DEV, generator=g)
        W = torch.randn(N, K, device=DEV, generator=g) * K ** -0.5
        b = torch.randn(N, device=DEV, generator=g)
        r = torch.randn(M, N, device=DEV, generator=g) * 4 if res else None
        with torch.no_grad():
            got = ops.linear(x.view(8, M // 8, K), W, b, r, act).reshape(M, N)
        F64 = x.double() @ W.double().t() + b.double()
        if act:
            F64 = F64.clamp_min(0)
        if res:
            F64 = F64 + r.double()
        S = x.double().abs() @ W.double().abs().t()
        bound = K * U23 * S + U23 * (S + b.double().abs())
        if res:
            bound = bound + U23 * (S + b.double().abs() + r.double().abs())
        tag = f'linear M {M} N {N} K {K} relu {act} residual {res}'
        worst[tag] = check_bound(got, F64, 1.001 * bound, tag, ('row', 'column'))
        print(f'{tag}: largest err/bound {worst[tag]:.3f}')
        del F64, S, bound
        if i == 2:          # misaligned views of every operand: the bits of aligned copies
            def mis(t):
                buf = torch.empty(t.numel() + 1, device=DEV)
                v = buf[1:].view(t.shape)
                v.copy_(t)
                assert v.data_ptr() % 16 != 0
                return v
            with torch.no_grad():
                got2 = ops.linear(mis(x), mis(W), mis(b), mis(r), act)
            assert torch.equal(got2.view(torch.int32), got.view(torch.int32)), f'{tag}: misaligned operands differ'
    g = torch.Generator(device=DEV).manual_seed(450)
    x = torch.randn(M, 256, device=DEV, generator=g) * 3 + torch.randn(M, 1, device=DEV, generator=g) * 8
    gamma = 0.5 + 1.5 * torch.rand(256, device=DEV, generator=g)
    beta = torch.rand(256, device=DEV, generator=g) * 2 - 1
    with torch.no_grad():
        y = ops.layer_norm(x.view(4, M // 4, 256), gamma, beta).view(M, 256)
    x64 = x.double()
    mu = x64.mean(1, keepdim=True)
    y64 = (x64 - mu) / torch.sqrt(((x64 - mu) ** 2).mean(1, keepdim=True) + 1e-5) * gamma.double() + beta.double()
    err = (y.double() - y64).abs()
    bad = ~(err <= LN_TOL)
    if bool(bad.any()):
        raise AssertionError(_named(f'layer_norm: |y - y64| > {LN_TOL}', bad, ('row', 'column'), y, y64))
    print(f'layer_norm M {M} C 256: largest |y - y64| {float(err.max()):.2e} (bar {LN_TOL})')

    def mis(t):
        buf = torch.empty(t.numel() + 2, device=DEV)
        v = buf[2:].view(t.shape)
        v.copy_(t)
        return v
    with torch.no_grad():
        y2 = ops.layer_norm(mis(x), mis(gamma), mis(beta))
    assert torch.equal(y2.view(torch.int32), y.view(torch.int32)), 'layer_norm: misaligned operands differ'
    print('linear / layer_norm: misaligned views give the bits of aligned copies')


# ---- (e) the wrappers' argument checks
def check_wrapper_rejections():
    from occnet_b200 import ops
    v = torch.zeros(2, 20, 2, 8, device=DEV)
    sh = torch.tensor([[4, 4], [2, 2]], device=DEV)
    ls = torch.tensor([0, 16], device=DEV)
    loc = torch.zeros(2, 3, 2, 2, 1, 2, device=DEV)
    w = torch.zeros(2, 3, 2, 2, 1, device=DEV)
    go = torch.zeros(2, 3, 16, device=DEV)
    ops.ms_deform_attn_forward(v, sh, ls, loc, w, 64)
    ops.ms_deform_attn_backward(v, sh, ls, loc, w, go, torch.zeros_like(v), torch.zeros_like(loc), torch.zeros_like(w), 64)
    z = torch.zeros
    fwd_bad = {
        'value 3-D': (v[0], sh, ls, loc, w), 'loc batch': (v, sh, ls, loc[:1], w), 'loc heads': (v, sh, ls, z(2, 3, 1, 2, 1, 2, device=DEV), w),
        'loc 5-D': (v, sh, ls, loc[..., 0].contiguous(), w), 'loc last dim': (v, sh, ls, z(2, 3, 2, 2, 1, 3, device=DEV), w),
        'weights shape': (v, sh, ls, loc, z(2, 3, 2, 2, 2, device=DEV)), 'shapes rows': (v, sh[:1], ls, loc, w),
        'shapes cols': (v, z(2, 3, dtype=torch.int64, device=DEV), ls, loc, w), 'lsi length': (v, sh, ls[:1], loc, w),
        'shapes on the CPU': (v, sh.cpu(), ls, loc, w), 'lsi int32': (v, sh, ls.int(), loc, w),
        'weights fp16': (v, sh, ls, loc, w.half()),
    }
    for name, args in fwd_bad.items():
        try:
            ops.ms_deform_attn_forward(*args, 64)
        except RuntimeError:
            continue
        raise AssertionError(f'ms_deform_attn_forward accepted {name}')
    grads = (torch.zeros_like(v), torch.zeros_like(loc), torch.zeros_like(w))
    bwd_bad = {
        'grad_output shape': (z(2, 2, 16, device=DEV), *grads), 'grad_output 2-D': (go.view(6, 16), *grads),
        'grad_value shape': (go, z(2, 10, 2, 8, device=DEV), grads[1], grads[2]),
        'grad_loc shape': (go, grads[0], z(2, 2, 2, 2, 1, 2, device=DEV), grads[2]),
        'grad_attn shape': (go, grads[0], grads[1], z(2, 3, 2, 2, 2, device=DEV)), 'grad_value on the CPU': (go, grads[0].cpu(), *grads[1:]),
        'grad_output fp64': (go.double(), *grads),
    }
    for name, (g_, a, b, c) in bwd_bad.items():
        try:
            ops.ms_deform_attn_backward(v, sh, ls, loc, w, g_, a, b, c, 64)
        except RuntimeError:
            continue
        raise AssertionError(f'ms_deform_attn_backward accepted {name}')
    x = torch.zeros(8, 64, device=DEV)
    W = torch.zeros(32, 64, device=DEV)
    lin_bad = {
        'weight K': dict(weight=torch.zeros(32, 48, device=DEV)), 'weight 1-D': dict(weight=torch.zeros(64, device=DEV)),
        'weight on the CPU': dict(weight=W.cpu()), 'weight fp16': dict(weight=W.half()),
        'bias length': dict(bias=torch.zeros(16, device=DEV)), 'bias 2-D': dict(bias=torch.zeros(1, 32, device=DEV)),
        'bias on the CPU': dict(bias=torch.zeros(32)), 'bias fp64': dict(bias=torch.zeros(32, device=DEV, dtype=torch.float64)),
        'broadcast residual (1, N)': dict(residual=torch.zeros(1, 32, device=DEV)),
        'residual non-contiguous': dict(residual=torch.zeros(32, 8, device=DEV).t()),
        'residual on the CPU': dict(residual=torch.zeros(8, 32)), 'act 2': dict(act=2),
    }
    for name, kw in lin_bad.items():
        args = dict(weight=W, bias=None, residual=None, act=0)
        args.update(kw)
        try:
            ops.linear(x, **args)
        except RuntimeError:
            continue
        raise AssertionError(f'linear accepted {name}')
    xl = torch.zeros(8, 256, device=DEV)
    gm = torch.ones(256, device=DEV)
    ln_bad = {'gamma on the CPU': (gm.cpu(), gm), 'beta length': (gm, gm[:128]), 'gamma fp16': (gm.half(), gm),
              'beta non-contiguous': (gm, torch.ones(512, device=DEV)[::2]), 'gamma None': (None, gm)}
    for name, (ga_, be) in ln_bad.items():
        try:
            ops.layer_norm(xl, ga_, be)
        except (RuntimeError, TypeError):
            continue
        raise AssertionError(f'layer_norm accepted {name}')
    torch.cuda.synchronize()
    print(f'wrappers: {len(fwd_bad) + len(bwd_bad) + len(lin_bad) + len(ln_bad)} bad calls refused before any kernel')


# ---- the GPU tests
@pytest.mark.gpu
def test_msda_bit_exact_on_dyadic_operands_both_forward_kernels_and_backward():
    _child('check_exact')


@pytest.mark.gpu
def test_msda_matches_fp64_at_the_plugins_production_shapes():
    _child('check_production')


@pytest.mark.gpu
def test_msda_accumulate_overwrite_outside_empty_misaligned_and_dtype_contracts():
    _child('check_contracts')


@pytest.mark.gpu
def test_ops_linear_and_layer_norm_at_the_plugins_shapes():
    _child('check_linear_layernorm')


@pytest.mark.gpu
def test_wrappers_refuse_mismatched_arguments():
    _child('check_wrapper_rejections')
