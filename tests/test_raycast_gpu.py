"""The ray caster at its edges (raycast.cu): render_forward_kernel through occb200_render_forward and ops.render_forward, and
the three metric-grid kernels (ray_metric_kernel, ray_records_kernel, ray_score_kernel) on adversarial origins and bundles.

(a) render_forward on every family of tests/golden/dvr_edges.py (exact tMax ties in every axis pair and octant, zero and
    zero-length directions, lattice origins, origins outside every face and in the (-1, 0) truncation band, entry after
    999 / 1000 / 1001 steps, the MAX_STEP cut-off inside a 1200-voxel grid, sigma 0.5 / nextafter / 1 / NaN / inf / -1 at
    the first and the last in-grid voxel, grids 200x200x16, 7x13x200 in every axis order, 1x1x1 and 1x9x1, and N = 3
    batches with sigma T in {1, 3} x origin To in {1, 3}, K = 4 points and padded tindex).  pred_dist, gt_dist and
    coord_index must equal, byte for byte, the reference kernel's outputs stored in tests/golden/ref_dvr_edges.npz (and
    the live reference kernel when oracle/_ref holds it), and the C oracle oracle/ray_dda.c bit for bit with NaN for NaN
    (the CPU's NaN payloads are not the GPU's).  Every input and output buffer lies between NaN guards: the outputs' must
    come back unchanged, the inputs' are what a wrong stride would read.
(b) ops.render_forward: the C entry's bytes on every family, and every shape / device error refused before a kernel runs.
(c) The metric grid (200x200x16, 0.4 m) from adversarial origins -- voxel-lattice planes (the dataset's y = 0 is 100.0
    exactly), the grid's faces, outside every face, the (-1, 0) band -- with the lidar bundle plus axis-parallel,
    diagonal and zero rays, f32 and f64 origins, T up to 8: the rows of ray_metric_kernel equal process_one_sample's
    restatement bit for bit (NaN for NaN), the records of ray_records_kernel equal numpy's narrowing of those rows, and
    the integer counters of ray_metric_kernel and ray_score_kernel equal ORM.accumulate; the `ave` sums lie within
    2^-21 sum(err) of the fp64 sum of fp64 norms (fp32 norm: a few units of 2^-24 each; fp64 atomics in any order).
Each test runs its checks in a child process, so that a device fault cannot poison this session.
"""
import ctypes
import glob
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
NAN32 = 0x7FA5A5A5
GUARD = 1024
NC = 17


def _run_isolated(fn, timeout=1200):
    code = f'import sys; sys.path.insert(0, "tests"); import test_raycast_gpu as t; t.{fn}(); print("OK")'
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-20000:])
    assert r.returncode == 0 and 'OK' in r.stdout, f'child failed ({r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'


def _edges():
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import dvr_edges
    return dvr_edges


def _lib():
    from occnet_b200 import _lib as L
    return L, L.load()


class Guarded:
    """a buffer of `n` elements of `dtype` with GUARD elements of the bits `fill` on each side (and in the body)"""

    def __init__(self, body_or_shape, dtype=torch.float32, fill=NAN32):
        shape = body_or_shape.shape if isinstance(body_or_shape, np.ndarray) else tuple(body_or_shape)
        self.shape, self.n = tuple(shape), int(np.prod(shape))
        itype = {torch.float32: torch.int32, torch.float64: torch.int64, torch.int8: torch.int8, torch.float16: torch.int16}[dtype]
        self.bits = torch.full((self.n + 2 * GUARD,), fill, dtype=itype, device=DEV)
        self.fill, self.dtype = fill, dtype
        self.buf = self.bits.view(dtype)
        if isinstance(body_or_shape, np.ndarray):
            self.value().copy_(torch.from_numpy(np.ascontiguousarray(body_or_shape)).to(DEV))

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + GUARD * self.buf.element_size())

    def value(self):
        return self.buf[GUARD:GUARD + self.n].view(self.shape)

    def check_guards(self, what):
        for name, p in (('leading', self.bits[:GUARD]), ('trailing', self.bits[GUARD + self.n:])):
            bad = (p != self.fill).nonzero()
            assert bad.numel() == 0, f'{what}: {bad.numel()} elements of the {name} guard were written'


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _first_mismatch(case, what, got, want, nan_equal):
    """None, or a message naming the ray (n, m), its origin and end point, and the element"""
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    same = _bits(g) == _bits(w)
    if nan_equal:
        same |= np.isnan(g) & np.isnan(w)
    if same.all():
        return None
    idx = np.argwhere(~same)[0]
    n, m = int(idx[0]), int(idx[1])
    ti = case['tindex'][n, m]
    o = case['origin'][n, max(int(ti), 0)] if ti >= 0 else None
    el = f'{what}[{n}][{m}]' + (f'[{int(idx[2])}]' if len(idx) > 2 else '')
    i = tuple(idx)
    return (f"{case['name']}: {int((~same).sum())} elements differ; first {el}: got {float(g[i])!r} (0x{int(_bits(g)[i]):08x}), "
            f"want {float(w[i])!r} (0x{int(_bits(w)[i]):08x}); ray (n={n}, m={m}) "
            f"tindex {ti} origin {None if o is None else tuple(map(float, o))} end {tuple(map(float, case['points'][n, m, :3]))}")


def _live_reference():
    so = glob.glob(os.path.join(ROOT, 'oracle', '_ref', 'dvr_ref*.so'))
    if not so:
        return None
    spec = importlib.util.spec_from_file_location('dvr_ref', so[0])
    dvr = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dvr)
    return dvr


def _render_entry(case):
    """occb200_render_forward on guarded copies of the inputs and NaN-guarded outputs -> (pred, gt, coord) numpy"""
    L, lib = _lib()
    N, T, Z, Y, X = case['sigma'].shape
    _, M, K = case['points'].shape
    To = case['origin'].shape[1]
    ins = [Guarded(case[k]) for k in ('sigma', 'origin', 'points', 'tindex')]
    outs = [Guarded((N, M)), Guarded((N, M)), Guarded((N, M, 3))]
    L.check(lib.occb200_render_forward(*[g.ptr() for g in ins], N, T, To, Z, Y, X, M, K, *[g.ptr() for g in outs],
                                       L.stream_ptr()))
    torch.cuda.synchronize()
    for g, name in zip(outs, ('pred_dist', 'gt_dist', 'coord_index')):
        g.check_guards(f"{case['name']}: {name}")
    for g, name in zip(ins, ('sigma', 'origin', 'points', 'tindex')):
        g.check_guards(f"{case['name']}: input {name}")
    return [g.value().cpu().numpy() for g in outs]


# --------------------------------------------------------------------------------------------------- (a) render_forward
def check_render_forward_families():
    from oracle import ray_metrics as ORM
    E = _edges()
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_dvr_edges.npz'))
    dvr = _live_reference()
    print('live reference kernel:', 'yes' if dvr is not None else 'not built')
    errors = []
    for case in E.cases():
        got = _render_entry(case)
        want = ORM.render_forward(case['sigma'], case['origin'], case['points'], case['tindex'])
        ref = None
        if dvr is not None:
            T, Z, Y, X = case['sigma'].shape[1:]
            r = dvr.render_forward(*[torch.from_numpy(case[k]).to(DEV) for k in ('sigma', 'origin', 'points', 'tindex')],
                                   [T, Z, Y, X], 'test')
            torch.cuda.synchronize()
            ref = [v.cpu().numpy() for v in r]
        for i, what in enumerate(('pred_dist', 'gt_dist', 'coord_index')):
            g = gold[f"{case['name']}/{what}"]
            for src, w, nan_eq in (('stored reference', g, False), ('C oracle', want[i], True),
                                   ('live reference', None if ref is None else ref[i], False)):
                if w is None:
                    continue
                msg = _first_mismatch(case, what, got[i], w, nan_eq)
                if msg:
                    errors.append(f'vs {src}: {msg}')
            msg = _first_mismatch(case, what, g, want[i], True)            # pins the C oracle against the stored reference
            if msg:
                errors.append(f'C oracle vs stored reference: {msg}')
        print(f"{case['name']}: {case['points'].shape[0] * case['points'].shape[1]} rays, "
              f"{int((got[0] != -1).sum())} entered the grid")
    assert not errors, '\n'.join(errors[:20])


def test_render_forward_families_match_the_reference_and_the_oracle():
    _run_isolated('check_render_forward_families')


# ------------------------------------------------------------------------------------------------ (b) ops.render_forward
def check_render_forward_wrapper():
    from occnet_b200 import ops
    E = _edges()
    for case in E.cases():
        T, Z, Y, X = case['sigma'].shape[1:]
        want = _render_entry(case)
        got = ops.render_forward(*[torch.from_numpy(case[k]).to(DEV) for k in ('sigma', 'origin', 'points', 'tindex')],
                                 [T, Z, Y, X], 'test')
        for i, what in enumerate(('pred_dist', 'gt_dist', 'coord_index')):
            msg = _first_mismatch(case, what, got[i].cpu().numpy(), want[i], False)
            assert msg is None, 'ops.render_forward vs the C entry: ' + msg
    # every shape / device / dtype error is refused before a kernel runs
    s = torch.zeros(2, 1, 4, 5, 6, device=DEV)
    o = torch.zeros(2, 3, 3, device=DEV)
    p = torch.zeros(2, 7, 4, device=DEV)
    ti = torch.zeros(2, 7, device=DEV)
    g = [1, 4, 5, 6]
    bad = [
        ((s, o, p, ti, [2, 4, 5, 6]), 'sigma has shape'), ((s, o, p, ti, [1, 4, 5]), 'grid'),
        ((s, o, p, ti, [1, 4, 5, 7]), 'sigma has shape'), ((s[:1], o, p, ti, g), 'sigma has shape'),
        ((s, o[:1], p, ti, g), 'origin must be'), ((s, o[:, :, :2].contiguous(), p, ti, g), 'origin must be'),
        ((s, o[:, :0], p, ti, g), 'origin must be'), ((s, o[0], p, ti, g), 'origin must be'),
        ((s, o, p[:, :, :2].contiguous(), ti, g), 'K >= 3'), ((s, o, p[0], ti, g), 'points must be'),
        ((s, o, p, ti[:, :6].contiguous(), g), 'tindex has shape'), ((s, o, p, ti[0], g), 'tindex has shape'),
        ((s, o, p, ti.double(), g), 'tindex must be'), ((s, o.cpu(), p, ti, g), 'CUDA'),
        ((s, o, p[:, :, :3], ti, g), 'contiguous'), ((s, o, p, ti, g, 'train'), 'PHASE'),
    ]
    if torch.cuda.device_count() > 1:
        bad.append(((s, o.to('cuda:1'), p, ti, g), 'one device'))
    for args, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            ops.render_forward(*args)
    torch.cuda.synchronize()
    print(f'{len(bad)} wrapper rejections')


def test_render_forward_wrapper_equals_the_entry_and_refuses_bad_shapes():
    _run_isolated('check_render_forward_wrapper')


# ------------------------------------------------------------------------------------------------ (c) the metric kernels
OFF = np.float32([-40, -40, -1])


def adversarial_origins():
    """origins in metres: voxel-lattice planes (y = 0 -> 40 / 0.4f = 100.0), the grid's faces, outside every face, the
    (-1, 0) band (x = -40.2 -> -0.5), and one inside off the lattice"""
    o = np.array([[0.98, 0.0, 1.84], [-40.0, 0.0, -1.0], [0.0, 0.0, 0.6], [-40.2, 3.1, 1.9], [12.3, 40.0, 2.2],
                  [-55.0, -47.0, 1.84], [3.3, -2.1, -1.3], [20.0, 45.0, 9.0]], np.float64)
    lat = ((o[:3].astype(np.float32) - OFF) / np.float32(0.4)).astype(np.float32)
    assert lat[0, 1] == 100.0 and (lat[1] == [0, 100, 0]).all() and lat[2, 0] == 100.0
    band = (np.float32(o[3, 0]) - OFF[0]) / np.float32(0.4)
    assert -1 < band < 0
    return o


def adversarial_rays():
    """the lidar bundle, then axis-parallel rays (both signs), xy / xz / yz / xyz diagonals with equal components (exact
    tMax ties from origins whose coordinates share their fraction), long rays, and the zero ray (a zero-length walk)"""
    from oracle import ray_metrics as ORM
    extra = []
    for k in range(3):
        for s in (1.0, -1.0):
            v = [0.0, 0.0, 0.0]; v[k] = s * 30.0
            extra.append(v)
    for sx in (1.0, -1.0):
        for sy in (1.0, -1.0):
            for sz in (1.0, -1.0):
                extra += [[sx * 10.0, sy * 10.0, 0.0], [sx * 10.0, 0.0, sz * 10.0], [0.0, sy * 10.0, sz * 10.0],
                          [sx * 4.0, sy * 4.0, sz * 4.0], [sx * 80.0, sy * 40.0, sz * 0.5]]
    extra.append([0.0, 0.0, 0.0])
    return np.concatenate([ORM.generate_lidar_rays(), np.asarray(extra, np.float32)]).astype(np.float32)


def _rows_restated(sem, flow, rays, orig):
    """process_one_sample's rows: its own float32 arithmetic, or with float64 origins the torch promotion restated in numpy
    (as tests/test_gpu_parity.py::test_ray_metric_counters_match_oracle does)"""
    from oracle import ray_metrics as ORM
    if orig.dtype != np.float64:
        return ORM.process_one_sample(sem, rays, orig, flow)
    T = orig.shape[1]
    lid = rays[None].astype(np.float64) + orig[:, :, None, :].reshape(1, T, 1, 3)
    off = OFF.astype(np.float64); sc = np.float64(np.float32(0.4))
    occ = np.ascontiguousarray(np.where(sem < 16, 1, 0).astype(np.float32).transpose(2, 1, 0))[None]
    out = []
    for t in range(T):
        o = ((orig[0, t] - off) / sc).astype(np.float32)
        p = ((lid[0, t] - off) / sc).astype(np.float32)
        pd, _, ci = ORM.render_forward(occ, o[None], p, np.zeros(len(rays), np.float32))
        ci = ci.astype(np.int32)
        out.append(np.concatenate([sem[ci[:, 0], ci[:, 1], ci[:, 2]].astype(np.float32)[:, None],
                                   (pd * np.float32(0.4))[:, None], flow[ci[:, 0], ci[:, 1], ci[:, 2]]], -1))
    return np.concatenate(out).astype(np.float32)


def _rows_equal(got, want, what):
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    same = (_bits(g) == _bits(w)) | (np.isnan(g) & np.isnan(w))
    if not same.all():
        i, c = np.argwhere(~same)[0]
        raise AssertionError(f'{what}: {int((~same).sum())} elements differ; first row {i} (origin {i // what[1]}, ray '
                             f'{i % what[1]}) column {c}: got {g[i]} want {w[i]}')


def _ave_sums(pp, pg):
    """per (threshold, class) the fp64 sum of the fp64 norms of the fp32 flow differences of the true positives"""
    from oracle import ray_metrics as ORM
    exact = np.zeros((3, NC))
    l1 = np.abs(pp[:, 1] - pg[:, 1])
    err = np.sqrt(((pg[:, 2:4] - pp[:, 2:4]).astype(np.float64) ** 2).sum(1))
    for j, thr in enumerate(ORM.THRESHOLDS):
        for i in range(ORM.FLOW_CLASSES):
            exact[j, i] = err[(pp[:, 0] == i) & (pg[:, 0] == i) & (l1 < thr)].sum()
    return exact


def check_metric_kernels():
    from oracle import ray_metrics as ORM
    L, lib = _lib()
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from test_score_gpu import metric_fixture
    sem_pred, flow_pred, sem_gt, flow_gt = metric_fixture()
    dev = [torch.from_numpy(a).to(DEV).contiguous() for a in (sem_pred, flow_pred, sem_gt, flow_gt)]
    rays = adversarial_rays()
    M = rays.shape[0]
    rays_d = torch.from_numpy(rays).to(DEV)
    allo = adversarial_origins()
    for dtype in (np.float32, np.float64):
        for T, pick in ((1, [0]), (3, [1, 3, 5]), (8, list(range(8)))):
            orig = np.ascontiguousarray(allo[pick][None], dtype)
            is64 = int(dtype == np.float64)
            what = (f'{np.dtype(dtype).name} origins, T={T}', M)
            o_dev = Guarded(orig[0], torch.float64 if is64 else torch.float32, fill=0x7FF4A5A5A5A5A5A5 if is64 else NAN32)
            pcd = [Guarded((T * M, 4)), Guarded((T * M, 4))]
            cnt = Guarded((187,), torch.float64, fill=0)
            L.check(lib.occb200_ray_metric_accumulate(*[L.ptr(t) for t in dev], o_dev.ptr(), is64, T, L.ptr(rays_d), M,
                                                      cnt.ptr(), pcd[0].ptr(), pcd[1].ptr(), L.stream_ptr()))
            torch.cuda.synchronize()
            for g, nm in zip(pcd + [cnt], ('pcd_pred', 'pcd_gt', 'counters')):
                g.check_guards(f'{what[0]}: {nm}')
            pp, pg = (g.value().cpu().numpy() for g in pcd)
            want_p = _rows_restated(sem_pred, flow_pred, rays, orig)
            want_g = _rows_restated(sem_gt, flow_gt, rays, orig)
            _rows_equal(pp, want_p, (what[0] + ' ray_metric_kernel pred rows', M))
            _rows_equal(pg, want_g, (what[0] + ' ray_metric_kernel gt rows', M))
            # the records: numpy's narrowing of the kernel's own rows
            rec = [Guarded((T * M,), torch.int8, fill=0x5A), Guarded((T * M,), torch.float16, fill=0x7E5A),
                   Guarded((T * M, 2), torch.float16, fill=0x7E5A)]
            L.check(lib.occb200_ray_records(L.ptr(dev[0]), L.ptr(dev[1]), L.ptr(orig[0]), is64, T, L.ptr(rays_d), M,
                                            *[g.ptr() for g in rec], L.stream_ptr()))
            torch.cuda.synchronize()
            for g, nm in zip(rec, ('cls', 'dist', 'flow')):
                g.check_guards(f'{what[0]}: records {nm}')
            cls, dist, fl = (g.value().cpu().numpy() for g in rec)
            for nm, g, w in (('cls', cls, pp[:, 0].astype(np.int8)), ('dist', dist.view(np.uint16), pp[:, 1].astype(np.float16).view(np.uint16)),
                             ('flow', fl.view(np.uint16), pp[:, 2:4].astype(np.float16).view(np.uint16))):
                if not np.array_equal(g, w):
                    i = int(np.argwhere(g != w)[0][0])
                    raise AssertionError(f'{what[0]}: ray_records_kernel {nm} row {i} (origin {i // M}, ray {i % M}): '
                                         f'got {g[i]} want {w[i]} from row {pp[i]}')
            # the counters: ray_metric_kernel's and ray_score_kernel's against ORM.accumulate on the restated rows
            valid = want_g[:, 0].astype(np.int32) != 16
            vec = ORM.counters_to_vector(ORM.accumulate(ORM.new_counters(), want_p[valid], want_g[valid]))
            exact = _ave_sums(want_p[valid], want_g[valid])
            lim = 2.0 ** -21 * exact
            sc = Guarded((187,), torch.float64, fill=0)
            L.check(lib.occb200_ray_score(*[L.ptr(t) for t in dev], L.ptr(orig[0]), is64, T, L.ptr(rays_d), M, sc.ptr(),
                                          L.stream_ptr()))
            torch.cuda.synchronize()
            sc.check_guards(f'{what[0]}: score counters')
            for nm, got in (('ray_metric_kernel', cnt.value().cpu().numpy()), ('ray_score_kernel', sc.value().cpu().numpy())):
                ints = np.r_[0:5 * NC, 8 * NC:11 * NC]
                bad = ints[got[ints] != vec[ints]]
                assert bad.size == 0, f'{what[0]}: {nm} counter {bad[0]}: got {got[bad[0]]} want {vec[bad[0]]}'
                ave = got[5 * NC:8 * NC].reshape(3, NC)
                assert (np.abs(ave - exact) <= lim).all(), (what[0], nm, np.abs(ave - exact).max())
                assert (np.abs(vec[5 * NC:8 * NC].reshape(3, NC) - exact) <= 2.0 ** -18 * exact).all()  # the oracle's fp32 sums
            print(f'{what[0]}: {T * M} rays, {int(valid.sum())} counted, rows / records / counters ok; '
                  f'ave err/bound {(np.abs(cnt.value().cpu().numpy()[5 * NC:8 * NC].reshape(3, NC) - exact) / np.maximum(lim, 1e-300)).max():.3f}')


def test_metric_kernels_on_adversarial_origins_and_bundles():
    _run_isolated('check_metric_kernels')
