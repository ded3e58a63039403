"""Ray-caster edge cases for `dvr.render_forward` ("test" phase) and a logging restatement of its walk.

The reference's traversal (tools/ray_iou/lib/dvr/dvr.cu:69-319, restated in oracle/ray_dda.c) goes wrong, if anywhere,
where its geometry is degenerate: exact tMax ties between axes (`<` against `<=` picks the voxel), axis-parallel and
zero-length rays, origins on lattice planes, origins outside the grid (between voxel coordinates -1 and 0, `int(xo)`
truncates towards the grid), the MAX_STEP = 1000 cut-off before and after the ray enters, sigma exactly 0.5, NaN and
inf, and grids whose three sizes differ.  `cases()` builds those families from closed forms and fixed seeds;
`walk()` restates the walk in Python doubles and logs every branch, so that `check_claims()` can prove each family
produces what it claims (tests/test_raycast_cpu.py).  tests/golden/gen_dvr_edges.py stores the reference kernel's
outputs for these inputs in ref_dvr_edges.npz; the inputs themselves are regenerated here, never stored.

A case is one render_forward call: sigma (N,T,Z,Y,X), origin (N,To,3), points (N,M,K), tindex (N,M) float32, and
`claims`: {(n, m): [tag, ...]} for the rays whose walk a family builds on purpose.  Tags:
  tie:xy / tie:xz / tie:yz / tie:xyz   an exact tie of those tMax values (finite) at a decision made inside the grid
  zero:<k>          k direction components are exactly 0 (the DBL_MAX branch); zero:len is a zero-length ray (NaN steps)
  face              the end point lies exactly on a voxel face
  lattice           the origin has an integer voxel coordinate
  outside:<face>    the origin lies outside the grid beyond that face (x-, x+, y-, y+, z-, z+)
  band              an origin coordinate lies in (-1, 0) and the start voxel int(o) is inside the grid
  entry:<s>         the walk is first inside after exactly s steps (999, 1000); entry:never -- it never is
  cut               the walk is still inside the grid when MAX_STEP ends it
  hit:first / hit:last   the first voxel with sigma > 0.5 is the first / the last in-grid voxel of the walk
  miss:<v>          the walk passes a voxel holding v (0.5, nan, -1) and hits nothing
  padded            tindex < 0: the outputs keep their -1 / 0 defaults
"""
import math
import sys
from fractions import Fraction

import numpy as np

MAX_STEP = 1000
DBL_MAX = sys.float_info.max
NEXT_HALF = float(np.nextafter(np.float32(0.5), np.float32(1)))


def _div(a, b):
    """IEEE double a / b (Python raises on a zero divisor)"""
    if b != 0 or math.isnan(b):
        return a / b
    if a == 0 or math.isnan(a):
        return math.nan
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def _fma(a, b, c):
    """correctly rounded a * b + c of finite doubles"""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def walk(o, e, size, occupied):
    """The reference's walk from voxel-unit origin o to end point e (float32 triples) through a grid of size (X, Y, Z);
    occupied(x, y, z) is sigma > 0.5.  Returns the outputs (pred_dist, gt_dist, coord as float32, or None when the ray
    never enters) and the log: entry step, in-grid count, hit index, exit reason and, per decision made inside the grid,
    the set of exact finite ties among the tMax values."""
    xo, yo, zo = (float(v) for v in o)
    xe, ye, ze = (float(v) for v in e)
    X, Y, Z = size
    v = [int(xo), int(yo), int(zo)]
    r = [xe - xo, ye - yo, ze - zo]
    gt_d = math.sqrt(_fma(r[2], r[2], _fma(r[1], r[1], r[0] * r[0])))     # nvcc contracts the norm (oracle/ray_dda.c)
    d = [_div(c, gt_d) for c in r]
    step_ = [1 if c >= 0 else -1 for c in d]
    o3 = (xo, yo, zo)
    tmax = [_div((v[k] + (0 if step_[k] < 0 else 1)) - o3[k], d[k]) if d[k] != 0 else DBL_MAX for k in range(3)]
    tdelta = [_div(step_[k], d[k]) if d[k] != 0 else DBL_MAX for k in range(3)]
    log = dict(entry=None, count=0, hit=None, exit='max_step', ties=[], inside0=None, zero=sum(c == 0 for c in d))
    step, count, was_inside = 0, 0, False
    hit = last = None
    while True:
        inside = 0 <= v[0] < X and 0 <= v[1] < Y and 0 <= v[2] < Z
        if log['inside0'] is None:
            log['inside0'] = inside
        cur = tuple(v)
        if inside:
            if not was_inside:
                log['entry'] = step
            was_inside = True
        elif was_inside:
            log['exit'] = 'left'
            break
        tx, ty, tz = tmax
        if inside:
            ties = set()
            for name, a, b in (('xy', tx, ty), ('xz', tx, tz), ('yz', ty, tz)):
                if a == b and a < DBL_MAX:
                    ties.add(name)
            if {'xy', 'xz', 'yz'} <= ties:
                ties.add('xyz')
            log['ties'].append(ties)
        if tx < ty:
            k = 0 if tx < tz else 2
        else:
            k = 1 if ty < tz else 2
        dist = tmax[k]
        v[k] += step_[k]
        tmax[k] += tdelta[k]
        if inside:
            last = (dist, cur)
            if hit is None and occupied(*cur):
                hit = (dist, cur)
                log['hit'] = count
            count += 1
        step += 1
        if step > MAX_STEP:
            log['cut_inside'] = inside
            break
    log['count'] = count
    if count == 0:
        return None, log
    dist, cur = hit if hit is not None else last
    return (np.float32(dist), np.float32(gt_d), np.float32(cur)), log


def _occupied(sigma_ntzyx, n, ts):
    s = sigma_ntzyx[n, ts]
    return lambda x, y, z: float(s[z, y, x]) > 0.5


def walk_case(case):
    """walk() for every ray of a case -> {(n, m): (outputs, log)}, the padded rays included (outputs None, log None)"""
    sig, org, pts, ti = case['sigma'], case['origin'], case['points'], case['tindex']
    N, T, Z, Y, X = sig.shape
    out = {}
    for n in range(N):
        for m in range(pts.shape[1]):
            if ti[n, m] < 0:
                out[(n, m)] = (None, None)
                continue
            t = int(ti[n, m])
            out[(n, m)] = walk(org[n, t], pts[n, m, :3], (X, Y, Z), _occupied(sig, n, 0 if T == 1 else t))
    return out


# ------------------------------------------------------------------------------------------------------------ families
def _rays_case(name, sigma_zyx, rays, K=3):
    """rays with their own origins through one static grid: N = 1, sigma T = 1, origin To = len(rays), ray m walks from
    origin[0][m] (tindex m) -- the reference's static-sigma, many-origins case.  rays: [(origin, end, tags)].  K > 3 pads
    each point with NaN columns that must not be read."""
    R = len(rays)
    pts = np.full((1, R, K), np.nan, np.float32)
    pts[0, :, :3] = np.asarray([r[1] for r in rays], np.float32)
    claims = {(0, i): list(r[2]) for i, r in enumerate(rays) if r[2]}
    return dict(name=name, sigma=np.asarray(sigma_zyx, np.float32)[None, None],
                origin=np.asarray([r[0] for r in rays], np.float32)[None], points=pts,
                tindex=np.arange(R, dtype=np.float32)[None], claims=claims)


def _bundle_case(name, sigma_zyx, origin, ends, tags, K=3):
    """one origin, M end points (N = 1, T = To = 1); tags per ray"""
    M = len(ends)
    pts = np.full((1, M, K), np.nan, np.float32)
    pts[0, :, :3] = np.asarray(ends, np.float32)
    claims = {(0, m): list(tg) for m, tg in enumerate(tags) if tg}
    return dict(name=name, sigma=np.asarray(sigma_zyx, np.float32)[None, None], origin=np.asarray(origin, np.float32)[None, None],
                points=pts, tindex=np.zeros((1, M), np.float32), claims=claims)


def _random_sigma(shape_zyx, density, seed):
    rng = np.random.RandomState(seed)
    return (rng.rand(*shape_zyx) < density).astype(np.float32)


_OCTANTS = [(sx, sy, sz) for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)]


def _tie_rays(size, kind, L, starts):
    """rays whose direction makes the `kind` tMax values tie: equal components (ratio 1:1) or 1:2, the other component
    chosen not to tie, in all 8 octants, from origins at voxel corners, edges and half-integers"""
    X, Y, Z = size
    rays = []
    axes = {'xy': (0, 1), 'xz': (0, 2), 'yz': (1, 2), 'xyz': (0, 1, 2)}[kind]
    for ratio in (1, 2):
        for octant in _OCTANTS:
            for o in starts:
                dvec = [0.3125, 0.3125, 0.3125]            # the third axis: 5/16, which never ties with 1 or 1/2 from these starts
                for i, a in enumerate(axes):
                    dvec[a] = 1.0 if (i == 0 or ratio == 1) else 0.5
                e = [o[k] + octant[k] * dvec[k] * L for k in range(3)]
                # ties recur when the tied axes start at the same offset from their next faces; at 1:2 only from faces
                # (offsets h and 2h then meet at 2h, 4h, ...; from half-integers they are h/2 (2k+1) and h (2j+1))
                same = len({o[a] % 1 for a in axes}) == 1 and (ratio == 1 or o[axes[0]] % 1 == 0)
                rays.append((o, e, ['tie:' + kind] if same else []))
    return rays


def cases():
    out = []
    # ---- ties, on the metric grid (200 x 200 x 16) and on a grid with three different sizes
    for size, L in (((200, 200, 16), 12.0), ((13, 7, 11), 6.0)):
        X, Y, Z = size
        cx, cy, cz = X // 2, Y // 2, Z // 2
        starts = [(cx, cy, cz), (cx + 0.5, cy + 0.5, cz + 0.5), (cx, cy, cz + 0.5), (cx + 0.5, cy, cz), (cx, cy + 0.5, cz)]
        sig = _random_sigma((Z, Y, X), 0.12, seed=11 + X)
        for kind in ('xy', 'xz', 'yz', 'xyz'):
            rays = _tie_rays(size, kind, L, starts)
            out.append(_rays_case(f'tie_{kind}_{X}x{Y}x{Z}', sig, rays))
    # ---- degenerate directions: one and two zero components, both signs; zero-length rays; ends exactly on a face
    size = (13, 7, 11)
    sig = _random_sigma((11, 7, 13), 0.1, seed=5)
    o = (6.3, 3.6, 5.2)
    rays = []
    for k in range(3):
        for s in (1, -1):
            e = list(o); e[k] += s * 9.0
            rays.append((o, e, ['zero:2']))
            for j in range(3):
                if j != k:
                    for s2 in (1, -1):
                        e2 = list(e); e2[j] += s2 * 4.5
                        rays.append((o, e2, ['zero:1']))
    for zo in ((6.3, 3.6, 5.2), (6.0, 3.0, 5.0), (0.0, 0.0, 0.0), (12.5, 6.5, 10.5)):
        rays.append((zo, zo, ['zero:len']))
    for e in ((13.0, 3.6, 5.2), (6.3, 0.0, 5.2), (6.3, 3.6, 11.0), (9.0, 5.0, 7.0), (0.0, 3.6, 5.2), (6.3, 7.0, 0.0)):
        rays.append((o, e, ['face']))
    out.append(_rays_case('degenerate_13x7x11', sig, rays))
    # ---- origins on lattice planes (the dataset's y = 0 lidar origin is 40 / 0.4f = 100.0 exactly)
    sig = _random_sigma((16, 200, 200), 0.05, seed=7)
    rng = np.random.RandomState(8)
    dirs = rng.normal(size=(24, 3)); dirs[:, 2] *= 0.2
    lat = [(100.0, 100.0, 7.0), (100.0, 73.4, 7.3), (51.7, 100.0, 7.3), (51.7, 73.4, 7.0), (0.0, 0.0, 0.0), (199.0, 37.0, 15.0)]
    rays = [(lo, tuple(np.float32(lo) + np.float32(dv * 30)), ['lattice']) for lo in lat for dv in dirs]
    out.append(_rays_case('lattice_200x200x16', sig, rays))
    # ---- origins outside each face, and in the (-1, 0) truncation band of each axis
    size = (13, 7, 11)
    sig = _random_sigma((11, 7, 13), 0.08, seed=9)
    X, Y, Z = size
    rays = []
    mid = (6.4, 3.3, 5.6)
    for k, (lo, hi) in enumerate(((-3.7, X + 2.2), (-4.1, Y + 1.6), (-2.6, Z + 3.3))):
        for far, face in ((lo, '-'), (hi, '+')):
            o = list(mid); o[k] = far
            for jit in ((0, 0, 0), (0.7, -0.4, 0.9), (-1.3, 0.8, -0.6)):
                e = [mid[j] + jit[j] for j in range(3)]
                rays.append((tuple(o), tuple(e), ['outside:' + 'xyz'[k] + face]))
            rays.append((tuple(o), tuple(2 * o[j] - mid[j] for j in range(3)), ['outside:' + 'xyz'[k] + face]))  # away
        for b in (-0.5, -0.25, -2.0 ** -20, -1.0 + 2.0 ** -10):
            o = list(mid); o[k] = b
            for e in (mid, tuple(m if j != k else -5.0 for j, m in enumerate(mid)),
                      tuple(m if j != k else b - 0.375 for j, m in enumerate(mid)), (mid[0] + 1.5, mid[1] - 2.5, mid[2] + 0.5)):
                rays.append((tuple(o), tuple(e), ['band']))
    out.append(_rays_case('outside_13x7x11', sig, rays))
    # ---- the MAX_STEP cut-off before the ray enters: first inside after exactly 999 and 1000 steps, never after 1001
    sig = _random_sigma((11, 7, 13), 0.0, seed=0)
    sig[5, 3, :] = 0.0
    rays = []
    for k in range(3):
        n = (X, Y, Z)[k]
        for s, tag in ((999, 'entry:999'), (1000, 'entry:1000'), (1001, 'entry:never')):
            for sign in (1, -1):
                o = [6.5, 3.5, 5.5]
                o[k] = -s - 0.5 if sign > 0 else n - 1 + s + 0.5           # int() truncates: voxel -s / n - 1 + s
                e = list(o); e[k] += sign * 2000.0
                rays.append((tuple(o), tuple(e), [tag]))
    out.append(_rays_case('max_step_entry_13x7x11', sig, rays))
    # ---- the cut-off inside: an in-grid path longer than MAX_STEP (X = 1200)
    sig = np.zeros((2, 3, 1200), np.float32)
    sig[1, 2, 1100] = 1.0
    rays = [((0.5, 0.5, 0.5), (1199.5, 0.5, 0.5), ['cut']), ((1199.5, 2.5, 1.5), (0.5, 2.5, 1.5), ['cut']),
            ((0.25, 1.5, 1.5), (1199.9, 1.5, 1.5), ['cut']), ((0.5, 2.5, 1.5), (1199.5, 2.5, 1.5), ['cut']),
            ((1150.5, 0.5, 0.5), (0.5, 0.5, 0.5), []), ((0.5, 0.5, 0.5), (1199.5, 2.5, 1.9), [])]
    out.append(_rays_case('cut_inside_1200x3x2', sig, rays))
    # ---- grids: X != Y != Z in each axis order, 1 x 1 x 1, 1 x Y x 1
    rng = np.random.RandomState(21)
    for size in ((7, 13, 200), (200, 7, 13), (13, 200, 7)):
        X, Y, Z = size
        sig = _random_sigma((Z, Y, X), 0.03, seed=X + 2 * Y)
        o = (X / 2 + 0.3, Y / 2 - 0.2, Z / 2 + 0.1)
        ends = [tuple(np.float32(o) + np.float32(dv * 260)) for dv in rng.normal(size=(48, 3))]
        ends += [(X - 0.5, Y - 0.5, Z - 0.5), (0.5, 0.5, 0.5), (X + 40.0, o[1], o[2]), (o[0], Y + 40.0, o[2]), (o[0], o[1], Z + 40.0)]
        out.append(_bundle_case(f'grid_{X}x{Y}x{Z}', sig, o, ends, [[]] * len(ends)))
    for size, sig in (((1, 1, 1), np.zeros((1, 1, 1), np.float32)), ((1, 9, 1), np.zeros((1, 9, 1), np.float32))):
        X, Y, Z = size
        if Y > 1:
            sig[0, 6, 0] = 1.0
        rays = [((0.5, 0.5, 0.5), (0.5, 0.5, 7.0), []), ((0.5, 0.5, 0.5), (-3.0, 2.5, 0.5), []), ((-0.5, -0.5, -0.5), (3.0, 8.0, 3.0), ['band']),
                ((0.5, Y + 2.5, 0.5), (0.5, -3.0, 0.5), ['outside:y+']), ((0.25, 0.75, 0.5), (0.75, Y - 0.25, 0.5), []),
                ((0.0, 0.0, 0.0), (1.0, Y + 0.0, 1.0), ['lattice']), ((0.5, 0.5, 0.5), (0.5, 0.5, 0.5), ['zero:len'])]
        out.append(_rays_case(f'grid_{X}x{Y}x{Z}', sig, rays))
    # ---- sigma values at the first and at the last in-grid voxel of each walk
    X, Y, Z = 9, 5, 4
    rays, sigs = [], []
    values = ((0.5, 'miss:0.5'), (NEXT_HALF, None), (1.0, None), (math.nan, 'miss:nan'), (math.inf, None), (-1.0, 'miss:-1'))
    for val, miss in values:
        for where in ('first', 'last'):
            for o, e, first, lastv in (((0.5, 2.5, 1.5), (8.7, 2.5, 1.5), (0, 2, 1), (8, 2, 1)),
                                       ((8.5, 4.5, 3.5), (-6.0, 0.4, 0.7), (8, 4, 3), None),
                                       ((4.5, 2.5, 1.5), (4.5, 2.5, 9.0), (4, 2, 1), (4, 2, 3))):
                s = np.zeros((Z, Y, X), np.float32)
                tgt = first if where == 'first' else lastv
                if tgt is None:
                    continue
                s[tgt[2], tgt[1], tgt[0]] = val
                sigs.append(s)
                rays.append((o, e, [miss if miss else 'hit:' + where]))
    N = len(rays)
    out.append(dict(name='sigma_values_9x5x4', sigma=np.stack(sigs)[:, None], origin=np.asarray([[r[0]] for r in rays], np.float32),
                    points=np.asarray([[r[1]] for r in rays], np.float32), tindex=np.zeros((N, 1), np.float32),
                    claims={(i, 0): r[2] for i, r in enumerate(rays)}))
    # ---- batch: N = 3, sigma T in {1, 3} x origin To in {1, 3}, tindex mixing t, fractional t, -0.0 and padding
    X, Y, Z = 11, 9, 6
    rng = np.random.RandomState(31)
    for T, To in ((1, 1), (1, 3), (3, 1), (3, 3)):
        N, M = 3, 40
        sigma = (rng.rand(N, T, Z, Y, X) < 0.12).astype(np.float32)
        origin = (rng.rand(N, To, 3) * [X, Y, Z]).astype(np.float32)
        pts = (rng.rand(N, M, 4) * [X + 6, Y + 6, Z + 6, 1] - [3, 3, 3, 0]).astype(np.float32)
        tmax = min(To, T) if T > 1 else To
        ti = rng.randint(0, tmax, size=(N, M)).astype(np.float32)
        ti[:, ::7] = -1.0
        ti[:, 3::11] = -0.5
        ti[:, 5::13] = -0.0
        if tmax > 1:
            ti[:, 2::9] = tmax - 1 + 0.75                          # a float index truncates: t = tmax - 1
        claims = {(n, m): ['padded'] for n in range(N) for m in range(M) if ti[n, m] < 0}
        out.append(dict(name=f'batch_T{T}_To{To}', sigma=sigma, origin=origin, points=pts, tindex=ti, claims=claims))
    for c in out:
        for k in ('sigma', 'origin', 'points', 'tindex'):
            c[k] = np.ascontiguousarray(c[k], np.float32)
    return out


# --------------------------------------------------------------------------------------------------------- the claims
def check_claims(case, walks=None):
    """Every tagged ray of the case does what its tag says; returns the per-tag counts.  Raises AssertionError naming
    the case, the ray and the tag otherwise."""
    walks = walk_case(case) if walks is None else walks
    counts = {}
    sig = case['sigma']
    X, Y, Z = sig.shape[4], sig.shape[3], sig.shape[2]
    for (n, m), tags in case['claims'].items():
        outp, log = walks[(n, m)]
        t = int(case['tindex'][n, m]) if case['tindex'][n, m] >= 0 else 0
        o = case['origin'][n, t]
        e = case['points'][n, m, :3]
        where = f"{case['name']}: ray (n={n}, m={m}) o={tuple(map(float, o))} e={tuple(map(float, e))}"
        for tag in tags:
            counts[tag] = counts.get(tag, 0) + 1
            kind, _, arg = tag.partition(':')
            if tag == 'padded':
                assert log is None and outp is None, (where, tag)
                continue
            if kind == 'tie':
                assert any(arg in s for s in log['ties']), (where, tag, 'no exact tie inside the grid')
            elif tag == 'zero:len':
                assert float(e[0]) == float(o[0]) and float(e[1]) == float(o[1]) and float(e[2]) == float(o[2]), (where, tag)
            elif kind == 'zero':
                assert log['zero'] == int(arg), (where, tag, log['zero'])
            elif tag == 'face':
                assert any(float(c) == int(float(c)) for c in e), (where, tag)
            elif tag == 'lattice':
                assert any(float(c) == int(float(c)) for c in o), (where, tag)
            elif kind == 'outside':
                k = 'xyz'.index(arg[0])
                size = (X, Y, Z)[k]
                assert (float(o[k]) <= -1.0) if arg[1] == '-' else (float(o[k]) >= size), (where, tag)
            elif tag == 'band':
                assert any(-1.0 < float(c) < 0.0 for c in o) and log['inside0'], (where, tag)
            elif kind == 'entry':
                want = None if arg == 'never' else int(arg)
                assert log['entry'] == want, (where, tag, log['entry'])
            elif tag == 'cut':
                assert log['exit'] == 'max_step' and log['cut_inside'] and log['count'] == MAX_STEP + 1 - log['entry'], \
                    (where, tag, log['exit'], log['count'])
            elif kind == 'hit':
                assert log['count'] >= 2 and log['hit'] == (0 if arg == 'first' else log['count'] - 1), (where, tag, log)
            elif kind == 'miss':
                assert log['count'] >= 2 and log['hit'] is None, (where, tag, log)
            else:
                raise AssertionError(f'unknown tag {tag}')
    return counts
