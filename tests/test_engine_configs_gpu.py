"""The frame engine against the oracles across the configurations occb200_engine_create accepts, not only the four shapes the
other engine tests run (toy, small6, 30 x 44 with eight cameras, full size).

The engine's code branches on its configuration: the head runs on the tensor cores only for num_classes + 2 <= 19, every dense
layer picks its GEMM route from M, N and K (ffn_dim is N of FFN1 and K of FFN2 and of the fused-LayerNorm GEMM), the T32
residual stream is padded to 128 rows and the merged TSA launch reads its T32 constant only when Nq % 32 == 0, the pack kernel
has scalar tails when a level's h * w is not a multiple of 4 (fp32 features) or 8 (bf16 features), and the SCA geometry depends on pc_range, the
image size, the pillar anchors and the cameras.  CONFIGS is a seeded table of configurations that each combine several unusual
values; test_engine_configs_cpu.py checks that the table covers every value it claims to and that create accepts it.

Every configuration runs on four plans (fp32 on CUDA cores, fp32 on the tensor cores as three bf16 passes, bf16 on CUDA cores,
bf16 on the tensor cores), each in self mode and with a prev_bev the engine rotates on the device by PREV_ANGLE about the
configuration's rotate_center.  The fp32 plans take fp32 feature levels; the bf16 plans take bf16 ones
(set_input_dtype(torch.bfloat16), the levels an on-device backbone hands over), and both oracles get the same rounded values:
  * fp32 plans, against oracle.bevformer_occ.head_forward: every layer's TSA / SCA / layer taps, the voxels, bev_embed, occ and
    flow within FP32_BAR; then a second frame with taps off, whose outputs must meet the same bar.
  * bf16 on the tensor cores, against the storage-rounding model oracle.bf16_model.head_forward: for bev_embed, occ and flow
    the engine's mean distance to the model must be below the model's own mean distance to the fp32 oracle, and the engine's
    distance to the model must stay under the six-layer bars of test_gpu_parity.py (BF16_MODEL_TOL_MAX / _MEAN).
  * bf16 on CUDA cores: the model does not describe this plan (it keeps fp32 weights and sampling projections; the engine
    lands about 1.15x the model's own distance from fp32 away from the model), so it is held to the fp32 oracle: mean
    distance below 1.25x the model's mean distance to fp32 + 1e-4, and the same BF16_MODEL_TOL_* bars.
  * classes, on every plan: occ_cls, occ_cls_i64 and argmax(occ) agree exactly, and every voxel whose reference top-2 logit gap
    exceeds twice the observed maximum logit error has the reference's class.
  * video: for VIDEO_CONFIGS, forward_video (scene start, then two frames with an angle each) is bit-identical to forward with
    the previous frame's bev_embed as prev_bev and the same angle.
The drop-in BEVFormerOccHead, built from a reference-style config dict (feedforward_channels=1024), must match the fp32 oracle.

Each plan runs in a child process, so a device fault cannot poison this session.  A failure names the configuration, the
plan, the output and its worst element; a pass prints one line per configuration and plan with each output's error / bar."""
import os
import subprocess
import sys

import pytest
import torch

from occnet_b200 import fixtures

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
FP32_BAR = 1e-3                     # the fp32 engine tests' bar (largest difference seen there: 1.1e-4)
PREV_ANGLE = 20.0                   # degrees: large enough to move cells of a 2 x 2 grid
VIDEO_ANGLES = (20.0, -11.0)
ASYM_PC = [-30.0, -50.0, -2.0, 50.0, 30.0, 4.4]

# (name, make_cfg overrides); num_cams > 6 takes fixtures.rig_metas' two extra cameras.  Level notes: h * w odd and < 64,
# h * w % 8 == 4 (a 4-pixel tail of the pack kernel's 8-pixel groups of bf16 features, the bf16 plans' input), wide
# (w >= 4 h) and tall (h >= 4 w) levels, partial 64-pixel pack tiles.
CONFIGS = [
    ('min2x2', dict(bev_h=2, bev_w=2, num_cams=1, num_points_in_pillar=1, num_layers=1, ffn_dim=64, num_classes=1,
                    level_shapes=[(2, 2)] * 4, pc_range=[-10.0, -4.0, -1.0, 30.0, 4.0, 5.4], rotate_center=[0, 1])),
    ('nq15', dict(bev_h=3, bev_w=5, num_cams=3, num_points_in_pillar=2, num_layers=2, ffn_dim=128, num_classes=2,
                  level_shapes=[(7, 9), (3, 5), (2, 6), (2, 2)], use_cams_embeds=False, pc_range=ASYM_PC, rotate_center=[4, 0])),
    ('tile128', dict(bev_h=8, bev_w=16, num_cams=5, num_points_in_pillar=4, num_layers=3, ffn_dim=576, num_classes=17,
                     level_shapes=[(3, 40), (2, 21), (2, 9), (2, 3)], img_shape=(480, 800, 3), rotate_center=[3, 6])),
    ('13x17', dict(bev_h=13, bev_w=17, num_cams=7, num_points_in_pillar=8, num_layers=1, ffn_dim=1024, num_classes=18,
                   level_shapes=[(40, 3), (21, 2), (9, 2), (3, 2)], pc_range=ASYM_PC, rotate_center=[40, -10])),
    ('17x13', dict(bev_h=17, bev_w=13, num_cams=8, num_points_in_pillar=2, num_layers=2, ffn_dim=576, num_classes=32,
                   level_shapes=[(9, 15), (5, 7), (3, 4), (2, 2)], use_cams_embeds=False, rotate_center=[9, 4])),
    ('thin2x63', dict(bev_h=2, bev_w=63, num_cams=8, num_points_in_pillar=1, num_layers=1, ffn_dim=64, num_classes=18,
                      level_shapes=[(29, 50), (15, 25), (8, 13), (4, 7)], rotate_center=[50, 1])),
    ('thin63x2', dict(bev_h=63, bev_w=2, num_cams=1, num_points_in_pillar=4, num_layers=3, ffn_dim=128, num_classes=17,
                      level_shapes=[(16, 16), (8, 8), (4, 4), (2, 2)], img_shape=(256, 704, 3), rotate_center=[1, 50])),
    ('nq15t', dict(bev_h=5, bev_w=3, num_cams=6, num_points_in_pillar=8, num_layers=1, ffn_dim=1024, num_classes=32,
                   level_shapes=[(2, 10), (3, 7), (5, 5), (2, 2)], use_cams_embeds=False, img_shape=(900, 1600, 3),
                   rotate_center=[-3, 7])),
]
VIDEO_CONFIGS = ('nq15', '17x13')
PLANS = {'fp32': ('fp32', False), 'fp32_tc': ('fp32', True), 'bf16': ('bf16', False), 'bf16_tc': ('bf16', True)}
WANT = ('bev_embed', 'occ', 'flow', 'occ_cls', 'occ_cls_i64')


def make_cfg(over):
    return fixtures.make_cfg('full', **over)


def metas_for(cfg, angle=None):
    return fixtures.rig_metas(cfg['num_cams'], tuple(cfg['img_shape'][:2]), can_bus_angle=angle)


def case(name):
    """-> cfg, params, feats (4 x (1, cams, 256, h, w)), prev (1, Nq, 256): seeded, the same for every plan"""
    cfg = make_cfg(dict(CONFIGS)[name])
    params = fixtures.init_params(cfg, seed=2)
    feats = fixtures.make_feats(cfg, bs=1, seed=1)
    prev = torch.randn(1, cfg['bev_h'] * cfg['bev_w'], cfg['embed_dims'], generator=torch.Generator().manual_seed(3))
    return cfg, params, feats, prev


# ------------------------------------------------------------------------------------------------ GPU checks (child process)
def _engine(cfg, params, precision, tc):
    """the plan's engine; bf16 plans take bf16 feature levels"""
    from occnet_b200.engine import OccEngine
    eng = OccEngine(cfg, params, precision=precision, use_tensor_cores=tc, device=DEV)
    eng.set_cameras(metas_for(cfg))
    if precision == 'bf16':
        eng.set_input_dtype(torch.bfloat16)
    return eng


def _rounded(feats):
    """the bf16 plans' feature levels, as the fp32 values the oracles read"""
    return [f.bfloat16().float() for f in feats]


def _worst(got, want):
    """-> (max |got - want|, index of that element); NaN counts as infinitely wrong"""
    d = (got.double() - want.double()).abs().nan_to_num(float('inf'))
    i = int(d.reshape(-1).argmax())
    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), d.shape))
    return d.reshape(-1)[i].item(), idx


def _outputs(out, cfg):
    """engine outputs in the oracles' layouts"""
    return {'bev_embed': out['bev_embed'].cpu().t().reshape(1, -1, cfg['bev_h'], cfg['bev_w']),
            'occ': out['occ'].cpu()[None], 'flow': out['flow'].cpu()[None]}


def _check_classes(tag, out, ref_occ, fails):
    """occ_cls / occ_cls_i64 / argmax(occ) identical; the class of every voxel whose reference top-2 gap exceeds twice the max
    logit error equals the reference's"""
    occ = out['occ'].cpu()
    am = occ.argmax(-1)
    for k in ('occ_cls', 'occ_cls_i64'):
        c = out[k].cpu().long()
        if not torch.equal(c, am):
            i = tuple(int(v) for v in (c != am).nonzero()[0])
            fails.append(f'{tag} {k}: differs from argmax(occ) in {int((c != am).sum())} voxels; first {i}: '
                         f'{int(c[i])} vs {int(am[i])}')
    ref = ref_occ[0]
    err = (occ - ref).abs().max().item()
    if ref.shape[-1] < 2:
        return
    top = ref.topk(2, -1).values
    sure = (top[..., 0] - top[..., 1]) > 2 * err
    bad = sure & (am != ref.argmax(-1))
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        fails.append(f'{tag} classes: {int(bad.sum())} of {int(sure.sum())} voxels with a top-2 gap > 2 x max logit error '
                     f'({err:.2e}) changed class; first {i}: {int(am[i])} vs {int(ref.argmax(-1)[i])}')


def _forward(eng, cfg, feats, prev):
    if prev is not None:
        eng.set_prev_rotation(PREV_ANGLE)
    out = eng.forward([f[0].to(DEV, eng.feat_dtype) for f in feats], prev_bev=None if prev is None else prev[0].to(DEV),
                      want=WANT)
    torch.cuda.synchronize()
    return out


def check_fp32(name, tc, fails):
    from oracle import bevformer_occ as O
    cfg, params, feats, prev = case(name)
    plan = 'fp32_tc' if tc else 'fp32'
    eng = _engine(cfg, params, 'fp32', tc)
    for with_prev in (False, True):
        metas = metas_for(cfg, PREV_ANGLE if with_prev else None)
        taps = {}
        with torch.no_grad():
            want = O.head_forward(params, cfg, feats, metas, prev_bev=prev.clone() if with_prev else None, taps=taps)
        pb = prev if with_prev else None
        tag = f'config {name} plan {plan} prev={with_prev}'
        summary = {}
        for frame, taps_on in ((0, True), (1, False)):
            eng.enable_taps(taps_on)
            out = _forward(eng, cfg, feats, pb)
            errs = {}
            if taps_on:
                for l in range(cfg['num_layers']):
                    for kind in ('tsa', 'sca', 'layer'):
                        key = f'layer{l}' + ('' if kind == 'layer' else '_' + kind)
                        errs[key] = _worst(eng.tap(kind, l).cpu(), taps[key][0])
                errs['voxel'] = _worst(eng.tap('voxel').cpu()[None], taps['voxel_feats'])
            got = _outputs(out, cfg)
            for k in ('bev_embed', 'occ', 'flow'):
                errs[k] = _worst(got[k], want[k])
            for k, (e, i) in errs.items():
                if not e < FP32_BAR:
                    fails.append(f'{tag} taps={taps_on} {k}: max |err| {e:.3e} >= {FP32_BAR} at {i}')
                summary[k] = max(summary.get(k, 0.0), e)
            _check_classes(f'{tag} taps={taps_on}', out, want['occ'], fails)
        k = max(summary, key=summary.get)
        print(f'{tag}: max |err| / bar {summary[k] / FP32_BAR:.3f} ({k} {summary[k]:.2e}); ' +
              ', '.join(f'{k} {v:.1e}' for k, v in summary.items() if not k.startswith('layer')))


def check_bf16(name, tc, fails):
    from oracle import bevformer_occ as O
    from oracle import bf16_model as BM
    from test_gpu_parity import BF16_MODEL_TOL_MAX, BF16_MODEL_TOL_MEAN
    cfg, params, feats, prev = case(name)
    feats = _rounded(feats)
    plan = 'bf16_tc' if tc else 'bf16'
    eng = _engine(cfg, params, 'bf16', tc)
    for with_prev in (False, True):
        metas = metas_for(cfg, PREV_ANGLE if with_prev else None)
        pb = prev.clone() if with_prev else None
        with torch.no_grad():
            want32 = O.head_forward(params, cfg, feats, metas, prev_bev=pb)
            model = BM.head_forward(params, cfg, feats, metas, prev_bev=pb)
        out = _forward(eng, cfg, feats, prev if with_prev else None)
        got = _outputs(out, cfg)
        tag = f'config {name} plan {plan} prev={with_prev}'
        # the model restates the tensor-core plan's storage points (bf16 weights, fp16 projections, folded layer-0 TSA); the
        # CUDA-core plan keeps fp32 weights and projections, so it is held to the fp32 oracle, no farther from it than the
        # model (the bar of the other bf16 engine tests, test_attention_gather_gpu.check_engine_bf16)
        ref = model if tc else want32
        worst, line = 0.0, []
        for k, t in got.items():
            d, d_mf = (t - ref[k]).abs(), (model[k] - want32[k]).abs()
            mx, i = _worst(t, ref[k])
            mean, mean_mf = d.mean().item(), d_mf.mean().item()
            mean_bar = mean_mf if tc else 1.25 * mean_mf + 1e-4
            vs = 'model' if tc else 'fp32'
            if not mean < mean_bar:
                fails.append(f'{tag} {k}: mean |engine - {vs}| {mean:.3e} >= {mean_bar:.3e} (model vs fp32 {mean_mf:.3e})')
            if not (mx < BF16_MODEL_TOL_MAX and mean < BF16_MODEL_TOL_MEAN):
                fails.append(f'{tag} {k}: |engine - {vs}| max {mx:.3e} (bar {BF16_MODEL_TOL_MAX}) at {i}, mean {mean:.3e} '
                             f'(bar {BF16_MODEL_TOL_MEAN})')
            r = max(mean / mean_bar, mx / BF16_MODEL_TOL_MAX, mean / BF16_MODEL_TOL_MEAN)
            worst = max(worst, r)
            line.append(f'{k} vs {vs} mean {mean:.1e} max {mx:.1e} (model vs fp32 mean {mean_mf:.1e})')
        _check_classes(tag, out, ref['occ'], fails)
        print(f'{tag}: max |err| / bar {worst:.3f}; ' + ', '.join(line))


def check_video(name, precision, tc, fails):
    """forward_video (scene start, then an angle per frame) == forward(prev_bev = the previous bev_embed), bit for bit"""
    cfg, params, _, _ = case(name)
    eng = _engine(cfg, params, precision, tc)
    frames = [[f[0].to(DEV, eng.feat_dtype) for f in fixtures.make_feats(cfg, bs=1, seed=50 + i)] for i in range(3)]
    angles = (None,) + VIDEO_ANGLES
    ref, prev = [], None
    for fr, a in zip(frames, angles):
        eng.set_prev_rotation(a)
        ref.append({k: v.clone() for k, v in eng.forward(fr, prev_bev=prev, want=WANT).items()})
        prev = ref[-1]['bev_embed']
    eng.set_prev_rotation(None)
    eng.set_history(True)
    tag = f'config {name} plan {PLAN_NAME[(precision, tc)]} video'
    for i, (fr, a) in enumerate(zip(frames, angles)):
        got = eng.forward_video(fr, rotation=a, scene_start=i == 0, want=WANT)
        for k in WANT:
            if not torch.equal(got[k], ref[i][k]):
                e, idx = _worst(got[k].cpu(), ref[i][k].cpu())
                fails.append(f'{tag} frame {i} {k}: differs from forward(prev_bev=...) by {e:.3e} at {idx}')
    torch.cuda.synchronize()
    print(f'{tag}: 3 frames bit-identical to forward(prev_bev=previous bev_embed)' if not any(tag in f for f in fails) else
          f'{tag}: FAILED')


PLAN_NAME = {v: k for k, v in PLANS.items()}


def check_plan(plan):
    precision, tc = PLANS[plan]
    fails = []
    for name, _ in CONFIGS:
        (check_fp32 if precision == 'fp32' else check_bf16)(name, tc, fails)
        if name in VIDEO_CONFIGS:
            check_video(name, precision, tc, fails)
    assert not fails, '\n'.join(fails)


def check_dropin_head():
    """BEVFormerOccHead built through the registry from a reference-style config: _engine_cfg must read
    feedforward_channels (1024 here), num_points_in_pillar, the cameras and the BEV shape"""
    import projects.mmdet3d_plugin  # noqa: F401  (registers the classes)
    from occnet_b200.mmcv_shim import build_head
    from oracle import bevformer_occ as O
    cfg = make_cfg(dict(bev_h=13, bev_w=17, num_cams=5, num_points_in_pillar=2, num_layers=2, ffn_dim=1024, num_classes=17,
                        level_shapes=[(9, 15), (5, 7), (3, 4), (2, 2)], rotate_center=[5, 9]))
    hc = fixtures.head_cfg(cfg)
    assert hc['transformer']['encoder']['transformerlayers']['feedforward_channels'] == 1024
    params = fixtures.init_params(cfg, seed=2)
    head = build_head(dict(hc, precision='fp32')).to(DEV).eval()
    head.load_state_dict(params, strict=True)
    feats = fixtures.make_feats(cfg, bs=1, seed=1)
    metas = metas_for(cfg)
    out = head([f.to(DEV) for f in feats], metas)
    with torch.no_grad():
        want = O.head_forward(params, cfg, feats, metas)
    ecfg = head._engine.cfg
    assert (ecfg['ffn_dim'], ecfg['num_points_in_pillar'], ecfg['num_cams'], ecfg['bev_h'], ecfg['bev_w']) == (1024, 2, 5, 13, 17)
    errs = {k: _worst(out[k].cpu(), want[k]) for k in ('bev_embed', 'occ', 'flow')}
    print('drop-in head 13x17, 5 cameras, D=2, feedforward_channels=1024: ' +
          ', '.join(f'{k} {e:.2e} / {FP32_BAR}' for k, (e, _) in errs.items()))
    for k, (e, i) in errs.items():
        assert e < FP32_BAR, f'drop-in head {k}: max |err| {e:.3e} at {i}'


def _run_isolated(call, timeout=1200):
    """Runs happen in a child process: a device fault there must not poison this session's context."""
    code = f'import sys; sys.path.insert(0, "tests"); import test_engine_configs_gpu as t; t.{call}; print("OK")'
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    print(r.stdout[-20000:])
    assert r.returncode == 0, f'child failed ({r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-6000:]}'
    assert 'OK' in r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize('plan', list(PLANS))
def test_engine_matches_oracle_over_config_table(plan):
    _run_isolated(f'check_plan({plan!r})')


@pytest.mark.gpu
def test_dropin_head_from_reference_config_matches_oracle():
    _run_isolated('check_dropin_head()')
