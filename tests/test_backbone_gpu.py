"""Parity of the image backbone + neck (ResNet-50 + FPN, SURVEY 8f rank 1) against its oracle (oracle/backbone.py, pinned
bit-exactly to torchvision's resnet50 / FeaturePyramidNetwork), and of the channels-last bf16 hand-over to the hot path.

On the tensor cores the stride-1 convolutions run on the TMA-im2col implicit-GEMM kernel (conv2d_tc.cu), the others on
explicit im2col + gemm_tc.  The bf16 backbone is held to the storage-rounding model (oracle.backbone.storage_model: exact
sums, the engine's roundings where it stores a value): per level its distance from the model, relative to the model's
distance from the fp32 oracle, is held to bars measured on an H100 (see BF16_BARS).  The single convolutions are tested one by
one in test_backbone_ops_gpu.py.
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'


def _run(precision, tc, hw=(128, 192), n=2, seed=5):
    from occnet_b200.backbone import BackboneEngine
    from oracle import backbone as OB
    p = OB.init_params(seed=seed)
    img = torch.randn(n, 3, *hw, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        want = OB.fpn(p, OB.resnet50(p, img))
    eng = BackboneEngine(p, n, hw, precision=precision, use_tensor_cores=tc)
    got = eng.forward(img.cuda())
    assert [tuple(g.shape) for g in got] == [tuple(w.shape) for w in want]
    return [(g.cpu() - w).abs().max().item() for g, w in zip(got, want)], [w.abs().max().item() for w in want]


def test_backbone_fp32_matches_oracle():
    err, mag = _run('fp32', False)
    assert max(err) < 1e-3 * max(1.0, max(mag)), (err, mag)


def _run_model(tc, hw=(128, 192), n=2, seed=5):
    """bf16 engine, fp32 oracle and storage-rounding model on the same input: per FPN level the (mean, max) distances
    engine-to-model and model-to-oracle, and the engine's largest error against the oracle relative to the level's magnitude"""
    from occnet_b200.backbone import BackboneEngine
    from oracle import backbone as OB
    p = OB.init_params(seed=seed)
    img = torch.randn(n, 3, *hw, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        want = OB.fpn(p, OB.resnet50(p, img))
        model = OB.storage_model(p, img.to(DEV), tensor_cores=tc)
    got = BackboneEngine(p, n, hw, precision='bf16', use_tensor_cores=tc).forward(img.cuda())
    em, mo, rel = [], [], []
    for g, m, w in zip(got, model, want):
        a, b = (g.double() - m).abs(), (m - w.to(DEV).double()).abs()
        em.append((a.mean().item(), a.max().item()))
        mo.append((b.mean().item(), b.max().item()))
        rel.append((g.cpu() - w).abs().max().item() / max(w.abs().max().item(), 1.0))
    for l in range(4):
        print(f'{"tensor cores" if tc else "CUDA cores"} level {l}: engine-model mean {em[l][0]:.3e} max {em[l][1]:.3e}; '
              f'model-fp32 mean {mo[l][0]:.3e} max {mo[l][1]:.3e}; ratios {em[l][0] / mo[l][0]:.3f} / {em[l][1] / mo[l][1]:.3f}')
    return em, mo, rel


# Engine-to-model distance over model-to-fp32 distance, (mean, max) per FPN level.  Measured on an H100 80GB HBM3 (700 W):
#   CUDA cores   (1.230, 1.258) (1.253, 1.097) (1.250, 1.196) (1.304, 1.183)
#   tensor cores (0.918, 0.959) (0.920, 0.981) (0.921, 0.751) (0.942, 1.022)
# The engine is NOT closer to the model than the model is to fp32: its fp32 accumulation order flips a bf16 rounding of the
# exact sum for a fraction of the elements of every layer (about K 2^-15 of them), and through 50-odd layers of a randomly
# initialised network those 1-ulp flips grow into bf16-sized noise that is independent of the model's.  At the whole-network
# level the model therefore bounds the size of the bf16 noise, not its values; each convolution is held bit-exactly and to a
# derived fp64 bound in test_backbone_ops_gpu.py.  Bars: 2x the measured ratios, rounded up to 0.1.
BF16_BARS = {False: ((2.5, 2.6), (2.6, 2.2), (2.5, 2.4), (2.7, 2.4)),
             True: ((1.9, 2.0), (1.9, 2.0), (1.9, 1.6), (1.9, 2.1))}


def _check_bf16_against_model(tc):
    em, mo, rel = _run_model(tc)
    assert max(rel) < 8e-2, rel                                      # sanity bound against the fp32 oracle
    for l, ((mean_bar, max_bar), (a_mean, a_max), (b_mean, b_max)) in enumerate(zip(BF16_BARS[tc], em, mo)):
        assert a_mean <= mean_bar * b_mean, (l, a_mean, b_mean)
        assert a_max <= max_bar * b_max, (l, a_max, b_max)


def test_backbone_bf16_simt_close_to_oracle():
    _check_bf16_against_model(False)


def test_backbone_bf16_tcgen05_close_to_oracle():
    _check_bf16_against_model(True)


def test_backbone_odd_sizes_fp32():
    err, mag = _run('fp32', False, hw=(232, 200), n=1)          # 29x25 / 15x13 / 8x7 / 4x4 levels: nearest-by-size upsample
    assert max(err) < 1e-3 * max(1.0, max(mag)), (err, mag)


def _small6_images():
    """6 camera images of 232x400 give exactly the `small6` FPN level shapes (29x50, 15x25, 8x13, 4x7)."""
    from occnet_b200 import fixtures
    from oracle import backbone as OB
    cfg = fixtures.make_cfg('small6', num_layers=1)
    params = fixtures.init_params(cfg, seed=2)
    bb = OB.init_params(seed=5)
    img = torch.randn(1, 6, 3, 232, 400, generator=torch.Generator().manual_seed(9))
    return cfg, params, bb, img, fixtures.make_img_metas(cfg)


def test_channels_last_bf16_handover_is_bit_identical():
    """bf16 backbone -> bf16 head: the last FPN convolutions write channels-last bf16 levels that the engine packs without a
    transpose (`occb200_backbone_forward_nhwc_bf16` + `occb200_engine_set_input_dtype(e, 2)`); the result must equal the
    NCHW fp32 hand-over of the same numbers bit for bit."""
    from occnet_b200.backbone import BackboneEngine
    from occnet_b200.engine import OccEngine
    cfg, params, bb, img, metas = _small6_images()
    be = BackboneEngine(bb, 6, (232, 400), precision='bf16')
    assert be.level_shapes == [tuple(s) for s in cfg['level_shapes']]
    x = img[0].to(DEV)
    nchw = be.forward(x)
    nhwc = be.forward(x, channels_last_bf16=True)
    for a, b in zip(nchw, nhwc):
        assert b.dtype == torch.bfloat16 and not b.is_contiguous() and torch.equal(a, b.float())
    eng = OccEngine(cfg, params, precision='bf16', use_tensor_cores=True, device=DEV)
    eng.set_cameras(metas)
    want = {k: v.clone() for k, v in eng.forward(nchw, want=('bev_embed', 'flow', 'occ_cls')).items()}
    eng.set_input_dtype(torch.bfloat16, channels_last=True)
    got = eng.forward(nhwc, want=('bev_embed', 'flow', 'occ_cls'))
    for k in want:
        assert torch.equal(want[k], got[k]), k


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_detector_images_to_voxels(precision):
    """`BEVFormerOcc(return_loss=False, img=[...], img_metas=...)`: images -> native ResNet-50 + FPN -> hot path, the
    reference's real inference call (bevformer_occ.py:231-270), against the oracle chain (backbone oracle -> head oracle)."""
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200 import fixtures
    from occnet_b200.mmcv_shim import build_detector
    from oracle import backbone as OB
    from oracle import bevformer_occ as O
    cfg, params, bb, img, metas = _small6_images()
    det = build_detector(dict(type='BEVFormerOcc', img_backbone=dict(type='ResNet', depth=50), img_neck=dict(type='FPN'),
                              pts_bbox_head=dict(fixtures.head_cfg(cfg), precision=precision))).to(DEV).eval()
    det.pts_bbox_head.load_state_dict(params, strict=True)
    missing = det.load_state_dict(bb, strict=False)
    assert not missing.unexpected_keys
    out = det(return_loss=False, rescale=True, img=[img.to(DEV)], img_metas=[metas])
    with torch.no_grad():
        feats = OB.fpn(bb, OB.resnet50(bb, img[0]))
        want = O.head_forward(params, cfg, [f[None] for f in feats], metas)
    tol, agree = (2e-3, 0.999) if precision == 'fp32' else (1.5e-1, 0.95)
    assert (out['flow_results'] - want['flow']).abs().max().item() < tol
    assert (out['occ_results'] == want['occ'].argmax(-1)).float().mean().item() > agree
