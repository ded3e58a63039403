"""Parity of the image backbone + neck (ResNet-50 + FPN, SURVEY 8f rank 1) against its oracle (oracle/backbone.py, pinned
bit-exactly to torchvision's resnet50 / FeaturePyramidNetwork), and of the channels-last bf16 hand-over to the hot path.

On the tensor cores the stride-1 convolutions run on the TMA-im2col implicit-GEMM kernel (conv2d_tc.cu), the others on
explicit im2col + gemm_tc.
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


def test_backbone_bf16_simt_close_to_oracle():
    err, mag = _run('bf16', False)
    assert max(e / max(m, 1.0) for e, m in zip(err, mag)) < 8e-2, (err, mag)


def test_backbone_bf16_tcgen05_close_to_oracle():
    err, mag = _run('bf16', True)
    assert max(e / max(m, 1.0) for e, m in zip(err, mag)) < 8e-2, (err, mag)


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
