"""uint8 camera frames as the input of the native backbone, the frame engine and the detector: the stem normalises and pads
them on the device (`occb200_backbone_forward_frames`, im2col_frames_kernel), and every result must equal, bit for bit, the
existing fp32-image path fed with the host pipeline's output as restated in oracle/image_pipeline.py."""
import numpy as np
import pytest
import torch

from oracle import image_pipeline as IP

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

NORMS = {'shipped': ((103.530, 116.280, 123.675), (1.0, 1.0, 1.0)),
         'imagenet': ((123.675, 116.28, 103.53), (58.395, 57.12, 57.375))}
# frame size, PadMultiViewImage arguments: 400 * 3 bytes per row take the 16-byte loads, 380 * 3 and 333 * 3 the byte loads
SIZES = {'220x400_size232x400': ((220, 400), dict(size=(232, 400))),
         '200x380_div32': ((200, 380), dict(size_divisor=32)),
         '201x333_div32': ((201, 333), dict(size_divisor=32))}
NORM_CASES = [('shipped', False), ('shipped', True), ('imagenet', True)]
BACKBONE_CASES = [(p, n, r, s, lay) for p in ('fp32', 'bf16') for (n, r) in NORM_CASES for s in SIZES
                  for lay in (('nchw', 'nhwc') if p == 'bf16' else ('nchw',))]

_ENGINES = {}


def _frames(n, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def _backbone(precision, n, hw):
    """fp32: CUDA-core GEMMs; bf16: tensor cores (cached per shape: building one folds all of ResNet-50)"""
    from occnet_b200 import fixtures
    from occnet_b200.backbone import BackboneEngine
    key = (precision, n, tuple(hw))
    if key not in _ENGINES:
        _ENGINES[key] = BackboneEngine(fixtures.init_backbone_params(seed=5), n, hw, precision=precision,
                                       use_tensor_cores=precision == 'bf16', device=DEV)
    return _ENGINES[key]


def check_backbone_case(precision, norm, to_rgb, size, layout, n=2):
    (h, w), pad = SIZES[size]
    mean, std = NORMS[norm]
    fr = _frames(n, h, w, seed=h + w)
    imgs, _ = IP.pipeline(fr, mean, std, to_rgb, **pad)
    be = _backbone(precision, n, imgs.shape[-2:])
    be.set_frame_format((h, w), mean, std, to_rgb)
    cl = layout == 'nhwc'
    want = [t.clone() for t in be.forward(torch.from_numpy(imgs).to(DEV), channels_last_bf16=cl)]
    got = be.forward_frames(torch.from_numpy(fr).to(DEV), channels_last_bf16=cl)
    for l, (a, b) in enumerate(zip(want, got)):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), (l, (a.float() - b.float()).abs().max().item())


@pytest.mark.parametrize('precision,norm,to_rgb,size,layout', BACKBONE_CASES)
def test_backbone_frames_bit_identical_to_restated_images(precision, norm, to_rgb, size, layout):
    check_backbone_case(precision, norm, to_rgb, size, layout)


def test_backbone_frames_full_size_bf16():
    """six 900 x 1600 frames, padded to 928 x 1600 (size_divisor 32): the shipped configuration's input"""
    mean, std = NORMS['shipped']
    fr = _frames(6, 900, 1600, seed=11)
    imgs, metas = IP.pipeline(fr, mean, std, False, size_divisor=32)
    assert metas['img_shape'][0] == (928, 1600, 3)
    be = _backbone('bf16', 6, (928, 1600))
    be.set_frame_format((900, 1600), mean, std, False)
    want = [t.clone() for t in be.forward(torch.from_numpy(imgs).to(DEV), channels_last_bf16=True)]
    del imgs
    got = be.forward_frames(torch.from_numpy(fr).to(DEV), channels_last_bf16=True)
    for a, b in zip(want, got):
        assert torch.equal(a, b)
    _ENGINES.pop(('bf16', 6, (928, 1600)))


# ------------------------------------------------------------------------------------------------ frame engine, code 3
def _small6(precision):
    """6 cameras of 220 x 400 frames padded to 232 x 400: the `small6` FPN level shapes"""
    from occnet_b200 import fixtures
    from occnet_b200.engine import OccEngine
    cfg = fixtures.make_cfg('small6', num_layers=1, img_shape=(232, 400, 3))
    params = fixtures.init_params(cfg, seed=2)
    metas = fixtures.make_img_metas(cfg)                            # camera rig scaled to 232 x 400
    be = _backbone(precision, 6, (232, 400))
    be.set_frame_format((220, 400), *NORMS['shipped'], False)
    eng = OccEngine(cfg, params, precision=precision, use_tensor_cores=precision == 'bf16', device=DEV)
    eng.set_cameras(metas)
    return cfg, params, metas, be, eng


WANT = ('bev_embed', 'flow', 'occ_cls', 'occ_cls_i64')


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_engine_frames_equal_backbone_then_levels(precision):
    cfg, _, _, be, eng = _small6(precision)
    fr = torch.from_numpy(_frames(6, 220, 400, seed=1)).to(DEV)
    cl = precision == 'bf16'                                       # both bf16: the channels-last hand-over
    levels = be.forward_frames(fr, channels_last_bf16=cl)
    eng.set_input_dtype(torch.bfloat16 if cl else torch.float32, channels_last=cl)
    want = {k: v.clone() for k, v in eng.forward(levels, want=WANT).items()}
    n_levels = eng.launches_per_frame
    eng.attach_backbone(be)
    eng.set_input_dtype(torch.uint8)
    got = eng.forward(fr, want=WANT)
    for k in WANT:
        assert torch.equal(want[k], got[k]), k
    assert eng.launches_per_frame > n_levels + 50                 # the backbone's ~60-90 kernels are counted too


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_engine_frames_host_paths(precision):
    """forward_host and the two-slot submit_host / wait_host pipeline upload the uint8 frames; five distinct frames, two in
    flight, and the caller's stream switches between submits: the shared backbone workspace must still be ordered."""
    _, _, _, be, eng = _small6(precision)
    eng.attach_backbone(be)
    eng.set_input_dtype(torch.uint8)
    frames = [torch.from_numpy(_frames(6, 220, 400, seed=20 + i)) for i in range(5)]
    dev = []
    for f in frames:
        o = eng.forward(f.to(DEV), want=('flow', 'occ_cls_i64'))
        dev.append((o['occ_cls_i64'].cpu(), o['flow'].cpu()))
    pinned = [f.pin_memory() for f in frames]
    occ_h, flow_h = eng.forward_host(pinned[2])
    assert torch.equal(occ_h, dev[2][0]) and torch.equal(flow_h, dev[2][1])
    got = [o.clone() for pair in eng.stream_host(pinned) for o in pair]
    for i in range(5):
        assert torch.equal(got[2 * i], dev[i][0]) and torch.equal(got[2 * i + 1], dev[i][1]), i
    streams = [torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)]
    X, Y, Z = eng.vox_shape
    outs = [(torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(), torch.empty((X, Y, Z, 2)).pin_memory()) for _ in range(2)]
    pending = []
    for i, f in enumerate(pinned):
        slot = i & 1
        if len(pending) == 2:
            j = pending.pop(0)
            eng.wait_host(j & 1)
            assert torch.equal(outs[j & 1][0], dev[j][0]) and torch.equal(outs[j & 1][1], dev[j][1]), j
        with torch.cuda.stream(streams[i % 2]):
            eng.submit_host(slot, f, *outs[slot])
        pending.append(i)
    for j in pending:
        eng.wait_host(j & 1)
        assert torch.equal(outs[j & 1][0], dev[j][0]) and torch.equal(outs[j & 1][1], dev[j][1]), j
    eng.attach_backbone(None)


# ---------------------------------------------------------------------------------------------------------- detector
@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_detector_frames_equal_restated_images(precision):
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200 import fixtures
    from occnet_b200.mmcv_shim import build_detector
    cfg, params, metas, _, _ = _small6(precision)
    det = build_detector(dict(type='BEVFormerOcc', img_backbone=dict(type='ResNet', depth=50), img_neck=dict(type='FPN'),
                              pts_bbox_head=dict(fixtures.head_cfg(cfg), precision=precision),
                              frame_pad=dict(size=(232, 400)))).to(DEV).eval()
    det.pts_bbox_head.load_state_dict(params, strict=True)
    assert not det.load_state_dict(fixtures.init_backbone_params(seed=5), strict=False).unexpected_keys
    seen = []
    head_forward = det.pts_bbox_head.forward
    det.pts_bbox_head.forward = lambda feats, img_metas, *a, **k: (seen.append(img_metas), head_forward(feats, img_metas, *a, **k))[1]
    fr = _frames(6, 220, 400, seed=3)
    imgs, pm = IP.pipeline(fr, *NORMS['shipped'], False, size=(232, 400))
    padded = [dict(metas[0], img_shape=pm['img_shape'])]
    bare = [{k: v for k, v in metas[0].items() if k != 'img_shape'}]
    want = det(return_loss=False, img=[torch.from_numpy(imgs)[None].to(DEV)], img_metas=[padded])
    for frames in (torch.from_numpy(fr)[None].to(DEV), torch.from_numpy(fr)[None]):          # CUDA, then CPU frames
        got = det(return_loss=False, img=[frames], img_metas=[bare])
        assert torch.equal(got['occ_results'], want['occ_results']) and torch.equal(got['flow_results'], want['flow_results'])
        assert seen[-1][0]['img_shape'] == [(232, 400, 3)] * 6 and seen[-1][0]['ori_shape'] == [(220, 400, 3)] * 6
    assert 'img_shape' not in bare[0]


# ------------------------------------------------------------------------------------------------------------ errors
def test_frame_errors_raise_before_any_launch():
    import ctypes
    from occnet_b200 import _lib
    from occnet_b200.backbone import BackboneEngine
    from occnet_b200 import fixtures
    cfg, _, _, be, eng = _small6('bf16')
    lib = _lib.load()
    fr = torch.from_numpy(_frames(6, 220, 400)).to(DEV)
    with pytest.raises(_lib.OccB200Error):
        be.set_frame_format((240, 400), *NORMS['shipped'], False)            # larger than the backbone's 232 x 400
    with pytest.raises(_lib.OccB200Error):
        be.set_frame_format((220, 404), *NORMS['shipped'], False)
    with pytest.raises(_lib.OccB200Error):
        be.set_frame_format((220, 400), NORMS['shipped'][0], (1.0, 0.0, 1.0), False)
    be.set_frame_format((220, 400), *NORMS['shipped'], False)
    with pytest.raises(ValueError):
        be.forward_frames(fr.float())                                          # dtype
    with pytest.raises(ValueError):
        be.forward_frames(torch.from_numpy(_frames(6, 220, 800)).to(DEV)[:, :, ::2])   # not contiguous
    with pytest.raises(ValueError):
        be.forward_frames(fr[:, :200].contiguous())                            # not the configured frame size
    with pytest.raises(ValueError):
        be.forward_frames(fr.cpu())
    # the C entries return an error and leave the outputs untouched: nothing was launched
    outs = [torch.full((6, 256, h, w), 7.0, device=DEV) for h, w in be.level_shapes]
    fresh = BackboneEngine(fixtures.init_backbone_params(seed=5), 6, (232, 400), precision='bf16', device=DEV)
    s = _lib.stream_ptr()
    assert lib.occb200_backbone_forward_frames(fresh._h, _lib.ptr(fr), *[_lib.ptr(o) for o in outs], 0, s) != 0   # no format
    assert lib.occb200_backbone_forward_frames(be._h, _lib.ptr(fr), *[_lib.ptr(o) for o in outs], 2, s) != 0      # layout
    torch.cuda.synchronize()
    assert all(bool((o == 7.0).all()) for o in outs)
    # engine, code 3: no backbone attached
    eng.set_input_dtype(torch.uint8)
    with pytest.raises(RuntimeError):
        eng.forward(fr)
    X, Y, Z = eng.vox_shape
    flow = torch.full((X, Y, Z, 2), 7.0, device=DEV)
    ptrs = (ctypes.c_void_p * 4)(fr.data_ptr(), 0, 0, 0)
    assert lib.occb200_engine_forward(eng._h, ptrs, None, None, None, _lib.ptr(flow), None, None, s) != 0
    torch.cuda.synchronize()
    assert bool((flow == 7.0).all())
    # mismatched backbones: num_images, level shapes, no frame format
    two = BackboneEngine(fixtures.init_backbone_params(seed=5), 2, (232, 400), precision='bf16', device=DEV)
    two.set_frame_format((220, 400), *NORMS['shipped'], False)
    taller = BackboneEngine(fixtures.init_backbone_params(seed=5), 6, (264, 400), precision='bf16', device=DEV)
    taller.set_frame_format((220, 400), *NORMS['shipped'], False)
    for bad in (two, taller, fresh):
        with pytest.raises(_lib.OccB200Error):
            eng.attach_backbone(bad)
    assert eng.backbone is None
    eng.attach_backbone(be)
    with pytest.raises(ValueError):
        eng.forward(fr.float())
    with pytest.raises(ValueError):
        eng.forward_host(fr.cpu()[:, :, :200].contiguous())
    eng.attach_backbone(None)
