"""JPEG camera files decoded on the GPU (occnet_b200/csrc/jpeg.cu) against cv2.imdecode(IMREAD_UNCHANGED), byte for byte, and
the frame engine / detector fed the encoded files against the same paths fed cv2's decoded frames."""
import itertools

import numpy as np
import pytest
import torch

from oracle import jpeg_decode as J

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

SIZES = [(900, 1600), (901, 1599), (9, 17), (8, 8), (1, 1)]
QUALITIES = [5, 50, 75, 95, 100]
SAMPLINGS = ['420', '444']
RESTARTS = [0, 1, 7, 'row']
OPTIMIZE = [False, True]


def _matrix(h, w):
    """every quality / sampling / restart / table / content combination at one size, seeded per case"""
    for i, (q, s, r, o, c) in enumerate(itertools.product(QUALITIES, SAMPLINGS, RESTARTS, OPTIMIZE, J.CONTENTS)):
        yield (q, s, r, o, c), J.encode(J.make_image(c, h, w, seed=i + h), q, s, r, o)


@pytest.mark.parametrize('size', SIZES, ids=lambda s: f'{s[1]}x{s[0]}')
def test_decoder_matches_cv2_on_the_matrix(size):
    """the full matrix at each size, six files per decode (consecutive cases: mixed qualities, samplings, restart intervals)"""
    from occnet_b200.jpeg import JpegDecoder
    dec = JpegDecoder(DEV)
    cases = list(_matrix(*size))
    for k in range(0, len(cases), 6):
        batch = cases[k:k + 6]
        got = dec.decode([b for _, b in batch]).cpu().numpy()
        torch.cuda.synchronize()
        assert dec.status() == 0
        for (case, buf), g in zip(batch, got):
            want = J.cv2_decode(buf)
            assert np.array_equal(g, want), (size, case, int(np.abs(g.astype(int) - want).max()))


def test_decoder_mixed_sizes_in_one_decode():
    from occnet_b200.jpeg import JpegDecoder
    dec = JpegDecoder(DEV)
    bufs = [J.encode(J.make_image(c, h, w, seed=h), q, s, r, o) for (h, w), c, q, s, r, o in
            zip(SIZES + [(33, 47)], J.CONTENTS * 2, [95, 5, 100, 50, 75, 90], SAMPLINGS * 3, RESTARTS + [3, 'row'],
                OPTIMIZE * 3)]
    got = dec.decode(bufs)
    torch.cuda.synchronize()
    assert dec.status() == 0
    for b, g in zip(bufs, got):
        assert np.array_equal(g.cpu().numpy(), J.cv2_decode(b))


def _corrupt(buf, seed):
    """flip bytes in the middle of the scan, never producing or removing a 0xFF (the markers stay where they were)"""
    b = bytearray(buf)
    sos = b.index(b'\xff\xda')
    rng = np.random.default_rng(seed)
    for p in rng.integers(sos + 20, len(b) - 4, 16):
        if b[p] != 0xFF and b[p - 1] != 0xFF:
            b[p] = (b[p] ^ 0x5A) if (b[p] ^ 0x5A) != 0xFF else b[p] ^ 0x0F
    return bytes(b)


def test_decoder_reports_a_corrupt_scan_and_recovers():
    from occnet_b200.jpeg import JpegDecoder
    dec = JpegDecoder(DEV)
    clean = [J.encode(J.make_image('noise', 64, 96, seed=i), 90, '420', r) for i, r in enumerate([0, 1, 0, 7, 0, 'row'])]
    for seed in range(4):
        bad = list(clean)
        bad[seed + 1] = _corrupt(clean[seed + 1], seed)
        dec.decode(bad)
        torch.cuda.synchronize()
        assert dec.status() & (1 << (seed + 1))
        got = dec.decode(clean)
        torch.cuda.synchronize()
        assert dec.status() == 0
        for b, g in zip(clean, got):
            assert np.array_equal(g.cpu().numpy(), J.cv2_decode(b))


# ------------------------------------------------------------------------------------------------ frame engine, code 4
SHIPPED_NORM = ((103.530, 116.280, 123.675), (1.0, 1.0, 1.0))
_BACKBONES = {}


def _camera_files(n_frames, seed=0):
    """frames of six 220 x 400 camera files: camera-like content, 4:2:0 at quality 90-95, mixed restart intervals"""
    out = []
    for i in range(n_frames):
        out.append([J.encode(J.make_image('camera' if c % 3 else 'noise', 220, 400, seed=seed + 10 * i + c), 90 + c,
                             '420', [0, 'row', 7][c % 3], bool(c % 2)) for c in range(6)])
    return out


def _engine(precision):
    """6 cameras of 220 x 400 frames padded to 232 x 400 (the small6 FPN level shapes) on the metric's 200 x 200 x 16 grid"""
    from occnet_b200 import fixtures
    from occnet_b200.backbone import BackboneEngine
    from occnet_b200.engine import OccEngine
    cfg = fixtures.make_cfg('small6', bev_h=200, bev_w=200, num_layers=1, img_shape=(232, 400, 3))
    if precision not in _BACKBONES:
        _BACKBONES[precision] = BackboneEngine(fixtures.init_backbone_params(seed=5), 6, (232, 400), precision=precision,
                                               use_tensor_cores=precision == 'bf16', device=DEV)
    be = _BACKBONES[precision]
    be.set_frame_format((220, 400), *SHIPPED_NORM, False)
    eng = OccEngine(cfg, fixtures.init_params(cfg, seed=2), precision=precision, use_tensor_cores=precision == 'bf16',
                    device=DEV)
    eng.set_cameras(fixtures.make_img_metas(cfg))
    eng.attach_backbone(be)
    return eng


def _origins(i):
    return np.random.default_rng(40 + i).uniform(-2, 2, (3, 3)).astype(np.float32)


def _gt(i):
    g = torch.Generator().manual_seed(50 + i)
    return (torch.randint(0, 17, (200, 200, 16), generator=g, dtype=torch.uint8),
            torch.randn((200, 200, 16, 2), generator=g))


WANT = ('bev_embed', 'flow', 'occ_cls', 'occ_cls_i64')


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_engine_from_jpeg_equals_engine_from_cv2_frames(precision):
    """every frame path fed the encoded files against the same path fed cv2's decoded uint8 frames: outputs, ray records and
    score counters byte-identical"""
    from occnet_b200.metric import RayMetric
    eng = _engine(precision)
    files = _camera_files(4, seed=7)
    frames = [torch.from_numpy(np.stack([J.cv2_decode(b) for b in f])) for f in files]
    rm_u8, rm_jpeg = RayMetric(DEV), RayMetric(DEV)

    def device_calls(dtype, inputs, rm):
        eng.set_input_dtype(dtype)
        outs = []
        for i, x in enumerate(inputs):
            x = x.to(DEV) if dtype == torch.uint8 else x
            o = eng.forward(x, want=WANT, ray_origins=_origins(i), score=(*[t.to(DEV) for t in _gt(i)], _origins(i)),
                            metric=rm)
            outs.append({k: v.clone() for k, v in o.items()})
        return outs, eng.launches_per_frame

    def video_calls(dtype, inputs):
        """device-side video frames with the rotation as an angle, on the engine's history"""
        eng.set_input_dtype(dtype)
        eng.set_history(True)
        outs = []
        for i, x in enumerate(inputs):
            x = x.to(DEV) if dtype == torch.uint8 else x
            o = eng.forward_video(x, rotation=2.5 * i - 1.0, scene_start=i == 0, want=WANT, ray_origins=_origins(i))
            outs.append({k: v.clone() for k, v in o.items()})
        eng.set_history(False)
        return outs

    want, n_u8 = device_calls(torch.uint8, frames, rm_u8)
    got, n_jpeg = device_calls('jpeg', files, rm_jpeg)
    want += video_calls(torch.uint8, frames)
    got += video_calls('jpeg', files)
    torch.cuda.synchronize()
    assert eng.jpeg_status() == 0
    assert n_jpeg == n_u8 + 3
    for w, g in zip(want, got):
        for k in w:
            assert torch.equal(w[k], g[k]), k
    assert torch.equal(rm_u8.counters, rm_jpeg.counters)

    def host_calls(dtype, inputs):
        eng.set_input_dtype(dtype)
        if dtype == torch.uint8:
            inputs = [x.pin_memory() for x in inputs]
        res = [tuple(t.clone() for t in eng.forward_host(inputs[0]))]
        res += [tuple(t.clone() for t in pair) for pair in eng.stream_host(inputs)]
        eng.set_history(True)
        items = [(x, 1.5 * i, i == 0, _origins(i)) for i, x in enumerate(inputs)]
        for occ, flow, rec in eng.stream_host_video(items):
            res.append((occ.clone(), flow.clone()) + tuple(v.clone() for v in rec.values()))
        eng.set_history(False)
        return res

    want_h = host_calls(torch.uint8, frames)
    got_h = host_calls('jpeg', files)
    assert len(want_h) == len(got_h) == 9
    for i, (w, g) in enumerate(zip(want_h, got_h)):
        for a, b in zip(w, g):
            assert torch.equal(a, b), i
    assert torch.equal(want_h[0][0], want[0]['occ_cls_i64'].cpu())


def test_engine_reports_a_corrupt_camera_file_and_recovers():
    """a host call whose camera file has a corrupt scan raises; the next frame is byte-identical again"""
    from occnet_b200 import _lib
    eng = _engine('bf16')
    files = _camera_files(2, seed=3)
    eng.set_input_dtype(torch.uint8)
    want = [tuple(t.clone() for t in eng.forward_host(torch.from_numpy(np.stack([J.cv2_decode(b) for b in f])).pin_memory()))
            for f in files]
    eng.set_input_dtype('jpeg')
    bad = list(files[0])
    bad[2] = _corrupt(bad[2], 1)
    with pytest.raises(_lib.OccB200Error, match='corrupt JPEG'):
        eng.forward_host(bad)
    got = eng.forward_host(files[1])
    assert torch.equal(got[0], want[1][0]) and torch.equal(got[1], want[1][1])
    X, Y, Z = eng.vox_shape
    outs = [(torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(), torch.empty((X, Y, Z, 2)).pin_memory()) for _ in range(2)]
    eng.submit_host(0, bad, *outs[0])
    eng.submit_host(1, files[0], *outs[1])
    with pytest.raises(_lib.OccB200Error, match='corrupt JPEG'):
        eng.wait_host(0)
    eng.wait_host(1)
    assert torch.equal(outs[1][0], want[0][0]) and torch.equal(outs[1][1], want[0][1])
    eng.forward(bad, want=('flow',))
    torch.cuda.synchronize()
    assert eng.jpeg_status() == 1 << 2
    eng.forward(files[0], want=('flow',))
    torch.cuda.synchronize()
    assert eng.jpeg_status() == 0


def test_backbone_forward_jpeg_equals_forward_frames():
    eng = _engine('bf16')
    be = eng.backbone
    files = _camera_files(1, seed=11)[0]
    want = [t.clone() for t in be.forward_frames(torch.from_numpy(np.stack([J.cv2_decode(b) for b in files])).to(DEV),
                                                 channels_last_bf16=True)]
    got = be.forward_jpeg(files, channels_last_bf16=True)
    torch.cuda.synchronize()
    assert be.jpeg_status() == 0
    for a, b in zip(want, got):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):                                   # another size: refused before any launch
        be.forward_jpeg(files[:5] + [J.encode(J.make_image('camera', 224, 400), 90)])


# ---------------------------------------------------------------------------------------------------------- detector
def _detector(precision, **kw):
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200 import fixtures
    from occnet_b200.mmcv_shim import build_detector
    cfg = fixtures.make_cfg('small6', bev_h=200, bev_w=200, num_layers=1, img_shape=(232, 400, 3))
    det = build_detector(dict(type='BEVFormerOcc', img_backbone=dict(type='ResNet', depth=50), img_neck=dict(type='FPN'),
                              pts_bbox_head=dict(fixtures.head_cfg(cfg), precision=precision),
                              frame_pad=dict(size=(232, 400)), **kw)).to(DEV).eval()
    det.pts_bbox_head.load_state_dict(fixtures.init_params(cfg, seed=2), strict=True)
    assert not det.load_state_dict(fixtures.init_backbone_params(seed=5), strict=False).unexpected_keys
    return cfg, det


def _bare_metas(cfg, bs, angle=None, token=None):
    from occnet_b200 import fixtures
    metas = [{k: v for k, v in m.items() if k != 'img_shape'} for m in fixtures.make_img_metas(cfg, bs=bs, can_bus_angle=angle)]
    if token is not None:
        for m in metas:
            m['scene_token'] = token
    return metas


def _same(a, b):
    assert set(a) == set(b)
    for k in a:
        if isinstance(a[k], dict):
            _same(a[k], b[k])
        elif a[k] is None:
            assert b[k] is None, k
        else:
            assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_detector_from_jpeg_equals_detector_from_frames(precision):
    """BEVFormerOcc.forward_test from the encoded files against the same detector given cv2's uint8 frames: batch 1 with ray
    records and with scoring, batch 2, and video frames on the engine history; the metas the uint8 path fills"""
    from occnet_b200.metric import RayMetric
    files = _camera_files(3, seed=21)
    frames = [torch.from_numpy(np.stack([J.cv2_decode(b) for b in f])) for f in files]
    cfg, det = _detector(precision)
    seen = []
    head_forward = det.pts_bbox_head.forward
    det.pts_bbox_head.forward = lambda feats, img_metas, *a, **k: (seen.append(img_metas), head_forward(feats, img_metas, *a, **k))[1]
    gt = [t.to(DEV) for t in _gt(0)]
    for kw in (dict(), dict(lidar_origins=_origins(0))):
        want = det(return_loss=False, img=[frames[0][None].to(DEV)], img_metas=[_bare_metas(cfg, 1)], **kw)
        got = det(return_loss=False, img=[[files[0]]], img_metas=[_bare_metas(cfg, 1)], **kw)
        _same(want, got)
        assert seen[-1][0]['ori_shape'] == [(220, 400, 3)] * 6 and seen[-1][0]['img_shape'] == [(232, 400, 3)] * 6
    rms = [RayMetric(DEV), RayMetric(DEV)]
    for rm, img in zip(rms, ([frames[1][None].to(DEV)], [files[1]])):
        det(return_loss=False, img=img, img_metas=[_bare_metas(cfg, 1)], lidar_origins=_origins(1), gt_semantics=gt[0][None],
            gt_flow=gt[1][None], ray_metric=rm)
    assert torch.equal(rms[0].counters, rms[1].counters)
    want = det(return_loss=False, img=[torch.stack(frames[:2]).to(DEV)], img_metas=[_bare_metas(cfg, 2)])
    got = det(return_loss=False, img=[[files[0], files[1]]], img_metas=[_bare_metas(cfg, 2)])
    _same(want, got)
    assert len(seen[-1]) == 2 and seen[-1][1]['ori_shape'] == [(220, 400, 3)] * 6

    results = []
    for inputs in (frames, files):
        _, vdet = _detector(precision, video_test_mode=True, temporal_test=True, engine_history=True)
        results.append([vdet(return_loss=False, img=[x[None].to(DEV)] if isinstance(x, torch.Tensor) else [[x]],
                             img_metas=[_bare_metas(cfg, 1, angle=3.0 * i, token='scene-a')]) for i, x in enumerate(inputs)])
    for a, b in zip(*results):
        _same(a, b)
    bad = list(files[2])
    bad[4] = _corrupt(bad[4], 2)
    with pytest.raises(RuntimeError, match='corrupt JPEG'):
        det(return_loss=False, img=[[bad]], img_metas=[_bare_metas(cfg, 1)])
