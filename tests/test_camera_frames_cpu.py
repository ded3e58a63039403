"""Camera frames (uint8, as decoded) as an input: the CPU restatement of the shipped test pipeline's image steps
(oracle/image_pipeline.py) and the detector's host-side handling of frames.  The GPU path is checked against this
restatement in test_camera_frames_gpu.py."""
import numpy as np
import pytest
import torch

from oracle import image_pipeline as IP

MEAN, STD = [103.530, 116.280, 123.675], [1.0, 1.0, 1.0]


def _frames(n, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


def test_full_size_pads_900_to_928_with_size_divisor_32():
    f = _frames(1, 900, 1600)
    imgs, metas = IP.pipeline(f, MEAN, STD, False, size_divisor=32)
    assert imgs.shape == (1, 3, 928, 1600) and imgs.dtype == np.float32
    assert metas['ori_shape'] == [(900, 1600, 3)]
    assert metas['img_shape'] == metas['pad_shape'] == [(928, 1600, 3)]
    assert metas['pad_size_divisor'] == 32 and metas['pad_fixed_size'] is None
    assert not imgs[:, :, 900:].any()                                     # the padded rows hold pad_val 0


def test_fixed_size_pads_to_exactly_that_size_and_pad_is_zero():
    f = _frames(2, 201, 333, seed=1)
    imgs, metas = IP.pipeline(f, MEAN, STD, False, size=(232, 400))
    assert imgs.shape == (2, 3, 232, 400)
    assert metas['img_shape'] == [(232, 400, 3)] * 2 and metas['ori_shape'] == [(201, 333, 3)] * 2
    assert metas['pad_fixed_size'] == (232, 400) and metas['pad_size_divisor'] is None
    assert not imgs[:, :, 201:, :].any() and not imgs[:, :, :, 333:].any()
    with pytest.raises(ValueError):
        IP.pipeline(f, MEAN, STD, False, size=(200, 400))                 # smaller than the frame


def test_size_divisor_rounds_each_side_up():
    assert IP.padded_shape(200, 380, size_divisor=32) == (224, 384)
    assert IP.padded_shape(201, 333, size_divisor=32) == (224, 352)
    assert IP.padded_shape(224, 384, size_divisor=32) == (224, 384)


def test_known_answer_std_one_is_one_subtraction_in_fp32_chw():
    f = _frames(3, 40, 56, seed=2)
    imgs, _ = IP.pipeline(f, MEAN, STD, False, size_divisor=32)
    assert imgs.shape == (3, 3, 64, 64)
    for c in range(3):                                                    # CHW: channel first, BGR order kept (to_rgb=False)
        want = np.float32(f[..., c]).astype(np.float32) - np.float32(MEAN[c])
        assert np.array_equal(imgs[:, c, :40, :56], want)


def test_to_rgb_swaps_before_the_mean_is_subtracted():
    f = _frames(1, 8, 8, seed=3)
    mean, std = (123.675, 116.28, 103.53), (58.395, 57.12, 57.375)
    imgs, metas = IP.pipeline(f, mean, std, True, size_divisor=8)
    for c in range(3):                                                    # output channel c = RGB c = BGR byte 2 - c
        inv = np.float32(1.0 / np.float64(np.float32(std[c])))
        want = (np.float32(f[0, ..., 2 - c]).astype(np.float32) - np.float32(mean[c])) * inv
        assert np.array_equal(imgs[0, c], want.astype(np.float32))
    # normalising in BGR order and swapping afterwards would pair byte 2 with mean[2], not mean[0]
    swap_last = (np.float32(f[0, ..., 2]).astype(np.float32) - np.float32(mean[2])) * np.float32(1.0 / np.float64(np.float32(std[2])))
    assert not np.array_equal(imgs[0, 0], swap_last.astype(np.float32))
    assert metas['img_norm_cfg']['to_rgb'] is True and metas['img_norm_cfg']['mean'].dtype == np.float32


# ---------------------------------------------------------------------------------------------------- detector, host side
def _shipped_detector(**kw):
    import projects.mmdet3d_plugin  # noqa: F401
    from occnet_b200.mmcv_shim import build_detector
    from test_dropin_cpu import shipped_config
    model = dict(shipped_config().model)
    model.update(kw)
    return build_detector(model)


def test_detector_frame_metas_match_the_pad_transform():
    det = _shipped_detector()
    assert det.frame_pad == dict(size=None, size_divisor=32)
    assert det.frame_norm_cfg == dict(mean=MEAN, std=STD, to_rgb=False)
    img = torch.zeros(1, 6, 900, 1600, 3, dtype=torch.uint8)
    metas = [dict(lidar2img=[np.eye(4)] * 6, scene_token='s')]
    got = det.frame_metas(metas, img)
    assert 'img_shape' not in metas[0]                                     # the caller's metas are not modified
    assert got[0]['img_shape'] == got[0]['pad_shape'] == [(928, 1600, 3)] * 6
    assert got[0]['ori_shape'] == [(900, 1600, 3)] * 6
    assert got[0]['pad_size_divisor'] == 32 and got[0]['pad_fixed_size'] is None
    assert np.array_equal(got[0]['img_norm_cfg']['mean'], np.float32(MEAN)) and got[0]['scene_token'] == 's'
    # metas that already carry the padded shape are accepted; a different one is an error
    det.frame_metas([dict(metas[0], img_shape=[(928, 1600, 3)] * 6)], img)
    with pytest.raises(ValueError):
        det.frame_metas([dict(metas[0], img_shape=[(900, 1600, 3)] * 6)], img)


def test_detector_frame_pad_options():
    det = _shipped_detector(frame_pad=dict(size=(232, 400)))
    assert det.frame_shape(220, 400) == (232, 400)
    with pytest.raises(ValueError):
        det.frame_shape(240, 400)
    with pytest.raises(NotImplementedError):
        _shipped_detector(frame_pad=dict(size_divisor=32, pad_val=114))
    with pytest.raises(ValueError):
        _shipped_detector(frame_pad=dict(size=(232, 400), size_divisor=32))


def test_detector_rejects_frames_without_gpu():
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    det = _shipped_detector().eval()
    img = torch.zeros(1, 6, 64, 96, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError):
        det(return_loss=False, img=[img], img_metas=[[dict(lidar2img=[np.eye(4)] * 6)]])
