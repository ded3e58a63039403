"""Image backbone + neck engine (ResNet-50 + FPN in front of the hot path; SURVEY 8f rank 1).

    reference: BEVFormerOcc.extract_img_feat, detectors/bevformer_occ.py:66-99
               (img_backbone / img_neck configured in projects/configs/bevformer/bevformer_base_occ.py:48-66)

Validated on the GPU against its oracle (tests/test_backbone_gpu.py; oracle/backbone.py is pinned bit-exactly to
torchvision's resnet50 / FeaturePyramidNetwork).  The arithmetic happens in libocc_b200 through the C ABI
(`occb200_backbone_*`); torch is only the tensor container.  There is no CPU or torch fallback.
"""
import ctypes

import numpy as np
import torch

from . import _lib


def _is_param(key):
    return (key.startswith('img_backbone.') or key.startswith('img_neck.')) and not key.endswith('num_batches_tracked')


class BackboneEngine:
    """state_dict: the detector's `state_dict()` (or any mapping holding its img_backbone.* / img_neck.* entries)."""

    def __init__(self, state_dict, num_images, img_hw, precision='fp32', use_tensor_cores=None, device='cuda:0'):
        if not torch.cuda.is_available():
            raise RuntimeError('libocc_b200 backbone needs a CUDA device (there is no CPU path)')
        assert precision in ('fp32', 'bf16')
        self.lib = _lib.load()
        self.precision = precision
        self.device = torch.device(device)
        self.num_images, (self.H, self.W) = int(num_images), (int(img_hw[0]), int(img_hw[1]))
        tc = (precision == 'bf16') if use_tensor_cores is None else bool(use_tensor_cores)
        with torch.cuda.device(self.device):
            self._h = self.lib.occb200_backbone_create(self.num_images, self.H, self.W, 1 if precision == 'bf16' else 0, int(tc))
            if not self._h:
                raise RuntimeError(self.lib.occb200_last_error().decode())
            for k, v in state_dict.items():
                if not _is_param(k):
                    continue
                a = np.ascontiguousarray(v.detach().float().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v, np.float32))
                _lib.check(self.lib.occb200_backbone_load_param(self._h, k.encode(), a.ctypes.data_as(ctypes.c_void_p), a.size))
            _lib.check(self.lib.occb200_backbone_finalize(self._h))
        self.level_shapes = []
        for l in range(4):
            h, w = ctypes.c_int(), ctypes.c_int()
            _lib.check(self.lib.occb200_backbone_level_shape(self._h, l, ctypes.byref(h), ctypes.byref(w)))
            self.level_shapes.append((h.value, w.value))

    def forward(self, img, channels_last_bf16=False):
        """img (num_images, 3, H, W) CUDA fp32 -> list of 4 x (num_images, 256, h_l, w_l) CUDA fp32; with
        `channels_last_bf16` (bf16 engines only) the levels come back as bf16 tensors of the same SHAPE whose memory is
        channels-last (num_images, h_l, w_l, 256) -- written directly by the last convolutions, and consumed as is by
        `OccEngine` (`set_input_dtype(torch.bfloat16, channels_last=True)`): no NCHW fp32 copy, no transpose."""
        if not (isinstance(img, torch.Tensor) and img.is_cuda):
            raise RuntimeError('img must be a CUDA tensor (libocc_b200 has no CPU path)')
        assert tuple(img.shape) == (self.num_images, 3, self.H, self.W), img.shape
        img = img.float().contiguous()
        if channels_last_bf16:
            if self.precision != 'bf16':
                raise RuntimeError('channels_last_bf16 output needs a bf16 backbone engine')
            outs = [torch.empty((self.num_images, h, w, 256), dtype=torch.bfloat16, device=img.device) for h, w in self.level_shapes]
            with torch.cuda.device(img.device):
                _lib.check(self.lib.occb200_backbone_forward_nhwc_bf16(self._h, _lib.ptr(img), *[_lib.ptr(o) for o in outs],
                                                                       _lib.stream_ptr()))
            return [o.permute(0, 3, 1, 2) for o in outs]
        outs = [torch.empty((self.num_images, 256, h, w), dtype=torch.float32, device=img.device) for h, w in self.level_shapes]
        with torch.cuda.device(img.device):
            _lib.check(self.lib.occb200_backbone_forward(self._h, _lib.ptr(img), *[_lib.ptr(o) for o in outs], _lib.stream_ptr()))
        return outs

    def set_frame_format(self, src_hw, mean, std, to_rgb):
        """Frames for `forward_frames` are uint8 (num_images, src_h, src_w, 3) in BGR order (as decoded by mmcv.imread); the
        stem normalises them like NormalizeMultiviewImage(mean, std, to_rgb) (swap first, then (x - mean[c]) * (1/std[c]) in
        fp32, mean / std in the normalised channel order) and pads them with 0 at the bottom / right to the engine's H x W
        like PadMultiViewImage(pad_val=0)."""
        src_h, src_w = int(src_hw[0]), int(src_hw[1])
        m = np.ascontiguousarray(np.asarray(mean, np.float32).reshape(3))
        s = np.ascontiguousarray(np.asarray(std, np.float32).reshape(3))
        _lib.check(self.lib.occb200_backbone_set_frame_format(self._h, src_h, src_w, _lib.ptr(m), _lib.ptr(s), int(bool(to_rgb))))
        self.frame_hw = (src_h, src_w)

    def check_frames(self, frames, cuda=True):
        """Host-side contract of a frame buffer: a wrong tensor would be an out-of-bounds read on the device."""
        hw = getattr(self, 'frame_hw', None)
        if hw is None:
            raise RuntimeError('BackboneEngine: call set_frame_format() before passing camera frames')
        want = (self.num_images, hw[0], hw[1], 3)
        if not isinstance(frames, torch.Tensor):
            raise TypeError('frames must be a torch.Tensor')
        if frames.dtype != torch.uint8:
            raise ValueError(f'frames must be uint8, got {frames.dtype}')
        if tuple(frames.shape) != want:
            raise ValueError(f'frames shape {tuple(frames.shape)} != {want} (num_images, src_h, src_w, 3)')
        if not frames.is_contiguous():
            raise ValueError('frames must be contiguous (num_images, src_h, src_w, 3)')
        if frames.is_cuda != cuda:
            raise ValueError(f'frames must be a {"CUDA" if cuda else "CPU (pinned)"} tensor')

    def forward_frames(self, frames, channels_last_bf16=False):
        """frames (num_images, src_h, src_w, 3) CUDA uint8, contiguous -> the same 4 levels as `forward` returns for the
        normalised, padded fp32 images, bit for bit (see `set_frame_format`)."""
        self.check_frames(frames, cuda=True)
        if channels_last_bf16 and self.precision != 'bf16':
            raise RuntimeError('channels_last_bf16 output needs a bf16 backbone engine')
        with torch.cuda.device(frames.device):
            if channels_last_bf16:
                outs = [torch.empty((self.num_images, h, w, 256), dtype=torch.bfloat16, device=frames.device) for h, w in self.level_shapes]
                _lib.check(self.lib.occb200_backbone_forward_frames(self._h, _lib.ptr(frames), *[_lib.ptr(o) for o in outs], 1,
                                                                    _lib.stream_ptr()))
                return [o.permute(0, 3, 1, 2) for o in outs]
            outs = [torch.empty((self.num_images, 256, h, w), dtype=torch.float32, device=frames.device) for h, w in self.level_shapes]
            _lib.check(self.lib.occb200_backbone_forward_frames(self._h, _lib.ptr(frames), *[_lib.ptr(o) for o in outs], 0,
                                                                _lib.stream_ptr()))
        return outs

    def forward_jpeg(self, files, channels_last_bf16=False):
        """files: the num_images encoded camera files (bytes-like, in image order; `occnet_b200.jpeg`) of the frame format's
        size -> decoded on the GPU into the frames cv2.imdecode(IMREAD_UNCHANGED) gives, then `forward_frames`.  The sizes are
        checked on the host before anything is launched; `jpeg_status()` after a synchronise reports a corrupt scan."""
        from .jpeg import JpegDecoder, image_size
        hw = getattr(self, 'frame_hw', None)
        if hw is None:
            raise RuntimeError('BackboneEngine: call set_frame_format() before passing camera files')
        files = list(files)
        if len(files) != self.num_images:
            raise ValueError(f'expected {self.num_images} camera files, got {len(files)}')
        for i, f in enumerate(files):
            if image_size(f) != tuple(hw):
                raise ValueError(f'camera file {i} is {image_size(f)} (h, w), the frame format is {tuple(hw)}')
        if getattr(self, '_jpeg', None) is None:
            self._jpeg = JpegDecoder(self.device)
        with torch.cuda.device(self.device):
            frames = self._jpeg.decode(files)
        return self.forward_frames(frames, channels_last_bf16=channels_last_bf16)

    def jpeg_status(self):
        """after `forward_jpeg` and a synchronise of its stream: bit i set = camera file i had a corrupt scan"""
        return self._jpeg.status()

    def __del__(self):
        h = getattr(self, '_h', None)
        if h:
            self.lib.occb200_backbone_destroy(h)
            self._h = None
