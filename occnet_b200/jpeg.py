"""JPEG camera files decoded on the GPU, byte-identical to `cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)` -- the decode
`mmcv.imread(name, 'unchanged')` runs in mmdet3d's LoadMultiViewImageFromFiles.

Baseline YCbCr files only (SOF0 / SOF1, 8-bit, one interleaved scan, 4:2:0 or 4:4:4, any restart interval): everything else
raises before any CUDA call.  EXIF orientation is ignored, as IMREAD_UNCHANGED ignores it.  The CPU restatement of the
arithmetic is oracle/jpeg_decode.py; the kernels are occnet_b200/csrc/jpeg.cu.
"""
import ctypes

import numpy as np
import torch

from . import _lib


def load_jpeg_frame(filenames):
    """the encoded bytes of one frame's camera files, in camera order (what `OccEngine` takes with set_input_dtype('jpeg'))"""
    return [open(f, 'rb').read() for f in filenames]


def is_buffer(buf):
    """whether `buf` is one encoded file as `host_buffer` takes it"""
    if isinstance(buf, (bytes, bytearray, memoryview)):
        return True
    if isinstance(buf, np.ndarray):
        return buf.dtype == np.uint8 and buf.ndim == 1
    return isinstance(buf, torch.Tensor) and buf.dtype == torch.uint8 and buf.dim() == 1 and not buf.is_cuda


def host_buffer(buf):
    """bytes-like (bytes, bytearray, 1-D uint8 numpy array, 1-D uint8 CPU tensor) -> (address, size, owner to keep alive)"""
    if isinstance(buf, torch.Tensor):
        if buf.is_cuda or buf.dtype != torch.uint8 or buf.dim() != 1 or not buf.is_contiguous():
            raise ValueError('an encoded image tensor must be a contiguous 1-D uint8 CPU tensor')
        return buf.data_ptr(), buf.numel(), buf
    if isinstance(buf, np.ndarray):
        if buf.dtype != np.uint8 or buf.ndim != 1 or not buf.flags['C_CONTIGUOUS']:
            raise ValueError('an encoded image array must be a contiguous 1-D uint8 array')
        return buf.ctypes.data, buf.size, buf
    if isinstance(buf, (bytes, bytearray, memoryview)):
        a = np.frombuffer(buf, np.uint8)
        return a.ctypes.data, a.size, a
    raise TypeError(f'an encoded image must be bytes-like, got {type(buf).__name__}')


def image_size(buf):
    """(h, w) of one encoded file after the decoder's header checks (host only; raises OccB200Error if unsupported)"""
    addr, n, _ = host_buffer(buf)
    h, w = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().occb200_jpeg_info(ctypes.c_void_p(addr), n, ctypes.byref(h), ctypes.byref(w)))
    return h.value, w.value


class JpegDecoder:
    """`decode(list of bytes-like)` -> CUDA uint8 (n, h, w, 3) BGR (a list of (h_i, w_i, 3) tensors when the sizes differ),
    decoded on the current stream.  `status()` after synchronising that stream: bit i set = image i's scan was corrupt."""

    def __init__(self, device='cuda:0'):
        if not torch.cuda.is_available():
            raise RuntimeError('JpegDecoder needs a CUDA device (there is no CPU path)')
        self.lib = _lib.load()
        self.device = torch.device(device)
        h = ctypes.c_void_p()
        _lib.check(self.lib.occb200_jpeg_create(ctypes.byref(h)))
        self._h = h

    def decode(self, bufs):
        bufs = list(bufs)
        hb = [host_buffer(b) for b in bufs]
        sizes = [image_size(b) for b in bufs]
        n = len(bufs)
        ptrs = (ctypes.c_void_p * n)(*[a for a, _, _ in hb])
        lens = (ctypes.c_int64 * n)(*[s for _, s, _ in hb])
        total = sum(h * w * 3 for h, w in sizes)
        out = torch.empty(total, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_jpeg_decode(self._h, n, ptrs, lens, _lib.ptr(out), total, _lib.stream_ptr()))
        if len(set(sizes)) == 1:
            h, w = sizes[0]
            return out.view(n, h, w, 3)
        views, o = [], 0
        for h, w in sizes:
            views.append(out[o:o + h * w * 3].view(h, w, 3))
            o += h * w * 3
        return views

    def status(self):
        s = ctypes.c_int()
        _lib.check(self.lib.occb200_jpeg_status(self._h, ctypes.byref(s)))
        return s.value

    def __del__(self):
        h = getattr(self, '_h', None)
        if h:
            self.lib.occb200_jpeg_destroy(h)
            self._h = None
