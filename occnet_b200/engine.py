"""Python handle of the libocc_b200 frame engine (C ABI: occb200_engine_*).

This is the host-side counterpart of `BEVFormerOccHead.forward` + `get_occ`
(reference: bevformer/dense_heads/bevformer_occ_head.py:99-160, 198-216): parameters come in under
their reference state_dict keys, camera geometry comes from `img_metas` exactly as
`BEVFormerEncoder.point_sampling` reads it (encoder.py:94-101, 133-134).
"""
import contextlib
import ctypes
import itertools
import numbers

import numpy as np
import torch

from . import _lib
from .jpeg import host_buffer
from .ops import ray_origins_host

PRECISIONS = {'fp32': 0, 'bf16': 1}


def _cfg_struct(cfg, precision, use_tensor_cores):
    c = _lib.OccConfig()
    c.bev_h, c.bev_w = cfg['bev_h'], cfg['bev_w']
    c.embed_dims, c.num_heads = cfg['embed_dims'], cfg['num_heads']
    c.num_layers, c.num_cams, c.num_levels = cfg['num_layers'], cfg['num_cams'], cfg['num_levels']
    for i, (h, w) in enumerate(cfg['level_shapes']):
        c.level_h[i], c.level_w[i] = h, w
    c.num_points_in_pillar = cfg['num_points_in_pillar']
    c.sca_points, c.tsa_points = cfg['sca_points'], cfg['tsa_points']
    c.ffn_dim, c.pillar_h, c.out_dim, c.num_classes = cfg['ffn_dim'], cfg['pillar_h'], cfg['out_dim'], cfg['num_classes']
    for i in range(6):
        c.pc_range[i] = cfg['pc_range'][i]
    c.precision = PRECISIONS[precision]
    c.use_tensor_cores = int(use_tensor_cores)
    c.use_cams_embeds = int(cfg.get('use_cams_embeds', True))
    rc = cfg.get('rotate_center', [100, 100])
    c.rotate_center[0], c.rotate_center[1] = int(rc[0]), int(rc[1])
    return c


def camera_params(cfg, img_metas):
    """-> (cam_mat (num_cams,16) f32, zs (D,) f32, img_h, img_w), with the reference's fp32 operation order:
    lidar2img / ego2lidar are cast to fp32 first, then multiplied (encoder.py:100-101, 126)."""
    l2i = torch.from_numpy(np.asarray(img_metas[0]['lidar2img'])).to(torch.float32)
    e2l = torch.from_numpy(np.asarray(img_metas[0]['ego2lidar'])).to(torch.float32)
    cam = torch.matmul(l2i, e2l).reshape(-1, 16).contiguous().numpy()
    Z = cfg['pc_range'][5] - cfg['pc_range'][2]
    D = cfg['num_points_in_pillar']
    zs = (torch.linspace(0.5, Z - 0.5, D, dtype=torch.float32) / Z).contiguous().numpy()
    h, w = img_metas[0]['img_shape'][0][:2]
    return cam, zs, int(h), int(w)


_ROT_CACHE = {}


def rotation_index_map(bev_h, bev_w, angle_deg, center):
    """Index map of the reference's prev_bev rotation (transformer_occ.py:195-205), obtained from the SAME torchvision
    call applied to an image of cell indices -- so ties, centre handling and out-of-image cells are torchvision's, not a
    re-derivation: returns (bev_h*bev_w,) int32, entry q = source cell of output cell q, -1 = outside (zero fill)."""
    key = (bev_h, bev_w, float(angle_deg), tuple(center))
    if key not in _ROT_CACHE:
        from torchvision.transforms.functional import rotate
        idx = torch.arange(1, bev_h * bev_w + 1, dtype=torch.float32).reshape(1, bev_h, bev_w)   # exact in fp32 (< 2^24)
        rot = rotate(idx, float(angle_deg), center=list(center))                                 # nearest, fill 0
        if len(_ROT_CACHE) > 64:
            _ROT_CACHE.clear()
        _ROT_CACHE[key] = (rot.reshape(-1).to(torch.int64) - 1).to(torch.int32).numpy()
    return _ROT_CACHE[key]


def score_args(score, metric, device, host):
    """The checks of a frame call's `score=(sem_gt, flow_gt, origins)` / `metric=` -> (sem_gt uint8 (200,200,16), flow_gt
    fp32 (200,200,16,2), origins numpy (T,3), is_f64).  The ground truth comes back on `device` for the device calls and on
    the CPU (`host`) for the host calls, converted only when it is not already a contiguous tensor of that kind."""
    if metric is None:
        raise ValueError('score= needs metric=, the RayMetric whose counters receive the frame')
    if metric.counters.device != device:
        raise ValueError(f'metric lives on {metric.counters.device}, the engine on {device}: its counters must be on the '
                         f"engine's device")
    sem_gt, flow_gt, origins = score
    where = torch.device('cpu') if host else device
    sem_gt = torch.as_tensor(sem_gt).to(where, torch.uint8).contiguous()
    flow_gt = torch.as_tensor(flow_gt).to(where, torch.float32).contiguous()
    if tuple(sem_gt.shape) != (200, 200, 16) or tuple(flow_gt.shape) != (200, 200, 16, 2):
        raise ValueError(f'score: ground truth {tuple(sem_gt.shape)} / {tuple(flow_gt.shape)}, need (200, 200, 16) / '
                         f'(200, 200, 16, 2)')
    return (sem_gt, flow_gt) + ray_origins_host(origins)


class OccEngine:
    def __init__(self, cfg, params, precision='fp32', use_tensor_cores=False, device='cuda:0'):
        if not torch.cuda.is_available():
            raise RuntimeError('OccEngine needs a CUDA device (no CPU fallback)')
        self.cfg = dict(cfg)
        self.precision = precision
        self.device = torch.device(device)
        self.lib = _lib.load()
        self._h = ctypes.c_void_p()
        c = _cfg_struct(cfg, precision, use_tensor_cores)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_engine_create(ctypes.byref(c), ctypes.byref(self._h)))
            for k, v in params.items():
                if k.endswith('num_batches_tracked'):
                    continue
                a = np.ascontiguousarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v, np.float32)
                _lib.check(self.lib.occb200_engine_load_param(self._h, k.encode(), _lib.ptr(a), a.size))
            _lib.check(self.lib.occb200_engine_finalize(self._h))
        self.Nq = cfg['bev_h'] * cfg['bev_w']
        self.vox_shape = (cfg['bev_w'], cfg['bev_h'], cfg['pillar_h'])
        self._pinned = None
        self.feat_dtype, self.feat_channels_last = torch.float32, False
        self.backbone = None
        self.history = False                                          # set_history(True) has allocated the BEV history
        self.num_rays = 0                                             # set_rays() has uploaded the ray bundle
        self._slot_gt = [None, None]                                  # a submitted frame's ground truth, alive while in flight

    def set_input_dtype(self, dtype, channels_last=False):
        """Feature levels are handed over as `dtype` from now on (torch.float32, the reference's, or torch.bfloat16);
        `channels_last` (bf16 only): tensors of shape (num_cams, C, h, w) whose MEMORY is (num_cams, h, w, C) -- the
        backbone engine's native output.  torch.uint8: each frame is ONE tensor of camera frames (num_cams, src_h, src_w, 3)
        that the attached backbone (`attach_backbone`) turns into the levels on the device first.  'jpeg': each frame is the
        num_cams encoded camera files in camera order (bytes, 1-D uint8 numpy arrays or CPU tensors; `load_jpeg_frame`), in
        host memory for every call, device or host; the engine decodes them on the GPU into the frames cv2.imdecode gives
        (occnet_b200/jpeg.py) and runs the attached backbone on them.  A host call whose file has a corrupt scan raises
        (forward_host, or wait_host for a slot); after a device call, `jpeg_status()` reports it."""
        assert dtype in (torch.float32, torch.bfloat16, torch.uint8, 'jpeg') and not (channels_last and dtype != torch.bfloat16)
        code = 4 if dtype == 'jpeg' else 3 if dtype == torch.uint8 else (2 if channels_last else int(dtype == torch.bfloat16))
        _lib.check(self.lib.occb200_engine_set_input_dtype(self._h, code))
        self.feat_dtype, self.feat_channels_last = dtype, bool(channels_last)

    def attach_backbone(self, backbone):
        """`backbone`: a `BackboneEngine` with one image per camera, this engine's level shapes and a frame format
        (`set_frame_format`), or None to detach.  Borrowed: the engine keeps a reference while it is attached."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_engine_attach_backbone(self._h, None if backbone is None else backbone._h))
        self.backbone = backbone

    def __del__(self):
        h = getattr(self, '_h', None)
        if h is not None and h.value:
            self.lib.occb200_engine_destroy(h)
            self._h = ctypes.c_void_p()

    def set_cameras(self, img_metas):
        cam, zs, h, w = camera_params(self.cfg, img_metas)
        _lib.check(self.lib.occb200_engine_set_cameras(self._h, _lib.ptr(cam), _lib.ptr(zs), h, w))

    def set_prev_rotation(self, index_map):
        """`index_map` (Nq,) int32 numpy / tensor: source BEV cell of every output cell (-1 = outside), e.g. from
        `rotation_index_map`; a real number: the angle in degrees (can_bus[-1]) about the config's rotate_center, whose
        source cells the engine computes on the device (the same cells as `rotation_index_map`); None = prev_bev arrives
        already rotated.  The last call wins."""
        if index_map is None:
            _lib.check(self.lib.occb200_engine_set_prev_rotation(self._h, None))
            return
        if isinstance(index_map, numbers.Real):
            _lib.check(self.lib.occb200_engine_set_prev_rotation_angle(self._h, float(index_map)))
            return
        m = np.ascontiguousarray(index_map.cpu().numpy() if isinstance(index_map, torch.Tensor) else index_map, np.int32)
        assert m.shape == (self.Nq,)
        _lib.check(self.lib.occb200_engine_set_prev_rotation(self._h, _lib.ptr(m)))

    # ------------------------------------------------------------------------------------------------------ ray records
    def set_rays(self, rays=None):
        """Upload the constant ray bundle, (M,3) float32 (default: `generate_lidar_rays()`), for `ray_origins=`; called on
        first use."""
        if rays is None:
            from .metric import generate_lidar_rays
            rays = generate_lidar_rays()
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 3)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_engine_set_rays(self._h, _lib.ptr(rays), rays.shape[0]))
        self.num_rays = rays.shape[0]

    def ray_buffers(self, T=8, host=False):
        """{'ray_cls' int8 (T*M,), 'ray_dist' fp16 (T*M,), 'ray_flow' fp16 (T*M,2)}: CUDA tensors, or pinned CPU tensors"""
        if not self.num_rays:
            self.set_rays()
        n = T * self.num_rays
        kw = dict(pin_memory=True) if host else dict(device=self.device)
        return {'ray_cls': torch.empty(n, dtype=torch.int8, **kw), 'ray_dist': torch.empty(n, dtype=torch.float16, **kw),
                'ray_flow': torch.empty((n, 2), dtype=torch.float16, **kw)}

    @contextlib.contextmanager
    def _ray_request(self, origins, bufs=None, host=False):
        """Arm the frame call made inside the block with `origins` ((T,3) or (1,T,3), float32 / float64, T <= 8; None: no
        request).  Yields the record tensors, the first T*M rows of `bufs` (allocated when None).  A frame call that raises
        leaves nothing armed."""
        if origins is None:
            yield {}
            return
        o, is64 = ray_origins_host(origins)
        if not self.num_rays:
            self.set_rays()
        if bufs is None:
            bufs = self.ray_buffers(o.shape[0], host=host)
        n = o.shape[0] * self.num_rays
        rec = {k: v[:n] for k, v in bufs.items()}
        _lib.check(self.lib.occb200_engine_request_rays(self._h, _lib.ptr(o), int(is64), o.shape[0], _lib.ptr(rec['ray_cls']),
                                                        _lib.ptr(rec['ray_dist']), _lib.ptr(rec['ray_flow'])))
        try:
            yield rec
        except BaseException:
            self.lib.occb200_engine_request_rays(self._h, None, 0, 0, None, None, None)
            raise

    @contextlib.contextmanager
    def _score_request(self, score, metric, slot=None, host=False):
        """Arm the frame call made inside the block to score itself: `score` = (sem_gt (200,200,16) uint8, flow_gt
        (200,200,16,2) fp32, origins as for `_ray_request`), CUDA tensors for the device calls and (pinned) CPU tensors for
        the host calls; the frame's 187 counters are added to `metric.counters` (a `RayMetric` on this device).  None: no
        request.  A frame call that raises leaves nothing armed."""
        if score is None:
            yield
            return
        sem_gt, flow_gt, o, is64 = score_args(score, metric, self.device, host)
        if not self.num_rays:
            self.set_rays()
        if slot is not None:
            self._slot_gt[slot] = (sem_gt, flow_gt)                   # the slot's upload reads them after the call returns
        _lib.check(self.lib.occb200_engine_request_score(self._h, _lib.ptr(sem_gt), _lib.ptr(flow_gt), _lib.ptr(o), int(is64),
                                                         o.shape[0], _lib.ptr(metric.counters)))
        try:
            yield
        except BaseException:
            self.lib.occb200_engine_request_score(self._h, None, None, None, 0, 0, None)
            raise

    def _check_feats(self, feats, cuda):
        """A mismatched tensor would be an out-of-bounds device read in the pack kernel: fail on the host instead."""
        if self.feat_dtype == 'jpeg':
            if self.backbone is None:
                raise RuntimeError("JPEG input ('jpeg') needs an attached backbone: call attach_backbone() first")
            if isinstance(feats, (bytes, bytearray, torch.Tensor, np.ndarray)) or len(feats) != self.cfg['num_cams']:
                raise ValueError(f'a JPEG frame is a sequence of {self.cfg["num_cams"]} encoded camera files')
            for f in feats:
                host_buffer(f)
            return
        if self.feat_dtype == torch.uint8:
            if self.backbone is None:
                raise RuntimeError('camera-frame input (torch.uint8) needs an attached backbone: call attach_backbone() first')
            self.backbone.check_frames(feats, cuda=cuda)
            return
        nc, C = self.cfg['num_cams'], self.cfg['embed_dims']
        if len(feats) != self.cfg['num_levels']:
            raise ValueError(f'expected {self.cfg["num_levels"]} feature levels, got {len(feats)}')
        for l, (f, (h, w)) in enumerate(zip(feats, self.cfg['level_shapes'])):
            if tuple(f.shape) != (nc, C, h, w):
                raise ValueError(f'feature level {l}: shape {tuple(f.shape)} != configured {(nc, C, h, w)}')
            dense = f.permute(0, 2, 3, 1).is_contiguous() if self.feat_channels_last else f.is_contiguous()
            if f.dtype != self.feat_dtype or f.is_cuda != cuda or not dense:
                raise ValueError(f'feature level {l}: need a {"channels-last" if self.feat_channels_last else "contiguous"} '
                                 f'{self.feat_dtype} {"CUDA" if cuda else "CPU (pinned)"} tensor')

    def _feat_ptrs(self, feats):
        if self.feat_dtype == 'jpeg':
            # feats[0] -> occb200_encoded_frame; the engine copies the files into its staging buffer before the call returns
            bufs = [host_buffer(f) for f in feats]
            desc = _lib.EncodedFrame()
            for c, (addr, n, _) in enumerate(bufs):
                desc.data[c], desc.size[c] = addr, n
            arr = (ctypes.c_void_p * 4)(ctypes.addressof(desc))
            arr._keep = (desc, bufs)
            return arr
        arr = (ctypes.c_void_p * 4)()
        for i, f in enumerate([feats] if self.feat_dtype == torch.uint8 else feats):
            arr[i] = f.data_ptr()
        return arr

    def _outputs(self, want):
        C = self.cfg['embed_dims']
        X, Y, Z = self.vox_shape
        dev = self.device
        out = {}
        if 'bev_embed' in want:
            out['bev_embed'] = torch.empty((self.Nq, C), dtype=torch.float32, device=dev)
        if 'occ' in want:
            out['occ'] = torch.empty((X, Y, Z, self.cfg['num_classes']), dtype=torch.float32, device=dev)
        if 'flow' in want:
            out['flow'] = torch.empty((X, Y, Z, 2), dtype=torch.float32, device=dev)
        if 'occ_cls' in want:
            out['occ_cls'] = torch.empty((X, Y, Z), dtype=torch.uint8, device=dev)
        if 'occ_cls_i64' in want:
            out['occ_cls_i64'] = torch.empty((X, Y, Z), dtype=torch.int64, device=dev)
        return out

    def forward(self, feats, prev_bev=None, want=('bev_embed', 'occ', 'flow', 'occ_cls'), ray_origins=None, score=None,
                metric=None):
        """feats: 4 CUDA fp32 tensors (num_cams, C, h, w) of one frame, or with `set_input_dtype(torch.uint8)` one CUDA
        uint8 tensor of camera frames (num_cams, src_h, src_w, 3).  Returns a dict of CUDA tensors.  `ray_origins` ((T,3) or
        (1,T,3), T <= 8): the frame also ray-casts its prediction and adds 'ray_cls' int8 (T*M,), 'ray_dist' fp16 (T*M,) and
        'ray_flow' fp16 (T*M,2), the challenge file's records (`ops.ray_records` of this frame's volumes).  `score` = (sem_gt
        (200,200,16) uint8 CUDA, flow_gt (200,200,16,2) fp32 CUDA, origins) with `metric`, a `RayMetric` on this device: the
        frame also scores itself, adding to `metric.counters` what `metric.add_frame` adds for this frame's 'occ_cls' and
        'flow'; the counters are complete when the frame is (stream order)."""
        C = self.cfg['embed_dims']
        dev = self.device
        if not self.feat_channels_last and self.feat_dtype in (torch.float32, torch.bfloat16):
            feats = [f.contiguous() for f in feats]
        self._check_feats(feats, cuda=True)
        out = self._outputs(want)
        if prev_bev is not None:
            prev_bev = prev_bev.to(device=dev, dtype=torch.float32).reshape(self.Nq, C).contiguous()
        with torch.cuda.device(dev), self._ray_request(ray_origins) as rec, self._score_request(score, metric):
            _lib.check(self.lib.occb200_engine_forward(
                self._h, self._feat_ptrs(feats), _lib.ptr(prev_bev), _lib.ptr(out.get('bev_embed')),
                _lib.ptr(out.get('occ')), _lib.ptr(out.get('flow')), _lib.ptr(out.get('occ_cls')),
                _lib.ptr(out.get('occ_cls_i64')), _lib.stream_ptr()))
        out.update(rec)
        return out

    def forward_host(self, feats_host, occ_out=None, flow_out=None, ray_origins=None, volumes=True, score=None, metric=None):
        """feats_host: 4 pinned CPU fp32 tensors (num_cams, C, h, w), or one pinned uint8 tensor of camera frames with
        `set_input_dtype(torch.uint8)` (25.9 MB per 6 x 900 x 1600 frame).  H2D + frame + D2H + sync inside.
        Returns (occ_cls int64 (X,Y,Z) CPU, flow fp32 (X,Y,Z,2) CPU); with `ray_origins` a third element, the frame's ray
        records as pinned CPU tensors (see `forward`).  `score` / `metric`: as for `forward`, with the ground truth as CPU
        tensors; the counters stay on the device.  With `volumes=False` (needs `ray_origins` or `score`) the two volumes are
        None and not copied."""
        X, Y, Z = self.vox_shape
        if not volumes:
            if ray_origins is None and score is None:
                raise ValueError('volumes=False needs ray_origins or score')
            occ_out = flow_out = None
        elif occ_out is None or flow_out is None:
            if self._pinned is None:
                self._pinned = (torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(),
                                torch.empty((X, Y, Z, 2), dtype=torch.float32).pin_memory())
            occ_out, flow_out = self._pinned
        self._check_feats(feats_host, cuda=False)
        arr = self._feat_ptrs(feats_host)
        with torch.cuda.device(self.device), self._ray_request(ray_origins, host=True) as rec, \
                self._score_request(score, metric, host=True):
            _lib.check(self.lib.occb200_engine_forward_host(self._h, arr, _lib.ptr(occ_out), _lib.ptr(flow_out),
                                                            _lib.stream_ptr()))
        return (occ_out, flow_out) if ray_origins is None else (occ_out, flow_out, rec)

    def submit_host(self, slot, feats_host, occ_out, flow_out, ray_origins=None, ray_out=None, score=None, metric=None):
        """Pipelined host-buffer call (slot 0/1): returns immediately; `wait_host(slot)` completes it.  With `ray_origins` the
        frame's ray records go to the pinned CPU tensors `ray_out` (`ray_buffers(host=True)`), whose first T*M rows are
        returned as a dict.  `score` / `metric`: as for `forward_host`; the counters are complete at `wait_host(slot)`.  With
        either request `occ_out` / `flow_out` may be None: that volume is then not copied."""
        self._check_feats(feats_host, cuda=False)
        arr = self._feat_ptrs(feats_host)
        with torch.cuda.device(self.device), self._ray_request(ray_origins, ray_out, host=True) as rec, \
                self._score_request(score, metric, slot, host=True):
            _lib.check(self.lib.occb200_engine_submit_host(self._h, slot, arr, _lib.ptr(occ_out), _lib.ptr(flow_out),
                                                           _lib.stream_ptr()))
        return rec

    def wait_host(self, slot):
        _lib.check(self.lib.occb200_engine_wait_host(self._h, slot))

    def jpeg_status(self):
        """After a device call ('jpeg' input) and a synchronise of its stream: bit c set = camera c's file had a corrupt
        scan (its frame was decoded from zero coefficients, so the outputs are not valid)."""
        s = ctypes.c_int()
        _lib.check(self.lib.occb200_engine_jpeg_status(self._h, ctypes.byref(s)))
        return s.value

    def stream_host(self, frames_host, ray_origins=None, volumes=True, score=None, metric=None):
        """Generator over an iterable of host frames with two frames in flight; yields (occ int64 CPU, flow CPU)
        views of the slot's pinned output buffers (valid until the slot is reused two frames later).  `ray_origins`: one
        origin set per frame ((T,3) or (1,T,3), T <= 8, T may differ between frames); every frame then yields (occ, flow,
        records) with the frame's ray records {'ray_cls', 'ray_dist', 'ray_flow'} as views of the slot's pinned record
        buffers (see `forward`).  `score`: one (sem_gt, flow_gt, origins) of CPU tensors per frame (None: that frame is not
        scored); every scored frame adds its counters to `metric` (see `forward_host`), complete when the frame is yielded.
        `volumes=False` (with `ray_origins` or `score`): occ and flow are None and never leave the device; 786 KB per frame
        cross the bus at T = 8 with ray records, 5.76 MB of ground truth go up with a score, instead of 10.24 MB."""
        if not volumes and ray_origins is None and score is None:
            raise ValueError('volumes=False needs ray_origins or score')
        rays = ray_origins is not None
        items = zip(frames_host, ray_origins if rays else itertools.repeat(None),
                    itertools.repeat(None) if score is None else score)
        return self._stream(items, lambda slot, it, outs, rb: self.submit_host(
            slot, it[0], *outs, ray_origins=it[1], ray_out=rb, score=it[2], metric=metric), volumes=volumes, rays=rays)

    def _stream(self, items, submit, volumes=True, rays=False):
        """submit(slot, item, (occ, flow) pinned or (None, None), the slot's pinned record buffers or None) -> the frame's
        records or None"""
        X, Y, Z = self.vox_shape
        if volumes and getattr(self, '_stream_outs', None) is None:  # pinned once: cudaHostAlloc costs milliseconds
            self._stream_outs = [(torch.empty((X, Y, Z), dtype=torch.int64).pin_memory(),
                                  torch.empty((X, Y, Z, 2)).pin_memory()) for _ in range(2)]
        if rays and getattr(self, '_stream_rays', None) is None:
            self._stream_rays = [self.ray_buffers(8, host=True) for _ in range(2)]
        outs = self._stream_outs if volumes else [(None, None)] * 2
        pending = []

        def finish(slot, rec):
            self.wait_host(slot)
            return outs[slot] + (rec,) if rays else outs[slot]

        for i, item in enumerate(items):
            slot = i & 1
            if len(pending) == 2:
                yield finish(*pending.pop(0))
            rec = submit(slot, item, outs[slot], self._stream_rays[slot] if rays else None)
            pending.append((slot, rec))
        for p in pending:
            yield finish(*p)

    # ---------------------------------------------------------------------------------------- video (temporal) inference
    def set_history(self, enabled=True):
        """Keep the BEV history inside the engine for `forward_video` / `submit_host_video`: one (Nq, 256) buffer in the
        storage precision, allocated (True) or freed (False).  Either way the next video frame starts a new scene."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_engine_set_history(self._h, int(enabled)))
        self.history = bool(enabled)

    def rotation_map(self, angle_deg):
        """-> CUDA int32 (Nq,): the source cell of every BEV cell (-1 = outside) that the engine computes on the device for a
        rotation by `angle_deg` about the config's rotate_center; equal to `rotation_index_map` of the same angle."""
        m = torch.empty(self.Nq, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_engine_rotation_map(self._h, float(angle_deg), _lib.ptr(m), _lib.stream_ptr()))
        return m

    def _rotation_host(self, rotation):
        """None or an index map (Nq,) -> int32 numpy (Nq,) or None.  `submit_host_video` hands the map to the engine, which
        rejects entries outside [-1, Nq)."""
        if rotation is None:
            return None
        m = np.ascontiguousarray(rotation.cpu().numpy() if isinstance(rotation, torch.Tensor) else rotation, np.int32)
        if m.shape != (self.Nq,):
            raise ValueError(f'rotation map: shape {m.shape} != ({self.Nq},)')
        return m

    def _rotation_dev(self, rotation):
        """the same as a CUDA int32 tensor on the current stream.  A CUDA map is used as given (the engine reads entries
        outside [-1, Nq) as -1); a host map is range-checked here and uploaded for this frame only: the upload and the frame
        are ordered on the current stream, so the temporary can be freed when the call returns."""
        if isinstance(rotation, torch.Tensor) and rotation.is_cuda:
            if rotation.dtype != torch.int32 or tuple(rotation.shape) != (self.Nq,) or not rotation.is_contiguous() \
                    or rotation.device != self.device:
                raise ValueError(f'rotation map: need a contiguous int32 ({self.Nq},) tensor on {self.device}')
            return rotation
        m = self._rotation_host(rotation)
        if m is None:
            return None
        if m.min() < -1 or m.max() >= self.Nq:
            raise ValueError(f'rotation map entry out of range: must be in [-1, {self.Nq})')
        return torch.from_numpy(m).pin_memory().to(self.device, non_blocking=True)

    def forward_video(self, feats, rotation=None, scene_start=False, want=('bev_embed', 'occ', 'flow', 'occ_cls'),
                      ray_origins=None, score=None, metric=None):
        """One frame of a video (needs `set_history()`): `feats` as for `forward`; the previous BEV is the engine's history,
        rotated by `rotation` (None, an angle in degrees or an index map), unless `scene_start` or this is the first frame
        since `set_history()` (self mode).  Equals `forward(feats, prev_bev=<previous frame's bev_embed>)` with the same
        rotation, bit for bit; the frame's BEV stays in the history whether or not 'bev_embed' is in `want`.  An angle
        costs no host work: the engine computes the cells of `rotation_index_map(angle)` on the device.  `ray_origins`,
        `score` and `metric`: as for `forward`."""
        if not self.feat_channels_last and self.feat_dtype in (torch.float32, torch.bfloat16):
            feats = [f.contiguous() for f in feats]
        self._check_feats(feats, cuda=True)
        out = self._outputs(want)
        outs = (_lib.ptr(out.get('bev_embed')), _lib.ptr(out.get('occ')), _lib.ptr(out.get('flow')),
                _lib.ptr(out.get('occ_cls')), _lib.ptr(out.get('occ_cls_i64')))
        with torch.cuda.device(self.device):
            rot = None if isinstance(rotation, numbers.Real) else self._rotation_dev(rotation)
            with self._ray_request(ray_origins) as rec, self._score_request(score, metric):
                if isinstance(rotation, numbers.Real):
                    _lib.check(self.lib.occb200_engine_forward_video_angle(
                        self._h, self._feat_ptrs(feats), float(rotation), int(bool(scene_start)), *outs, _lib.stream_ptr()))
                else:
                    _lib.check(self.lib.occb200_engine_forward_video(
                        self._h, self._feat_ptrs(feats), _lib.ptr(rot), int(bool(scene_start)), *outs, _lib.stream_ptr()))
        out.update(rec)
        return out

    def submit_host_video(self, slot, feats_host, occ_out, flow_out, rotation=None, scene_start=False, ray_origins=None,
                          ray_out=None, score=None, metric=None):
        """Pipelined host-buffer video frame (slot 0/1; `submit_host` + the history of `forward_video`): returns
        immediately, `wait_host(slot)` completes it.  An index map is copied before the call returns; an angle needs no
        map at all.  `ray_origins` / `ray_out`, the returned records, `score` and `metric`: as for `submit_host`."""
        self._check_feats(feats_host, cuda=False)
        arr = self._feat_ptrs(feats_host)
        rot = None if isinstance(rotation, numbers.Real) else self._rotation_host(rotation)
        with torch.cuda.device(self.device), self._ray_request(ray_origins, ray_out, host=True) as rec, \
                self._score_request(score, metric, slot, host=True):
            if isinstance(rotation, numbers.Real):
                _lib.check(self.lib.occb200_engine_submit_host_video_angle(
                    self._h, slot, arr, float(rotation), int(bool(scene_start)), _lib.ptr(occ_out), _lib.ptr(flow_out),
                    _lib.stream_ptr()))
            else:
                _lib.check(self.lib.occb200_engine_submit_host_video(self._h, slot, arr, _lib.ptr(rot), int(bool(scene_start)),
                                                                     _lib.ptr(occ_out), _lib.ptr(flow_out), _lib.stream_ptr()))
        return rec

    def stream_host_video(self, items, volumes=True, score=None, metric=None):
        """`stream_host` for video: items are (feats_host, rotation, scene_start); two frames in flight, yields
        (occ int64 CPU, flow CPU) views of the slot's pinned output buffers, frame by frame.  Items with a fourth element,
        the frame's ray origins, make every frame yield (occ, flow, records) as `stream_host(ray_origins=...)` does;
        `score` (one ground truth per item) and `metric`: as for `stream_host`.  `volumes=False` (with ray origins or
        `score`) keeps the volumes on the device."""
        items = iter(items)
        first = next(items, None)
        if first is None:
            return iter(())
        rays = len(first) > 3
        if not volumes and not rays and score is None:
            raise ValueError('volumes=False needs ray origins (a fourth element in every item) or score')
        scored = zip(itertools.chain([first], items), itertools.repeat(None) if score is None else score)
        return self._stream(scored, lambda slot, p, outs, rb: self.submit_host_video(
            slot, p[0][0], *outs, rotation=p[0][1], scene_start=p[0][2], ray_origins=p[0][3] if rays else None, ray_out=rb,
            score=p[1], metric=metric), volumes=volumes, rays=rays)

    def enable_taps(self, on=True):
        _lib.check(self.lib.occb200_engine_enable_taps(self._h, int(on)))

    def tap(self, which, layer=0):
        names = {'layer': 0, 'tsa': 1, 'sca': 2, 'voxel': 3, 'tokens': 4}
        w = names[which]
        if w == 4:
            nv = sum(h * w_ for h, w_ in self.cfg['level_shapes'])
            dst = torch.empty((self.cfg['num_cams'], nv, self.cfg['embed_dims']), dtype=torch.float32, device=self.device)
        elif w == 3:
            X, Y, Z = self.vox_shape
            dst = torch.empty((X, Y, Z, self.cfg['out_dim']), dtype=torch.float32, device=self.device)
        else:
            dst = torch.empty((self.Nq, self.cfg['embed_dims']), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_engine_copy_tap(self._h, w, layer, _lib.ptr(dst), _lib.stream_ptr()))
        return dst

    def project_pillars(self):
        D = self.cfg['num_points_in_pillar']
        nc = self.cfg['num_cams']
        ref = torch.empty((nc, self.Nq, D, 2), dtype=torch.float32, device=self.device)
        mask = torch.empty((nc, self.Nq, D), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.occb200_engine_project_pillars(self._h, _lib.ptr(ref), _lib.ptr(mask), _lib.stream_ptr()))
        return ref, mask

    CATEGORIES = ('pack', 'gemm', 'tsa_gather', 'sca_gather', 'layernorm', 'bev_to_voxel', 'conv3d', 'occ_head')

    def profile(self, on=True):
        _lib.check(self.lib.occb200_engine_profile(self._h, int(on)))

    def profile_read(self):
        """-> {category: (milliseconds, launches)} since the last read (synchronises the device)."""
        ms = np.zeros(8, np.float32)
        n = np.zeros(8, np.int32)
        _lib.check(self.lib.occb200_engine_profile_read(self._h, _lib.ptr(ms), _lib.ptr(n), 8))
        return {c: (float(ms[i]), int(n[i])) for i, c in enumerate(self.CATEGORIES)}

    @property
    def launches_per_frame(self):
        """kernels the last forward launched; with camera frames (torch.uint8) the backbone's kernels are included"""
        return int(self.lib.occb200_engine_launches_per_frame(self._h))
