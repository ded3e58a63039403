"""Operator-level API mirroring what the reference binds from mmcv's compiled extension.

  ext_module.ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_locations,
                                    attention_weights, im2col_step=...)
      reference call site: bevformer/modules/multi_scale_deformable_attn_function.py:118-124
  MultiScaleDeformableAttnFunction_fp32.apply(...)                     :90-128
  dvr.render_forward(sigma, origin, points, tindex, grid, phase)       tools/ray_iou/lib/dvr/dvr.cpp:39-48
  ray_records(sem_u8, flow, origins): the prediction half of NuSceneOcc.format_results, datasets/nuscenes_occ.py:230-255

Same argument meaning and error behaviour (RuntimeError on non-CUDA / non-contiguous input or a batch
that does not divide im2col_step).  torch is only the tensor container: the arithmetic happens in
libocc_b200 through the C ABI.
"""
import numpy as np
import torch

from . import _lib


def _require(t, name, dtype=None):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f'{name} must be a torch.Tensor')
    if not t.is_cuda:
        raise RuntimeError(f'{name} must be a CUDA tensor (libocc_b200 has no CPU path)')
    if not t.is_contiguous():
        raise RuntimeError(f'{name} tensor has to be contiguous')
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError(f'{name} must be {dtype}, got {t.dtype}')


def _same_device(ref, *tensors):
    for t, name in tensors:
        if t.device != ref.device:
            raise RuntimeError(f'{name} is on {t.device}, value on {ref.device}: all tensors must be on one device')


def _check_shape(t, name, shape):
    if tuple(t.shape) != tuple(shape):
        raise RuntimeError(f'{name} has shape {tuple(t.shape)}, expected {tuple(shape)}')


def _msda_sizes(value, spatial_shapes, level_start_index, sampling_locations, attention_weights):
    """(B, Nv, M, C, Nq, L, P) after cross-checking every tensor's shape against value [B, Nv, M, C] and sampling_locations
    [B, Nq, M, L, P, 2].  The kernels index every buffer with these sizes, so a mismatch would read or write outside it.
    The CONTENTS of spatial_shapes and level_start_index (each level inside value's Nv rows) stay unchecked, as in mmcv:
    checking them would need a device-to-host copy and a sync on every call."""
    if value.dim() != 4:
        raise RuntimeError(f'value must be [B, Nv, M, C], got shape {tuple(value.shape)}')
    B, Nv, M, C = value.shape
    if sampling_locations.dim() != 6:
        raise RuntimeError(f'sampling_loc must be [B, Nq, M, L, P, 2], got shape {tuple(sampling_locations.shape)}')
    Nq, L, P = sampling_locations.shape[1], sampling_locations.shape[3], sampling_locations.shape[4]
    _check_shape(sampling_locations, 'sampling_loc', (B, Nq, M, L, P, 2))
    _check_shape(attention_weights, 'attn_weight', (B, Nq, M, L, P))
    _check_shape(spatial_shapes, 'spatial_shapes', (L, 2))
    _check_shape(level_start_index, 'level_start_index', (L,))
    _same_device(value, (spatial_shapes, 'spatial_shapes'), (level_start_index, 'level_start_index'),
                 (sampling_locations, 'sampling_loc'), (attention_weights, 'attn_weight'))
    return B, Nv, M, C, Nq, L, P


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights,
                           im2col_step=64):
    """mmcv `_ext.ms_deform_attn_forward` drop-in -> out [B, Nq, M*C] fp32.  Any contiguous value is accepted: a view whose
    storage is not 16-byte aligned runs the per-channel kernel instead of the 8-channel one."""
    _require(value, 'value', torch.float32)
    _require(spatial_shapes, 'spatial_shapes', torch.int64)
    _require(level_start_index, 'level_start_index', torch.int64)
    _require(sampling_locations, 'sampling_loc', torch.float32)
    _require(attention_weights, 'attn_weight', torch.float32)
    B, Nv, M, C, Nq, L, P = _msda_sizes(value, spatial_shapes, level_start_index, sampling_locations, attention_weights)
    out = torch.empty((B, Nq, M * C), dtype=torch.float32, device=value.device)
    lib = _lib.load()
    with torch.cuda.device(value.device):
        _lib.check(lib.occb200_ms_deform_attn_forward(
            _lib.ptr(value), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(sampling_locations),
            _lib.ptr(attention_weights), B, Nv, M, C, Nq, L, P, int(im2col_step), _lib.ptr(out), _lib.stream_ptr()))
    return out


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights,
                            grad_output, grad_value, grad_sampling_loc, grad_attn_weight, im2col_step=64):
    """mmcv `_ext.ms_deform_attn_backward` drop-in, in place: grad_value is ACCUMULATED into (pass it zeroed for the
    gradient alone), grad_sampling_loc and grad_attn_weight are OVERWRITTEN.  Shapes and devices are checked as in
    `ms_deform_attn_forward`; grad_output must be [B, Nq, M*C] and each gradient the shape of its input."""
    for t, n in ((value, 'value'), (sampling_locations, 'sampling_loc'), (attention_weights, 'attn_weight'),
                 (grad_output, 'grad_output'), (grad_value, 'grad_value'), (grad_sampling_loc, 'grad_sampling_loc'),
                 (grad_attn_weight, 'grad_attn_weight')):
        _require(t, n, torch.float32)
    _require(spatial_shapes, 'spatial_shapes', torch.int64)
    _require(level_start_index, 'level_start_index', torch.int64)
    B, Nv, M, C, Nq, L, P = _msda_sizes(value, spatial_shapes, level_start_index, sampling_locations, attention_weights)
    _check_shape(grad_output, 'grad_output', (B, Nq, M * C))
    _check_shape(grad_value, 'grad_value', value.shape)
    _check_shape(grad_sampling_loc, 'grad_sampling_loc', sampling_locations.shape)
    _check_shape(grad_attn_weight, 'grad_attn_weight', attention_weights.shape)
    _same_device(value, (grad_output, 'grad_output'), (grad_value, 'grad_value'),
                 (grad_sampling_loc, 'grad_sampling_loc'), (grad_attn_weight, 'grad_attn_weight'))
    lib = _lib.load()
    with torch.cuda.device(value.device):
        _lib.check(lib.occb200_ms_deform_attn_backward(
            _lib.ptr(value), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(sampling_locations),
            _lib.ptr(attention_weights), _lib.ptr(grad_output), B, Nv, M, C, Nq, L, P, int(im2col_step),
            _lib.ptr(grad_value), _lib.ptr(grad_sampling_loc), _lib.ptr(grad_attn_weight), _lib.stream_ptr()))


class MultiScaleDeformableAttnFunction_fp32(torch.autograd.Function):
    """Drop-in for the reference autograd Function, forward and backward (inputs are cast to fp32 like
    `custom_fwd(cast_inputs=torch.float32)`, multi_scale_deformable_attn_function.py:93)."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights,
                im2col_step):
        value = value.float().contiguous()
        sampling_locations = sampling_locations.float().contiguous()
        attention_weights = attention_weights.float().contiguous()
        value_spatial_shapes = value_spatial_shapes.contiguous()
        value_level_start_index = value_level_start_index.contiguous()
        ctx.im2col_step = im2col_step
        out = ms_deform_attn_forward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                                     attention_weights, im2col_step)
        ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_output):
        value, shapes, lsi, loc, aw = ctx.saved_tensors
        grad_value = torch.zeros_like(value)
        grad_loc = torch.zeros_like(loc)
        grad_aw = torch.zeros_like(aw)
        ms_deform_attn_backward(value, shapes, lsi, loc, aw, grad_output.float().contiguous(), grad_value, grad_loc,
                                grad_aw, ctx.im2col_step)
        return grad_value, None, None, grad_loc, grad_aw, None


MultiScaleDeformableAttnFunction_fp16 = MultiScaleDeformableAttnFunction_fp32   # reference: both branches pick fp32


def render_forward(sigma, origin, points, tindex, grid, phase='test'):
    """dvr.render_forward drop-in: -> [pred_dist (N,M), gt_dist (N,M), coord_index (N,M,3)] fp32 CUDA tensors."""
    for t, n in ((sigma, 'sigma'), (origin, 'origin'), (points, 'points'), (tindex, 'tindex')):
        _require(t, n, torch.float32)
    if phase != 'test':
        raise RuntimeError(f'UNKNOWN / unsupported PHASE NAME: {phase} (only "test" is on the metric path)')
    N, M = points.shape[0], points.shape[1]
    T, Z, Y, X = [int(g) for g in grid]
    assert tuple(sigma.shape) == (N, T, Z, Y, X), (sigma.shape, grid)
    pred = torch.empty((N, M), dtype=torch.float32, device=sigma.device)
    gt = torch.empty_like(pred)
    coord = torch.empty((N, M, 3), dtype=torch.float32, device=sigma.device)
    lib = _lib.load()
    with torch.cuda.device(sigma.device):
        _lib.check(lib.occb200_render_forward(_lib.ptr(sigma), _lib.ptr(origin), _lib.ptr(points), _lib.ptr(tindex),
                                              N, T, Z, Y, X, M, _lib.ptr(pred), _lib.ptr(gt), _lib.ptr(coord),
                                              _lib.stream_ptr()))
    torch.cuda.current_stream().synchronize()      # the reference op returns after cudaDeviceSynchronize (dvr.cu:384)
    return [pred, gt, coord]


def ray_origins_host(origins):
    """(T,3) or (1,T,3) lidar origins -> (contiguous numpy (T,3) float32 or float64, is_f64).  float64 origins keep their
    dtype (process_one_sample's arithmetic then runs in double, torch's type promotion); everything else is cast to float32."""
    o = origins.detach().cpu().numpy() if isinstance(origins, torch.Tensor) else np.asarray(origins)
    o = np.ascontiguousarray(o.reshape(-1, 3), np.float64 if o.dtype == np.float64 else np.float32)
    if not 1 <= o.shape[0] <= 8:
        raise ValueError(f'ray records take 1..8 lidar origins, got {o.shape[0]}')
    return o, o.dtype == np.float64


_RAYS = {}


def lidar_rays(device):
    """generate_lidar_rays() as a CUDA tensor, uploaded once per device"""
    from .metric import generate_lidar_rays
    device = torch.device(device)
    if device not in _RAYS:
        _RAYS[device] = torch.from_numpy(generate_lidar_rays()).to(device)
    return _RAYS[device]


def ray_records(sem_u8, flow, origins):
    """The challenge file's records of one predicted volume: sem_u8 (200,200,16) uint8 and flow (200,200,16,2) fp32 CUDA
    tensors, origins (T,3) or (1,T,3) float32 / float64 with T <= 8 -> (pcd_cls int8 (T*M,), pcd_dist fp16 (T*M,), pcd_flow
    fp16 (T*M,2)) CUDA tensors, M = 14040 rays: `process_one_sample`'s rows narrowed as numpy's astype narrows them, from
    one walk per ray."""
    _require(sem_u8, 'sem_u8', torch.uint8)
    _require(flow, 'flow', torch.float32)
    if tuple(sem_u8.shape) != (200, 200, 16) or tuple(flow.shape) != (200, 200, 16, 2):
        raise ValueError(f'ray_records needs (200,200,16) classes and (200,200,16,2) flow, got {tuple(sem_u8.shape)} / '
                         f'{tuple(flow.shape)}')
    o, is64 = ray_origins_host(origins)
    rays = lidar_rays(sem_u8.device)
    n = o.shape[0] * rays.shape[0]
    cls = torch.empty(n, dtype=torch.int8, device=sem_u8.device)
    dist = torch.empty(n, dtype=torch.float16, device=sem_u8.device)
    fl = torch.empty((n, 2), dtype=torch.float16, device=sem_u8.device)
    lib = _lib.load()
    with torch.cuda.device(sem_u8.device):
        _lib.check(lib.occb200_ray_records(_lib.ptr(sem_u8), _lib.ptr(flow), _lib.ptr(o), int(is64), o.shape[0], _lib.ptr(rays),
                                           rays.shape[0], _lib.ptr(cls), _lib.ptr(dist), _lib.ptr(fl), _lib.stream_ptr()))
    return cls, dist, fl


def ray_score(sem_pred, flow_pred, sem_gt, flow_gt, origins, counters):
    """ray_score_kernel on its own: adds to `counters` (187 float64, CUDA) what `RayMetric.add_frame` adds for the same
    (200,200,16) uint8 / (200,200,16,2) fp32 CUDA volumes and origins ((T,3) or (1,T,3), T <= 8); rays whose ground-truth
    hit is free skip their walk through the prediction.  The frame engine launches the same kernel for `score=`."""
    for t, name, dt, shape in ((sem_pred, 'sem_pred', torch.uint8, (200, 200, 16)), (sem_gt, 'sem_gt', torch.uint8, (200, 200, 16)),
                               (flow_pred, 'flow_pred', torch.float32, (200, 200, 16, 2)),
                               (flow_gt, 'flow_gt', torch.float32, (200, 200, 16, 2)), (counters, 'counters', torch.float64, (187,))):
        _require(t, name, dt)
        if tuple(t.shape) != shape:
            raise ValueError(f'ray_score: {name} has shape {tuple(t.shape)}, need {shape}')
    o, is64 = ray_origins_host(origins)
    rays = lidar_rays(sem_pred.device)
    lib = _lib.load()
    with torch.cuda.device(sem_pred.device):
        _lib.check(lib.occb200_ray_score(_lib.ptr(sem_pred), _lib.ptr(flow_pred), _lib.ptr(sem_gt), _lib.ptr(flow_gt), _lib.ptr(o),
                                         int(is64), o.shape[0], _lib.ptr(rays), rays.shape[0], _lib.ptr(counters),
                                         _lib.stream_ptr()))
    return counters


def _no_autograd(name, *tensors):
    """The module-level mirror is an INFERENCE path: these two building blocks have no backward.  Silently cutting the
    graph would leave projection / FFN / norm weights without gradients, so a training-mode call fails loudly instead
    (only `MultiScaleDeformableAttnFunction_fp32` is differentiable, as the reference's op is)."""
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise RuntimeError(f'occnet_b200.ops.{name}: no autograd support (inference path); wrap the call in '
                           f'torch.no_grad() or detach the inputs')


def _aligned(t):
    """t itself when its storage is 16-byte aligned (the kernels move it with 16-byte vector accesses), otherwise an
    aligned copy"""
    return t if t is None or t.data_ptr() % 16 == 0 else t.clone()


def _operand(t, name, shape, x):
    """fp32, CUDA, contiguous, on x's device, of `shape`"""
    _require(t, name, torch.float32)
    if t.device != x.device:
        raise RuntimeError(f'{name} is on {t.device}, x on {x.device}')
    _check_shape(t, name, shape)


def linear(x, weight, bias=None, residual=None, act=0):
    """fp32 y = act(x W^T + b) (+ residual) through the CUDA-core GEMM (module-level API mirror).  x [..., K], weight
    [N, K], bias [N], residual with the M*N elements of the output (it is read as [M, N], it does not broadcast); all fp32,
    contiguous, on one CUDA device.  K must be a multiple of 16 and N of 4."""
    _no_autograd('linear', x, weight, bias, residual)
    _require(x, 'x', torch.float32)
    K = x.shape[-1]
    if weight is None or getattr(weight, 'dim', lambda: 0)() != 2:
        raise RuntimeError(f'weight must be [N, K], got {None if weight is None else tuple(weight.shape)}')
    N = weight.shape[0]
    _operand(weight, 'weight', (N, K), x)
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    if bias is not None:
        _operand(bias, 'bias', (N,), x)
    res = None
    if residual is not None:
        _require(residual, 'residual', torch.float32)
        if residual.numel() != M * N:
            raise RuntimeError(f'residual has shape {tuple(residual.shape)} ({residual.numel()} elements), the output '
                               f'[{M}, {N}] has {M * N}')
        res = residual.reshape(M, N)
        _operand(res, 'residual', (M, N), x)
    if act not in (0, 1):
        raise RuntimeError(f'act must be 0 (none) or 1 (ReLU), got {act}')
    out = torch.empty((M, N), dtype=torch.float32, device=x.device)
    x2, weight, bias, res = (_aligned(t) for t in (x2, weight, bias, res))     # copies stay alive until the launch
    lib = _lib.load()
    with torch.cuda.device(x.device):
        _lib.check(lib.occb200_linear_f32(_lib.ptr(x2), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(res), _lib.ptr(out), M, N,
                                          K, act, _lib.stream_ptr()))
    return out.reshape(*x.shape[:-1], N)


def layer_norm(x, gamma, beta):
    """fp32 LayerNorm over the last dimension (eps 1e-5), C = 256: x [..., 256], gamma and beta [256], all fp32,
    contiguous, on one CUDA device."""
    _no_autograd('layer_norm', x, gamma, beta)
    _require(x, 'x', torch.float32)
    C = x.shape[-1]
    _operand(gamma, 'gamma', (C,), x)
    _operand(beta, 'beta', (C,), x)
    x2 = x.reshape(-1, C)
    out = torch.empty_like(x2)
    x2, gamma, beta = (_aligned(t) for t in (x2, gamma, beta))                  # copies stay alive until the launch
    lib = _lib.load()
    with torch.cuda.device(x.device):
        _lib.check(lib.occb200_layernorm_f32(_lib.ptr(x2), _lib.ptr(gamma), _lib.ptr(beta), _lib.ptr(out), x2.shape[0], C,
                                             _lib.stream_ptr()))
    return out.reshape(x.shape)
