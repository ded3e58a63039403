"""Host-side mirror of the reference's module / registry API for the occupancy hot path.

Same registered type names, constructor kwargs, forward signatures and state_dict keys as
`projects/mmdet3d_plugin/bevformer/{modules,dense_heads,detectors}` in the reference, so the shipped
configs (`projects/configs/bevformer/bevformer_base_occ.py:45-135`) build these classes unchanged and
reference checkpoints load with `strict=True`.  The modules are parameter containers: arithmetic runs
in libocc_b200 through the C ABI --

  * `BEVFormerOccHead.forward` / `TransformerOcc.forward` : the fused frame engine (occnet_b200.engine)
  * stand-alone attention modules                         : the operator-level entry points
    (`ops.ms_deform_attn_forward`, `ops.linear`, `ops.layer_norm`) with torch only as tensor plumbing.

There is no CPU path: calling a forward with CPU tensors raises.
"""
import copy
import math
import warnings

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..engine import OccEngine, rotation_index_map
from ..mmcv_shim import (ATTENTION, BACKBONES, DETECTORS, HEADS, NECKS, TRANSFORMER, TRANSFORMER_LAYER, TRANSFORMER_LAYER_SEQUENCE,
                         BaseModule, ConfigDict, ConvModule, ModuleList, TransformerLayerSequence, build_attention,
                         build_feedforward_network, build_head, build_loss, build_norm_layer,
                         build_positional_encoding, build_transformer, build_transformer_layer_sequence,
                         constant_init, xavier_init)


def _need_cuda(t, who):
    if not t.is_cuda:
        raise RuntimeError(f'{who}: CUDA tensors required (libocc_b200 has no CPU fallback)')


def _inference_forward(fn):
    """The stand-alone modules run their projections / norms / FFN through `ops.linear` / `ops.layer_norm`, which have no
    backward: in eval mode the forward runs under `no_grad`; in training mode with autograd on it raises instead of
    silently returning a graph that is cut at every projection (only the MSDA operator itself is differentiable)."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *args, **kwargs):
        if self.training and torch.is_grad_enabled():
            raise RuntimeError(f'{type(self).__name__}: the libocc_b200 module mirror is an inference path (its linear / '
                               f'norm building blocks have no autograd); call .eval() or use torch.no_grad()')
        with torch.no_grad():
            return fn(self, *args, **kwargs)
    return wrapped


def _offset_grid_bias(num_heads, num_levels, num_points):
    """Reference init of `sampling_offsets.bias`: head h looks along angle 2*pi*h/num_heads, point i at radius i+1."""
    thetas = torch.arange(num_heads, dtype=torch.float32) * (2.0 * math.pi / num_heads)
    g = torch.stack([thetas.cos(), thetas.sin()], -1)
    g = (g / g.abs().max(-1, keepdim=True)[0]).view(num_heads, 1, 1, 2).repeat(1, num_levels, num_points, 1)
    for i in range(num_points):
        g[:, :, i, :] *= i + 1
    return g.view(-1)


@ATTENTION.register_module()
class MSDeformableAttention3D(BaseModule):
    """reference: modules/spatial_cross_attention.py:178-400"""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=8, im2col_step=64, dropout=0.1,
                 batch_first=True, norm_cfg=None, init_cfg=None):
        super().__init__(init_cfg)
        if embed_dims % num_heads != 0:
            raise ValueError(f'embed_dims must be divisible by num_heads, but got {embed_dims} and {num_heads}')
        self.embed_dims, self.num_heads, self.num_levels, self.num_points = embed_dims, num_heads, num_levels, num_points
        self.im2col_step, self.batch_first, self.norm_cfg, self.output_proj = im2col_step, batch_first, norm_cfg, None
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.init_weights()

    def init_weights(self):
        constant_init(self.sampling_offsets, 0.)
        self.sampling_offsets.bias.data = _offset_grid_bias(self.num_heads, self.num_levels, self.num_points)
        constant_init(self.attention_weights, val=0., bias=0.)
        xavier_init(self.value_proj, distribution='uniform', bias=0.)
        self._is_init = True

    @_inference_forward
    def forward(self, query, key=None, value=None, identity=None, query_pos=None, key_padding_mask=None,
                reference_points=None, spatial_shapes=None, level_start_index=None, **kwargs):
        _need_cuda(query, 'MSDeformableAttention3D')
        value = query if value is None else value
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        bs, nq, _ = query.shape
        nv = value.shape[1]
        assert int((spatial_shapes[:, 0] * spatial_shapes[:, 1]).sum()) == nv
        M, L, P = self.num_heads, self.num_levels, self.num_points
        v = ops.linear(value.float().contiguous(), self.value_proj.weight, self.value_proj.bias)
        if key_padding_mask is not None:
            v = v.masked_fill(key_padding_mask[..., None], 0.0)
        v = v.view(bs, nv, M, -1)
        q = query.float().contiguous()
        off = ops.linear(q, self.sampling_offsets.weight, self.sampling_offsets.bias).view(bs, nq, M, L, P, 2)
        aw = ops.linear(q, self.attention_weights.weight, self.attention_weights.bias).view(bs, nq, M, L * P)
        aw = aw.softmax(-1).view(bs, nq, M, L, P)
        if reference_points.shape[-1] != 2:
            raise ValueError(f'Last dim of reference_points must be 2, but get {reference_points.shape[-1]} instead.')
        D = reference_points.shape[2]
        assert P % D == 0
        norm = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
        off = (off / norm[None, None, None, :, None, :]).view(bs, nq, M, L, P // D, D, 2)
        loc = (reference_points[:, :, None, None, None, :, :] + off).view(bs, nq, M, L, P, 2)
        out = ops.ms_deform_attn_forward(v.contiguous(), spatial_shapes.contiguous(), level_start_index.contiguous(),
                                         loc.contiguous(), aw.contiguous(), self.im2col_step)
        return out if self.batch_first else out.permute(1, 0, 2)


@ATTENTION.register_module()
class SpatialCrossAttention(BaseModule):
    """reference: modules/spatial_cross_attention.py:31-175.  The per-camera rebatch of the reference is a memory
    optimisation; the result is  q + W_o(sum_{cams seeing q} MSDA_cam(q) / max(1, #cams)) + b_o  (SURVEY a6)."""

    def __init__(self, embed_dims=256, num_cams=6, pc_range=None, dropout=0.1, init_cfg=None, batch_first=False,
                 deformable_attention=dict(type='MSDeformableAttention3D', embed_dims=256, num_levels=4), **kwargs):
        super().__init__(init_cfg)
        self.dropout = nn.Dropout(dropout)
        self.pc_range, self.embed_dims, self.num_cams, self.batch_first = pc_range, embed_dims, num_cams, batch_first
        self.deformable_attention = build_attention(deformable_attention)
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.init_weight()

    def init_weight(self):
        xavier_init(self.output_proj, distribution='uniform', bias=0.)

    @_inference_forward
    def forward(self, query, key, value, residual=None, query_pos=None, key_padding_mask=None, reference_points=None,
                spatial_shapes=None, reference_points_cam=None, bev_mask=None, level_start_index=None, flag='encoder',
                **kwargs):
        _need_cuda(query, 'SpatialCrossAttention')
        key = query if key is None else key
        value = key if value is None else value
        inp_residual = query if residual is None else residual
        if query_pos is not None:
            query = query + query_pos
        bs, nq, C = query.shape
        ncam = self.num_cams
        vis = (bev_mask.sum(-1) > 0)                                     # (cam, bs, nq)
        v = value.permute(2, 0, 1, 3).reshape(bs * ncam, -1, C)
        q_all = query[:, None].expand(bs, ncam, nq, C).reshape(bs * ncam, nq, C)
        ref = reference_points_cam.permute(1, 0, 2, 3, 4).reshape(bs * ncam, nq, -1, 2)
        out = self.deformable_attention(query=q_all, key=v, value=v, reference_points=ref, spatial_shapes=spatial_shapes,
                                        level_start_index=level_start_index).view(bs, ncam, nq, C)
        slots = (out * vis.permute(1, 0, 2)[..., None].to(out.dtype)).sum(1)
        count = torch.clamp(vis.permute(1, 2, 0).sum(-1), min=1.0)
        slots = slots / count[..., None]
        slots = ops.linear(slots.contiguous(), self.output_proj.weight, self.output_proj.bias)
        return self.dropout(slots) + inp_residual


@ATTENTION.register_module()
class TemporalSelfAttention(BaseModule):
    """reference: modules/temporal_self_attention.py:25-272"""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, num_bev_queue=2, im2col_step=64,
                 dropout=0.1, batch_first=True, norm_cfg=None, init_cfg=None):
        super().__init__(init_cfg)
        if embed_dims % num_heads != 0:
            raise ValueError(f'embed_dims must be divisible by num_heads, but got {embed_dims} and {num_heads}')
        self.embed_dims, self.num_heads, self.num_levels, self.num_points = embed_dims, num_heads, num_levels, num_points
        self.num_bev_queue, self.im2col_step, self.batch_first, self.norm_cfg = num_bev_queue, im2col_step, batch_first, norm_cfg
        self.dropout = nn.Dropout(dropout)
        Q = num_bev_queue
        self.sampling_offsets = nn.Linear(embed_dims * Q, Q * num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims * Q, Q * num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.init_weights()

    def init_weights(self):
        constant_init(self.sampling_offsets, 0.)
        self.sampling_offsets.bias.data = _offset_grid_bias(self.num_heads, self.num_levels * self.num_bev_queue,
                                                            self.num_points)
        constant_init(self.attention_weights, val=0., bias=0.)
        xavier_init(self.value_proj, distribution='uniform', bias=0.)
        xavier_init(self.output_proj, distribution='uniform', bias=0.)
        self._is_init = True

    @_inference_forward
    def forward(self, query, key=None, value=None, identity=None, query_pos=None, key_padding_mask=None,
                reference_points=None, spatial_shapes=None, level_start_index=None, flag='decoder', **kwargs):
        _need_cuda(query, 'TemporalSelfAttention')
        if value is None:
            assert self.batch_first
            bs, n, c = query.shape
            value = torch.stack([query, query], 1).reshape(bs * 2, n, c)
        identity = query if identity is None else identity
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        bs, nq, C = query.shape
        nv = value.shape[1]
        assert int((spatial_shapes[:, 0] * spatial_shapes[:, 1]).sum()) == nv
        assert self.num_bev_queue == 2
        M, Q, L, P = self.num_heads, self.num_bev_queue, self.num_levels, self.num_points
        qcat = torch.cat([value[:bs], query], -1).float().contiguous()
        v = ops.linear(value.float().contiguous(), self.value_proj.weight, self.value_proj.bias)
        if key_padding_mask is not None:
            v = v.masked_fill(key_padding_mask[..., None], 0.0)
        v = v.reshape(bs * Q, nv, M, -1)
        off = ops.linear(qcat, self.sampling_offsets.weight, self.sampling_offsets.bias).view(bs, nq, M, Q, L, P, 2)
        aw = ops.linear(qcat, self.attention_weights.weight, self.attention_weights.bias).view(bs, nq, M, Q, L * P)
        aw = aw.softmax(-1).view(bs, nq, M, Q, L, P)
        aw = aw.permute(0, 3, 1, 2, 4, 5).reshape(bs * Q, nq, M, L, P).contiguous()
        off = off.permute(0, 3, 1, 2, 4, 5, 6).reshape(bs * Q, nq, M, L, P, 2)
        if reference_points.shape[-1] != 2:
            raise ValueError(f'Last dim of reference_points must be 2, but get {reference_points.shape[-1]} instead.')
        norm = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
        loc = reference_points[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
        out = ops.ms_deform_attn_forward(v.contiguous(), spatial_shapes.contiguous(), level_start_index.contiguous(),
                                         loc.contiguous(), aw, self.im2col_step)
        out = out.permute(1, 2, 0).view(nq, C, bs, Q).mean(-1).permute(2, 0, 1)
        out = ops.linear(out.contiguous(), self.output_proj.weight, self.output_proj.bias)
        if not self.batch_first:
            out = out.permute(1, 0, 2)
        return self.dropout(out) + identity


@TRANSFORMER_LAYER.register_module()
class MyCustomBaseTransformerLayer(BaseModule):
    """reference: modules/custom_base_transformer_layer.py:37-262 (constructor contract: attentions / ffns / norms)."""

    def __init__(self, attn_cfgs=None, ffn_cfgs=dict(type='FFN', embed_dims=256, feedforward_channels=1024, num_fcs=2,
                                                     ffn_drop=0., act_cfg=dict(type='ReLU', inplace=True)),
                 operation_order=None, norm_cfg=dict(type='LN'), init_cfg=None, batch_first=True, **kwargs):
        ffn_cfgs = copy.deepcopy(ffn_cfgs)
        for old, new in dict(feedforward_channels='feedforward_channels', ffn_dropout='ffn_drop', ffn_num_fcs='num_fcs').items():
            if old in kwargs:
                ffn_cfgs[new] = kwargs[old]
        super().__init__(init_cfg)
        self.batch_first = batch_first
        assert set(operation_order) <= {'self_attn', 'norm', 'ffn', 'cross_attn'}
        num_attn = operation_order.count('self_attn') + operation_order.count('cross_attn')
        if isinstance(attn_cfgs, dict):
            attn_cfgs = [copy.deepcopy(attn_cfgs) for _ in range(num_attn)]
        assert num_attn == len(attn_cfgs)
        self.num_attn, self.operation_order, self.norm_cfg = num_attn, operation_order, norm_cfg
        self.pre_norm = operation_order[0] == 'norm'
        self.attentions = ModuleList()
        idx = 0
        for name in operation_order:
            if name in ('self_attn', 'cross_attn'):
                cfg = dict(attn_cfgs[idx])
                cfg.setdefault('batch_first', self.batch_first)
                assert cfg['batch_first'] == self.batch_first
                att = build_attention(cfg)
                att.operation_name = name
                self.attentions.append(att)
                idx += 1
        self.embed_dims = self.attentions[0].embed_dims
        self.ffns = ModuleList()
        n_ffn = operation_order.count('ffn')
        if isinstance(ffn_cfgs, dict):
            ffn_cfgs = [copy.deepcopy(ffn_cfgs) for _ in range(n_ffn)]
        for c in ffn_cfgs:
            c = dict(c)
            c.setdefault('embed_dims', self.embed_dims)
            assert c['embed_dims'] == self.embed_dims
            self.ffns.append(build_feedforward_network(c))
        self.norms = ModuleList()
        for _ in range(operation_order.count('norm')):
            self.norms.append(build_norm_layer(norm_cfg, self.embed_dims)[1])


@TRANSFORMER_LAYER.register_module()
class BEVFormerLayer(MyCustomBaseTransformerLayer):
    """reference: modules/encoder.py:242-406"""

    def __init__(self, attn_cfgs, feedforward_channels, ffn_dropout=0.0, operation_order=None,
                 act_cfg=dict(type='ReLU', inplace=True), norm_cfg=dict(type='LN'), ffn_num_fcs=2, **kwargs):
        super().__init__(attn_cfgs=attn_cfgs, feedforward_channels=feedforward_channels, ffn_dropout=ffn_dropout,
                         operation_order=operation_order, act_cfg=act_cfg, norm_cfg=norm_cfg, ffn_num_fcs=ffn_num_fcs,
                         **kwargs)
        assert len(operation_order) == 6
        assert set(operation_order) == {'self_attn', 'norm', 'cross_attn', 'ffn'}

    @_inference_forward
    def forward(self, query, key=None, value=None, bev_pos=None, query_pos=None, key_pos=None, attn_masks=None,
                query_key_padding_mask=None, key_padding_mask=None, ref_2d=None, ref_3d=None, bev_h=None, bev_w=None,
                reference_points_cam=None, mask=None, spatial_shapes=None, level_start_index=None, prev_bev=None,
                **kwargs):
        ni = ai = fi = 0
        for op in self.operation_order:
            if op == 'self_attn':
                query = self.attentions[ai](query, prev_bev, prev_bev, None, query_pos=bev_pos, key_pos=bev_pos,
                                            reference_points=ref_2d,
                                            spatial_shapes=torch.tensor([[bev_h, bev_w]], device=query.device),
                                            level_start_index=torch.tensor([0], device=query.device), **kwargs)
                ai += 1
            elif op == 'norm':
                n = self.norms[ni]
                query = ops.layer_norm(query.float().contiguous(), n.weight, n.bias)
                ni += 1
            elif op == 'cross_attn':
                query = self.attentions[ai](query, key, value, None, query_pos=query_pos, key_pos=key_pos,
                                            reference_points=ref_3d, reference_points_cam=reference_points_cam, mask=mask,
                                            spatial_shapes=spatial_shapes, level_start_index=level_start_index, **kwargs)
                ai += 1
            elif op == 'ffn':
                f = self.ffns[fi]
                h = ops.linear(query.float().contiguous(), f.layers[0][0].weight, f.layers[0][0].bias, act=1)
                query = ops.linear(h, f.layers[1].weight, f.layers[1].bias, residual=query.float().contiguous())
                fi += 1
        return query


@TRANSFORMER_LAYER_SEQUENCE.register_module()
class BEVFormerEncoder(TransformerLayerSequence):
    """reference: modules/encoder.py:28-239"""

    def __init__(self, *args, pc_range=None, num_points_in_pillar=4, return_intermediate=False,
                 dataset_type='nuscenes', **kwargs):
        super().__init__(*args, **kwargs)
        self.return_intermediate, self.num_points_in_pillar, self.pc_range = return_intermediate, num_points_in_pillar, pc_range

    @staticmethod
    def get_reference_points(H, W, Z=8, num_points_in_pillar=4, dim='3d', bs=1, device='cuda', dtype=torch.float):
        if dim == '3d':
            D = num_points_in_pillar
            zs = torch.linspace(0.5, Z - 0.5, D, dtype=dtype, device=device).view(-1, 1, 1).expand(D, H, W) / Z
            xs = torch.linspace(0.5, W - 0.5, W, dtype=dtype, device=device).view(1, 1, W).expand(D, H, W) / W
            ys = torch.linspace(0.5, H - 0.5, H, dtype=dtype, device=device).view(1, H, 1).expand(D, H, W) / H
            ref = torch.stack((xs, ys, zs), -1).permute(0, 3, 1, 2).flatten(2).permute(0, 2, 1)
            return ref[None].repeat(bs, 1, 1, 1)
        ry, rx = torch.meshgrid(torch.linspace(0.5, H - 0.5, H, dtype=dtype, device=device),
                                torch.linspace(0.5, W - 0.5, W, dtype=dtype, device=device), indexing='ij')
        ref = torch.stack((rx.reshape(-1)[None] / W, ry.reshape(-1)[None] / H), -1)
        return ref.repeat(bs, 1, 1).unsqueeze(2)

    def point_sampling(self, reference_points, pc_range, img_metas):
        """Camera projection of the pillar points (reference :92-151), fp32, same `img_metas[0]` conventions."""
        dev = reference_points.device
        l2i = reference_points.new_tensor(np.asarray([m['lidar2img'] for m in img_metas]))       # (B, N, 4, 4)
        e2l = reference_points.new_tensor(np.asarray(img_metas[0]['ego2lidar']))
        p = reference_points.clone()
        for i in range(3):
            p[..., i] = p[..., i] * (pc_range[i + 3] - pc_range[i]) + pc_range[i]
        p = torch.cat((p, torch.ones_like(p[..., :1])), -1).permute(1, 0, 2, 3)                 # (D, B, Nq, 4)
        D, B, nq = p.shape[:3]
        ncam = l2i.size(1)
        mat = torch.matmul(l2i.float(), e2l.float())                                             # (B, N, 4, 4)
        cam = torch.einsum('bnij,dbqj->dbnqi', mat, p.float())
        eps = 1e-5
        m = cam[..., 2:3] > eps
        xy = cam[..., 0:2] / torch.maximum(cam[..., 2:3], torch.ones_like(cam[..., 2:3]) * eps)
        xy[..., 0] /= img_metas[0]['img_shape'][0][1]
        xy[..., 1] /= img_metas[0]['img_shape'][0][0]
        m = m & (xy[..., 1:2] > 0.0) & (xy[..., 1:2] < 1.0) & (xy[..., 0:1] < 1.0) & (xy[..., 0:1] > 0.0)
        return xy.permute(2, 1, 3, 0, 4), torch.nan_to_num(m).permute(2, 1, 3, 0, 4).squeeze(-1)

    @_inference_forward
    def forward(self, bev_query, key, value, *args, bev_h=None, bev_w=None, bev_pos=None, spatial_shapes=None,
                level_start_index=None, valid_ratios=None, prev_bev=None, **kwargs):
        _need_cuda(bev_query, 'BEVFormerEncoder')
        bs = bev_query.size(1)
        pc = self.pc_range
        ref_3d = self.get_reference_points(bev_h, bev_w, pc[5] - pc[2], self.num_points_in_pillar, '3d', bs,
                                           bev_query.device, bev_query.dtype)
        ref_2d = self.get_reference_points(bev_h, bev_w, dim='2d', bs=bs, device=bev_query.device, dtype=bev_query.dtype)
        rpc, mask = self.point_sampling(ref_3d, pc, kwargs['img_metas'])
        bev_query, bev_pos = bev_query.permute(1, 0, 2), bev_pos.permute(1, 0, 2)
        n = ref_2d.shape[1]
        if prev_bev is not None:
            prev_bev = torch.stack([prev_bev.permute(1, 0, 2), bev_query], 1).reshape(bs * 2, n, -1)
        hybrid = torch.stack([ref_2d, ref_2d], 1).reshape(bs * 2, n, 1, 2)
        inter = []
        for layer in self.layers:
            bev_query = layer(bev_query, key, value, *args, bev_pos=bev_pos, ref_2d=hybrid, ref_3d=ref_3d, bev_h=bev_h,
                              bev_w=bev_w, spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                              reference_points_cam=rpc, bev_mask=mask, prev_bev=prev_bev, **kwargs)
            if self.return_intermediate:
                inter.append(bev_query)
        return torch.stack(inter) if self.return_intermediate else bev_query


def _engine_cfg(head):
    """The C-ABI engine configuration implied by a built `BEVFormerOccHead`."""
    t = head.transformer
    enc = t.encoder
    lay = enc.layers[0]
    tsa, sca = lay.attentions[0], lay.attentions[1]
    da = sca.deformable_attention
    return dict(bev_h=head.bev_h, bev_w=head.bev_w, embed_dims=t.embed_dims, num_heads=da.num_heads,
                num_layers=len(enc.layers), num_cams=t.num_cams, num_levels=da.num_levels,
                num_points_in_pillar=enc.num_points_in_pillar, sca_points=da.num_points, tsa_points=tsa.num_points,
                num_bev_queue=tsa.num_bev_queue, ffn_dim=lay.ffns[0].feedforward_channels, pillar_h=t.pillar_h,
                out_dim=t.out_dim, num_classes=head.num_classes, pc_range=list(enc.pc_range),
                use_cams_embeds=bool(t.use_cams_embeds), rotate_center=list(t.rotate_center))


@TRANSFORMER.register_module()
class TransformerOcc(BaseModule):
    """reference: modules/transformer_occ.py:26-321 (use_3d voxel decoder; parameter containers + `rotate_prev_bev`)."""

    def __init__(self, num_feature_levels=4, num_cams=6, two_stage_num_proposals=300, encoder=None, decoder=None,
                 embed_dims=256, rotate_prev_bev=True, use_shift=True, use_can_bus=True, can_bus_norm=True,
                 use_cams_embeds=True, use_3d=False, use_conv=False, rotate_center=[100, 100], num_classes=18,
                 out_dim=32, pillar_h=16, act_cfg=dict(type='ReLU', inplace=True), norm_cfg=dict(type='BN'),
                 norm_cfg_3d=dict(type='BN3d'), **kwargs):
        super().__init__(**kwargs)
        if not use_3d:
            raise NotImplementedError('libocc_b200 implements the use_3d=True voxel decoder of the shipped configs '
                                      '(bevformer_base_occ.py:95); use_conv / MLP variants are not on the hot path')
        self.encoder = build_transformer_layer_sequence(encoder)
        self.embed_dims, self.num_feature_levels, self.num_cams = embed_dims, num_feature_levels, num_cams
        self.rotate_prev_bev, self.use_shift, self.use_can_bus, self.can_bus_norm = rotate_prev_bev, use_shift, use_can_bus, can_bus_norm
        self.use_cams_embeds, self.use_3d, self.use_conv = use_cams_embeds, use_3d, use_conv
        self.pillar_h, self.out_dim, self.rotate_center = pillar_h, out_dim, rotate_center
        self.two_stage_num_proposals = two_stage_num_proposals
        mid = embed_dims // pillar_h
        mk = lambda cin: ConvModule(cin, out_dim, kernel_size=3, stride=1, padding=1, bias=norm_cfg_3d is None,
                                    conv_cfg=dict(type='Conv3d'), norm_cfg=norm_cfg_3d, act_cfg=act_cfg)
        self.decoder = nn.Sequential(mk(mid), mk(out_dim))
        self.predicter = nn.Sequential(nn.Linear(out_dim, out_dim * 2), nn.Softplus(), nn.Linear(out_dim * 2, num_classes))
        self.flow_predicter = nn.Sequential(nn.Linear(out_dim, out_dim * 2), nn.ReLU(), nn.Linear(out_dim * 2, 2))
        self.level_embeds = nn.Parameter(torch.Tensor(num_feature_levels, embed_dims))
        self.cams_embeds = nn.Parameter(torch.Tensor(num_cams, embed_dims))
        nn.init.normal_(self.level_embeds)
        nn.init.normal_(self.cams_embeds)

    def init_weights(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, (MSDeformableAttention3D, TemporalSelfAttention)):
                m.init_weights()
        nn.init.normal_(self.level_embeds)
        nn.init.normal_(self.cams_embeds)

    def rotate_prev(self, prev_bev, bev_h, bev_w, img_metas):
        """reference :189-205: prev_bev (bs, Nq, C) rotated by can_bus[-1] degrees about `rotate_center` (nearest, zero
        fill), as a row gather with torchvision's own index map (`occnet_b200.engine.rotation_index_map`)."""
        out = torch.zeros_like(prev_bev)
        for i in range(prev_bev.shape[0]):
            m = torch.from_numpy(rotation_index_map(bev_h, bev_w, img_metas[i]['can_bus'][-1], self.rotate_center)).to(prev_bev.device)
            ok = m >= 0
            out[i, ok] = prev_bev[i, m[ok].long()]
        return out


@HEADS.register_module()
class BEVFormerOccHead(BaseModule):
    """reference: dense_heads/bevformer_occ_head.py:32-216.  `forward` runs the libocc_b200 frame engine."""

    def __init__(self, *args, with_box_refine=False, as_two_stage=False, transformer=None, bbox_coder=None,
                 num_cls_fcs=2, code_weights=None, pc_range=[-40, -40, -1.0, 40, 40, 5.4], bev_h=30, bev_w=30,
                 loss_occ=None, loss_flow=None, use_mask=False, positional_encoding=None, precision='fp32',
                 use_tensor_cores=None, test_logits=True, **kwargs):
        super().__init__()
        self.bev_h, self.bev_w, self.num_classes, self.use_mask = bev_h, bev_w, kwargs['num_classes'], use_mask
        self.with_box_refine, self.as_two_stage, self.pc_range = with_box_refine, as_two_stage, pc_range
        self.real_w, self.real_h = pc_range[3] - pc_range[0], pc_range[4] - pc_range[1]
        self.loss_occ = build_loss(loss_occ) if loss_occ else None
        self.loss_flow = build_loss(loss_flow) if loss_flow else None
        self.positional_encoding = build_positional_encoding(positional_encoding)
        self.transformer = build_transformer(transformer)
        self.embed_dims = self.transformer.embed_dims
        self.bev_embedding = nn.Embedding(bev_h * bev_w, self.embed_dims)
        self.precision = precision                       # 'fp32' (reference arithmetic) or 'bf16' (throughput config)
        self.use_tensor_cores = (precision == 'bf16') if use_tensor_cores is None else use_tensor_cores
        # test_logits=False: `forward(test=True)` (the detector's inference call) does not materialise the 43 MB of fp32
        # semantic logits -- `get_occ` only needs their argmax, which the head kernel emits fused ('occ' is then None)
        self.test_logits = test_logits
        self._engine, self._engine_key = None, None

    def init_weights(self):
        self.transformer.init_weights()

    def _get_engine(self, device, level_shapes):
        key = (str(device), tuple(level_shapes), self.precision, self.use_tensor_cores,
               tuple(p._version for p in self.parameters()), tuple(b._version for b in self.buffers()))
        if self._engine is None or key != self._engine_key:
            cfg = dict(_engine_cfg(self), level_shapes=list(level_shapes))
            self._engine = OccEngine(cfg, self.state_dict(), precision=self.precision,
                                     use_tensor_cores=self.use_tensor_cores, device=str(device))
            self._engine_key = key
        return self._engine

    def forward(self, mlvl_feats, img_metas, prev_bev=None, only_bev=False, test=False, ray_origins=None, score=None,
                metric=None):
        """mlvl_feats: 4 x (B, num_cams, C, h, w) CUDA fp32 -> {'bev_embed','occ','flow'} in the reference layouts.
        Frames of a batch are processed independently (== the reference at samples_per_gpu=1, its only shipped mode;
        the reference's batch>1 cross-item quirks, SURVEY a2/a5/a6, are not reproduced).
        `ray_origins` ((1,T,3) or (T,3) lidar origins, batch 1): the frame's engine call also ray-casts the prediction and
        the result carries 'ray_cls' / 'ray_dist' / 'ray_flow' (`OccEngine.forward`).  `score` = (sem_gt, flow_gt, origins)
        with `metric` (batch 1): the frame's engine call also scores the prediction into `metric.counters`."""
        _need_cuda(mlvl_feats[0], 'BEVFormerOccHead')
        bs = mlvl_feats[0].shape[0]
        if (ray_origins is not None or score is not None) and (bs != 1 or only_bev):
            raise ValueError('ray_origins / score take one frame (batch 1) that runs the heads')
        eng = self._get_engine(mlvl_feats[0].device, [tuple(f.shape[-2:]) for f in mlvl_feats])
        rot_maps = None
        if prev_bev is not None:
            if prev_bev.dim() == 4:                                            # (B, C, H, W) = a previous 'bev_embed' (:193-194)
                prev_bev = prev_bev.reshape(bs, -1, self.bev_h * self.bev_w).permute(0, 2, 1)
            elif prev_bev.shape[1] != self.bev_h * self.bev_w:
                prev_bev = prev_bev.permute(1, 0, 2)
            if self.transformer.rotate_prev_bev:
                # nearest-neighbour rotation = a row permutation: torchvision computes the index map (160 KB, cached per
                # angle), the engine applies it while casting prev_bev to its operand type (no 41 MB torch round trip)
                rot_maps = [rotation_index_map(self.bev_h, self.bev_w, img_metas[b]['can_bus'][-1], self.transformer.rotate_center)
                            for b in range(bs)]
        bevs, occs, flows, clss = [], [], [], []
        want = ('bev_embed', 'occ', 'flow', 'occ_cls_i64') if (self.test_logits or not test) else ('bev_embed', 'flow', 'occ_cls_i64')
        for b in range(bs):
            eng.set_cameras([img_metas[b] if b == 0 else dict(img_metas[b], ego2lidar=img_metas[0]['ego2lidar'],
                                                              img_shape=img_metas[0]['img_shape'])])
            eng.set_prev_rotation(None if rot_maps is None else rot_maps[b])
            fb = self._engine_feats(eng, [f[b] for f in mlvl_feats])
            out = eng.forward(fb, prev_bev=None if prev_bev is None else prev_bev[b],
                              want=('bev_embed',) if only_bev else want, ray_origins=ray_origins, score=score, metric=metric)
            rays = {k: v for k, v in out.items() if k.startswith('ray_')}
            bevs.append(out['bev_embed'])
            if not only_bev:
                flows.append(out['flow']); clss.append(out['occ_cls_i64'])
                if 'occ' in out:
                    occs.append(out['occ'])
        bev = torch.stack(bevs)                                               # (B, Nq, C)
        if only_bev:
            return bev
        bev_embed = bev.permute(0, 2, 1).reshape(bs, -1, self.bev_h, self.bev_w)
        # 'occ_cls' is the head kernel's fused argmax (int64, first-max tie rule like torch.argmax): `get_occ` returns it
        # instead of re-reading the 43 MB of logits (reference: softmax(-1).argmax(-1), bevformer_occ_head.py:211-212)
        return dict({'bev_embed': bev_embed, 'occ': torch.stack(occs) if occs else None, 'flow': torch.stack(flows),
                     'occ_cls': torch.stack(clss)}, **rays)

    @staticmethod
    def _engine_feats(eng, fb):
        """one batch item's levels as the engine takes them: fp32 (the reference's dtype), bf16, or bf16 whose memory is
        channels-last (the native backbone's output); the engine's input dtype follows them"""
        cl = fb[0].dtype == torch.bfloat16 and all((not f.is_contiguous()) and f.permute(0, 2, 3, 1).is_contiguous() for f in fb)
        want_dt = torch.bfloat16 if fb[0].dtype == torch.bfloat16 else torch.float32
        if want_dt != eng.feat_dtype or cl != eng.feat_channels_last:
            eng.set_input_dtype(want_dt, channels_last=cl)
        if fb[0].dtype != eng.feat_dtype:
            fb = [f.float() for f in fb]
        return fb

    def forward_video(self, mlvl_feats, img_metas, scene_start, ray_origins=None, score=None, metric=None):
        """One video frame of batch 1 with the BEV history kept inside the engine (`OccEngine.forward_video`): the previous
        frame's BEV never leaves the engine, and the rotation by can_bus[-1] degrees (none when the transformer's
        rotate_prev_bev is False) is computed on the device.  `scene_start` (or the first frame after the engine is built)
        runs without a previous BEV.  Bit-identical to `forward(mlvl_feats, img_metas, prev_bev=<previous frame's
        bev_embed>, test=True)`; the result's 'bev_embed' is None.  `ray_origins`, `score` and `metric`: as for `forward`."""
        _need_cuda(mlvl_feats[0], 'BEVFormerOccHead')
        if mlvl_feats[0].shape[0] != 1:
            raise ValueError(f'forward_video takes batch 1, got {mlvl_feats[0].shape[0]}')
        eng = self._get_engine(mlvl_feats[0].device, [tuple(f.shape[-2:]) for f in mlvl_feats])
        if not eng.history:
            eng.set_history(True)
        eng.set_cameras([img_metas[0]])
        rotation = float(img_metas[0]['can_bus'][-1]) if self.transformer.rotate_prev_bev else None
        want = ('occ', 'flow', 'occ_cls_i64') if self.test_logits else ('flow', 'occ_cls_i64')
        out = eng.forward_video(self._engine_feats(eng, [f[0] for f in mlvl_feats]), rotation=rotation,
                                scene_start=scene_start, want=want, ray_origins=ray_origins, score=score, metric=metric)
        return dict({'bev_embed': None, 'occ': out['occ'][None] if 'occ' in out else None, 'flow': out['flow'][None],
                     'occ_cls': out['occ_cls_i64'][None]}, **{k: v for k, v in out.items() if k.startswith('ray_')})

    def get_occ(self, preds_dicts, img_metas, rescale=False):
        cls = preds_dicts.get('occ_cls')
        if cls is None:                                                       # a dict that did not come from forward()
            cls = preds_dicts['occ'].argmax(-1)                               # argmax(softmax(x)) == argmax(x)
        return cls, preds_dicts['flow']


class _Bottleneck(nn.Module):
    """Parameter container of one ResNet bottleneck (names = mmdet / torchvision: conv1..3, bn1..3, downsample.{0,1})."""

    def __init__(self, inplanes, planes, stride, downsample):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False); self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False); self.bn2 = nn.BatchNorm2d(planes)   # style 'pytorch'
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False); self.bn3 = nn.BatchNorm2d(planes * 4)
        if downsample:
            self.downsample = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride, bias=False), nn.BatchNorm2d(planes * 4))


@BACKBONES.register_module()
class ResNet(BaseModule):
    """mmdet `ResNet` as the shipped config uses it (bevformer_base_occ.py:48-58): depth 50, out_indices (1,2,3), style
    'pytorch', norm_eval.  A PARAMETER CONTAINER with the reference's `state_dict` keys (= torchvision's resnet50, which
    `pretrained='torchvision://resnet50'` loads unchanged); the arithmetic is `occnet_b200.backbone.BackboneEngine`."""

    def __init__(self, depth=50, num_stages=4, out_indices=(1, 2, 3), frozen_stages=-1, norm_cfg=None, norm_eval=True,
                 style='pytorch', with_cp=False, pretrained=None, init_cfg=None, **kwargs):
        super().__init__()
        if depth != 50 or num_stages != 4 or style != 'pytorch' or tuple(out_indices) != (1, 2, 3):
            raise NotImplementedError('libocc_b200 backbone: ResNet-50, 4 stages, style pytorch, out_indices (1,2,3) only')
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        inplanes = 64
        for s, (nblk, planes) in enumerate(zip((3, 4, 6, 3), (64, 128, 256, 512))):
            blocks = [_Bottleneck(inplanes if i == 0 else planes * 4, planes, 2 if (i == 0 and s > 0) else 1, i == 0)
                      for i in range(nblk)]
            setattr(self, f'layer{s + 1}', nn.Sequential(*blocks))
            inplanes = planes * 4

    def forward(self, x):
        raise RuntimeError('ResNet here is a parameter container; run BEVFormerOcc.extract_feat (BackboneEngine)')


@NECKS.register_module()
class FPN(BaseModule):
    """mmdet `FPN` as configured in bevformer_base_occ.py:59-66 (start_level 0, add_extra_convs 'on_output', num_outs 4):
    parameter container with the reference keys lateral_convs.{i}.conv.*, fpn_convs.{i}.conv.*."""

    def __init__(self, in_channels=(512, 1024, 2048), out_channels=256, num_outs=4, start_level=0, end_level=-1,
                 add_extra_convs='on_output', relu_before_extra_convs=True, no_norm_on_lateral=False, conv_cfg=None,
                 norm_cfg=None, act_cfg=None, upsample_cfg=None, init_cfg=None, **kwargs):
        super().__init__()
        if (list(in_channels) != [512, 1024, 2048] or num_outs != 4 or start_level != 0 or add_extra_convs != 'on_output'
                or norm_cfg is not None or act_cfg is not None or out_channels != 256):
            raise NotImplementedError('libocc_b200 neck: the shipped FPN configuration only')

        def cm(ci, co, k, stride=1):
            m = nn.Module()
            m.conv = nn.Conv2d(ci, co, k, stride, k // 2)
            return m
        self.lateral_convs = nn.ModuleList([cm(c, out_channels, 1) for c in in_channels])
        self.fpn_convs = nn.ModuleList([cm(out_channels, out_channels, 3) for _ in in_channels] + [cm(out_channels, out_channels, 3, 2)])

    def forward(self, feats):
        raise RuntimeError('FPN here is a parameter container; run BEVFormerOcc.extract_feat (BackboneEngine)')


@DETECTORS.register_module()
class BEVFormerOcc(BaseModule):
    """reference: detectors/bevformer_occ.py:20-270 (inference shell).  `img_backbone` / `img_neck` are built as
    parameter containers (so reference checkpoints load with their own keys).  Features come from, in this order:
    `img_feats=` handed to forward / simple_test; a `feature_extractor(img)` callable; or the native ResNet-50 + FPN
    (`occnet_b200.backbone.BackboneEngine`, SURVEY 8f rank 1; `native_backbone=False` turns it off) when the config builds
    `img_backbone` / `img_neck` -- images then go to voxels without leaving the device (bf16: channels-last hand-over).

    `img` may also be the camera frames themselves, uint8 (B, N, h, w, 3) in BGR order as decoded, on CUDA or CPU: the native
    backbone's stem then does the test pipeline's NormalizeMultiviewImage(**frame_norm_cfg) + PadMultiViewImage(**frame_pad)
    + DefaultFormatBundle3D on the device (bit-identical to running them on the host in fp32), and copies of the metas get
    the keys those transforms set.  The defaults are the shipped config's (bevformer_base_occ.py:14-15, 166-171).

    `img` may also be the cameras' encoded JPEG files (LoadMultiViewImageFromFiles' input): `[frames]` with `frames` a list of
    B batch items, each a sequence of N bytes-like files (bytes, 1-D uint8 numpy arrays or CPU tensors) in camera order, or
    one item's N files directly.  They are decoded on the GPU into the uint8 frames cv2.imdecode(IMREAD_UNCHANGED) gives
    (`occnet_b200.jpeg`), which then take the uint8 path above, metas included; a corrupt scan raises once the frame has run."""

    def __init__(self, pts_bbox_head=None, img_backbone=None, img_neck=None, use_grid_mask=False, video_test_mode=False,
                 train_cfg=None, test_cfg=None, pretrained=None, feature_extractor=None, native_backbone=True,
                 backbone_precision=None, temporal_test=False, engine_history=False, ray_only=False, score_only=False,
                 frame_norm_cfg=dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False),
                 frame_pad=dict(size_divisor=32), **kwargs):
        super().__init__()
        self.frame_norm_cfg = dict(mean=[float(v) for v in frame_norm_cfg['mean']],
                                   std=[float(v) for v in frame_norm_cfg['std']], to_rgb=bool(frame_norm_cfg.get('to_rgb', True)))
        frame_pad = dict(frame_pad)
        if frame_pad.pop('pad_val', 0) != 0:
            raise NotImplementedError('frame_pad: only pad_val=0 (the shipped value and the default) is supported')
        if (frame_pad.get('size') is None) == (frame_pad.get('size_divisor') is None) or set(frame_pad) - {'size', 'size_divisor'}:
            raise ValueError(f'frame_pad takes exactly one of size=(H, W) / size_divisor=d, got {frame_pad}')
        self.frame_pad = dict(size=frame_pad.get('size'), size_divisor=frame_pad.get('size_divisor'))
        if pts_bbox_head is not None:
            pts_bbox_head = dict(pts_bbox_head)
            pts_bbox_head.pop('train_cfg', None); pts_bbox_head.pop('test_cfg', None)
        self.pts_bbox_head = build_head(pts_bbox_head)
        self.img_backbone_cfg, self.img_neck_cfg = img_backbone, img_neck
        if img_backbone is not None and img_backbone.get('type') == 'ResNet':
            self.img_backbone = BACKBONES.build(dict(img_backbone))
        if img_neck is not None and img_neck.get('type') == 'FPN':
            self.img_neck = NECKS.build(dict(img_neck))
        self.feature_extractor = feature_extractor
        # the backbone runs in the head's precision unless told otherwise (fp32: the reference's arithmetic, CUDA-core GEMMs)
        if backbone_precision is None:
            backbone_precision = getattr(self.pts_bbox_head, 'precision', 'fp32')
        self.native_backbone, self.backbone_precision = native_backbone, backbone_precision
        self._backbone_engine, self._backbone_key = None, None
        self.video_test_mode = video_test_mode
        # temporal_test=False reproduces the reference exactly: its forward_test always passes prev_bev=None
        # (bevformer_occ.py:243-244), `prev_frame_info` is dead state there.  temporal_test=True (with video_test_mode)
        # turns the cache on the way upstream BEVFormer uses it: the previous frame's BEV (kept on the device) feeds the
        # next frame of the SAME scene; a new `scene_token` (or prev_bev_exists=False) resets it (SURVEY 8f rank 3).
        self.temporal_test = temporal_test
        # engine_history=True (with temporal_test and video_test_mode): batch-1 frames keep that BEV inside the head's frame
        # engine instead (`BEVFormerOccHead.forward_video`): no fp32 bev_embed round trip and the rotation is computed on
        # the device.  The outputs are bit-identical to the cache's; `prev_frame_info['prev_bev']` then stays None.
        # Batch > 1 keeps the cache, and a batch > 1 call in the middle of a scene makes the next batch-1 frame start anew.
        self.engine_history = engine_history
        self._engine_history_valid = False
        # ray_only=True: `forward_test(lidar_origins=...)` returns the frame's ray records only; 'occ_results' and
        # 'flow_results' are None and the 10.24 MB of volumes stay on the device
        self.ray_only = ray_only
        # score_only=True: `forward_test(gt_semantics=..., gt_flow=..., lidar_origins=..., ray_metric=...)` only scores the
        # frame into `ray_metric`; 'occ_results' and 'flow_results' are None and nothing is copied to the host
        self.score_only = score_only
        self.prev_frame_info = {'prev_bev': None, 'scene_token': None, 'prev_pos': 0, 'prev_angle': 0}

    @staticmethod
    def _encoded_batch(img):
        """`img` as the encoded files of B batch items (a list of B lists of N bytes-like), or None if it holds tensors"""
        from ..jpeg import is_buffer
        if not isinstance(img, (list, tuple)) or not img:
            return None
        if is_buffer(img[0]):                                            # one item's N files
            return [list(img)]
        if isinstance(img[0], (list, tuple)) and img[0] and is_buffer(img[0][0]):
            return [list(x) for x in img]
        if isinstance(img[0], (list, tuple)) and img[0] and isinstance(img[0][0], (list, tuple)):
            return BEVFormerOcc._encoded_batch(img[0])                     # [frames]: the outer test-time list
        return None

    def _decode_jpeg(self, batch):
        """B items x N encoded files -> uint8 CUDA frames (B, N, h, w, 3), decoded on the GPU on the current stream"""
        from ..jpeg import JpegDecoder
        if not torch.cuda.is_available():
            raise RuntimeError('BEVFormerOcc: JPEG camera files need a CUDA device (libocc_b200 has no CPU path)')
        B, N = len(batch), len(batch[0])
        if any(len(x) != N for x in batch):
            raise ValueError('every batch item must hold the same number of camera files')
        p = next(self.pts_bbox_head.parameters())
        dev = p.device if p.is_cuda else torch.device('cuda', torch.cuda.current_device())
        if getattr(self, '_jpeg', None) is None or self._jpeg.device != dev:
            self._jpeg = JpegDecoder(str(dev))
        with torch.cuda.device(dev):
            frames = self._jpeg.decode([f for x in batch for f in x])
        if isinstance(frames, list):
            raise ValueError('the camera files of one call must all have the same size')
        return frames.view(B, N, *frames.shape[1:])

    def _get_backbone_engine(self, device, shape):
        """the native backbone engine for images of `shape` (B*N, 3, H, W) on `device`, rebuilt when a parameter changes"""
        from ..backbone import BackboneEngine
        key = (str(device), tuple(shape), self.backbone_precision,
               tuple(p._version for p in self.img_backbone.parameters()), tuple(p._version for p in self.img_neck.parameters()))
        if self._backbone_engine is None or key != self._backbone_key:
            sd = {k: v for k, v in self.state_dict().items() if k.startswith(('img_backbone.', 'img_neck.'))}
            self._backbone_engine = BackboneEngine(sd, shape[0], shape[-2:], precision=self.backbone_precision, device=str(device))
            self._backbone_key = key
        return self._backbone_engine

    def extract_img_feat(self, img, img_metas=None, len_queue=None):
        """reference :66-99 (eval: GridMask is the identity).  img (B, N, 3, H, W) -> list of (B, N, 256, h_l, w_l)."""
        if img.dim() == 4:
            img = img.unsqueeze(0)
        B, N = img.shape[:2]
        x = img.reshape(B * N, *img.shape[2:])
        be = self._get_backbone_engine(x.device, x.shape)
        cl = self.backbone_precision == 'bf16' and getattr(self.pts_bbox_head, 'precision', 'fp32') == 'bf16'
        feats = be.forward(x, channels_last_bf16=cl)                           # bf16 head: channels-last hand-over, no copies
        if len_queue is not None:
            return [f.view(B // len_queue, len_queue, N, *f.shape[1:]) for f in feats]
        return [f.view(B, N, *f.shape[1:]) for f in feats]

    def frame_shape(self, h, w):
        """(H, W) that PadMultiViewImage(**frame_pad) pads an h x w frame to"""
        size, d = self.frame_pad['size'], self.frame_pad['size_divisor']
        if size is not None:
            H, W = int(size[0]), int(size[1])
            if H < h or W < w:
                raise ValueError(f'frame_pad size {(H, W)} is smaller than the {h}x{w} camera frames')
            return H, W
        return -(-h // d) * d, -(-w // d) * d

    @staticmethod
    def _check_frames(img):
        if img.dim() == 4:
            img = img.unsqueeze(0)
        if img.dim() != 5 or img.shape[-1] != 3:
            raise ValueError(f'camera frames must be uint8 (B, N, h, w, 3), got shape {tuple(img.shape)}')
        return img

    def frame_metas(self, img_metas, img):
        """Copies of `img_metas` with the keys NormalizeMultiviewImage + PadMultiViewImage set for uint8 frames `img`
        (B, N, h, w, 3): ori_shape (h, w, 3), img_shape = pad_shape (H, W, 3) per camera, pad_fixed_size, pad_size_divisor,
        img_norm_cfg.  A meta that already carries a different img_shape is an error: the camera projection normalises by
        it (encoder.py:133-134)."""
        img = self._check_frames(img)
        N, h, w = img.shape[1:4]
        H, W = self.frame_shape(h, w)
        nc = self.frame_norm_cfg
        out = []
        for m in img_metas:
            have = m.get('img_shape')
            if have is not None and any(tuple(s[:2]) != (H, W) for s in have):
                raise ValueError(f"img_metas carry img_shape {list(have)[:1]}... but the {h}x{w} frames pad to {(H, W)}")
            m = dict(m)
            m.update(ori_shape=[(h, w, 3)] * N, img_shape=[(H, W, 3)] * N, pad_shape=[(H, W, 3)] * N,
                     pad_fixed_size=self.frame_pad['size'], pad_size_divisor=self.frame_pad['size_divisor'],
                     img_norm_cfg=dict(mean=np.asarray(nc['mean'], np.float32), std=np.asarray(nc['std'], np.float32),
                                       to_rgb=nc['to_rgb']))
            out.append(m)
        return out

    def extract_frame_feat(self, img):
        """uint8 camera frames (B, N, h, w, 3), CUDA or CPU -> list of (B, N, 256, h_l, w_l), normalised and padded by the
        native backbone's stem."""
        if not torch.cuda.is_available():
            raise RuntimeError('BEVFormerOcc: camera frames need a CUDA device (libocc_b200 has no CPU path)')
        if not (self.native_backbone and hasattr(self, 'img_backbone') and hasattr(self, 'img_neck')):
            raise RuntimeError('BEVFormerOcc: uint8 camera frames need the native backbone (img_backbone=ResNet, img_neck=FPN)')
        img = self._check_frames(img)
        if not img.is_cuda:
            p = next(self.pts_bbox_head.parameters())
            dev = p.device if p.is_cuda else torch.device('cuda', torch.cuda.current_device())
            img = img.to(dev, non_blocking=img.is_pinned())
        B, N, h, w = img.shape[:4]
        H, W = self.frame_shape(h, w)
        be = self._get_backbone_engine(img.device, (B * N, 3, H, W))
        nc = self.frame_norm_cfg
        be.set_frame_format((h, w), nc['mean'], nc['std'], nc['to_rgb'])
        cl = self.backbone_precision == 'bf16' and getattr(self.pts_bbox_head, 'precision', 'fp32') == 'bf16'
        feats = be.forward_frames(img.reshape(B * N, h, w, 3).contiguous(), channels_last_bf16=cl)
        return [f.view(B, N, *f.shape[1:]) for f in feats]

    def extract_feat(self, img, img_metas=None, len_queue=None):
        if self.feature_extractor is not None:
            return self.feature_extractor(img)
        if self.native_backbone and hasattr(self, 'img_backbone') and hasattr(self, 'img_neck'):
            return self.extract_img_feat(img, img_metas, len_queue=len_queue)
        raise RuntimeError('BEVFormerOcc: pass img_feats=..., set feature_extractor, or configure img_backbone=ResNet / '
                           'img_neck=FPN with native_backbone=True (the default)')

    def obtain_history_bev(self, feats_queue, img_metas_list):
        """reference: detectors/bevformer_occ.py:159-178 -- run the encoder over the history frames (oldest first), each
        frame's BEV feeding the next as `prev_bev`; a frame flagged `prev_bev_exists=False` restarts the recurrence.
        `feats_queue[i]` are the FPN features of history frame i (the reference extracts them from `imgs_queue`)."""
        prev_bev = None
        with torch.no_grad():
            for feats, metas in zip(feats_queue, img_metas_list):
                if not metas[0].get('prev_bev_exists', True):
                    prev_bev = None
                prev_bev = self.pts_bbox_head(feats, metas, prev_bev, only_bev=True)
        return prev_bev

    @staticmethod
    def _ray_results(outs):
        """the head's ray records (CUDA) under the challenge file's names"""
        return {'pcd_cls': outs['ray_cls'], 'pcd_dist': outs['ray_dist'], 'pcd_flow': outs['ray_flow']}

    def simple_test_pts(self, x, img_metas, prev_bev=None, rescale=False, ray_origins=None, score=None, metric=None):
        """-> (bev_embed, occ, flow), and with `ray_origins` a fourth element: the frame's ray records (CUDA tensors);
        `score` / `metric`: the frame scores itself (`BEVFormerOccHead.forward`)"""
        outs = self.pts_bbox_head(x, img_metas, prev_bev=prev_bev, test=True, ray_origins=ray_origins, score=score,
                                  metric=metric)
        occ, flow = self.pts_bbox_head.get_occ(outs, img_metas, rescale=rescale)
        if ray_origins is not None:
            return outs['bev_embed'], occ, flow, self._ray_results(outs)
        return outs['bev_embed'], occ, flow

    def simple_test(self, img_metas, img=None, img_feats=None, prev_bev=None, rescale=False, ray_origins=None, score=None,
                    metric=None, **kwargs):
        if img_feats is None and isinstance(img, torch.Tensor) and img.dtype == torch.uint8:
            img_metas = self.frame_metas(img_metas, img)                       # before any launch: shape errors are free
            return self.simple_test_pts(self.extract_frame_feat(img), img_metas, prev_bev, rescale=rescale,
                                        ray_origins=ray_origins, score=score, metric=metric)
        feats = img_feats if img_feats is not None else self.extract_feat(img, img_metas)
        return self.simple_test_pts(feats, img_metas, prev_bev, rescale=rescale, ray_origins=ray_origins, score=score,
                                    metric=metric)

    def simple_test_video(self, img_metas, img=None, img_feats=None, scene_start=False, rescale=False, ray_origins=None,
                          score=None, metric=None, **kwargs):
        """`simple_test` of one batch-1 video frame on the head engine's BEV history (`BEVFormerOccHead.forward_video`)
        -> (occ, flow), and with `ray_origins` a third element: the frame's ray records (CUDA tensors)"""
        if img_feats is None and isinstance(img, torch.Tensor) and img.dtype == torch.uint8:
            img_metas = self.frame_metas(img_metas, img)
            feats = self.extract_frame_feat(img)
        else:
            feats = img_feats if img_feats is not None else self.extract_feat(img, img_metas)
        outs = self.pts_bbox_head.forward_video(feats, img_metas, scene_start, ray_origins=ray_origins, score=score,
                                                metric=metric)
        occ, flow = self.pts_bbox_head.get_occ(outs, img_metas, rescale=rescale)
        return (occ, flow) if ray_origins is None else (occ, flow, self._ray_results(outs))

    @staticmethod
    def _batch_size(img, img_feats):
        if img_feats is not None:
            return img_feats[0].shape[0]
        return 1 if img is None or img.dim() == 4 else img.shape[0]

    def _results(self, occ, flow, rays):
        """the result dict of `forward_test`: CPU tensors, no volumes for a `ray_only` / `score_only` detector; `rays` (None when the frame
        made no ray records) adds 'ray_results'"""
        res = {'occ_results': None, 'flow_results': None} if self.score_only or self.ray_only else \
            {'occ_results': occ.cpu(), 'flow_results': flow.cpu()}
        if rays is not None:
            res['ray_results'] = {k: v.cpu() for k, v in rays.items()}
        return res

    def forward_test(self, img_metas, img=None, img_feats=None, lidar_origins=None, gt_semantics=None, gt_flow=None,
                     ray_metric=None, **kwargs):
        """`lidar_origins` ((1,T,3) or (T,3), T <= 8, batch 1): the frame's engine call also ray-casts its prediction and
        the result carries 'ray_results' {'pcd_cls' int8, 'pcd_dist' fp16, 'pcd_flow' fp16}, the records
        `datasets.submission.format_results` writes as they are.  Without it the result is {'occ_results', 'flow_results'}.
        `gt_semantics` ((200,200,16) or (1,200,200,16)), `gt_flow` (.., 2) and `ray_metric` (a `RayMetric` on the frame's
        device) together with `lidar_origins` (batch 1): the frame's engine call scores its prediction against that ground
        truth into `ray_metric.counters` instead, what `evaluate_miou` + `ray_based_miou` do with the volumes on the host;
        the result carries ray records only if the detector is `ray_only`."""
        metas = img_metas[0] if isinstance(img_metas[0], (list, tuple)) else img_metas
        encoded = self._encoded_batch(img)
        if encoded is not None:
            img = self._decode_jpeg(encoded)
            res = self._forward_test(metas, img, img_feats, lidar_origins, gt_semantics, gt_flow, ray_metric, **kwargs)
            torch.cuda.current_stream(img.device).synchronize()
            bad = self._jpeg.status()
            if bad:
                raise RuntimeError(f'BEVFormerOcc: corrupt JPEG scan in camera file(s) with bit mask {bad} (item-major '
                                   'order); the results are not valid')
            return res
        if isinstance(img, (list, tuple)):
            img = img[0]
        return self._forward_test(metas, img, img_feats, lidar_origins, gt_semantics, gt_flow, ray_metric, **kwargs)

    def _forward_test(self, metas, img, img_feats, lidar_origins, gt_semantics, gt_flow, ray_metric, **kwargs):
        if self.ray_only and lidar_origins is None:
            raise ValueError('ray_only=True needs lidar_origins for every frame')
        score = None
        if gt_semantics is not None or gt_flow is not None or ray_metric is not None:
            if gt_semantics is None or gt_flow is None or ray_metric is None or lidar_origins is None:
                raise ValueError('scoring a frame needs gt_semantics, gt_flow, lidar_origins and ray_metric together')
            score = (torch.as_tensor(gt_semantics).reshape(200, 200, 16), torch.as_tensor(gt_flow).reshape(200, 200, 16, 2),
                     lidar_origins)
            if not self.ray_only:
                lidar_origins = None
        elif self.score_only:
            raise ValueError('score_only=True needs gt_semantics, gt_flow, lidar_origins and ray_metric for every frame')
        prev_bev = None                                                                             # reference: prev_bev=None
        video = self.temporal_test and self.video_test_mode
        if video:
            info = self.prev_frame_info
            tok = metas[0].get('scene_token')
            new_scene = tok != info['scene_token'] or not metas[0].get('prev_bev_exists', True)
            if new_scene:
                info['prev_bev'] = None                                                             # first frame of a scene
            info['scene_token'] = tok
            prev_bev = info['prev_bev']
            if self.engine_history and self._batch_size(img, img_feats) == 1:
                occ, flow, *rays = self.simple_test_video(metas, img, img_feats=img_feats, ray_origins=lidar_origins,
                                                          score=score, metric=ray_metric,
                                                          scene_start=new_scene or not self._engine_history_valid, **kwargs)
                self._engine_history_valid = True
                return self._results(occ, flow, rays[0] if rays else None)
        new_prev_bev, occ, flow, *rays = self.simple_test(metas, img, img_feats=img_feats, prev_bev=prev_bev,
                                                          ray_origins=lidar_origins, score=score, metric=ray_metric, **kwargs)
        if video:
            self.prev_frame_info['prev_bev'] = new_prev_bev                                         # (B, C, H, W), stays on the device
            self._engine_history_valid = False
        return self._results(occ, flow, rays[0] if rays else None)

    def forward(self, return_loss=False, **kwargs):
        if return_loss:
            raise NotImplementedError('training is outside the inference hot path (SURVEY 8f rank 4)')
        return self.forward_test(**kwargs)
