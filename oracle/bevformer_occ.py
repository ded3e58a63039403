"""ORACLE (test infrastructure only -- never imported by the product path).

Plain-torch CPU restatement of the reference's camera->occupancy hot path, function by
function (SURVEY section 8a rows a1-a13).  Each function cites the reference lines it
follows (paths relative to projects/mmdet3d_plugin/bevformer/ of the reference tree).  All
arithmetic is fp32, eval mode (dropout = identity, BatchNorm uses running statistics).

Parameters travel in a flat dict keyed exactly like the reference's
`pts_bbox_head.state_dict()` (e.g. 'transformer.encoder.layers.0.attentions.1.output_proj.weight'),
so a reference checkpoint can be fed to the oracle and to the CUDA path unchanged.

Third-party pieces restated from their published semantics (absent from the reference tree):
mmcv FFN / LayerNorm / ConvModule, mmdet LearnedPositionalEncoding, mmcv MSDA (oracle/msda.py).

Parity status: pinned against the UNMODIFIED reference modules, imported through an mmcv stand-in (tests/golden/gen_golden.py -> tests/golden/ref_*.npz); the
reference itself ships no golden vectors, so there is no upstream pin beyond that.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .msda import msda_grid_sample

DEFAULT_CFG = dict(
    bev_h=200, bev_w=200, embed_dims=256, num_heads=8, num_layers=4,
    num_points_in_pillar=8, sca_points=8, num_levels=4, tsa_points=4, num_bev_queue=2,
    ffn_dim=512, pillar_h=16, out_dim=32, num_classes=17, num_cams=6,
    pc_range=[-40, -40, -1.0, 40, 40, 5.4],
)


def make_cfg(**kw):
    c = dict(DEFAULT_CFG)
    c.update(kw)
    return c


# ------------------------------------------------------------------ a1  encoder.py:50-89
def get_reference_points(H, W, Z=8, num_points_in_pillar=4, dim='3d', bs=1, dtype=torch.float32, device='cpu'):
    """`device`: the reference builds these on the query's device (encoder.py:64); 'cuda' is used by bench.py's
    gpu_eager_baseline leg only (the restated modules on stock torch kernels)."""
    if dim == '3d':
        zs = torch.linspace(0.5, Z - 0.5, num_points_in_pillar, dtype=dtype, device=device).view(-1, 1, 1) \
            .expand(num_points_in_pillar, H, W) / Z
        xs = torch.linspace(0.5, W - 0.5, W, dtype=dtype, device=device).view(1, 1, W).expand(num_points_in_pillar, H, W) / W
        ys = torch.linspace(0.5, H - 0.5, H, dtype=dtype, device=device).view(1, H, 1).expand(num_points_in_pillar, H, W) / H
        ref_3d = torch.stack((xs, ys, zs), -1)
        ref_3d = ref_3d.permute(0, 3, 1, 2).flatten(2).permute(0, 2, 1)
        return ref_3d[None].repeat(bs, 1, 1, 1)                      # (bs, D, H*W, 3)
    ref_y, ref_x = torch.meshgrid(torch.linspace(0.5, H - 0.5, H, dtype=dtype, device=device),
                                  torch.linspace(0.5, W - 0.5, W, dtype=dtype, device=device), indexing='ij')
    ref_y = ref_y.reshape(-1)[None] / H
    ref_x = ref_x.reshape(-1)[None] / W
    ref_2d = torch.stack((ref_x, ref_y), -1)
    return ref_2d.repeat(bs, 1, 1).unsqueeze(2)                      # (bs, H*W, 1, 2)


# ------------------------------------------------------------------ a2  encoder.py:92-151
def point_sampling(reference_points, pc_range, img_metas):
    ego2lidar = img_metas[0]['ego2lidar']                            # batch item 0 only (:94)
    lidar2img = np.asarray([m['lidar2img'] for m in img_metas])
    lidar2img = reference_points.new_tensor(lidar2img)               # (B, N, 4, 4)
    ego2lidar = reference_points.new_tensor(np.asarray(ego2lidar))
    reference_points = reference_points.clone()
    reference_points[..., 0:1] = reference_points[..., 0:1] * (pc_range[3] - pc_range[0]) + pc_range[0]
    reference_points[..., 1:2] = reference_points[..., 1:2] * (pc_range[4] - pc_range[1]) + pc_range[1]
    reference_points[..., 2:3] = reference_points[..., 2:3] * (pc_range[5] - pc_range[2]) + pc_range[2]
    reference_points = torch.cat((reference_points, torch.ones_like(reference_points[..., :1])), -1)
    reference_points = reference_points.permute(1, 0, 2, 3)          # (D, B, Nq, 4)
    D, B, num_query = reference_points.size()[:3]
    num_cam = lidar2img.size(1)
    reference_points = reference_points.view(D, B, 1, num_query, 4).repeat(1, 1, num_cam, 1, 1).unsqueeze(-1)
    lidar2img = lidar2img.view(1, B, num_cam, 1, 4, 4).repeat(D, 1, 1, num_query, 1, 1)
    ego2lidar = ego2lidar.view(1, 1, 1, 1, 4, 4).repeat(D, 1, num_cam, num_query, 1, 1)
    reference_points_cam = torch.matmul(torch.matmul(lidar2img.to(torch.float32), ego2lidar.to(torch.float32)),
                                        reference_points.to(torch.float32)).squeeze(-1)
    eps = 1e-5
    bev_mask = (reference_points_cam[..., 2:3] > eps)
    reference_points_cam = reference_points_cam[..., 0:2] / torch.maximum(
        reference_points_cam[..., 2:3], torch.ones_like(reference_points_cam[..., 2:3]) * eps)
    reference_points_cam[..., 0] /= img_metas[0]['img_shape'][0][1]  # padded W of batch item 0 (:133)
    reference_points_cam[..., 1] /= img_metas[0]['img_shape'][0][0]  # padded H of batch item 0 (:134)
    bev_mask = (bev_mask & (reference_points_cam[..., 1:2] > 0.0) & (reference_points_cam[..., 1:2] < 1.0)
                & (reference_points_cam[..., 0:1] < 1.0) & (reference_points_cam[..., 0:1] > 0.0))
    bev_mask = torch.nan_to_num(bev_mask)
    reference_points_cam = reference_points_cam.permute(2, 1, 3, 0, 4)   # (cam, B, Nq, D, 2)
    bev_mask = bev_mask.permute(2, 1, 3, 0, 4).squeeze(-1)               # (cam, B, Nq, D)
    return reference_points_cam, bev_mask


def _lin(p, prefix, x):
    return F.linear(x, p[prefix + '.weight'], p[prefix + '.bias'])


# ------------------------------------------------------------------ a5  temporal_self_attention.py:128-272
def temporal_self_attention(p, prefix, cfg, query, value=None, query_pos=None, reference_points=None,
                            spatial_shapes=None, level_start_index=None, msda=msda_grid_sample):
    M = cfg['num_heads']; Q = cfg['num_bev_queue']; P = cfg['tsa_points']; L = 1
    if value is None:
        bs, len_bev, c = query.shape
        value = torch.stack([query, query], 1).reshape(bs * 2, len_bev, c)      # :177-180
    identity = query                                                             # :184-185
    if query_pos is not None:
        query = query + query_pos
    bs, num_query, embed_dims = query.shape
    _, num_value, _ = value.shape
    assert int((spatial_shapes[:, 0] * spatial_shapes[:, 1]).sum()) == num_value
    assert Q == 2
    query = torch.cat([value[:bs], query], -1)                                   # :197 (value[:bs] quirk)
    value = _lin(p, prefix + '.value_proj', value)
    value = value.reshape(bs * Q, num_value, M, -1)
    so = _lin(p, prefix + '.sampling_offsets', query).view(bs, num_query, M, Q, L, P, 2)
    aw = _lin(p, prefix + '.attention_weights', query).view(bs, num_query, M, Q, L * P)
    aw = aw.softmax(-1).view(bs, num_query, M, Q, L, P)
    aw = aw.permute(0, 3, 1, 2, 4, 5).reshape(bs * Q, num_query, M, L, P).contiguous()
    so = so.permute(0, 3, 1, 2, 4, 5, 6).reshape(bs * Q, num_query, M, L, P, 2)
    offset_normalizer = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
    loc = reference_points[:, :, None, :, None, :] + so / offset_normalizer[None, None, None, :, None, :]
    out = msda(value, spatial_shapes, loc, aw)                                   # (bs*Q, Nq, C)
    out = out.permute(1, 2, 0).view(num_query, embed_dims, bs, Q).mean(-1).permute(2, 0, 1)
    out = _lin(p, prefix + '.output_proj', out)
    return out + identity                                                        # dropout = identity (eval)


# ------------------------------------------------------------------ a7  spatial_cross_attention.py:273-400
def msda3d(p, prefix, cfg, query, value, reference_points, spatial_shapes, level_start_index,
           msda=msda_grid_sample):
    M = cfg['num_heads']; L = cfg['num_levels']; P = cfg['sca_points']
    bs, num_query, _ = query.shape
    bs, num_value, _ = value.shape
    assert int((spatial_shapes[:, 0] * spatial_shapes[:, 1]).sum()) == num_value
    value = _lin(p, prefix + '.value_proj', value).view(bs, num_value, M, -1)
    so = _lin(p, prefix + '.sampling_offsets', query).view(bs, num_query, M, L, P, 2)
    aw = _lin(p, prefix + '.attention_weights', query).view(bs, num_query, M, L * P)
    aw = aw.softmax(-1).view(bs, num_query, M, L, P)
    offset_normalizer = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
    bs, num_query, num_Z_anchors, xy = reference_points.shape
    ref = reference_points[:, :, None, None, None, :, :]
    so = so / offset_normalizer[None, None, None, :, None, :]
    so = so.view(bs, num_query, M, L, P // num_Z_anchors, num_Z_anchors, xy)     # :366-367 Z-anchor interleave
    loc = (ref + so).view(bs, num_query, M, L, P, xy)
    return msda(value, spatial_shapes, loc, aw)                                  # no output_proj / residual


# ------------------------------------------------------------------ a6  spatial_cross_attention.py:75-175
def spatial_cross_attention(p, prefix, cfg, query, key, value, reference_points_cam, bev_mask,
                            spatial_shapes, level_start_index, msda=msda_grid_sample):
    num_cams = cfg['num_cams']; C = cfg['embed_dims']
    inp_residual = query
    slots = torch.zeros_like(query)
    bs, num_query, _ = query.size()
    D = reference_points_cam.size(3)
    indexes = []
    for i, mask_per_img in enumerate(bev_mask):
        indexes.append(mask_per_img[0].sum(-1).nonzero().squeeze(-1))            # batch-0 mask for all b (:139)
    max_len = max(len(e) for e in indexes)
    queries_rebatch = query.new_zeros([bs, num_cams, max_len, C])
    ref_rebatch = reference_points_cam.new_zeros([bs, num_cams, max_len, D, 2])
    for j in range(bs):
        for i, ref_per_img in enumerate(reference_points_cam):
            idx = indexes[i]
            queries_rebatch[j, i, :len(idx)] = query[j, idx]
            ref_rebatch[j, i, :len(idx)] = ref_per_img[j, idx]
    num_cams_k, l, bs_k, embed_dims = key.shape
    value = value.permute(2, 0, 1, 3).reshape(bs * num_cams, l, C)
    queries = msda3d(p, prefix + '.deformable_attention', cfg,
                     queries_rebatch.view(bs * num_cams, max_len, C), value,
                     ref_rebatch.view(bs * num_cams, max_len, D, 2), spatial_shapes, level_start_index,
                     msda=msda).view(bs, num_cams, max_len, C)
    for j in range(bs):
        for i, idx in enumerate(indexes):
            slots[j, idx] += queries[j, i, :len(idx)]
    count = bev_mask.sum(-1) > 0
    count = count.permute(1, 2, 0).sum(-1)
    count = torch.clamp(count, min=1.0)
    slots = slots / count[..., None]
    slots = _lin(p, prefix + '.output_proj', slots)
    return slots + inp_residual


def spatial_cross_attention_direct(p, prefix, cfg, query, value, reference_points_cam, bev_mask,
                                   spatial_shapes, level_start_index, msda=msda_grid_sample):
    """Same math without the rebatch (SURVEY a6: `out_q = q + W_o (sum_{c visible} MSDA_c(q) / max(1,#c)) + b_o`).
    Used by tests to show that a no-rebatch fused kernel is semantically exact for B == 1."""
    num_cams = cfg['num_cams']; C = cfg['embed_dims']
    bs, num_query, _ = query.shape
    vis = bev_mask.sum(-1) > 0                                                    # (cam, B, Nq)
    v = value.permute(2, 0, 1, 3).reshape(bs * num_cams, -1, C)
    q_all = query[:, None].expand(bs, num_cams, num_query, C).reshape(bs * num_cams, num_query, C)
    ref = reference_points_cam.permute(1, 0, 2, 3, 4).reshape(bs * num_cams, num_query, -1, 2)
    out = msda3d(p, prefix + '.deformable_attention', cfg, q_all, v, ref, spatial_shapes,
                 level_start_index, msda=msda).view(bs, num_cams, num_query, C)
    visb = vis.permute(1, 0, 2)[..., None].to(out.dtype)                          # (B, cam, Nq, 1)
    slots = (out * visb).sum(1)
    count = torch.clamp(vis.permute(1, 2, 0).sum(-1), min=1.0)
    slots = slots / count[..., None]
    return _lin(p, prefix + '.output_proj', slots) + query


# ------------------------------------------------------------------ a4  encoder.py:287-406, custom_base_transformer_layer.py:72-165
def ffn(p, prefix, x):
    h = F.relu(_lin(p, prefix + '.layers.0.0', x))
    return x + _lin(p, prefix + '.layers.1', h)


def layer_norm(p, prefix, x):
    return F.layer_norm(x, (x.shape[-1],), p[prefix + '.weight'], p[prefix + '.bias'], 1e-5)


def bevformer_layer(p, prefix, cfg, query, key, value, bev_pos, ref_2d, bev_h, bev_w,
                    reference_points_cam, bev_mask, spatial_shapes, level_start_index, prev_bev=None,
                    msda=msda_grid_sample, taps=None):
    # operation_order ('self_attn','norm','cross_attn','norm','ffn','norm')  (bevformer_base_occ.py:127-128)
    q = temporal_self_attention(p, prefix + '.attentions.0', cfg, query, prev_bev, bev_pos, ref_2d,
                                torch.tensor([[bev_h, bev_w]], device=query.device), torch.tensor([0], device=query.device),
                                msda=msda)
    if taps is not None:
        taps['tsa'] = q
    q = layer_norm(p, prefix + '.norms.0', q)
    q = spatial_cross_attention(p, prefix + '.attentions.1', cfg, q, key, value, reference_points_cam,
                                bev_mask, spatial_shapes, level_start_index, msda=msda)
    if taps is not None:
        taps['sca'] = q
    q = layer_norm(p, prefix + '.norms.1', q)
    q = ffn(p, prefix + '.ffns.0', q)
    q = layer_norm(p, prefix + '.norms.2', q)
    return q


# ------------------------------------------------------------------ a3  encoder.py:153-239
def bevformer_encoder(p, prefix, cfg, bev_query, key, value, bev_h, bev_w, bev_pos, spatial_shapes,
                      level_start_index, img_metas, prev_bev=None, msda=msda_grid_sample, taps=None):
    pc = cfg['pc_range']
    bs = bev_query.size(1)
    ref_3d = get_reference_points(bev_h, bev_w, pc[5] - pc[2], cfg['num_points_in_pillar'], '3d', bs,
                                  bev_query.dtype, bev_query.device)
    ref_2d = get_reference_points(bev_h, bev_w, dim='2d', bs=bs, dtype=bev_query.dtype, device=bev_query.device)
    reference_points_cam, bev_mask = point_sampling(ref_3d, pc, img_metas)
    shift_ref_2d = ref_2d.clone()
    bev_query = bev_query.permute(1, 0, 2)
    bev_pos = bev_pos.permute(1, 0, 2)
    bs, len_bev, num_bev_level, _ = ref_2d.shape
    if prev_bev is not None:
        prev_bev = prev_bev.permute(1, 0, 2)
        prev_bev = torch.stack([prev_bev, bev_query], 1).reshape(bs * 2, len_bev, -1)   # once, before the loop
        hybird_ref_2d = torch.stack([shift_ref_2d, ref_2d], 1).reshape(bs * 2, len_bev, num_bev_level, 2)
    else:
        hybird_ref_2d = torch.stack([ref_2d, ref_2d], 1).reshape(bs * 2, len_bev, num_bev_level, 2)
    if taps is not None:
        taps['reference_points_cam'] = reference_points_cam
        taps['bev_mask'] = bev_mask
    for lid in range(cfg['num_layers']):
        lt = {} if taps is not None else None
        bev_query = bevformer_layer(p, f'{prefix}.layers.{lid}', cfg, bev_query, key, value, bev_pos,
                                    hybird_ref_2d, bev_h, bev_w, reference_points_cam, bev_mask,
                                    spatial_shapes, level_start_index, prev_bev=prev_bev, msda=msda, taps=lt)
        if taps is not None:
            taps[f'layer{lid}'] = bev_query
            taps[f'layer{lid}_tsa'] = lt['tsa']
            taps[f'layer{lid}_sca'] = lt['sca']
    return bev_query


# ------------------------------------------------------------------ a9  transformer_occ.py:170-242
def pack_camera_features(p, prefix, cfg, mlvl_feats):
    feat_flatten, spatial_shapes = [], []
    for lvl, feat in enumerate(mlvl_feats):
        bs, num_cam, c, h, w = feat.shape
        spatial_shapes.append((h, w))
        feat = feat.flatten(3).permute(1, 0, 3, 2)                               # (cam, B, hw, C)
        if cfg.get('use_cams_embeds', True):                                     # :214-215
            feat = feat + p[prefix + '.cams_embeds'][:, None, None, :]
        feat = feat + p[prefix + '.level_embeds'][None, None, lvl:lvl + 1, :]
        feat_flatten.append(feat)
    feat_flatten = torch.cat(feat_flatten, 2)
    spatial_shapes = torch.as_tensor(spatial_shapes, dtype=torch.long, device=feat_flatten.device)
    level_start_index = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))
    return feat_flatten.permute(0, 2, 1, 3), spatial_shapes, level_start_index  # (cam, Nv, B, C)


def rotate_prev_bev(prev_bev, bev_h, bev_w, angle_deg, center):
    """transformer_occ.py:195-205 (torchvision `rotate`, nearest, about `rotate_center`)."""
    from torchvision.transforms.functional import rotate
    t = prev_bev.reshape(bev_h, bev_w, -1).permute(2, 0, 1)
    t = rotate(t, angle_deg, center=center)
    return t.permute(1, 2, 0).reshape(bev_h * bev_w, -1)


def get_bev_features(p, prefix, cfg, mlvl_feats, bev_queries, bev_h, bev_w, bev_pos, img_metas,
                     prev_bev=None, msda=msda_grid_sample, taps=None):
    bs = mlvl_feats[0].size(0)
    bev_queries = bev_queries.unsqueeze(1).repeat(1, bs, 1)
    bev_pos = bev_pos.flatten(2).permute(2, 0, 1)
    if prev_bev is not None:
        if prev_bev.shape[1] == bev_h * bev_w:
            prev_bev = prev_bev.permute(1, 0, 2)
        prev_bev = prev_bev.clone()
        for i in range(bs):
            ang = img_metas[i]['can_bus'][-1]
            prev_bev[:, i] = rotate_prev_bev(prev_bev[:, i], bev_h, bev_w, ang, cfg.get('rotate_center', [100, 100]))
    feat_flatten, spatial_shapes, level_start_index = pack_camera_features(p, prefix, cfg, mlvl_feats)
    return bevformer_encoder(p, prefix + '.encoder', cfg, bev_queries, feat_flatten, feat_flatten, bev_h, bev_w,
                             bev_pos, spatial_shapes, level_start_index, img_metas, prev_bev=prev_bev,
                             msda=msda, taps=taps)


# ------------------------------------------------------------------ a10 transformer_occ.py:106-131, 305-308
def voxel_decoder(p, prefix, cfg, bev_embed, bev_h, bev_w):
    """bev_embed (B, Nq, C) -> (B, X, Y, Z, out_dim).  Conv3d(k3,p1,bias=False)+BN3d(eval)+ReLU twice."""
    bs = bev_embed.shape[0]
    x = bev_embed.permute(0, 2, 1).reshape(bs, -1, bev_h, bev_w)
    x = x.view(bs, -1, cfg['pillar_h'], bev_h, bev_w)
    for i in range(2):
        x = F.conv3d(x, p[f'{prefix}.{i}.conv.weight'], None, stride=1, padding=1)
        x = F.batch_norm(x, p[f'{prefix}.{i}.bn.running_mean'], p[f'{prefix}.{i}.bn.running_var'],
                         p[f'{prefix}.{i}.bn.weight'], p[f'{prefix}.{i}.bn.bias'], False, 0.1, 1e-5)
        x = F.relu(x)
    return x.permute(0, 4, 3, 2, 1)


# ------------------------------------------------------------------ a11 transformer_occ.py:132-141, 318-319
def occ_heads(p, prefix, voxel_feats):
    occ = _lin(p, prefix + '.predicter.2', F.softplus(_lin(p, prefix + '.predicter.0', voxel_feats)))
    flow = _lin(p, prefix + '.flow_predicter.2', F.relu(_lin(p, prefix + '.flow_predicter.0', voxel_feats)))
    return occ, flow


# ------------------------------------------------------------------ a12 bevformer_occ_head.py:99-160, 198-216
def positional_encoding(p, prefix, bs, h, w):
    x_embed = p[prefix + '.col_embed.weight'][:w]
    y_embed = p[prefix + '.row_embed.weight'][:h]
    pos = torch.cat((x_embed.unsqueeze(0).repeat(h, 1, 1), y_embed.unsqueeze(1).repeat(1, w, 1)), dim=-1)
    return pos.permute(2, 0, 1).unsqueeze(0).repeat(bs, 1, 1, 1)


def head_forward(p, cfg, mlvl_feats, img_metas, prev_bev=None, only_bev=False, msda=msda_grid_sample,
                 taps=None):
    """`p` is keyed like pts_bbox_head.state_dict().  Returns dict(bev_embed, occ, flow)."""
    bev_h, bev_w = cfg['bev_h'], cfg['bev_w']
    bs = mlvl_feats[0].shape[0]
    bev_queries = p['bev_embedding.weight']
    bev_pos = positional_encoding(p, 'positional_encoding', bs, bev_h, bev_w)
    bev = get_bev_features(p, 'transformer', cfg, mlvl_feats, bev_queries, bev_h, bev_w, bev_pos, img_metas,
                           prev_bev=prev_bev, msda=msda, taps=taps)              # (B, Nq, C)
    if only_bev:
        return bev
    vox = voxel_decoder(p, 'transformer.decoder', cfg, bev, bev_h, bev_w)
    if taps is not None:
        taps['voxel_feats'] = vox
    occ, flow = occ_heads(p, 'transformer', vox)
    bev_embed = bev.permute(0, 2, 1).reshape(bs, -1, bev_h, bev_w)
    return {'bev_embed': bev_embed, 'occ': occ, 'flow': flow}


def get_occ(preds):
    occ_score = preds['occ'].softmax(-1).argmax(-1)
    return occ_score, preds['flow']


# ------------------------------------------------------------------ parameter construction
# Seeded synthetic weights are a fixture shared with the product-side benchmark: see occnet_b200/fixtures.py.
from occnet_b200.fixtures import init_params  # noqa: E402,F401
