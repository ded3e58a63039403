"""Seeded synthetic inputs for the occupancy hot path (SURVEY section 8d).

There is no nuScenes data (and no network) in this environment, so every test and the
benchmark run on these fixtures.  Matrix conventions follow the reference's dataset
class: `lidar2img = viewpad @ lidar2cam_rt.T` (datasets/nuscenes_occ.py:96-113) and
`ego2lidar = inv(pseudo_lidar2ego)` (tools/ray_iou/ego_pose_extractor.py:24-28).
"""
import math

import numpy as np
import torch

PC_RANGE = [-40.0, -40.0, -1.0, 40.0, 40.0, 5.4]

# (yaw deg, focal, translation) for a nuScenes-like 6-camera rig
_RIG = [(0.0, 1266.0, (1.7, 0.0, 1.5)), (-55.0, 1266.0, (1.5, -0.5, 1.5)), (55.0, 1266.0, (1.5, 0.5, 1.5)),
        (180.0, 809.0, (0.0, 0.0, 1.5)), (110.0, 1266.0, (1.0, 0.5, 1.5)), (-110.0, 1266.0, (1.0, -0.5, 1.5))]

# tools/ray_iou/ego_pose_extractor.py:24-28 (constant of the reference; lidar -> ego)
PSEUDO_LIDAR2EGO = np.array([[0.0, 1.0, 0.0, 0.9858], [-1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 1.0, 1.8402],
                             [0.0, 0.0, 0.0, 1.0]])

CFG_FULL = dict(bev_h=200, bev_w=200, embed_dims=256, num_heads=8, num_layers=4, num_points_in_pillar=8,
                sca_points=8, num_levels=4, tsa_points=4, num_bev_queue=2, ffn_dim=512, pillar_h=16,
                out_dim=32, num_classes=17, num_cams=6, pc_range=PC_RANGE,
                img_shape=(928, 1600, 3), level_shapes=[(116, 200), (58, 100), (29, 50), (15, 25)])

CFG_TOY = dict(CFG_FULL, bev_h=50, bev_w=50, num_layers=1, num_cams=1, img_shape=(256, 256, 3),
               level_shapes=[(32, 32), (16, 16), (8, 8), (4, 4)])

CFG_SMALL6 = dict(CFG_FULL, bev_h=40, bev_w=40, num_layers=2, img_shape=(928, 1600, 3),
                  level_shapes=[(29, 50), (15, 25), (8, 13), (4, 7)])


def make_cfg(base='full', **kw):
    c = dict({'full': CFG_FULL, 'toy': CFG_TOY, 'small6': CFG_SMALL6}[base])
    c.update(kw)
    return c


def camera_rig(num_cams=6, img_hw=(928, 1600)):
    """-> (lidar2img (num_cams,4,4) float64, ego2lidar (4,4) float64)."""
    R0 = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])        # cam (z fwd, x right, y down) -> ego
    lidar2ego = PSEUDO_LIDAR2EGO
    ego2lidar = np.linalg.inv(lidar2ego)
    out = []
    sx = img_hw[1] / 1600.0
    sy = img_hw[0] / 928.0
    for yaw, f, t in _RIG[:num_cams]:
        a = math.radians(yaw)
        Rz = np.array([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])
        cam2ego = np.eye(4)
        cam2ego[:3, :3] = Rz @ R0
        cam2ego[:3, 3] = t
        sensor2lidar = ego2lidar @ cam2ego
        s2l_R, s2l_t = sensor2lidar[:3, :3], sensor2lidar[:3, 3]
        lidar2cam_r = np.linalg.inv(s2l_R)
        lidar2cam_t = s2l_t @ lidar2cam_r.T
        rt = np.eye(4)
        rt[:3, :3] = lidar2cam_r.T
        rt[3, :3] = -lidar2cam_t
        K = np.array([[f * sx, 0.0, 816.0 * sx], [0.0, f * sy, 491.0 * sy], [0.0, 0.0, 1.0]], dtype=np.float32)
        viewpad = np.eye(4)
        viewpad[:3, :3] = K
        out.append(viewpad @ rt.T)
    return np.stack(out), ego2lidar


IMG_RIG = (928, 1600)


def _camera(yaw, f, t, img_hw):
    """lidar2img of one camera built like fixtures.camera_rig"""
    R0 = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
    ego2lidar = np.linalg.inv(PSEUDO_LIDAR2EGO)
    a = math.radians(yaw)
    Rz = np.array([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])
    cam2ego = np.eye(4)
    cam2ego[:3, :3] = Rz @ R0
    cam2ego[:3, 3] = t
    s2l = ego2lidar @ cam2ego
    r = np.linalg.inv(s2l[:3, :3])
    rt = np.eye(4)
    rt[:3, :3] = r.T
    rt[3, :3] = -(s2l[:3, 3] @ r.T)
    sx, sy = img_hw[1] / 1600.0, img_hw[0] / 928.0
    K = np.array([[f * sx, 0.0, 816.0 * sx], [0.0, f * sy, 491.0 * sy], [0.0, 0.0, 1.0]], dtype=np.float32)
    vp = np.eye(4)
    vp[:3, :3] = K
    return vp @ rt.T


# two extra cameras of the eight-camera rig: they overlap the front-left / rear-right cameras of the fixture rig
EXTRA_CAMS = [(28.0, 1000.0, (1.6, 0.3, 1.6)), (-150.0, 900.0, (-0.4, -0.4, 1.4))]


def rig_metas(num_cams, img_hw=IMG_RIG, can_bus_angle=None):
    """img_metas of the first num_cams cameras of the fixture rig, extended by EXTRA_CAMS beyond six"""
    l2i, e2l = camera_rig(min(num_cams, 6), img_hw)
    mats = [l2i[i] for i in range(min(num_cams, 6))] + [_camera(*c, img_hw) for c in EXTRA_CAMS[:max(0, num_cams - 6)]]
    m = dict(lidar2img=mats, ego2lidar=e2l, img_shape=[tuple(img_hw) + (3,)] * num_cams)
    if can_bus_angle is not None:
        m['can_bus'] = np.zeros(18)
        m['can_bus'][-1] = can_bus_angle
    return [m]


def make_img_metas(cfg, bs=1, can_bus_angle=None):
    l2i, e2l = camera_rig(cfg['num_cams'], cfg['img_shape'][:2])
    metas = []
    for _ in range(bs):
        m = dict(lidar2img=[l2i[i] for i in range(cfg['num_cams'])], ego2lidar=e2l,
                 img_shape=[tuple(cfg['img_shape'])] * cfg['num_cams'])
        if can_bus_angle is not None:
            cb = np.zeros(18)
            cb[-1] = can_bus_angle
            m['can_bus'] = cb
        metas.append(m)
    return metas


def make_feats(cfg, bs=1, seed=1, device='cpu', dtype=torch.float32):
    """FPN-like multi-level camera features ~ N(0,1): list of (B, num_cams, C, h, w)."""
    g = torch.Generator().manual_seed(seed)
    feats = []
    for (h, w) in cfg['level_shapes']:
        feats.append(torch.randn(bs, cfg['num_cams'], cfg['embed_dims'], h, w, generator=g).to(device=device, dtype=dtype))
    return feats


def make_occ_scene(seed=4, size=(200, 200, 16), num_boxes=40):
    """Synthetic GT semantics (X,Y,Z) uint8 + flow (X,Y,Z,2) fp32 (SURVEY 8d 'metric fixture')."""
    rng = np.random.RandomState(seed)
    X, Y, Z = size
    sem = np.full(size, 16, np.uint8)
    flow = np.zeros(size + (2,), np.float32)
    sem[:, :, 0:2] = 10                                                            # ground slab
    sem[: X // 10, :, 2:10] = 14                                                   # manmade wall
    sem[:, : Y // 12, 2:7] = 15                                                    # vegetation wall
    for _ in range(num_boxes):
        c = rng.randint(0, 10)
        sx, sy, sz = rng.randint(2, 12), rng.randint(2, 12), rng.randint(2, 6)
        x0, y0 = rng.randint(0, X - sx), rng.randint(0, Y - sy)
        sem[x0:x0 + sx, y0:y0 + sy, 2:2 + sz] = c
        if c < 8:
            flow[x0:x0 + sx, y0:y0 + sy, 2:2 + sz] = rng.uniform(-5, 5, 2).astype(np.float32)
    return sem, flow


def make_ray_origins(T=8, z=1.84):
    """(1, T, 3) fp32 ego-frame origins along x in [-20, 20] (all pass ego_pose_extractor's |x|,|y| < 39)."""
    xs = np.linspace(-20.0, 20.0, T)
    o = np.stack([xs, np.zeros(T), np.full(T, z)], -1).astype(np.float32)
    return o[None]


FREE_BIAS = 1.25      # see init_params(free_bias=...)


def init_params(cfg, seed=2, perturb=True, num_embed_levels=None, free_bias=0.0):
    """Reference `init_weights` (spatial_cross_attention.py:253-271, temporal_self_attention.py:107-126,
    transformer_occ.py:154-167) followed by the SURVEY 8d perturbation so that offsets / weights are
    query-dependent (the stock init zeroes `sampling_offsets.weight` and `attention_weights.weight`).
    `free_bias` is added to the bias of the 'free' class (index num_classes-1) of the semantic head: with purely random
    weights only ~1 % of the voxels come out free, every metric ray then stops in its first voxel and Ray-mIoU is
    degenerate; FREE_BIAS = 1.25 makes ~78 % of the full-size fixture's voxels free (rays travel, classes compete)."""
    g = torch.Generator().manual_seed(seed)
    C = cfg['embed_dims']; M = cfg['num_heads']; L = cfg['num_levels']; P = cfg['sca_points']
    Pt = cfg['tsa_points']; Q = cfg['num_bev_queue']; F_ = cfg['ffn_dim']
    p = {}

    def xavier(o, i):
        a = math.sqrt(6.0 / (i + o))
        return (torch.rand(o, i, generator=g) * 2 - 1) * a

    def grid_bias(levels, points):
        thetas = torch.arange(M, dtype=torch.float32) * (2.0 * math.pi / M)
        gi = torch.stack([thetas.cos(), thetas.sin()], -1)
        gi = (gi / gi.abs().max(-1, keepdim=True)[0]).view(M, 1, 1, 2).repeat(1, levels, points, 1)
        for i in range(points):
            gi[:, :, i, :] *= i + 1
        return gi.reshape(-1)

    Nq = cfg['bev_h'] * cfg['bev_w']
    p['bev_embedding.weight'] = torch.randn(Nq, C, generator=g)
    p['positional_encoding.row_embed.weight'] = torch.rand(cfg['bev_h'], C // 2, generator=g)
    p['positional_encoding.col_embed.weight'] = torch.rand(cfg['bev_w'], C // 2, generator=g)
    p['transformer.level_embeds'] = torch.randn(L, C, generator=g)
    p['transformer.cams_embeds'] = torch.randn(cfg['num_cams'], C, generator=g)
    for l in range(cfg['num_layers']):
        pre = f'transformer.encoder.layers.{l}'
        a0 = pre + '.attentions.0'
        p[a0 + '.sampling_offsets.weight'] = torch.randn(Q * M * 1 * Pt * 2, C * Q, generator=g) * (0.02 if perturb else 0)
        p[a0 + '.sampling_offsets.bias'] = grid_bias(1 * Q, Pt)
        p[a0 + '.attention_weights.weight'] = torch.randn(Q * M * 1 * Pt, C * Q, generator=g) * (0.1 if perturb else 0)
        p[a0 + '.attention_weights.bias'] = torch.zeros(Q * M * 1 * Pt)
        p[a0 + '.value_proj.weight'] = xavier(C, C); p[a0 + '.value_proj.bias'] = torch.zeros(C)
        p[a0 + '.output_proj.weight'] = xavier(C, C); p[a0 + '.output_proj.bias'] = torch.zeros(C)
        a1 = pre + '.attentions.1'
        d = a1 + '.deformable_attention'
        p[d + '.sampling_offsets.weight'] = torch.randn(M * L * P * 2, C, generator=g) * (0.02 if perturb else 0)
        p[d + '.sampling_offsets.bias'] = grid_bias(L, P)
        p[d + '.attention_weights.weight'] = torch.randn(M * L * P, C, generator=g) * (0.1 if perturb else 0)
        p[d + '.attention_weights.bias'] = torch.zeros(M * L * P)
        p[d + '.value_proj.weight'] = xavier(C, C); p[d + '.value_proj.bias'] = torch.zeros(C)
        p[a1 + '.output_proj.weight'] = xavier(C, C); p[a1 + '.output_proj.bias'] = torch.zeros(C)
        f = pre + '.ffns.0'
        p[f + '.layers.0.0.weight'] = xavier(F_, C); p[f + '.layers.0.0.bias'] = torch.randn(F_, generator=g) * 0.02
        p[f + '.layers.1.weight'] = xavier(C, F_); p[f + '.layers.1.bias'] = torch.randn(C, generator=g) * 0.02
        for n in range(3):
            p[f'{pre}.norms.{n}.weight'] = 1 + 0.1 * torch.randn(C, generator=g) if perturb else torch.ones(C)
            p[f'{pre}.norms.{n}.bias'] = 0.1 * torch.randn(C, generator=g) if perturb else torch.zeros(C)
    mid = C // cfg['pillar_h']; od = cfg['out_dim']
    for i, cin in enumerate((mid, od)):
        pre = f'transformer.decoder.{i}'
        fan = cin * 27
        p[pre + '.conv.weight'] = torch.randn(od, cin, 3, 3, 3, generator=g) * math.sqrt(2.0 / fan)
        p[pre + '.bn.weight'] = 1 + 0.1 * torch.randn(od, generator=g) if perturb else torch.ones(od)
        p[pre + '.bn.bias'] = 0.1 * torch.randn(od, generator=g) if perturb else torch.zeros(od)
        p[pre + '.bn.running_mean'] = 0.1 * torch.randn(od, generator=g) if perturb else torch.zeros(od)
        p[pre + '.bn.running_var'] = 0.5 + torch.rand(od, generator=g) if perturb else torch.ones(od)
        p[pre + '.bn.num_batches_tracked'] = torch.zeros((), dtype=torch.long)
    for name, out in (('predicter', cfg['num_classes']), ('flow_predicter', 2)):
        p[f'transformer.{name}.0.weight'] = xavier(od * 2, od)
        p[f'transformer.{name}.0.bias'] = torch.randn(od * 2, generator=g) * 0.05
        p[f'transformer.{name}.2.weight'] = xavier(out, od * 2)
        p[f'transformer.{name}.2.bias'] = torch.randn(out, generator=g) * 0.05
    if free_bias:
        p['transformer.predicter.2.bias'][cfg['num_classes'] - 1] += free_bias
    return p


# ---- image backbone + neck (ResNet-50 + FPN, reference config bevformer_base_occ.py:48-66): synthetic parameters
_RESNET50_BLOCKS, _RESNET50_PLANES = (3, 4, 6, 3), (64, 128, 256, 512)


def init_backbone_params(seed=5, out_channels=256, bn_stats=True):
    """Random parameters with the reference's `state_dict` key names (img_backbone.* / img_neck.*): Kaiming-normal
    convolutions (mmdet `ResNet.init_weights`), BatchNorm gamma=1 / beta=0 perturbed, running statistics perturbed so
    that a BN-folding bug cannot hide; FPN convs Xavier-uniform with perturbed biases."""
    g = torch.Generator().manual_seed(seed)
    p = {}

    def conv(name, co, ci, k):
        fan_out = co * k * k
        p[name + '.weight'] = torch.randn(co, ci, k, k, generator=g) * (2.0 / fan_out) ** 0.5

    def bn(name, c):
        p[name + '.weight'] = 1.0 + 0.1 * torch.randn(c, generator=g)
        p[name + '.bias'] = 0.1 * torch.randn(c, generator=g)
        p[name + '.running_mean'] = (0.1 * torch.randn(c, generator=g)) if bn_stats else torch.zeros(c)
        p[name + '.running_var'] = (0.5 + torch.rand(c, generator=g)) if bn_stats else torch.ones(c)

    b = 'img_backbone.'
    conv(b + 'conv1', 64, 3, 7); bn(b + 'bn1', 64)
    inplanes = 64
    for s, (nblk, planes) in enumerate(zip(_RESNET50_BLOCKS, _RESNET50_PLANES)):
        for i in range(nblk):
            pre = f'{b}layer{s + 1}.{i}.'
            conv(pre + 'conv1', planes, inplanes, 1); bn(pre + 'bn1', planes)
            conv(pre + 'conv2', planes, planes, 3); bn(pre + 'bn2', planes)
            conv(pre + 'conv3', planes * 4, planes, 1); bn(pre + 'bn3', planes * 4)
            if i == 0:
                conv(pre + 'downsample.0', planes * 4, inplanes, 1); bn(pre + 'downsample.1', planes * 4)
            inplanes = planes * 4
    nk = 'img_neck.'
    for i, ci in enumerate((512, 1024, 2048)):
        w = torch.empty(out_channels, ci, 1, 1)
        bound = (6.0 / (ci + out_channels)) ** 0.5
        p[f'{nk}lateral_convs.{i}.conv.weight'] = (torch.rand(w.shape, generator=g) * 2 - 1) * bound
        p[f'{nk}lateral_convs.{i}.conv.bias'] = 0.05 * torch.randn(out_channels, generator=g)
    for i in range(4):
        bound = (6.0 / (out_channels * 9 * 2)) ** 0.5
        p[f'{nk}fpn_convs.{i}.conv.weight'] = (torch.rand(out_channels, out_channels, 3, 3, generator=g) * 2 - 1) * bound
        p[f'{nk}fpn_convs.{i}.conv.bias'] = 0.05 * torch.randn(out_channels, generator=g)
    return p


def head_cfg(cfg):
    """mmcv-style config dict of `BEVFormerOccHead` (same keys as bevformer_base_occ.py:67-135) for a fixture geometry."""
    C = cfg['embed_dims']
    return dict(
        type='BEVFormerOccHead', pc_range=cfg['pc_range'], bev_h=cfg['bev_h'], bev_w=cfg['bev_w'],
        num_classes=cfg['num_classes'], in_channels=C, sync_cls_avg_factor=True, with_box_refine=True, as_two_stage=False,
        use_mask=False, loss_occ=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
        loss_flow=dict(type='L1Loss', loss_weight=0.25),
        transformer=dict(
            type='TransformerOcc', pillar_h=cfg['pillar_h'], num_classes=cfg['num_classes'], norm_cfg=dict(type='BN'),
            norm_cfg_3d=dict(type='BN3d'), use_3d=True, use_conv=False, rotate_prev_bev=True, use_shift=True,
            use_can_bus=True, embed_dims=C, num_cams=cfg['num_cams'], rotate_center=cfg.get('rotate_center', [100, 100]),
            encoder=dict(
                type='BEVFormerEncoder', num_layers=cfg['num_layers'], pc_range=cfg['pc_range'],
                num_points_in_pillar=cfg['num_points_in_pillar'], return_intermediate=False,
                transformerlayers=dict(
                    type='BEVFormerLayer',
                    attn_cfgs=[dict(type='TemporalSelfAttention', embed_dims=C, num_levels=1),
                               dict(type='SpatialCrossAttention', pc_range=cfg['pc_range'], num_cams=cfg['num_cams'],
                                    deformable_attention=dict(type='MSDeformableAttention3D', embed_dims=C,
                                                              num_points=cfg['sca_points'], num_levels=cfg['num_levels']),
                                    embed_dims=C)],
                    feedforward_channels=cfg['ffn_dim'], ffn_dropout=0.1,
                    operation_order=('self_attn', 'norm', 'cross_attn', 'norm', 'ffn', 'norm')))),
        positional_encoding=dict(type='LearnedPositionalEncoding', num_feats=C // 2, row_num_embed=cfg['bev_h'],
                                 col_num_embed=cfg['bev_w']))
