"""CPU suite (-m "not gpu"): the oracle against the committed goldens (generated from the unmodified
reference modules by tests/golden/gen_golden.py), independent cross-checks, host logic, and the C ABI surface."""
import os
import re

import numpy as np
import pytest
import torch

from occnet_b200 import fixtures
from oracle import bevformer_occ as O
from oracle import msda as OM
from oracle import ray_metrics as ORM

CASES = {
    'toy': (fixtures.make_cfg('toy'), 1, False, None),
    'small6': (fixtures.make_cfg('small6'), 1, False, None),
    'small6_b2': (fixtures.make_cfg('small6', num_layers=1), 2, False, None),
    'small6_prev': (fixtures.make_cfg('small6', rotate_center=[20, 20]), 1, True, 3.0),
}


def run_oracle_case(name):
    cfg, bs, with_prev, ang = CASES[name]
    params = O.init_params(cfg, seed=2)
    feats = fixtures.make_feats(cfg, bs=bs, seed=1)
    metas = fixtures.make_img_metas(cfg, bs=bs, can_bus_angle=ang)
    prev = None
    if with_prev:
        g = torch.Generator().manual_seed(3)
        prev = torch.randn(bs, cfg['bev_h'] * cfg['bev_w'], cfg['embed_dims'], generator=g)
    with torch.no_grad():
        out = O.head_forward(params, cfg, feats, metas, prev_bev=prev)
    return cfg, out


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_matches_reference_golden(name, golden_dir):
    """Oracle == unmodified reference modules (goldens), incl. batch-2 quirks and the temporal path."""
    g = np.load(os.path.join(golden_dir, f'ref_model_{name}.npz'))
    _, out = run_oracle_case(name)
    for k in ('bev_embed', 'occ', 'flow'):
        assert tuple(out[k].shape) == tuple(g[k + '_shape'])
        sub = out[k].reshape(-1)[torch.from_numpy(g[k + '_idx'])].numpy()
        np.testing.assert_allclose(sub, g[k + '_sub'], rtol=0, atol=2e-5)
        assert abs(out[k].abs().double().mean().item() - float(g[k + '_absmean'])) < 1e-5
    cls = out['occ'].softmax(-1).argmax(-1).numpy().astype(np.uint8)
    assert (cls == g['occ_cls']).mean() > 0.9999


def test_msda_three_way():
    """grid_sample restatement == scalar CUDA-kernel formulation == transformers' independent implementation."""
    torch.manual_seed(0)
    B, M, C, L, P, Nq = 2, 4, 8, 3, 4, 37
    shapes = torch.tensor([[7, 9], [4, 5], [2, 3]])
    lsi = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
    Nv = int(shapes.prod(1).sum())
    value = torch.randn(B, Nv, M, C)
    loc = torch.rand(B, Nq, M, L, P, 2) * 1.4 - 0.2          # some samples fall outside the maps
    w = torch.rand(B, Nq, M, L, P)
    a = OM.msda_grid_sample(value, shapes, loc, w)
    b = OM.msda_loops(value, shapes, lsi, loc, w)
    np.testing.assert_allclose(a.numpy(), b.numpy(), atol=2e-5, rtol=0)
    from transformers.models.mask2former.modeling_mask2former import multi_scale_deformable_attention
    c = multi_scale_deformable_attention(value, [(int(h), int(wd)) for h, wd in shapes], loc, w)
    np.testing.assert_allclose(a.numpy(), c.numpy(), atol=2e-5, rtol=0)


def test_sca_rebatch_equals_direct_formula():
    """SURVEY a6: the reference's rebatch is a memory optimisation; the fused per-(query,camera) sum is exact (B=1)."""
    cfg = fixtures.make_cfg('small6')
    p = O.init_params(cfg, seed=2)
    feats = fixtures.make_feats(cfg, bs=1, seed=1)
    metas = fixtures.make_img_metas(cfg, bs=1)
    pc = cfg['pc_range']
    Nq = cfg['bev_h'] * cfg['bev_w']
    ref_3d = O.get_reference_points(cfg['bev_h'], cfg['bev_w'], pc[5] - pc[2], cfg['num_points_in_pillar'], '3d', 1)
    rpc, mask = O.point_sampling(ref_3d, pc, metas)
    value, shapes, lsi = O.pack_camera_features(p, 'transformer', cfg, feats)
    q = torch.randn(1, Nq, 256, generator=torch.Generator().manual_seed(7))
    pre = 'transformer.encoder.layers.0.attentions.1'
    with torch.no_grad():
        a = O.spatial_cross_attention(p, pre, cfg, q, value, value, rpc, mask, shapes, lsi)
        b = O.spatial_cross_attention_direct(p, pre, cfg, q, value, rpc, mask, shapes, lsi)
    assert mask.any() and (mask.sum(-1) > 0).sum() > 100
    np.testing.assert_allclose(a.numpy(), b.numpy(), atol=1e-5, rtol=0)


def test_reference_points_closed_form():
    r3 = O.get_reference_points(4, 5, 6.4, 8, '3d', 1)
    assert r3.shape == (1, 8, 20, 3)
    np.testing.assert_allclose(r3[0, 0, :5, 0].numpy(), (np.arange(5) + 0.5) / 5, atol=1e-7)
    np.testing.assert_allclose(r3[0, :, 0, 2].numpy(), np.linspace(0.5, 5.9, 8) / 6.4, atol=1e-6)
    r2 = O.get_reference_points(4, 5, dim='2d', bs=1)
    assert r2.shape == (1, 20, 1, 2)
    np.testing.assert_allclose(r2[0, 7, 0].numpy(), [(7 % 5 + 0.5) / 5, (7 // 5 + 0.5) / 4], atol=1e-7)


def test_rig_statistics_full_size():
    """SURVEY 8d fixture numbers: visible queries per camera at 200x200, D=8, img (928,1600)."""
    cfg = fixtures.make_cfg('full')
    metas = fixtures.make_img_metas(cfg)
    pc = cfg['pc_range']
    ref_3d = O.get_reference_points(200, 200, pc[5] - pc[2], 8, '3d', 1)
    _, mask = O.point_sampling(ref_3d, pc, metas)
    per_cam = (mask[:, 0].sum(-1) > 0).sum(-1).tolist()
    assert per_cam == [5790, 7339, 7334, 9893, 7148, 7090]


def test_metric_oracle_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'ref_metric.npz'))
    rays = ORM.generate_lidar_rays()
    assert rays.shape == (14040, 3)
    np.testing.assert_array_equal(rays[:4], g['rays_first'])
    np.testing.assert_array_equal(rays[-4:], g['rays_last'])
    sem_gt, flow_gt = fixtures.make_occ_scene(seed=4)
    rng = np.random.RandomState(5)
    sem_pred = np.roll(sem_gt, 1, axis=0).copy()
    flip = rng.rand(*sem_pred.shape) < 0.03
    sem_pred[flip] = rng.randint(0, 17, int(flip.sum())).astype(np.uint8)
    flow_pred = (np.roll(flow_gt, 1, axis=0) + rng.normal(0, 0.5, flow_gt.shape)).astype(np.float32)
    orig = fixtures.make_ray_origins(T=2)
    pp = ORM.process_one_sample(sem_pred, rays, orig, flow_pred)
    pg = ORM.process_one_sample(sem_gt, rays, orig, flow_gt)
    np.testing.assert_array_equal(pp, g['pcd_pred'])
    np.testing.assert_array_equal(pg[:, 0].astype(np.uint8), g['pcd_gt_cls'])
    np.testing.assert_array_equal(pg[:, 1], g['pcd_gt_dist'])
    valid = pg[:, 0].astype(np.int32) != 16
    cnt = ORM.accumulate(ORM.new_counters(), pp[valid], pg[valid])
    np.testing.assert_allclose(ORM.counters_to_vector(cnt), g['counters'], rtol=1e-12)
    fin = ORM.finalize(cnt)
    np.testing.assert_allclose(fin['iou'], g['iou'], equal_nan=True)
    np.testing.assert_allclose(fin['ave'], g['ave'], equal_nan=True)
    # empty / degenerate: no origins -> no rays -> empty result; a ray bundle that never enters the grid
    far = np.array([[[500.0, 500.0, 50.0]]], np.float32)
    out = ORM.process_one_sample(sem_gt, rays[:16], far, flow_gt)
    assert out.shape == (16, 4) and np.allclose(out[:, 1], -0.4) and (out[:, 0] == sem_gt[0, 0, 0]).all()


def test_host_metric_finalize_matches_oracle(golden_dir):
    from occnet_b200 import metric
    g = np.load(os.path.join(golden_dir, 'ref_metric.npz'))
    fin = metric.finalize_counters(g['counters'])
    np.testing.assert_allclose(fin['iou'], g['iou'], equal_nan=True)
    np.testing.assert_allclose(fin['ave'], g['ave'], equal_nan=True)
    np.testing.assert_array_equal(metric.generate_lidar_rays(), ORM.generate_lidar_rays())


def test_c_abi_exports_every_declared_symbol(lib_built):
    import ctypes
    from occnet_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'occ_b200.h')).read()
    declared = set(re.findall(r'\b(occb200_\w+)\s*\(', hdr))
    assert len(declared) >= 18
    lib = ctypes.CDLL(lib_built)
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in include/occ_b200.h but not exported'
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert b'sm_90a' in _lib.load().occb200_version()


def test_product_path_fails_loudly_without_gpu():
    from occnet_b200 import ops
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    with pytest.raises(RuntimeError):
        ops.ms_deform_attn_forward(torch.zeros(1, 4, 1, 8), torch.tensor([[2, 2]]), torch.tensor([0]),
                                   torch.zeros(1, 1, 1, 1, 1, 2), torch.zeros(1, 1, 1, 1, 1))
    from occnet_b200.engine import OccEngine
    with pytest.raises(RuntimeError):
        OccEngine(fixtures.make_cfg('toy'), {}, 'fp32')


def test_no_oracle_import_in_product():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for d, _, files in os.walk(os.path.join(root, 'occnet_b200')):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh')):
                src = open(os.path.join(d, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', src, re.M), f'{f} imports the oracle'


# ---- image backbone + neck (SURVEY 8f rank 1): oracle pinned against torchvision's independent implementations
def test_backbone_resnet50_matches_torchvision():
    from torchvision.models import resnet50
    from oracle import backbone as OB
    p = OB.init_params(seed=5)
    m = resnet50(weights=None).eval()
    sd = {k[len('img_backbone.'):]: v for k, v in p.items() if k.startswith('img_backbone.')}
    missing = m.load_state_dict(sd, strict=False)
    assert not missing.unexpected_keys
    assert all(k.startswith('fc.') or k.endswith('num_batches_tracked') for k in missing.missing_keys), missing.missing_keys
    got = {}
    for name in ('layer2', 'layer3', 'layer4'):
        getattr(m, name).register_forward_hook(lambda mod, i, o, n=name: got.__setitem__(n, o))
    img = torch.randn(2, 3, 72, 104, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        m(img)
        outs = OB.resnet50(p, img)
    assert [tuple(o.shape) for o in outs] == [(2, 512, 9, 13), (2, 1024, 5, 7), (2, 2048, 3, 4)]
    for o, name in zip(outs, ('layer2', 'layer3', 'layer4')):
        assert torch.equal(o, got[name]), (name, (o - got[name]).abs().max())


def test_backbone_fpn_matches_torchvision():
    from collections import OrderedDict
    from torchvision.ops import FeaturePyramidNetwork
    from torchvision.ops.feature_pyramid_network import LastLevelP6P7
    from oracle import backbone as OB
    p = OB.init_params(seed=6)
    m = FeaturePyramidNetwork([512, 1024, 2048], 256, extra_blocks=LastLevelP6P7(256, 256)).eval()
    sd = m.state_dict()
    for i in range(3):
        sd[f'inner_blocks.{i}.0.weight'] = p[f'img_neck.lateral_convs.{i}.conv.weight']
        sd[f'inner_blocks.{i}.0.bias'] = p[f'img_neck.lateral_convs.{i}.conv.bias']
        sd[f'layer_blocks.{i}.0.weight'] = p[f'img_neck.fpn_convs.{i}.conv.weight']
        sd[f'layer_blocks.{i}.0.bias'] = p[f'img_neck.fpn_convs.{i}.conv.bias']
    sd['extra_blocks.p6.weight'] = p['img_neck.fpn_convs.3.conv.weight']
    sd['extra_blocks.p6.bias'] = p['img_neck.fpn_convs.3.conv.bias']
    m.load_state_dict(sd)
    g = torch.Generator().manual_seed(1)
    feats = [torch.randn(2, 512, 29, 50, generator=g), torch.randn(2, 1024, 15, 25, generator=g),
             torch.randn(2, 2048, 8, 13, generator=g)]                       # odd sizes: top-down resize is by SIZE
    with torch.no_grad():
        ref = m(OrderedDict((str(i), f) for i, f in enumerate(feats)))
        outs = OB.fpn(p, feats)
    assert [tuple(o.shape[2:]) for o in outs] == [(29, 50), (15, 25), (8, 13), (4, 7)]
    for o, k in zip(outs, ('0', '1', '2', 'p6')):
        assert torch.equal(o, ref[k]), (k, (o - ref[k]).abs().max())


def test_backbone_extract_img_feat_shapes():
    from oracle import backbone as OB
    p = OB.init_params(seed=5)
    img = torch.randn(1, 2, 3, 64, 96, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        feats = OB.extract_img_feat(p, img)
    assert [tuple(f.shape) for f in feats] == [(1, 2, 256, 8, 12), (1, 2, 256, 4, 6), (1, 2, 256, 2, 3), (1, 2, 256, 1, 2)]
    # the shipped configuration's level shapes (928 x 1600 padded input): strides 8 / 16 / 32 / 64
    h, w = 928, 1600
    shapes = []
    for s in (8, 16, 32):
        shapes.append((-(-h // s), -(-w // s)))
    shapes.append((-(-shapes[-1][0] // 2), -(-shapes[-1][1] // 2)))
    assert shapes == [tuple(s) for s in fixtures.CFG_FULL['level_shapes']]


def test_backbone_engine_schedule_emulated_on_cpu():
    """The backbone engine (csrc/backbone.cu) could not be run on a GPU in round 1.  This test re-states its SCHEDULE in
    numpy -- NHWC activations, BN folded into tap-major weights [co][(ky*KW+kx)*Cin + c] zero-padded to 64, explicit
    im2col with the same index arithmetic, GEMM, add+ReLU, nearest-by-size top-down add, extra stride-2 level on the last
    output -- and checks it against the oracle, so that layout / ordering mistakes cannot hide behind CUDA syntax."""
    from oracle import backbone as OB
    p = {k: v.numpy() for k, v in OB.init_params(seed=7).items()}
    pt = {k: torch.from_numpy(v) for k, v in p.items()}

    def fold(conv, bn, k, conv_bias=False):
        w = p[conv + '.weight']; co, ci = w.shape[:2]
        scale, shift = np.ones(co, np.float32), np.zeros(co, np.float32)
        if bn:
            scale = p[bn + '.weight'] / np.sqrt(p[bn + '.running_var'] + np.float32(1e-5))
            shift = p[bn + '.bias'] - p[bn + '.running_mean'] * scale
        if conv_bias:
            shift = shift + p[conv + '.bias'] * scale
        kpad = (k * k * ci + 63) // 64 * 64
        W = np.zeros((co, kpad), np.float32)
        W[:, :k * k * ci] = (w.transpose(0, 2, 3, 1) * scale[:, None, None, None]).reshape(co, -1)   # (ky, kx, ci) order
        return W, shift.astype(np.float32), kpad

    def im2col(x, k, stride, pad, kpad):                       # x [N,H,W,C] -> [N*Ho*Wo, kpad]
        N, H, W, C = x.shape
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        out = np.zeros((N, Ho, Wo, kpad), np.float32)
        for kk in range(kpad):
            tap, c = divmod(kk, C)
            if tap >= k * k:
                continue
            ky, kx = divmod(tap, k)
            ys, xs = np.arange(Ho) * stride + ky - pad, np.arange(Wo) * stride + kx - pad
            vy, vx = (ys >= 0) & (ys < H), (xs >= 0) & (xs < W)
            out[:, vy[:, None] & vx[None, :], kk] = x[:, ys[vy]][:, :, xs[vx]][..., c].reshape(N, -1)
        return out.reshape(-1, kpad), Ho, Wo

    def conv(x, conv_key, bn_key, k, stride, pad, relu, conv_bias=False):
        W, b, kpad = fold(conv_key, bn_key, k, conv_bias)
        N, H, Wd, C = x.shape
        if k == 1 and stride == 1 and kpad == C:
            A, Ho, Wo = x.reshape(-1, C), H, Wd
        else:
            A, Ho, Wo = im2col(x, k, stride, pad, kpad)
        y = A @ W.T + b
        return (np.maximum(y, 0) if relu else y).reshape(N, Ho, Wo, -1)

    img = torch.randn(1, 3, 72, 104, generator=torch.Generator().manual_seed(4))
    x = img.numpy().transpose(0, 2, 3, 1)                                            # nchw_to_nhwc_small
    x = conv(x, 'img_backbone.conv1', 'img_backbone.bn1', 7, 2, 3, True)
    x = torch.nn.functional.max_pool2d(torch.from_numpy(x).permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).numpy()
    stage_out = []
    for s, nblk in enumerate((3, 4, 6, 3)):
        for i in range(nblk):
            pre = f'img_backbone.layer{s + 1}.{i}.'
            stride = 2 if (i == 0 and s > 0) else 1
            t = conv(x, pre + 'conv1', pre + 'bn1', 1, 1, 0, True)
            t = conv(t, pre + 'conv2', pre + 'bn2', 3, stride, 1, True)
            t = conv(t, pre + 'conv3', pre + 'bn3', 1, 1, 0, False)
            idn = conv(x, pre + 'downsample.0', pre + 'downsample.1', 1, stride, 0, False) if i == 0 else x
            x = np.maximum(t + idn, 0)
        if s >= 1:
            stage_out.append(x)
    lat = [conv(c, f'img_neck.lateral_convs.{i}.conv', None, 1, 1, 0, False, True) for i, c in enumerate(stage_out)]
    for i in (2, 1):
        Hf, Wf, Hc, Wc = lat[i - 1].shape[1], lat[i - 1].shape[2], lat[i].shape[1], lat[i].shape[2]
        sy = np.minimum(np.floor(np.arange(Hf, dtype=np.float32) * (np.float32(Hc) / np.float32(Hf))).astype(int), Hc - 1)
        sx = np.minimum(np.floor(np.arange(Wf, dtype=np.float32) * (np.float32(Wc) / np.float32(Wf))).astype(int), Wc - 1)
        lat[i - 1] = lat[i - 1] + lat[i][:, sy][:, :, sx]
    outs = [conv(l, f'img_neck.fpn_convs.{i}.conv', None, 3, 1, 1, False, True) for i, l in enumerate(lat)]
    outs.append(conv(outs[2], 'img_neck.fpn_convs.3.conv', None, 3, 2, 1, False, True))
    with torch.no_grad():
        want = OB.fpn(pt, OB.resnet50(pt, img))
    for o, w in zip(outs, want):
        got = torch.from_numpy(o).permute(0, 3, 1, 2)                                # nhwc_to_nchw_f32
        assert got.shape == w.shape
        assert (got - w).abs().max().item() < 2e-3 * max(1.0, w.abs().max().item()), (got - w).abs().max()


@pytest.mark.parametrize('X,Y,grid', [(200, 200, 148), (50, 50, 148), (40, 40, 148), (7, 9, 3), (5, 8, 1), (33, 17, 20)])
def test_conv3d_plane_major_schedule_covers_every_tap_once(X, Y, grid):
    """Python mirror of the MMA loop of csrc/conv3d_tc.cu (plane-major, one N = 96 MMA per tap pair into a sliding window of
    three accumulators: columns [0,32) / [32,64) / [64,96) hold outputs p-1 / p / p+1): every output tile must receive each
    of its 27 taps exactly once, with the weight sub-tile of that tap, before its epilogue, in the CTA's tile order, for any
    volume size and grid."""
    TILE_Y = 8
    y_tiles = (Y + TILE_Y - 1) // TILE_Y
    total = X * y_tiles
    grid = min(grid, total)
    for cta in range(grid):
        t_begin, t_end = total * cta // grid, total * (cta + 1) // grid
        acc = {}                                                # output n -> list of (plane, t9, resident weight tile)
        written = []                                            # epilogue order
        n_base, t = 0, t_begin
        while t < t_end:
            xa = t % X
            xb = min(X, xa + (t_end - t))
            for p in range(xa - 1, xb + 1):
                if 0 <= p < X:                                  # planes outside the volume are the zero padding
                    for t9 in range(9):
                        for j in range(3):                      # window column block j: output p - 1 + j, weight sub-tile j
                            x = p - 1 + j
                            if xa <= x < xb:
                                n = n_base + (x - xa)
                                assert n not in written, 'tap after the epilogue'
                                acc.setdefault(n, []).append((p, t9, t9 * 3 + j))
                if p - 1 >= xa:                                 # output p - 1 is complete: epilogue, window slides
                    written.append(n_base + (p - 1 - xa))
            n_base += xb - xa
            t += xb - xa
        assert written == list(range(t_end - t_begin)) and set(acc) == set(written)
        for i, tt in enumerate(range(t_begin, t_end)):          # epilogue order: n-th tile of the CTA = tile t_begin + n
            x = tt % X
            want = sorted((x + dx - 1, t9, t9 * 3 + (2 - dx)) for dx in range(3) for t9 in range(9) if 0 <= x + dx - 1 < X)
            assert sorted(acc[i]) == want, (cta, tt)


@pytest.mark.parametrize('M,n_tiles,sms', [(40000, 1, 148), (40000, 3, 148), (184950, 6, 148), (130, 1, 148), (31, 1, 148),
                                           (2227200, 8, 148), (4097, 2, 7)])
def test_gemm_row_ranges_cover_every_row_once(M, n_tiles, sms):
    """Python mirror of gemm_tc.cu's CTA -> (n block, row range) mapping: ranges are dealt in 32-row blocks, every row of
    every n-block is owned by exactly one CTA, every CTA owns at least one block, and the spread is at most one block."""
    m_tiles = (M + 127) // 128
    per_n = max(1, min(sms // n_tiles, m_tiles))
    grid = per_n * n_tiles
    nb32 = (M + 31) >> 5
    owned = {n: [] for n in range(n_tiles)}
    for cta in range(grid):
        n_blk, grp, ngrp = cta % n_tiles, cta // n_tiles, grid // n_tiles
        row_begin = ((nb32 * grp) // ngrp) << 5
        row_end = min(M, ((nb32 * (grp + 1)) // ngrp) << 5)
        assert row_begin < row_end and row_begin % 32 == 0
        owned[n_blk].append((row_begin, row_end))
    for n, rs in owned.items():
        rs.sort()
        assert rs[0][0] == 0 and rs[-1][1] == M
        assert all(a[1] == b[0] for a, b in zip(rs, rs[1:]))
        blocks = [(e - b + 31) // 32 for b, e in rs]
        assert max(blocks) - min(blocks) <= 1


def test_clamped_2x2_fetch_block_equals_zero_padded_bilinear():
    """Python mirror of msda.cu `prep_sample`: the gather kernels always fetch the 2x2 pixel block whose top-left corner is
    clamped to [0,H-2]x[0,W-2] and re-assign the bilinear corner weights to the positions of that block that coincide with
    in-bounds true corners.  Must equal zero-padded bilinear sampling (mmcv ms_deform_attn_im2col_bilinear) everywhere,
    including the one-pixel border band and fully outside positions."""
    rng = np.random.default_rng(0)
    for H, W in ((2, 2), (3, 5), (15, 25), (116, 200)):
        img = rng.standard_normal((H, W)).astype(np.float64)
        pts = np.concatenate([rng.uniform(-2.5, max(H, W) + 1.5, size=(4000, 2)),
                              np.array([[-1.0, -1.0], [-0.999, 0.3], [H - 1, W - 1], [H - 0.001, W - 0.001], [H, 0], [0, W],
                                        [-0.5, -0.5], [H - 0.5, W - 0.5], [0.0, 0.0], [H - 1.0, 0.0]])])
        for h_im, w_im in pts:
            valid = h_im > -1 and w_im > -1 and h_im < H and w_im < W
            # reference: zero padding outside, corners (h_lo, w_lo) .. (h_lo+1, w_lo+1)
            want = 0.0
            if valid:
                h_lo, w_lo = int(np.floor(h_im)), int(np.floor(w_im))
                lh, lw = h_im - h_lo, w_im - w_lo
                for dy, dx, wt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
                    y, x = h_lo + dy, w_lo + dx
                    if 0 <= y < H and 0 <= x < W:
                        want += wt * img[y, x]
            # kernel: clamped block + re-assigned weights
            hf, wf = (np.floor(h_im), np.floor(w_im)) if valid else (0.0, 0.0)
            h_lo, w_lo = int(hf), int(wf)
            lh, lw = h_im - hf, w_im - wf
            hh, hw = 1 - lh, 1 - lw
            hb, wb = min(max(h_lo, 0), H - 2), min(max(w_lo, 0), W - 2)
            rw0 = hh if h_lo == hb else (lh if h_lo + 1 == hb else 0.0)
            rw1 = hh if h_lo == hb + 1 else (lh if h_lo == hb else 0.0)
            cw0 = hw if w_lo == wb else (lw if w_lo + 1 == wb else 0.0)
            cw1 = hw if w_lo == wb + 1 else (lw if w_lo == wb else 0.0)
            g = 1.0 if valid else 0.0
            got = g * (rw0 * cw0 * img[hb, wb] + rw0 * cw1 * img[hb, wb + 1] + rw1 * cw0 * img[hb + 1, wb] + rw1 * cw1 * img[hb + 1, wb + 1])
            assert abs(got - want) < 1e-12, (H, W, h_im, w_im, got, want)


# ------------------------------------------------------------------------------------------ storage-rounding model
@pytest.mark.parametrize('base,prev', [('toy', False), ('small6', False), ('small6', True)])
def test_bf16_model_without_rounding_equals_fp32_oracle(base, prev):
    """oracle/bf16_model.py is the oracle's algorithm in the engine's formulation (direct masked SCA, index gather, folded
    BN): with every rounding switched off it must reproduce the reference-pinned fp32 oracle to round-off; with the
    roundings on it must sit at bf16 distance from it (this is the distance the bf16 engine is allowed)."""
    from oracle import bf16_model as B
    cfg = fixtures.make_cfg(base, rotate_center=[20, 20]) if prev else fixtures.make_cfg(base)
    params = O.init_params(cfg, seed=2)
    feats = fixtures.make_feats(cfg, bs=1, seed=1)
    metas = fixtures.make_img_metas(cfg, bs=1, can_bus_angle=3.0 if prev else None)
    pb = torch.randn(1, cfg['bev_h'] * cfg['bev_w'], 256, generator=torch.Generator().manual_seed(3)) if prev else None
    with torch.no_grad():
        want = O.head_forward(params, cfg, feats, metas, prev_bev=None if pb is None else pb.clone())
    exact = B.head_forward(params, cfg, feats, metas, prev_bev=pb, quant=False)
    rounded = B.head_forward(params, cfg, feats, metas, prev_bev=pb, quant=True)
    for k in ('bev_embed', 'occ', 'flow'):
        assert (exact[k] - want[k]).abs().max().item() < 2e-4, k
        d = (rounded[k] - want[k]).abs()
        assert 1e-3 < d.max().item() < 6e-2 and d.mean().item() < 6e-3, k


def test_full_size_goldens_are_committed_and_consistent(golden_dir):
    """tests/golden/gen_fullsize.py outputs (full size, 6 layers; regenerating takes ~1 min and is not done here)."""
    import sys
    sys.path.insert(0, golden_dir)
    from sampling import N_OUT, N_TAP, sub_idx
    n_tap, n_out = len(sub_idx('x', 10 ** 6, N_TAP)), len(sub_idx('x', 10 ** 6, N_OUT))
    g = np.load(os.path.join(golden_dir, 'full6_fp32.npz'))
    assert g['occ_cls'].shape == (200, 200, 16) and g['flow_f16'].shape == (200, 200, 16, 2) and g['counters'].shape == (187,)
    for l in range(6):
        for sfx in ('', '_tsa', '_sca'):
            assert g[f'layer{l}{sfx}_sub'].shape == (n_tap,)
    for tag in ('full6_bf16', 'full6_prev_fp32', 'full6_prev_bf16'):
        h = np.load(os.path.join(golden_dir, tag + '.npz'))
        assert h['occ_sub'].shape == (n_out,) and h['occ_cls'].shape == (200, 200, 16)
    free = (g['occ_cls'] == 16).mean()
    assert 0.6 < free < 0.9                                          # FREE_BIAS keeps the metric rays travelling
    assert not g['flow_f16'][g['occ_cls'] >= 8].any()               # flow stored only where the metric reads it
    b = np.load(os.path.join(golden_dir, 'full6_bf16.npz'))
    assert (b['occ_cls'] == g['occ_cls']).mean() > 0.99 and np.abs(b['occ_sub'] - g['occ_sub']).max() < 6e-2


@pytest.mark.parametrize('hw,center', [((40, 40), [20, 20]), ((200, 200), [100, 100]), ((30, 50), [25, 15])])
def test_rotation_index_map_is_torchvisions_rotation(hw, center):
    """The engine rotates prev_bev by gathering rows through `rotation_index_map` (host side, torchvision applied to an
    image of cell indices).  Applying that map must equal the reference's rotation of the feature map itself
    (transformer_occ.py:195-205) bit for bit, including zero fill and ties."""
    from occnet_b200.engine import rotation_index_map
    h, w = hw
    prev = torch.randn(h * w, 16, generator=torch.Generator().manual_seed(0))
    for ang in (0.0, 3.0, -17.5, 90.0, 181.3, 45.0):
        want = O.rotate_prev_bev(prev.clone(), h, w, ang, center)
        m = torch.from_numpy(rotation_index_map(h, w, ang, center)).long()
        got = torch.zeros_like(prev)
        got[m >= 0] = prev[m[m >= 0]]
        assert torch.equal(got, want), ang
        if ang == 0.0:
            assert torch.equal(m, torch.arange(h * w))
