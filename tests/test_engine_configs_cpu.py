"""occb200_engine_create's argument checks, and the coverage of the configuration table of test_engine_configs_gpu.py.

Every refusal returns 1 with a message naming the field, before any CUDA call: on a machine without a GPU a configuration that
got past the checks returns 4 ('no CUDA device') instead, and every entry of the table does.  The coverage test computes each
property the GPU test's docstring claims from the table itself, so an edit that drops one fails here."""
import ctypes
import math

import pytest
import torch

from test_engine_configs_gpu import ASYM_PC, CONFIGS, PLANS, VIDEO_CONFIGS, make_cfg


def _struct(cfg, precision='bf16', tc=True):
    from occnet_b200.engine import _cfg_struct
    return _cfg_struct(cfg, precision, tc)


def _create(lib, c):
    h = ctypes.c_void_p()
    rc = lib.occb200_engine_create(ctypes.byref(c), ctypes.byref(h))
    err = lib.occb200_last_error().decode()
    if h.value:
        lib.occb200_engine_destroy(h)
    return rc, err


def _set(c, field, value):
    if isinstance(field, tuple):                      # (array field, index)
        getattr(c, field[0])[field[1]] = value
    else:
        setattr(c, field, value)


# (field, value, message fragment): each breaks one field of a valid configuration
REJECTIONS = [
    # existing checks
    ('embed_dims', 128, 'embed_dims'), ('num_heads', 4, 'num_heads'), ('num_levels', 3, 'num_levels'),
    ('sca_points', 4, 'SCA num_points'), ('tsa_points', 8, 'TSA num_points'),
    ('num_cams', 0, 'num_cams'), ('num_cams', 9, 'num_cams'),
    ('num_points_in_pillar', 0, 'num_points_in_pillar'), ('num_points_in_pillar', 3, 'num_points_in_pillar'),
    ('num_points_in_pillar', 16, 'num_points_in_pillar'),
    ('pillar_h', 8, 'pillar_h'), ('out_dim', 64, 'out_dim'),
    ('precision', 2, 'precision'),
    # ffn_dim, num_classes, num_layers: one message per field with its range
    ('ffn_dim', 96, 'ffn_dim must be a positive multiple of 64, got 96'),
    ('ffn_dim', 0, 'ffn_dim must be a positive multiple of 64, got 0'),
    ('ffn_dim', -64, 'ffn_dim must be a positive multiple of 64, got -64'),
    ('num_classes', 33, 'num_classes must be in [1,32], got 33'), ('num_classes', 0, 'num_classes must be in [1,32], got 0'),
    ('num_classes', -1, 'num_classes must be in [1,32], got -1'),
    ('num_layers', 0, 'num_layers must be >= 1, got 0'), ('num_layers', -2, 'num_layers must be >= 1, got -2'),
    # BEV and levels: the gathers sample 2 x 2 neighbourhoods
    ('bev_h', 1, 'bev_h and bev_w must be >= 2'), ('bev_w', 1, 'bev_h and bev_w must be >= 2'),
    ('bev_h', 0, 'bev_h and bev_w must be >= 2'), ('bev_w', -3, 'bev_h and bev_w must be >= 2'),
    (('level_h', 0), 1, 'level 0 must be >= 2'), (('level_w', 1), 1, 'level 1 must be >= 2'),
    (('level_h', 2), 0, 'level 2 must be >= 2'), (('level_w', 3), -2, 'level 3 must be >= 2'),
]
for _ax in range(3):
    REJECTIONS += [(('pc_range', _ax), 40.0 + 100, f'pc_range must be finite with max > min on every axis (axis {_ax})'),
                   (('pc_range', _ax + 3), -1e3, f'pc_range must be finite with max > min on every axis (axis {_ax})'),
                   (('pc_range', _ax), math.nan, f'(axis {_ax})'), (('pc_range', _ax + 3), math.inf, f'(axis {_ax})'),
                   (('pc_range', _ax), -math.inf, f'(axis {_ax})')]
REJECTIONS += [(('pc_range', 5), ASYM_PC[2], '(axis 2)')]              # max == min (the base configuration's pc_range is ASYM_PC)


def _size_cases():
    """configurations just over each element-count bound"""
    base = make_cfg(dict(CONFIGS)['13x17'])
    return [
        (dict(base, bev_h=4096, bev_w=2048), 'bev_h * bev_w * 256'),                          # 2^31 elements
        (dict(base, bev_h=2048, bev_w=2048), 'bev_h * bev_w * pillar_h * out_dim'),           # Nq * 256 = 2^30 fits
        (dict(base, num_cams=8, level_shapes=[(1024, 1024)] + [(2, 2)] * 3), 'num_cams * (sum of level h * w) * 256'),
    ]


@pytest.mark.parametrize('case', range(len(REJECTIONS)))
def test_engine_create_rejects_bad_configuration_before_any_cuda_call(case, lib_built):
    from occnet_b200 import _lib
    lib = _lib.load()
    field, value, msg = REJECTIONS[case]
    c = _struct(make_cfg(dict(CONFIGS)['13x17']))
    _set(c, field, value)
    rc, err = _create(lib, c)
    assert rc == 1, (field, value, rc, err)
    assert msg in err, (field, value, err)


@pytest.mark.parametrize('case', range(3))
def test_engine_create_rejects_sizes_whose_element_counts_overflow_int(case, lib_built):
    from occnet_b200 import _lib
    lib = _lib.load()
    cfg, msg = _size_cases()[case]
    rc, err = _create(lib, _struct(cfg))
    assert rc == 1 and msg in err, (rc, err)


@pytest.mark.parametrize('plan', list(PLANS))
@pytest.mark.parametrize('name', [n for n, _ in CONFIGS])
def test_engine_create_accepts_every_table_entry(name, plan, lib_built):
    """past every check: 0 with a GPU, 4 ('no CUDA device') without one"""
    from occnet_b200 import _lib
    lib = _lib.load()
    rc, err = _create(lib, _struct(make_cfg(dict(CONFIGS)[name]), *PLANS[plan]))
    if torch.cuda.is_available():
        assert rc == 0, err
    else:
        assert rc == 4 and 'no CUDA device' in err, (rc, err)


def test_config_table_covers_every_claimed_value():
    cfgs = {n: make_cfg(o) for n, o in CONFIGS}
    assert 8 <= len(cfgs) <= 10 and len(cfgs) == len(CONFIGS)
    vals = lambda k: {c[k] for c in cfgs.values()}                                   # noqa: E731
    bevs = {(c['bev_h'], c['bev_w']) for c in cfgs.values()}
    assert {(2, 2), (3, 5), (8, 16), (13, 17), (17, 13), (2, 63), (63, 2)} <= bevs
    nq = {(c['bev_h'], c['bev_w']): c['bev_h'] * c['bev_w'] for c in cfgs.values()}
    assert nq[(3, 5)] < 32 and nq[(8, 16)] == 128 and nq[(8, 16)] % 128 == 0
    assert nq[(13, 17)] % 32 != 0 and nq[(17, 13)] % 32 != 0
    assert any(n < 32 for n in nq.values()) and any(n % 32 for n in nq.values()) and any(n % 128 == 0 for n in nq.values())
    assert {1, 3, 5, 7, 8} <= vals('num_cams')
    assert {1, 2, 4, 8} <= vals('num_points_in_pillar')
    assert {1, 2, 3} <= vals('num_layers')
    assert {64, 128, 576, 1024} <= vals('ffn_dim')
    assert {1, 2, 17, 18, 32} <= vals('num_classes')
    # the head route: tensor cores for num_classes + 2 <= 19 (largest 17), CUDA cores above (smallest 18)
    assert max(n for n in vals('num_classes') if n + 2 <= 19) == 17 and min(n for n in vals('num_classes') if n + 2 > 19) == 18
    levels = [lv for c in cfgs.values() for lv in c['level_shapes']]
    assert any(all(lv == (2, 2) for lv in c['level_shapes']) for c in cfgs.values())
    assert any(h * w % 2 == 1 and h * w < 64 for h, w in levels)
    assert any(h * w % 8 == 4 for h, w in levels)                                    # bf16 features: a 4-pixel tail
    assert any(h * w % 4 for h, w in levels)                                         # fp32 features: a scalar tail
    assert {PLANS[p][0] for p in PLANS} == {'fp32', 'bf16'}                          # fp32 and bf16 features both run
    assert any(w >= 4 * h for h, w in levels) and any(h >= 4 * w for h, w in levels)
    assert any(h * w > 64 and h * w % 64 for h, w in levels)                         # a partial 64-pixel tile after full ones
    assert {False, True} <= {bool(c.get('use_cams_embeds', True)) for c in cfgs.values()}
    pcs = [c['pc_range'] for c in cfgs.values()]
    assert ASYM_PC in pcs and ASYM_PC[3] != -ASYM_PC[0] and ASYM_PC[4] != -ASYM_PC[1]                # not centred on the ego
    assert any(tuple(c['img_shape']) != (928, 1600, 3) for c in cfgs.values())
    centres = [(c['rotate_center'], c['bev_h'], c['bev_w']) for c in cfgs.values()]
    assert all(rc != [w // 2, h // 2] for rc, h, w in centres)                       # every one off-centre
    assert sum(rc[0] != rc[1] for rc, h, w in centres) >= len(centres) - 1          # a swapped x / y moves the centre
    assert any(not (0 <= rc[0] < w and 0 <= rc[1] < h) for rc, h, w in centres)      # outside the grid
    assert len(VIDEO_CONFIGS) == 2 and set(VIDEO_CONFIGS) <= set(cfgs)
    assert set(PLANS.values()) == {('fp32', False), ('fp32', True), ('bf16', False), ('bf16', True)}
    # each configuration combines several unusual values: at least three of these per entry
    for n, c in cfgs.items():
        unusual = [c['bev_h'] != c['bev_w'] or c['bev_h'] < 8, c['num_cams'] not in (6,), c['num_points_in_pillar'] != 8,
                   c['ffn_dim'] != 512, c['num_classes'] != 17, c['pc_range'] != make_cfg({})['pc_range'],
                   not c.get('use_cams_embeds', True), tuple(c['img_shape']) != (928, 1600, 3)]
        assert sum(unusual) >= 3, n


def test_every_config_has_pillars_some_camera_sees():
    """an SCA stage whose cameras see nothing would leave the pack stage, the levels and cams_embeds untested"""
    from oracle import bevformer_occ as O
    from test_engine_configs_gpu import metas_for
    for n, o in CONFIGS:
        c = make_cfg(o)
        pc = c['pc_range']
        ref = O.get_reference_points(c['bev_h'], c['bev_w'], pc[5] - pc[2], c['num_points_in_pillar'], '3d', 1)
        _, mask = O.point_sampling(ref, pc, metas_for(c))
        seen = mask[:, 0].any(-1).any(0)
        assert 0.1 < seen.float().mean().item(), (n, seen.float().mean().item())
