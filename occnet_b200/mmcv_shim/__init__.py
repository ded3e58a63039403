"""Minimal stand-in for the parts of mmcv / mmdet the occupancy hot path touches.

mmcv-full, mmdet and mmdet3d are third-party dependencies of the reference that are
neither vendored under the reference tree nor installable here (no network).  The
shipped configs (`projects/configs/bevformer/bevformer_base_occ.py`) are plain Python
files read by `mmcv.Config` and built through mmcv registries, so the drop-in needs:

  * `Config.fromfile` with `_base_` inheritance              (reference: tools/test.py:128)
  * `Registry` / `build_from_cfg`                             (reference: encoder.py:13-16, 28)
  * `BaseModule`, `ModuleList`, `Sequential`                  (spatial_cross_attention.py:21)
  * `FFN`, `build_norm_layer`, `ConvModule`                   (custom_base_transformer_layer.py:150-165,
                                                               transformer_occ.py:110-131)
  * `xavier_init`, `constant_init`                            (spatial_cross_attention.py:13)
  * `LearnedPositionalEncoding` (mmdet)                       (bevformer_base_occ.py:130-135)
  * no-op `auto_fp16` / `force_fp32` (no cfg.fp16 in the shipped configs: SURVEY section 0 row 4)

Everything here is a behavioural restatement of the published mmcv 1.x / mmdet 2.x
semantics (parameter names, init rules, forward arithmetic), written from scratch.
`install_as_mmcv()` additionally registers these objects under the `mmcv.*` / `mmdet.*`
module names; only `tests/golden/gen_golden.py` uses that, to import the *unmodified*
reference modules from the reference tree and pin the oracle against them.
"""
from __future__ import annotations

import copy
import functools
import importlib.util
import math
import os
import sys
import types
import warnings

import torch
import torch.nn as nn

# --------------------------------------------------------------------------- config


class ConfigDict(dict):
    """dict with attribute access (nested dicts are converted on construction)."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        for k, v in dict(*args, **kwargs).items():
            self[k] = v

    @staticmethod
    def _wrap(v):
        if isinstance(v, dict) and not isinstance(v, ConfigDict):
            return ConfigDict(v)
        if isinstance(v, (list, tuple)):
            return type(v)(ConfigDict._wrap(x) for x in v)
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, ConfigDict._wrap(v))

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:  # mirror mmcv: attribute error on missing key
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def __deepcopy__(self, memo):
        return ConfigDict({k: copy.deepcopy(v, memo) for k, v in self.items()})


def _merge(base: dict, child: dict) -> dict:
    out = dict(base)
    for k, v in child.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict) and not v.get('_delete_', False):
            out[k] = _merge(out[k], v)
        else:
            if isinstance(v, dict):
                v = {kk: vv for kk, vv in v.items() if kk != '_delete_'}
            out[k] = v
    return out


def _exec_cfg_file(path: str) -> dict:
    path = os.path.abspath(path)
    ns: dict = {'__file__': path}
    with open(path, 'r') as f:
        code = compile(f.read(), path, 'exec')
    exec(code, ns)  # the config language *is* python (mmcv semantics)
    cfg = {k: v for k, v in ns.items()
           if not k.startswith('__') and not isinstance(v, (types.ModuleType, types.FunctionType))}
    bases = cfg.pop('_base_', [])
    if isinstance(bases, str):
        bases = [bases]
    merged: dict = {}
    for b in bases:
        merged = _merge(merged, _exec_cfg_file(os.path.join(os.path.dirname(path), b)))
    return _merge(merged, cfg)


class Config:
    """`Config.fromfile(path)` -> attribute-accessible nested config (mmcv semantics)."""

    def __init__(self, cfg_dict=None, filename=None):
        object.__setattr__(self, '_cfg_dict', ConfigDict(cfg_dict or {}))
        object.__setattr__(self, 'filename', filename)

    @staticmethod
    def fromfile(filename):
        return Config(_exec_cfg_file(filename), filename=filename)

    def __getattr__(self, k):
        return getattr(self._cfg_dict, k)

    def __getitem__(self, k):
        return self._cfg_dict[k]

    def __contains__(self, k):
        return k in self._cfg_dict

    def get(self, k, default=None):
        return self._cfg_dict.get(k, default)

    def merge_from_dict(self, options: dict):
        for key, v in options.items():
            d = self._cfg_dict
            parts = key.split('.')
            for p in parts[:-1]:
                d = d[int(p)] if isinstance(d, (list, tuple)) else d.setdefault(p, ConfigDict())
            if isinstance(d, list):
                d[int(parts[-1])] = v
            else:
                d[parts[-1]] = v


# --------------------------------------------------------------------------- registry


class Registry:
    def __init__(self, name, build_func=None, parent=None, scope=None):
        self.name = name
        self._module_dict: dict = {}
        self.parent = parent
        self.build_func = build_func or build_from_cfg

    @property
    def module_dict(self):
        return self._module_dict

    def get(self, key):
        if key in self._module_dict:
            return self._module_dict[key]
        if self.parent is not None:
            return self.parent.get(key)
        return None

    def __contains__(self, key):
        return self.get(key) is not None

    def _register(self, cls, name=None, force=False):
        name = name or cls.__name__
        names = [name] if isinstance(name, str) else list(name)
        for n in names:
            if not force and n in self._module_dict and self._module_dict[n] is not cls:
                raise KeyError(f'{n} is already registered in {self.name}')
            self._module_dict[n] = cls

    def register_module(self, name=None, force=False, module=None):
        if module is not None:
            self._register(module, name, force)
            return module

        def deco(cls):
            self._register(cls, name, force)
            return cls
        return deco

    def build(self, *args, **kwargs):
        return self.build_func(*args, **kwargs, registry=self)


def build_from_cfg(cfg, registry, default_args=None):
    if not isinstance(cfg, dict):
        raise TypeError(f'cfg must be a dict, got {type(cfg)}')
    if 'type' not in cfg and not (default_args and 'type' in default_args):
        raise KeyError(f'`cfg` or `default_args` must contain the key "type", got {cfg}')
    args = dict(cfg)
    if default_args:
        for k, v in default_args.items():
            args.setdefault(k, v)
    typ = args.pop('type')
    if isinstance(typ, str):
        cls = registry.get(typ)
        if cls is None:
            raise KeyError(f'{typ} is not in the {registry.name} registry')
    else:
        cls = typ
    return cls(**args)


ATTENTION = Registry('attention')
FEEDFORWARD_NETWORK = Registry('feed-forward Network')
TRANSFORMER_LAYER = Registry('transformerLayer')
TRANSFORMER_LAYER_SEQUENCE = Registry('transformer-layers sequence')
POSITIONAL_ENCODING = Registry('position encoding')
PLUGIN_LAYERS = Registry('plugin layer')
NORM_LAYERS = Registry('norm layer')
ACTIVATION_LAYERS = Registry('activation layer')
CONV_LAYERS = Registry('conv layer')
DROPOUT_LAYERS = Registry('drop out layers')
TRANSFORMER = Registry('Transformer')          # mmdet.models.utils.builder.TRANSFORMER
HEADS = Registry('head')                       # mmdet.models.HEADS
DETECTORS = Registry('detector')               # mmdet.models.DETECTORS
LOSSES = Registry('loss')
BACKBONES = Registry('backbone')
NECKS = Registry('neck')


def build_attention(cfg, default_args=None):
    return build_from_cfg(cfg, ATTENTION, default_args)


def build_feedforward_network(cfg, default_args=None):
    return build_from_cfg(cfg, FEEDFORWARD_NETWORK, default_args)


def build_transformer_layer(cfg, default_args=None):
    return build_from_cfg(cfg, TRANSFORMER_LAYER, default_args)


def build_transformer_layer_sequence(cfg, default_args=None):
    return build_from_cfg(cfg, TRANSFORMER_LAYER_SEQUENCE, default_args)


def build_positional_encoding(cfg, default_args=None):
    return build_from_cfg(cfg, POSITIONAL_ENCODING, default_args)


def build_transformer(cfg, default_args=None):
    return build_from_cfg(cfg, TRANSFORMER, default_args)


def build_loss(cfg):
    return build_from_cfg(cfg, LOSSES)


def build_head(cfg):
    return build_from_cfg(cfg, HEADS)


def build_detector(cfg, train_cfg=None, test_cfg=None):
    return build_from_cfg(cfg, DETECTORS, dict(train_cfg=train_cfg, test_cfg=test_cfg))


# --------------------------------------------------------------------------- modules / init


class BaseModule(nn.Module):
    def __init__(self, init_cfg=None):
        super().__init__()
        self._is_init = False
        self.init_cfg = copy.deepcopy(init_cfg)

    def init_weights(self):
        for m in self.children():
            if hasattr(m, 'init_weights'):
                m.init_weights()
        self._is_init = True


class Sequential(BaseModule, nn.Sequential):
    def __init__(self, *args, init_cfg=None):
        BaseModule.__init__(self, init_cfg)
        nn.Sequential.__init__(self, *args)


class ModuleList(BaseModule, nn.ModuleList):
    def __init__(self, modules=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg)
        nn.ModuleList.__init__(self, modules)


def xavier_init(module, gain=1, bias=0, distribution='normal'):
    assert distribution in ('uniform', 'normal')
    if hasattr(module, 'weight') and module.weight is not None:
        if distribution == 'uniform':
            nn.init.xavier_uniform_(module.weight, gain=gain)
        else:
            nn.init.xavier_normal_(module.weight, gain=gain)
    if hasattr(module, 'bias') and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def constant_init(module, val, bias=0):
    if hasattr(module, 'weight') and module.weight is not None:
        nn.init.constant_(module.weight, val)
    if hasattr(module, 'bias') and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def caffe2_xavier_init(module, bias=0):
    nn.init.kaiming_uniform_(module.weight, a=1, mode='fan_in', nonlinearity='leaky_relu')
    if getattr(module, 'bias', None) is not None:
        nn.init.constant_(module.bias, bias)


def bias_init_with_prob(prior_prob):
    return float(-math.log((1 - prior_prob) / prior_prob))


def _passthrough_decorator(*dargs, **dkwargs):
    """`auto_fp16` / `force_fp32`: identity unless `fp16_enabled` -- never set by the shipped configs."""
    if len(dargs) == 1 and callable(dargs[0]) and not dkwargs:
        return dargs[0]

    def deco(fn):
        return fn
    return deco


auto_fp16 = _passthrough_decorator
force_fp32 = _passthrough_decorator


def deprecated_api_warning(name_dict, cls_name=None):
    def deco(fn):
        return fn
    return deco


def to_2tuple(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x, x)


def digit_version(version_str):
    out = []
    for p in str(version_str).split('+')[0].split('.'):
        num = ''.join(ch for ch in p if ch.isdigit())
        out.append(int(num) if num else 0)
    return tuple(out)


TORCH_VERSION = torch.__version__

Linear = nn.Linear
Conv2d = nn.Conv2d
Conv3d = nn.Conv3d

for _n, _c in (('BN', nn.BatchNorm2d), ('BN1d', nn.BatchNorm1d), ('BN2d', nn.BatchNorm2d),
               ('BN3d', nn.BatchNorm3d), ('LN', nn.LayerNorm), ('GN', nn.GroupNorm)):
    NORM_LAYERS.register_module(_n, module=_c)
for _n, _c in (('ReLU', nn.ReLU), ('Softplus', nn.Softplus), ('GELU', nn.GELU), ('Sigmoid', nn.Sigmoid)):
    ACTIVATION_LAYERS.register_module(_n, module=_c)
for _n, _c in (('Conv1d', nn.Conv1d), ('Conv2d', nn.Conv2d), ('Conv3d', nn.Conv3d), ('Conv', nn.Conv2d)):
    CONV_LAYERS.register_module(_n, module=_c)
DROPOUT_LAYERS.register_module('Dropout', module=nn.Dropout)


def build_norm_layer(cfg, num_features, postfix=''):
    """-> (name, layer); name abbreviations follow mmcv ('bn', 'ln', 'gn')."""
    cfg = dict(cfg)
    typ = cfg.pop('type')
    cls = NORM_LAYERS.get(typ)
    if cls is None:
        raise KeyError(f'Unrecognized norm type {typ}')
    requires_grad = cfg.pop('requires_grad', True)
    cfg.setdefault('eps', 1e-5)
    abbr = {'BN': 'bn', 'BN1d': 'bn', 'BN2d': 'bn', 'BN3d': 'bn', 'LN': 'ln', 'GN': 'gn'}[typ]
    if typ == 'GN':
        layer = cls(num_channels=num_features, **cfg)
    else:
        layer = cls(num_features, **cfg)
    for p in layer.parameters():
        p.requires_grad = requires_grad
    return abbr + str(postfix), layer


def build_activation_layer(cfg):
    cfg = dict(cfg)
    return ACTIVATION_LAYERS.get(cfg.pop('type'))(**cfg)


def build_conv_layer(cfg, *args, **kwargs):
    cfg = dict(cfg) if cfg is not None else dict(type='Conv2d')
    return CONV_LAYERS.get(cfg.pop('type'))(*args, **kwargs, **cfg)


def build_dropout(cfg):
    cfg = dict(cfg)
    return DROPOUT_LAYERS.get(cfg.pop('type'))(**cfg)


class ConvModule(nn.Module):
    """conv -> norm -> act bundle; attribute names `conv`, `bn`, `activate` are part of the
    checkpoint key contract (`...decoder.{0,1}.conv.weight`, `...decoder.{0,1}.bn.*`)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                 groups=1, bias='auto', conv_cfg=None, norm_cfg=None, act_cfg=dict(type='ReLU'),
                 inplace=True, order=('conv', 'norm', 'act'), **kwargs):
        super().__init__()
        self.with_norm = norm_cfg is not None
        self.with_activation = act_cfg is not None
        if bias == 'auto':
            bias = not self.with_norm
        self.order = order
        self.conv = build_conv_layer(conv_cfg, in_channels, out_channels, kernel_size, stride=stride,
                                     padding=padding, dilation=dilation, groups=groups, bias=bias)
        self.norm_name = None
        if self.with_norm:
            self.norm_name, norm = build_norm_layer(norm_cfg, out_channels)
            self.add_module(self.norm_name, norm)
        if self.with_activation:
            act_cfg = dict(act_cfg)
            if act_cfg['type'] in ('ReLU',):
                act_cfg.setdefault('inplace', inplace)
            self.activate = build_activation_layer(act_cfg)
        # mmcv default init: kaiming_normal(fan_out, relu) on conv, constant 1/0 on norm
        nn.init.kaiming_normal_(self.conv.weight, a=0, mode='fan_out', nonlinearity='relu')
        if self.conv.bias is not None:
            nn.init.constant_(self.conv.bias, 0)

    @property
    def norm(self):
        return getattr(self, self.norm_name) if self.norm_name else None

    def forward(self, x):
        for layer in self.order:
            if layer == 'conv':
                x = self.conv(x)
            elif layer == 'norm' and self.with_norm:
                x = self.norm(x)
            elif layer == 'act' and self.with_activation:
                x = self.activate(x)
        return x


@FEEDFORWARD_NETWORK.register_module()
class FFN(BaseModule):
    """x + drop(W2 . drop(act(W1 . x)))  -- parameter keys `layers.0.0.*`, `layers.1.*`."""

    def __init__(self, embed_dims=256, feedforward_channels=1024, num_fcs=2,
                 act_cfg=dict(type='ReLU', inplace=True), ffn_drop=0., dropout_layer=None,
                 add_identity=True, init_cfg=None, **kwargs):
        super().__init__(init_cfg)
        assert num_fcs >= 2
        self.embed_dims = embed_dims
        self.feedforward_channels = feedforward_channels
        self.num_fcs = num_fcs
        self.activate = build_activation_layer(act_cfg)
        layers = []
        in_ch = embed_dims
        for _ in range(num_fcs - 1):
            layers.append(Sequential(Linear(in_ch, feedforward_channels), self.activate, nn.Dropout(ffn_drop)))
            in_ch = feedforward_channels
        layers.append(Linear(feedforward_channels, embed_dims))
        layers.append(nn.Dropout(ffn_drop))
        self.layers = Sequential(*layers)
        self.dropout_layer = build_dropout(dropout_layer) if dropout_layer else nn.Identity()
        self.add_identity = add_identity

    def forward(self, x, identity=None):
        out = self.layers(x)
        if not self.add_identity:
            return self.dropout_layer(out)
        if identity is None:
            identity = x
        return identity + self.dropout_layer(out)


class TransformerLayerSequence(BaseModule):
    def __init__(self, transformerlayers=None, num_layers=None, init_cfg=None):
        super().__init__(init_cfg)
        if isinstance(transformerlayers, dict):
            transformerlayers = [copy.deepcopy(transformerlayers) for _ in range(num_layers)]
        else:
            assert isinstance(transformerlayers, list) and len(transformerlayers) == num_layers
        self.num_layers = num_layers
        self.layers = ModuleList()
        for i in range(num_layers):
            self.layers.append(build_transformer_layer(transformerlayers[i]))
        self.embed_dims = self.layers[0].embed_dims
        self.pre_norm = self.layers[0].pre_norm


@POSITIONAL_ENCODING.register_module()
class LearnedPositionalEncoding(BaseModule):
    """mmdet: pos[b, :, y, x] = cat(col_embed[x], row_embed[y]); Embedding weights ~ U(0,1)."""

    def __init__(self, num_feats, row_num_embed=50, col_num_embed=50, init_cfg=None):
        super().__init__(init_cfg)
        self.row_embed = nn.Embedding(row_num_embed, num_feats)
        self.col_embed = nn.Embedding(col_num_embed, num_feats)
        self.num_feats = num_feats
        self.row_num_embed = row_num_embed
        self.col_num_embed = col_num_embed
        nn.init.uniform_(self.row_embed.weight)
        nn.init.uniform_(self.col_embed.weight)

    def forward(self, mask):
        h, w = mask.shape[-2:]
        x = torch.arange(w, device=mask.device)
        y = torch.arange(h, device=mask.device)
        x_embed = self.col_embed(x)
        y_embed = self.row_embed(y)
        pos = torch.cat((x_embed.unsqueeze(0).repeat(h, 1, 1),
                         y_embed.unsqueeze(1).repeat(1, w, 1)), dim=-1)
        return pos.permute(2, 0, 1).unsqueeze(0).repeat(mask.shape[0], 1, 1, 1)


@LOSSES.register_module()
class CrossEntropyLoss(nn.Module):
    def __init__(self, use_sigmoid=False, use_mask=False, reduction='mean', class_weight=None,
                 loss_weight=1.0, **kwargs):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, cls_score, label, weight=None, avg_factor=None, **kwargs):
        loss = nn.functional.cross_entropy(cls_score, label, reduction='none')
        if weight is not None:
            loss = loss * weight.float()
        loss = loss.sum() / avg_factor if avg_factor is not None else loss.mean()
        return self.loss_weight * loss


@LOSSES.register_module()
class L1Loss(nn.Module):
    def __init__(self, reduction='mean', loss_weight=1.0):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, **kwargs):
        return self.loss_weight * (pred - target).abs().mean()


class _ExtLoader:
    """`mmcv.utils.ext_loader`: the reference calls `load_ext('_ext', [...])` at import time
    (encoder.py:24-25).  `provider(name)` supplies the compiled-op namespace."""
    provider = None

    @classmethod
    def load_ext(cls, name, funcs):
        if cls.provider is None:
            raise ImportError('no ms_deform_attn extension provider registered')
        ext = cls.provider(name)
        for f in funcs:
            assert hasattr(ext, f), f'{f} missing in {name}'
        return ext


ext_loader = _ExtLoader


# --------------------------------------------------------------------------- sys.modules installation


def install_as_mmcv(msda_pytorch=None, ext_provider=None, extra_stub_modules=()):
    """Expose this shim as `mmcv.*` / `mmdet.*` so the unmodified reference modules import.

    Only tests/golden/gen_golden.py calls this (the product imports `occnet_b200.mmcv_shim`
    directly).  `msda_pytorch` is the restated `multi_scale_deformable_attn_pytorch`.
    """
    me = sys.modules[__name__]

    def mod(name, **attrs):
        m = sys.modules.get(name)
        if m is None:
            m = types.ModuleType(name)
            m.__path__ = []  # behave as a package
            sys.modules[name] = m
            if '.' in name:
                parent, _, leaf = name.rpartition('.')
                setattr(mod(parent), leaf, m)
        for k, v in attrs.items():
            setattr(m, k, v)
        return m

    public = {k: getattr(me, k) for k in dir(me) if not k.startswith('_')}
    mod('mmcv', **public)
    mod('mmcv.cnn', **public)
    mod('mmcv.cnn.bricks', **public)
    mod('mmcv.cnn.bricks.registry', **public)
    mod('mmcv.cnn.bricks.transformer', **public)
    mod('mmcv.runner', **public)
    mod('mmcv.runner.base_module', **public)
    mod('mmcv.utils', **public)
    if ext_provider is not None:
        _ExtLoader.provider = ext_provider
    ops = mod('mmcv.ops')
    mod('mmcv.ops.multi_scale_deform_attn',
        multi_scale_deformable_attn_pytorch=msda_pytorch,
        MultiScaleDeformableAttention=type('MultiScaleDeformableAttention', (nn.Module,), {}))
    ops.multi_scale_deformable_attn_pytorch = msda_pytorch
    mod('mmdet')
    mod('mmdet.core', multi_apply=None, reduce_mean=None)
    mod('mmdet.models', HEADS=HEADS, DETECTORS=DETECTORS, build_loss=build_loss)
    mod('mmdet.models.builder', build_loss=build_loss, HEADS=HEADS, DETECTORS=DETECTORS)
    mod('mmdet.models.utils', build_transformer=build_transformer)
    mod('mmdet.models.utils.builder', TRANSFORMER=TRANSFORMER)
    mod('mmdet.models.utils.transformer', inverse_sigmoid=None)
    mod('mmdet.models.dense_heads', DETRHead=type('DETRHead', (BaseModule,), {}))
    mod('mmdet3d')
    mod('mmdet3d.core')
    mod('mmdet3d.core.bbox')
    mod('mmdet3d.core.bbox.coders', build_bbox_coder=None)
    for name in extra_stub_modules:
        mod(name)
    return me
