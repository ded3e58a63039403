"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement of the image backbone + neck that FEED the hot path (SURVEY section 8f rank 1, "next"):

    BEVFormerOcc.extract_img_feat           detectors/bevformer_occ.py:66-99
      img (B, N, 3, H, W) -> (B*N, 3, H, W) -> [GridMask: identity in eval, models/utils/grid_mask.py:85-87]
      -> img_backbone -> img_neck -> 4 x (B, N, 256, h_l, w_l)

configured by projects/configs/bevformer/bevformer_base_occ.py:48-66:

    img_backbone = ResNet(depth=50, num_stages=4, out_indices=(1,2,3), norm_eval=True, style='pytorch')
    img_neck     = FPN(in_channels=[512,1024,2048], out_channels=256, start_level=0,
                       add_extra_convs='on_output', num_outs=4, relu_before_extra_convs=True)

Both are THIRD-PARTY mmdet modules (mmdet is absent from the reference tree; BEVFormer's install page pins
mmdet 2.14.0), so the algorithm is restated from its published form:

  * ResNet-50, bottleneck blocks, style='pytorch' (the stride-2 convolution is the 3x3 one, i.e. torchvision's
    "v1.5"); parameter names equal torchvision's (`pretrained='torchvision://resnet50'` loads them unchanged):
    conv1/bn1, layer{1..4}.{i}.conv{1,2,3}/bn{1,2,3}, layer{k}.0.downsample.{0,1}.
  * mmdet FPN: lateral 1x1 convs (bias, no norm/act); top-down `laterals[i-1] += interpolate(laterals[i],
    size=shape(i-1), mode='nearest')`; 3x3 output convs; extra level = `fpn_convs[3]` (3x3, stride 2, pad 1) applied to
    the last OUTPUT (add_extra_convs='on_output'); `relu_before_extra_convs` only affects levels after the first extra
    one, so with num_outs=4 no ReLU is applied.  Parameter names: lateral_convs.{i}.conv.{weight,bias},
    fpn_convs.{i}.conv.{weight,bias}.

Parity status: PINNED against independent implementations of the same published architectures that ARE installed here
-- torchvision.models.resnet50 (same parameter names) and torchvision.ops.FeaturePyramidNetwork + LastLevelP6P7
(tests/test_oracle_cpu.py::test_backbone_*): bit-identical on CPU.  Not pinned against mmdet itself (absent).

All arithmetic fp32, eval mode (BatchNorm uses running statistics).
"""
import torch
import torch.nn.functional as F

STAGE_BLOCKS = (3, 4, 6, 3)          # ResNet-50
STAGE_PLANES = (64, 128, 256, 512)
EXPANSION = 4
BN_EPS = 1e-5


def _bn(p, name, x):
    return F.batch_norm(x, p[name + '.running_mean'], p[name + '.running_var'], p[name + '.weight'], p[name + '.bias'],
                        training=False, eps=BN_EPS)


def bottleneck(p, pre, x, stride):
    """mmdet `Bottleneck.forward` (style='pytorch') == torchvision `Bottleneck.forward`."""
    out = F.relu(_bn(p, pre + 'bn1', F.conv2d(x, p[pre + 'conv1.weight'])))
    out = F.relu(_bn(p, pre + 'bn2', F.conv2d(out, p[pre + 'conv2.weight'], stride=stride, padding=1)))
    out = _bn(p, pre + 'bn3', F.conv2d(out, p[pre + 'conv3.weight']))
    if pre + 'downsample.0.weight' in p:
        x = _bn(p, pre + 'downsample.1', F.conv2d(x, p[pre + 'downsample.0.weight'], stride=stride))
    return F.relu(out + x)


def resnet50(p, img, prefix='img_backbone.', out_indices=(1, 2, 3), taps=None):
    """img (BN, 3, H, W) fp32 -> tuple of stage outputs selected by `out_indices` (mmdet `ResNet.forward`)."""
    x = F.conv2d(img, p[prefix + 'conv1.weight'], stride=2, padding=3)
    x = F.relu(_bn(p, prefix + 'bn1', x))
    if taps is not None:
        taps['stem'] = x
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    outs = []
    for s, nblk in enumerate(STAGE_BLOCKS):
        for b in range(nblk):
            stride = 2 if (b == 0 and s > 0) else 1
            x = bottleneck(p, f'{prefix}layer{s + 1}.{b}.', x, stride)
        if taps is not None:
            taps[f'layer{s + 1}'] = x
        if s in out_indices:
            outs.append(x)
    return tuple(outs)


def fpn(p, feats, prefix='img_neck.', num_outs=4):
    """mmdet `FPN.forward` for start_level=0, add_extra_convs='on_output', upsample mode 'nearest'."""
    n = len(feats)
    lat = [F.conv2d(f, p[f'{prefix}lateral_convs.{i}.conv.weight'], p[f'{prefix}lateral_convs.{i}.conv.bias'])
           for i, f in enumerate(feats)]
    for i in range(n - 1, 0, -1):
        lat[i - 1] = lat[i - 1] + F.interpolate(lat[i], size=lat[i - 1].shape[2:], mode='nearest')
    outs = [F.conv2d(lat[i], p[f'{prefix}fpn_convs.{i}.conv.weight'], p[f'{prefix}fpn_convs.{i}.conv.bias'], padding=1)
            for i in range(n)]
    for i in range(n, num_outs):
        src = outs[-1] if i == n else F.relu(outs[-1])           # relu_before_extra_convs: only from the 2nd extra level on
        outs.append(F.conv2d(src, p[f'{prefix}fpn_convs.{i}.conv.weight'], p[f'{prefix}fpn_convs.{i}.conv.bias'],
                             stride=2, padding=1))
    return tuple(outs)


def extract_img_feat(p, img, taps=None):
    """detectors/bevformer_occ.py:66-99 (eval): img (B, N, 3, H, W) -> list of (B, N, 256, h_l, w_l)."""
    B, N = img.shape[:2]
    x = img.reshape(B * N, *img.shape[2:])
    feats = fpn(p, resnet50(p, x, taps=taps))
    return [f.view(B, N, *f.shape[1:]) for f in feats]


from occnet_b200.fixtures import init_backbone_params as init_params  # noqa: E402,F401  (synthetic weights live with the fixtures)
