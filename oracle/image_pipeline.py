"""CPU restatement of the shipped test pipeline's image steps (test infrastructure only, like the rest of oracle/).

    reference: projects/configs/bevformer/bevformer_base_occ.py:166-183 (test_pipeline)
               projects/mmdet3d_plugin/datasets/pipelines/transform_3d.py:11-99 (PadMultiViewImage, NormalizeMultiviewImage)

Steps, per camera, on the HWC uint8 image in BGR order that mmcv.imread returns:

1. LoadMultiViewImageFromFiles(to_float32=True) (mmdet3d, not in the reference tree) only casts to float32: the values stay
   integral, 0..255.
2. NormalizeMultiviewImage(mean, std, to_rgb) stores mean / std as float32 arrays and calls mmcv.imnormalize: the BGR->RGB
   swap first (so mean / std are indexed in RGB order when to_rgb), then cv2.subtract(img, float64(mean)) and
   cv2.multiply(img, 1 / float64(std)).  Restated in fp32 as

       y = (f32(x) - f32(mean[c])) * f32(1 / f64(f32(std[c])))

   two separately rounded operations (the device kernel uses __fsub_rn / __fmul_rn so nothing is contracted into an FMA).
   mmcv and OpenCV are not available here, so whether OpenCV rounds its float64 scalar operands to float32 exactly like this
   before operating on a CV_32F image is NOT checked; either way a difference would be at most one ulp of the normalised
   value.  With the shipped std = 1 the multiply is exact and y = f32(x) - f32(mean[c]).
3. PadMultiViewImage(size | size_divisor, pad_val=0) pads at the bottom and right AFTER normalisation (padded pixels hold
   pad_val, not a normalised 0); size_divisor d pads (h, w) to (ceil(h/d)*d, ceil(w/d)*d) (mmcv.impad_to_multiple), size
   pads to exactly (H, W) (mmcv.impad, which rejects a smaller size).  It sets the per-camera lists ori_shape (unpadded),
   img_shape and pad_shape (both padded) and pad_fixed_size / pad_size_divisor.
4. DefaultFormatBundle3D transposes every camera HWC -> CHW and stacks them: (N, 3, H, W) float32.
"""
import numpy as np

SHIPPED_NORM = dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False)   # bevformer_base_occ.py:14-15
SHIPPED_PAD = dict(size_divisor=32)                                                         # :170


def padded_shape(h, w, size=None, size_divisor=None):
    """(H, W) after PadMultiViewImage; exactly one of size / size_divisor."""
    assert (size is None) != (size_divisor is None), 'PadMultiViewImage takes exactly one of size / size_divisor'
    if size is not None:
        H, W = int(size[0]), int(size[1])
        if H < h or W < w:
            raise ValueError(f'pad size {(H, W)} is smaller than the image {(h, w)}')
        return H, W
    d = int(size_divisor)
    return int(np.ceil(h / d)) * d, int(np.ceil(w / d)) * d


def normalize(img, mean, std, to_rgb):
    """mmcv.imnormalize(img, float32 mean, float32 std, to_rgb) restated in fp32: HWC uint8/float -> HWC float32."""
    x = np.asarray(img).astype(np.float32)
    if to_rgb:
        x = x[..., ::-1]
    m = np.asarray(mean, np.float32).reshape(1, 1, 3)
    inv = (1.0 / np.asarray(std, np.float32).astype(np.float64)).astype(np.float32).reshape(1, 1, 3)
    return np.ascontiguousarray((x - m) * inv, dtype=np.float32)


def pad(img, H, W, pad_val=0):
    """bottom / right padding of an HWC image to (H, W) with pad_val"""
    h, w = img.shape[:2]
    out = np.full((H, W) + img.shape[2:], pad_val, dtype=img.dtype)
    out[:h, :w] = img
    return out


def pipeline(frames, mean=SHIPPED_NORM['mean'], std=SHIPPED_NORM['std'], to_rgb=SHIPPED_NORM['to_rgb'], size=None,
             size_divisor=None, pad_val=0):
    """frames: N HWC uint8 BGR images (an (N, h, w, 3) array or a list).  Returns (imgs (N, 3, H, W) float32, metas) where
    metas holds what NormalizeMultiviewImage + PadMultiViewImage add to the results dict."""
    if size is None and size_divisor is None:
        size_divisor = SHIPPED_PAD['size_divisor']
    frames = [np.asarray(f) for f in frames]
    normed = [normalize(f, mean, std, to_rgb) for f in frames]
    padded = []
    for f in normed:
        H, W = padded_shape(f.shape[0], f.shape[1], size=size, size_divisor=size_divisor)
        padded.append(pad(f, H, W, pad_val))
    metas = dict(ori_shape=[f.shape for f in normed], img_shape=[f.shape for f in padded],
                 pad_shape=[f.shape for f in padded], pad_fixed_size=size, pad_size_divisor=size_divisor,
                 img_norm_cfg=dict(mean=np.asarray(mean, np.float32), std=np.asarray(std, np.float32), to_rgb=to_rgb))
    imgs = np.stack([np.ascontiguousarray(f.transpose(2, 0, 1)) for f in padded]).astype(np.float32)
    return imgs, metas
