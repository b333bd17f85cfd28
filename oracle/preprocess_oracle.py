"""CPU restatement of the reference's per-frame input stage -- TEST INFRASTRUCTURE ONLY
(see oracle/planesweep_oracle.py header for who may import oracle/).

Follows mdataloader/scanNet.py:368-369 (PIL.Image.resize(img_size, NEAREST)) and mdataloader/m_preprocess.py:15-21
(torchvision ToTensor + Normalize(ImageNet)). PIL and torchvision are third-party dependencies of the reference that are
not vendored under /root/reference (requirements.txt pins no versions); their algorithms restated here:
  * Pillow libImaging/Geometry.c ImagingScaleAffine, nearest filter: xo = 0.5*scale; for each output sample take
    (int)xo, then xo += scale (double accumulation);
  * torchvision to_tensor: uint8 HWC -> float32 CHW, .div(255); Normalize: .sub_(mean).div_(std), fp32.
Pinned bit-exactly against Pillow 12.2 / torchvision 0.26 run here: tests/golden/make_golden.py preprocess.
"""
import numpy as np

IMAGENET = {'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225]}


def nearest_index(n_out, n_in):
    a = n_in / n_out
    xo = a * 0.5
    out = np.empty(n_out, np.int64)
    for x in range(n_out):
        out[x] = min(int(xo), n_in - 1)
        xo += a
    return out


def resize_nearest(img_u8_hwc, size_wh):
    W, H = size_wh
    a = np.asarray(img_u8_hwc)
    return a[nearest_index(H, a.shape[0])][:, nearest_index(W, a.shape[1])]


def to_tensor_normalize(img_u8_hwc, stats=IMAGENET):
    f = (np.asarray(img_u8_hwc).astype(np.float32) / np.float32(255)).transpose(2, 0, 1)
    mean = np.asarray(stats['mean'], np.float32)[:, None, None]
    std = np.asarray(stats['std'], np.float32)[:, None, None]
    return ((f - mean).astype(np.float32) / std).astype(np.float32)[None]


def preprocess(img_u8_hwc, size_wh=None):
    a = np.asarray(img_u8_hwc)
    if size_wh is not None:
        a = resize_nearest(a, size_wh)
    return to_tensor_normalize(a)
