"""CPU oracle of KVNET.forward in conv_math='f16' (numpy float32, TEST INFRASTRUCTURE ONLY): oracle/kvnet_oracle.py's
KVNET with every convolution that the engine runs on tensor cores computed on RN_f16-rounded operands,
sum RN_f16(x) * RN_f16(w) accumulated in fp32. The 3-input-channel first layer of the feature CNN stays fp32. Everything
else (bias, BatchNorm, residual adds, the sweep, softmax, R-Net's activations) is the fp32 oracle unchanged.

The oracle's convolution primitives (oracle/kvnet_oracle.py) are wrapped only while kvnet_forward runs; oracle/ is not
modified.
"""
import contextlib

import numpy as np

from oracle import kvnet_oracle as N

f32 = np.float32


def rn_f16(a):
    return np.asarray(a, f32).astype(np.float16).astype(f32)


@contextlib.contextmanager
def f16_convolutions():
    conv2d, conv3d, convT = N.conv2d, N.conv3d, N.conv_transpose2d

    def c2(x, w, *a, **k):
        if np.asarray(w).shape[1] == 3:            # the feature CNN's first layer: fp32 on the device too
            return conv2d(x, w, *a, **k)
        return conv2d(rn_f16(x), rn_f16(w), *a, **k)

    def c3(x, w, *a, **k):
        return conv3d(rn_f16(x), rn_f16(w), *a, **k)

    def ct(x, w, *a, **k):
        return convT(rn_f16(x), rn_f16(w), *a, **k)

    N.conv2d, N.conv3d, N.conv_transpose2d = c2, c3, ct
    try:
        yield
    finally:
        N.conv2d, N.conv3d, N.conv_transpose2d = conv2d, conv3d, convT


def kvnet_forward(sd, ref_frame, src_frames, src_cam_poses, cam, d_candi, sigma, BV_predict=None, training=False):
    """kvnet_oracle.kvnet_forward with conv_math='f16' convolutions."""
    with f16_convolutions():
        return N.kvnet_forward(sd, ref_frame, src_frames, src_cam_poses, cam, d_candi, sigma, BV_predict=BV_predict,
                               training=training)
