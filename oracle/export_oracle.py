"""CPU restatement of the reference's output stage -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product path never does (see oracle/planesweep_oracle.py header).

Follows /root/reference/code/test_utils/export_res.py:
  depth_regression            :37-41   sum_d exp(BV) * Depth_Indx_vol
  export_res_img (maps part)  :43-75   Depth_val_vol[0, d] = 1 * d_candi[d] (:49-52); conf = exp(max_d BV) (:56-59);
                                       (map * scale).astype(np.uint16) (:74-75)
  export2pgm                  mio/imgIO.py:9-10  PIL fromarray(uint16).convert('I').save('*.pgm')
Pinned against the live reference by tests/golden/make_golden.py export -> tests/golden/export_outputs.npz
(floating point: torch's vectorised exp / sum order differ from the plain loops here by <= 2 ulp, so the
uint16 maps are pinned to +-1 LSB and the float maps to 2e-6 relative; the PGM byte format is pinned exactly).
"""
import numpy as np


def depth_regression(bv_log, d_candi):
    """bv_log: [D, H, W] float32 log-probabilities -> expected depth [H, W] float32 (sequential fp32 sum over d,
    products rounded before they are added, as the materialised exp(BV) * Depth_val_vol of the reference)."""
    bv = np.asarray(bv_log, np.float32)
    w = np.asarray(d_candi, np.float64).astype(np.float32)     # torch.ones(...) * d_candi[i]: float32 planes
    acc = np.zeros(bv.shape[1:], np.float32)
    for d in range(bv.shape[0]):
        acc = (acc + (np.exp(bv[d]).astype(np.float32) * w[d]).astype(np.float32)).astype(np.float32)
    return acc


def confidence(bv_log):
    """exp(max_d BV) [H, W] float32."""
    return np.exp(np.max(np.asarray(bv_log, np.float32), axis=0)).astype(np.float32)


def to_u16(x, scale):
    """(x * scale).astype(np.uint16): float32 product, truncation toward zero."""
    return (np.asarray(x, np.float32) * np.float32(scale)).astype(np.float32).astype(np.uint16)


def pgm16_bytes(im_u16):
    """Bytes of the .pgm PIL writes for a uint16 image converted to mode 'I': P5, maxval 65535, big-endian."""
    im = np.ascontiguousarray(im_u16, np.uint16)
    h, w = im.shape
    return b'P5\n%d %d\n65535\n' % (w, h) + im.astype('>u2').tobytes()


def export_maps(bv_log, d_candi, depth_scale=1000, conf_scale=1000):
    d = depth_regression(bv_log, d_candi)
    c = confidence(bv_log)
    return d, c, to_u16(d, depth_scale), to_u16(c, conf_scale)
