"""Golden gradients of the geometry mirrors: torch autograd through the UNMODIFIED reference (CPU) for
warp_img_feats_v3 (list and tensor forms), resample_vol_cuda (+ the clamp of test_utils/test_KVNet.py:58-59) and
mutils.misc.depth_val_regression, on the seeded cases of tests/cases_grad.py.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_grad.py
Stored per case (tests/golden/grad_outputs.npz): the gradient as a strided sample (cases_grad.sub) and its full-array
statistics (cases_grad.summary). tests/golden/PINNING_grad.json holds tests/oracle_grad.py's deviation from the full
reference gradients. Both files are written with fixed member order and timestamps, so a re-run reproduces them.
"""
import io
import json
import os
import sys
import warnings
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, '/root/reference/code')
warnings.filterwarnings('ignore')

torch.Tensor.cuda = lambda s, *a, **k: s
torch.nn.Module.cuda = lambda s, *a, **k: s
torch.cuda.current_device = lambda: 0
torch.Tensor.get_device = lambda s: 0

import warping.homography as wh                      # noqa: E402  (reference)
import mutils.misc as m_misc                         # noqa: E402  (reference)

from oracle import planesweep_oracle as O            # noqa: E402
from tests import cases, cases_grad as CG            # noqa: E402
from tests import oracle_grad as OG                  # noqa: E402

T = torch.from_numpy


def save_npz(path, arrays):
    """np.savez_compressed with a fixed member order and timestamp."""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def cam_torch(w, h):
    cam = cases.cam_for(O.make_cam_intrinsics, w, h)
    camt = dict(cam, unit_ray_array_2D=T(cam['unit_ray_array_2D']), intrinsic_M_cuda=T(cam['intrinsic_M_cuda']))
    return cam, camt


def record(out, pin, name, ref_grad, orc_grad):
    out[name + '/g'] = CG.sub(ref_grad)
    out[name + '/stats'] = CG.summary(ref_grad)
    pin['cases'][name] = {'maxabs_oracle': float(np.abs(orc_grad.astype(np.float64) - ref_grad).max()),
                          'max_ref': float(np.abs(ref_grad).max()), 'shape': list(ref_grad.shape)}
    print(name, pin['cases'][name], flush=True)


def warp(out, pin):
    for name in CG.WARP_CASES:
        c = CG.warp_case(name)
        cam, camt = cam_torch(c['w'], c['h'])
        if c['tensor']:
            img = T(c['imgs']).clone().requires_grad_(True)
            res = wh.warp_img_feats_v3(img, c['d'], T(c['R']), T(c['t']), camt)
            (res * T(c['grads'])).sum().backward()
            g = img.grad.numpy()
            o = OG.warp_img_feats_backward([c['grads']], c['d'], [c['R']], [c['t']], cam, c['h'], c['w'])[0]
        else:
            imgs = [T(i).clone().requires_grad_(True) for i in c['imgs']]
            res = wh.warp_img_feats_v3(imgs, c['d'], [T(r) for r in c['R']], [T(t) for t in c['t']], camt)
            sum((r * T(gv)).sum() for r, gv in zip(res, c['grads'])).backward()
            g = np.concatenate([i.grad.numpy() for i in imgs])
            o = np.concatenate(OG.warp_img_feats_backward(c['grads'], c['d'], c['R'], c['t'], cam, c['h'], c['w']))
        del res
        record(out, pin, 'warp/' + name, g, o)


def resample(out, pin):
    for name in CG.RESAMPLE_CASES:
        c = CG.resample_case(name)
        cam, camt = cam_torch(c['w'], c['h'])
        vol = T(c['vol']).clone().requires_grad_(True)
        res = wh.resample_vol_cuda(vol, T(c['rel']), camt, c['d'], c['d_new'], padding_value=c['pad'])
        if c['clamp'] is not None:
            res = res.clamp(min=c['clamp'][0], max=c['clamp'][1])
        res.backward(T(c['grad']))
        o = OG.resample_vol_cuda_backward(c['grad'], c['vol'], c['rel'], cam, c['d'], c['d_new'], c['pad'], c['clamp'])
        record(out, pin, 'resample/' + name, vol.grad.numpy(), o)


def regression(out, pin):
    for name in CG.REGRESSION_CASES:
        c = CG.regression_case(name)
        bv = T(c['bv']).clone().requires_grad_(True)
        m_misc.depth_val_regression(bv, c['d'], BV_log=c['log']).backward(T(c['grad']))
        o = OG.depth_val_regression_backward(c['grad'], c['bv'], c['d'], c['log'])
        record(out, pin, 'regression/' + name, bv.grad.numpy(), o)


def main():
    torch.set_num_threads(8)
    out, pin = {}, {'torch': torch.__version__, 'numpy': np.__version__, 'cases': {}}
    warp(out, pin)
    resample(out, pin)
    regression(out, pin)
    save_npz(os.path.join(HERE, 'grad_outputs.npz'), out)
    with open(os.path.join(HERE, 'PINNING_grad.json'), 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=True)
        f.write('\n')


if __name__ == '__main__':
    main()
