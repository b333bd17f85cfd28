"""Golden outputs and gradients of the DPV statistics: the UNMODIFIED reference's mutils.misc.depth_var and
dpv_statistics on CPU, forward and torch autograd, on the seeded cases of tests/cases_stats.py.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_stats.py
Stored per case (tests/golden/stats_outputs.npz): each output and gradient as a strided sample (cases_stats.sub) with its
full-array statistics (cases_stats.summary), and the plane indices torch.max / torch.min select inside dpv_statistics
(misc.py:600-603) as uint8, in full for the tie case. tests/golden/PINNING_stats.json holds tests/oracle_stats.py's deviation from the
full reference arrays. Both files are written with fixed member order and timestamps, so a re-run reproduces them.
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

import mutils.misc as m_misc                         # noqa: E402  (reference)

from tests import cases_stats as CS                  # noqa: E402
from tests import oracle_stats as OS                 # noqa: E402

T = torch.from_numpy
FULL_INDEX = ('prior_pad_120x160_d64',)     # the tie case keeps every index, its border pixels included


def save_npz(path, arrays):
    """np.savez_compressed with a fixed member order and timestamp."""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def record(out, pin, key, ref, orc):
    ref = np.asarray(ref)
    out[key] = CS.sub(ref)
    out[key + '/stats'] = CS.summary(ref)
    pin['cases'][key] = {'maxabs_oracle': float(np.abs(np.asarray(orc, np.float64) - ref).max()),
                         'max_ref': float(np.abs(ref).max()), 'shape': list(ref.shape)}
    print(key, pin['cases'][key], flush=True)


def main():
    torch.set_num_threads(8)
    out, pin = {}, {'torch': torch.__version__, 'numpy': np.__version__, 'cases': {}}
    for name in CS.CASES:
        c = CS.case(name)
        bv0, d, log = c['bv'], c['d'], c['log']
        # depth_var with the expected depth as its mean, as train_utils/train_KVNet.py:137-138 calls it
        mean0 = c['mean']
        bv, mean = T(bv0).clone().requires_grad_(True), T(mean0).clone().requires_grad_(True)
        var = m_misc.depth_var(bv, mean, d, BV_log=log, d_sigma=c['sigma'])
        var.backward(T(c['g_var']))
        key = 'var/' + name
        record(out, pin, key + '/out', var.detach().numpy(), OS.depth_var(bv0, mean0, d, log, c['sigma']))
        g_bv, g_mu = OS.depth_var_backward(c['g_var'], bv0, mean0, d, log, c['sigma'])
        record(out, pin, key + '/g_bv', bv.grad.numpy(), g_bv)
        record(out, pin, key + '/g_mean', mean.grad.numpy(), g_mu.reshape(mean0.shape))

        # dpv_statistics, differentiated through every channel (the variance's mean included)
        bv = T(bv0).clone().requires_grad_(True)
        feats = m_misc.dpv_statistics(bv, d, c['stats'], BV_log=log)
        feats.backward(T(c['g_stats']))
        of, parts = OS.dpv_statistics(bv0, d, c['stats'], log)
        key = 'stats/' + name
        record(out, pin, key + '/out', feats.detach().numpy(), of)
        record(out, pin, key + '/g_bv', bv.grad.numpy(), OS.dpv_statistics_backward(c['g_stats'], bv0, d, parts, log))
        # the planes the reference's max / min pick (misc.py:600-603 compute them and drop them)
        p = torch.exp(T(bv0)) if log else T(bv0)
        for kind, fn in (('argmax', torch.max), ('argmin', torch.min if log else torch.max)):
            idx = fn(p, dim=1)[1].numpy()
            out[key + '/' + kind] = idx.astype(np.uint8) if name in FULL_INDEX else CS.sub(idx).astype(np.uint8)
            orc = OS.extreme(bv0, log, kind == 'argmin' and log)[1]
            pin['cases'][key + '/' + kind] = {'mismatch_oracle': int((orc != idx).sum()), 'shape': list(idx.shape)}
            print(key + '/' + kind, pin['cases'][key + '/' + kind], flush=True)
    save_npz(os.path.join(HERE, 'stats_outputs.npz'), out)
    with open(os.path.join(HERE, 'PINNING_stats.json'), 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=True)
        f.write('\n')


if __name__ == '__main__':
    main()
