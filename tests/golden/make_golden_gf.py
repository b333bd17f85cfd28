"""Golden outputs and gradients of the guided filter: the UNMODIFIED reference's models/GF GuidedFilter and BoxFilter on
CPU, forward and torch autograd, on the seeded cases of tests/cases_gf.py.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_gf.py
Stored per case (tests/golden/gf_outputs.npz): GuidedFilter's output and the gradients of x and y, BoxFilter(r)'s output
on y and its gradient, each as a strided sample (cases_gf.sub) with its full-array statistics (cases_gf.summary).
tests/golden/PINNING_gf.json holds tests/oracle_gf.py's deviation from the full reference arrays. Both files are written
with fixed member order and timestamps, so a re-run reproduces them.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, '/root/reference/code')
warnings.filterwarnings('ignore')

from models.GF.guided_filter import GuidedFilter            # noqa: E402  (reference)
from models.GF.box_filter import BoxFilter                  # noqa: E402  (reference)

from tests import cases_gf as CG                            # noqa: E402
from tests import oracle_gf as OG                           # noqa: E402
from tests.golden.make_golden_stats import save_npz         # noqa: E402

T = torch.from_numpy


def record(out, pin, key, ref, orc):
    ref = np.asarray(ref)
    out[key] = CG.sub(ref)
    out[key + '/stats'] = CG.summary(ref)
    pin['cases'][key] = {'maxabs_oracle': float(np.abs(np.asarray(orc, np.float64) - ref).max()),
                         'max_ref': float(np.abs(ref).max()), 'shape': list(ref.shape)}
    print(key, pin['cases'][key], flush=True)


def main():
    torch.set_num_threads(8)
    out, pin = {}, {'torch': torch.__version__, 'numpy': np.__version__, 'cases': {}}
    for name in CG.CASES:
        c = CG.case(name)
        x, y = T(c['x']).clone().requires_grad_(True), T(c['y']).clone().requires_grad_(True)
        o = GuidedFilter(c['r'], c['eps'])(x, y)
        o.backward(T(c['g']))
        key = 'gf/' + name
        record(out, pin, key + '/out', o.detach().numpy(), OG.guided_filter(c['x'], c['y'], c['r'], c['eps']))
        gx, gy = OG.guided_filter_backward(c['g'], c['x'], c['y'], c['r'], c['eps'])
        record(out, pin, key + '/g_x', x.grad.numpy(), gx)
        record(out, pin, key + '/g_y', y.grad.numpy(), gy)

        yb = T(c['y']).clone().requires_grad_(True)
        ob = BoxFilter(c['r'])(yb)
        ob.backward(T(c['g_box']))
        key = 'box/' + name
        record(out, pin, key + '/out', ob.detach().numpy(), OG.box_filter(c['y'], c['r']))
        record(out, pin, key + '/g_x', yb.grad.numpy(), OG.box_filter_backward(c['g_box'], c['r']))
    save_npz(os.path.join(HERE, 'gf_outputs.npz'), out)
    with open(os.path.join(HERE, 'PINNING_gf.json'), 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=True)
        f.write('\n')


if __name__ == '__main__':
    main()
