"""Times models.GF GuidedFilter(r=1, eps=1e-8), forward and forward + backward, through the mirror
(neuralrgbd_b200.models.GF) and through the reference's own module (the copy in oracle/_ref) on the same GPU. Reports
CUDA-event times (median of rounds), device operations per call (torch.profiler: kernels, memsets and copies), the
library's own launches for the mirror, and the bytes a call must move, computed from the shapes. Records the card's name
and power limit in the same run.

    python tools/bench_gf.py [iters=50] [rounds=5] [out=PATH]

Workloads: N = 1, C_x = C_y = 1 at 480x640 (KVNET-DGF's refined output) and 120x160; x and y seeded on the device, the
upstream gradient a seeded tensor of the output's shape.
Bytes: the compulsory traffic of the filter, not of its intermediates: the forward reads x and y and writes the output
(3 planes); the backward reads the upstream gradient, x and y and writes both gradients (5 more planes). GB/s is that
over the measured time, an effective rate: the kernels also stream their box-sum planes through L2 and HBM.
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralrgbd_b200.models.GF.guided_filter import GuidedFilter      # noqa: E402
from oracle import fetch_reference                                     # noqa: E402
from tools.bench_refine import card                                    # noqa: E402
from tools.bench_stats import _device_ops, _launches, _time           # noqa: E402


def _reference_gf():
    code = fetch_reference.code_dir()
    if not code:
        raise SystemExit('no copy of the reference in oracle/_ref: run __graft_entry__.build() first')
    sys.path.insert(1, code)
    import importlib
    m = importlib.import_module('models.GF.guided_filter')
    assert m.__file__.startswith(os.path.abspath(code)), m.__file__
    return m


def workloads(ref, h, w):
    g = torch.Generator(device='cuda').manual_seed(h * w)
    x = torch.randn((1, 1, h, w), device='cuda', generator=g)
    y = 2.5 + torch.randn((1, 1, h, w), device='cuda', generator=g)
    go = torch.randn((1, 1, h, w), device='cuda', generator=g)
    plane = 4 * h * w
    out = {}
    for impl, mod in (('mirror', GuidedFilter(1, 1e-8)), ('reference', ref.GuidedFilter(1, 1e-8))):
        xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
        out[impl] = {
            'gf_fwd': (lambda mod=mod: mod(x, y), 3 * plane),
            'gf_fwd_bwd': (lambda mod=mod, xg=xg, yg=yg: mod(xg, yg).backward(go), 8 * plane),
        }
    return out


def main():
    args = dict(a.split('=', 1) for a in sys.argv[1:])
    iters, rounds = int(args.get('iters', 50)), int(args.get('rounds', 5))
    ref = _reference_gf()
    res = {'card': card(), 'iters': iters, 'rounds': rounds, 'shapes': {}}
    for h, w in ((120, 160), (480, 640)):
        rows = {}
        for impl, ops in workloads(ref, h, w).items():
            for name, (fn, nbytes) in ops.items():
                med, ts = _time(fn, iters, rounds)
                row = {'us': med, 'rounds_us': ts, 'device_ops': _device_ops(fn), 'bytes': nbytes,
                       'GB_per_s': nbytes / (med * 1e-6) / 1e9}
                if impl == 'mirror':
                    row['nrgbd_launches'] = _launches(fn)
                rows.setdefault(name, {})[impl] = row
        for r in rows.values():
            r['speedup'] = r['reference']['us'] / r['mirror']['us']
        res['shapes']['%dx%d' % (h, w)] = rows
    res['card_after'] = card()
    print(json.dumps(res))
    if args.get('out'):
        with open(args['out'], 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
