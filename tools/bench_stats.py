"""Times mutils.misc.depth_var and dpv_statistics(['E_mean', 'variance', 'max', 'min']), forward and forward + backward,
through the mirrors and through the reference's own eager ATen code (the copy in oracle/_ref) on the same GPU. Reports
CUDA-event times (median of rounds), device operations per call (torch.profiler: kernels, memsets and copies), the
library's own launches, and the bytes each mirror call must move, computed from the shapes. Records the card's name and
power limit in the same run.

    python tools/bench_stats.py [iters=50] [rounds=5] [out=PATH]

Workloads: a log-DPV with D = 64 at 120x160 (the 640x480 stream's quarter resolution, where the reference's training loss
takes these statistics) and at 480x640. The upstream gradient is a seeded tensor of the output's shape.
Bytes (mirror): the forward reads BV once per statistic (D·hw·4 each) and the mean map, and writes hw·4 per channel. The
backward kernels read BV again (and the upstream gradient, index and mean maps) and write one D·hw gradient per
statistic; autograd then sums the per-statistic gradients (3 adds of D·hw·4 · 3 for dpv_statistics), counted too.
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralrgbd_b200 import _lib, synth                             # noqa: E402
from neuralrgbd_b200.mutils import misc as M                         # noqa: E402
from oracle import fetch_reference                                   # noqa: E402
from tools.bench_refine import card                                  # noqa: E402

STATS = ['E_mean', 'variance', 'max', 'min']


def _time(fn, iters, rounds):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(rounds):
        a.record()
        for _ in range(iters):
            fn()
        b.record(); b.synchronize()
        ts.append(a.elapsed_time(b) / iters * 1e3)          # us per call
    return statistics.median(ts), ts


def _device_ops(fn):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def _launches(fn):
    L = _lib.lib()
    torch.cuda.synchronize()
    L.nrgbd_reset_launch_count()
    fn(); torch.cuda.synchronize()
    return L.nrgbd_launch_count()


def _reference_misc():
    code = fetch_reference.code_dir()
    if not code:
        raise SystemExit('no copy of the reference in oracle/_ref: run __graft_entry__.build() first')
    sys.path.insert(1, code)
    import importlib
    m = importlib.import_module('mutils.misc')
    assert m.__file__.startswith(os.path.abspath(code)), m.__file__
    return m


def workloads(ref, h, w, D=64):
    g = torch.Generator(device='cuda').manual_seed(h * w)
    bv0 = torch.log_softmax(10.0 * torch.randn((1, D, h, w), device='cuda', generator=g), 1).contiguous()
    d = synth.d_candidates(D)
    mean = M.depth_val_regression(bv0, d)
    g_var = torch.randn((1, h, w), device='cuda', generator=g)
    g_st = torch.randn((1, len(STATS), h, w), device='cuda', generator=g)
    hw, Dhw = h * w, D * h * w
    bytes_var = 4 * (Dhw + 2 * hw)
    bytes_var_bwd = 4 * (Dhw + 3 * hw + Dhw + hw)
    bytes_st = 4 * (4 * Dhw + hw + 4 * hw)
    bytes_st_bwd = 4 * (2 * Dhw + hw) + 4 * (2 * Dhw + 3 * hw) + 2 * 4 * (Dhw + 3 * hw) + 3 * 3 * 4 * Dhw
    out = {}
    for impl, mod in (('mirror', M), ('reference', ref)):
        bv_g = bv0.clone().requires_grad_(True)
        out[impl] = {
            'depth_var_fwd': (lambda mod=mod: mod.depth_var(bv0, mean, d), bytes_var),
            'depth_var_fwd_bwd': (lambda mod=mod, bv_g=bv_g: mod.depth_var(bv_g, mean, d).backward(g_var), bytes_var + bytes_var_bwd),
            'dpv_statistics_fwd': (lambda mod=mod: mod.dpv_statistics(bv0, d, STATS), bytes_st),
            'dpv_statistics_fwd_bwd': (lambda mod=mod, bv_g=bv_g: mod.dpv_statistics(bv_g, d, STATS).backward(g_st), bytes_st + bytes_st_bwd),
        }
    return out


def main():
    args = dict(a.split('=', 1) for a in sys.argv[1:])
    iters, rounds = int(args.get('iters', 50)), int(args.get('rounds', 5))
    ref = _reference_misc()
    res = {'card': card(), 'iters': iters, 'rounds': rounds, 'shapes': {}}
    for h, w in ((120, 160), (480, 640)):
        key = '%dx%d_d64' % (h, w)
        rows = {}
        for impl, ops in workloads(ref, h, w).items():
            for name, (fn, nbytes) in ops.items():
                med, ts = _time(fn, iters, rounds)
                row = {'us': med, 'rounds_us': ts, 'device_ops': _device_ops(fn)}
                if impl == 'mirror':
                    row.update(bytes=nbytes, GB_per_s=nbytes / (med * 1e-6) / 1e9, nrgbd_launches=_launches(fn))
                rows.setdefault(name, {})[impl] = row
        for r in rows.values():
            r['speedup'] = r['reference']['us'] / r['mirror']['us']
        res['shapes'][key] = rows
    res['card_after'] = card()
    print(json.dumps(res))
    if args.get('out'):
        with open(args['out'], 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
