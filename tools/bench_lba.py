#!/usr/bin/env python
"""tools/bench_lba.py - ms per call of the LBA pose optimiser, ICP.opt_pose_numerical.local_BA_direct_parallel.

    python tools/bench_lba.py [--impl engine|reference-gpu|reference] [--steps K] [--warmup W] [--dump-outputs DIR]

Workload: the docs/LBA.md command - 384x256 frames, 4 source views, dw_scales [4, 2, 1], max_iter 20, step 0.01,
opt_vars [0, 1] - on the seeded textured-plane scene of tests/cases_lba_opt.py (seed 71, initial translations perturbed).
value = median ms per call, torch.cuda.synchronize() after every call (the call itself ends with its device-to-host read).
  engine        : the device mirror (csrc/lba_opt.cu); also reports launches per call and the final-pose difference to the
                  unmodified reference run once on the same GPU
  reference-gpu : the unmodified reference (oracle/_ref, copied by build(); $NRGBD_REFERENCE_CODE overrides), eager ATen
  reference     : the same on the host cores (the 4-line .cuda() shim); at most 3 timed calls
Prints one JSON line with the card name and its power limit. --dump-outputs DIR writes the engine's final poses as
DIR/poses.npy.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_CODE = os.environ.get('NRGBD_REFERENCE_CODE') or os.path.join(ROOT, 'oracle', '_ref', 'code')
CFG = dict(H=256, W=384, V=4, dw_scales=[4, 2, 1], max_iter=20, step=0.01, opt_vars=[0, 1], seed=71)


def inputs(torch):
    """The scene (initial poses perturbed in t) and the intrinsics of the three levels (torch members, as the reference's)."""
    from tests import cases, cases_lba_opt as LC
    from oracle.planesweep_oracle import make_cam_intrinsics
    c = LC.lba_scene(CFG['seed'], CFG['H'], CFG['W'], CFG['V'], perturb_R=False, perturb_t=True)
    cams = []
    for d in CFG['dw_scales']:
        k = cases.cam_for(make_cam_intrinsics, CFG['W'] // d, CFG['H'] // d)
        cams.append(dict(k, unit_ray_array_2D=torch.from_numpy(k['unit_ray_array_2D']), intrinsic_M_cuda=torch.from_numpy(k['intrinsic_M_cuda'])))
    return c, cams


def gpu_identity(torch):
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'], capture_output=True,
                             text=True, timeout=10).stdout.strip()
        power = float(out) if out else None
    except Exception:           # noqa: BLE001
        power = None
    return {'name': name, 'power_limit_w': power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--impl', default='engine', choices=['engine', 'reference-gpu', 'reference'])
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--dump-outputs', default=None, metavar='DIR')
    args = ap.parse_args()
    if args.dump_outputs and args.impl != 'engine':
        ap.error('--dump-outputs writes the engine\'s outputs: it needs --impl engine')
    on_gpu = args.impl != 'reference'
    if not on_gpu:
        os.environ['CUDA_VISIBLE_DEVICES'] = ''
    import torch
    if not on_gpu:                                     # the reference hard-codes .cuda()
        torch.Tensor.cuda = lambda s_, *a, **k: s_
        torch.nn.Module.cuda = lambda s_, *a, **k: s_
    else:
        assert torch.cuda.is_available(), 'tools/bench_lba.py --impl %s needs a CUDA device' % args.impl
    c, cams = inputs(torch)
    have_ref = bool(REF_CODE) and os.path.isdir(os.path.join(REF_CODE, 'ICP'))

    def reference_fn():
        if not have_ref:
            raise RuntimeError('the reference copy (oracle/_ref, made by build()) is not present')
        sys.path.insert(0, REF_CODE)
        import ICP.opt_pose_numerical as ref_opn                  # reference
        return ref_opn.local_BA_direct_parallel
    if args.impl == 'engine':
        from neuralrgbd_b200 import _lib
        from neuralrgbd_b200.ICP import opt_pose_numerical as M
        fn = M.local_BA_direct_parallel
        L = _lib.lib()
    else:
        fn = reference_fn()
    dev = torch.device('cuda', 0) if on_gpu else torch.device('cpu')
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    frames = (T(c['ref']), [T(s) for s in c['srcs']], T(c['dmap']), T(c['conf']))

    def call(f=fn):
        with contextlib.redirect_stdout(io.StringIO()):
            return f(*frames, cams, CFG['dw_scales'], list(c['poses_init']), CFG['max_iter'], CFG['step'], CFG['opt_vars'])
    for _ in range(args.warmup):
        call()
    if on_gpu:
        torch.cuda.synchronize()
    if args.impl == 'engine':
        L.nrgbd_reset_launch_count()
    ts = []
    for _ in range(max(1, args.steps if on_gpu else min(args.steps, 3))):
        t0 = time.perf_counter()
        poses = call()
        if on_gpu:
            torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    P = np.stack([p.numpy() for p in poses])
    line = {'impl': args.impl, 'metric': 'ms per ICP.opt_pose_numerical.local_BA_direct_parallel call (device-synchronised)',
            'value': 1e3 * float(np.median(ts)), 'unit': 'ms/call', 'higher_is_better': False, 'steps': len(ts), 'warmup': args.warmup,
            'ms_mean': 1e3 * float(np.mean(ts)), 'ms_min': 1e3 * float(np.min(ts)), 'dtype': 'f32',
            'config': dict(CFG, workload='docs/LBA.md setting on tests/cases_lba_opt.py lba_scene'),
            'pose_error_vs_true': {'initial': float(np.abs(c['poses_init'] - c['poses_true']).max()),
                                   'final': float(np.abs(P - c['poses_true']).max())}}
    if on_gpu:
        line['gpu'] = gpu_identity(torch)
    if args.impl == 'engine':
        line['gpu_launches_per_call'] = int(L.nrgbd_launch_count()) / len(ts)
        try:
            ref_P = np.stack([p.cpu().numpy() for p in call(reference_fn())])
            line['final_pose_maxabs_vs_reference_gpu'] = float(np.abs(P - ref_P).max())
        except RuntimeError as e:
            line['final_pose_maxabs_vs_reference_gpu'] = None
            line['reference_note'] = str(e)
        if args.dump_outputs:
            os.makedirs(args.dump_outputs, exist_ok=True)
            np.save(os.path.join(args.dump_outputs, 'poses.npy'), P.astype(np.float32))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
