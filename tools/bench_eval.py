"""Train-mode against eval-mode KVNET on one GPU, alternating in one job.

Workloads: the C3 stream (640x480, D=64, V=4, the 30 steps of tests/cases.py 'c23_640x480_d64_v4_stream30' through
test_utils.test_KVNet.test with R_net=True: D-Net + K-Net + 2x R-Net + propagation per frame) and the C2 first window
(one forward without a prior). Eval mode uses the running statistics the reference produced for that case
(tests/golden/eval_outputs.npz). Reports, per mode, frames/s (median of the rounds, CUDA events, profiler off), then in a
separate profiled round the per-frame time and launch count of the convolution kernels and of the BatchNorm-pass kernels
(torch.profiler, CUDA activities); the card name and power limit; and dumps both modes' C3 outputs (the last frame's refined
DPV, every frame's depth) to <out>/bench_eval_outputs.npz so that train mode can be compared bit for bit with another build.
usage: bench_eval.py [rounds=3] [out=DIR]
"""
import contextlib
import io
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralrgbd_b200 import synth                                    # noqa: E402
from neuralrgbd_b200.models.KVNET import KVNET                       # noqa: E402
from neuralrgbd_b200.test_utils import test_KVNet as TK              # noqa: E402
from neuralrgbd_b200.mutils import misc                              # noqa: E402
from oracle import planesweep_oracle as O                            # noqa: E402
from tests import cases                                              # noqa: E402

NAME = 'c23_640x480_d64_v4_stream30'
dev = torch.device('cuda:0')


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def setup():
    c = cases.big_case(NAME)
    cam = cases.big_cam(O.make_cam_intrinsics, c)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']), intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_outputs.npz'))
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in c['sd'].items()}
    pre = 'eval/%s/rs/' % NAME
    sd.update({k[len(pre):]: torch.from_numpy(np.asarray(gold[k])) for k in gold.files if k.startswith(pre)})
    with contextlib.redirect_stdout(io.StringIO()):
        m = KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                  d_upsample_ratio_KV_net=None, t_win_r=2, if_refined=True)
    m.load_state_dict(sd)
    m = m.to(dev)
    fr = [{'img': torch.from_numpy(f[None]).to(dev)} for f in c['frames']]
    return c, cam, m, fr


def stream(c, cam, m, fr, n=None, keep=False):
    """C3: the whole stream; returns (frames, per-frame depth list, last refined DPV) when keep."""
    r = c['t_win_r']
    n = n or c['n_steps']
    bv, deps, dmap = None, [], None
    for i in range(n):
        poses, idx = synth.window_rel_poses(c['exts'], r + i, r)
        src = torch.from_numpy(poses[None]).to(dev)
        dmap, bv = TK.test(m, c['d'], [cam], r, [fr[r + i]], [[fr[j] for j in idx]], src, bv, R_net=True)
        if keep:
            deps.append(misc.depth_val_regression(dmap, c['d']).cpu().numpy())
    return n, deps, dmap


def first_window(c, cam, m, fr):
    r = c['t_win_r']
    poses, idx = synth.window_rel_poses(c['exts'], r, r)
    src_f = torch.cat([fr[j]['img'] for j in idx])[None]
    with torch.no_grad():
        return m(fr[r]['img'], src_f, torch.from_numpy(poses[None]).to(dev), torch.zeros(1), cam_intrinsics=[cam])


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); n = fn(); b.record(); torch.cuda.synchronize()
    return n, a.elapsed_time(b)


def main():
    args = dict(a.split('=', 1) for a in sys.argv[1:] if '=' in a)
    rounds = int(args.get('rounds', 3))
    out = args.get('out', os.environ.get('NRGBD_BENCH_OUT', '.'))
    c, cam, m, fr = setup()
    res = {'card': card(), 'workloads': {}}
    modes = {'train': True, 'eval': False}
    for mode, tr in modes.items():                          # warm-up: eager step of each branch and graph capture
        m.train(tr)
        stream(c, cam, m, fr, n=4)
        for _ in range(3):
            first_window(c, cam, m, fr)
    fps = {('c3', k): [] for k in modes}
    fps.update({('c2', k): [] for k in modes})
    for _ in range(rounds):
        for mode, tr in modes.items():                      # alternating
            m.train(tr)
            n, ms = timed(lambda: stream(c, cam, m, fr)[0])
            fps[('c3', mode)].append(1e3 * n / ms)
            n, ms = timed(lambda: [first_window(c, cam, m, fr) for _ in range(20)] and 20)
            fps[('c2', mode)].append(1e3 * n / ms)
    for (w, mode), v in fps.items():
        res['workloads'].setdefault(w, {})[mode] = {'frames_per_s_median': float(np.median(v)), 'rounds': v}
    # profiled round (separate): per-frame time and launches of the convolution and BatchNorm-pass kernels, C3 stream
    from torch.profiler import profile, ProfilerActivity
    for mode, tr in modes.items():
        m.train(tr)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            n = stream(c, cam, m, fr, n=10)[0]
            torch.cuda.synchronize()
        agg = {'conv': [0, 0.0], 'bn_pass': [0, 0.0]}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            k = 'conv' if 'conv_wg_kernel' in e.name else 'bn_pass' if 'bn_apply' in e.name else None
            if k:
                agg[k][0] += 1; agg[k][1] += e.time_range.elapsed_us() / 1e3
        res['workloads']['c3'][mode]['profiled_per_frame'] = {k: {'launches': v[0] / n, 'ms': v[1] / n} for k, v in agg.items()}
    # outputs of both modes at C3 (fresh run of the whole stream each)
    dump = {}
    for mode, tr in modes.items():
        m.train(tr)
        _, deps, dmap = stream(c, cam, m, fr, keep=True)
        dump['%s/depth' % mode] = np.stack(deps)
        dump['%s/last_dmap_refined' % mode] = dmap.cpu().numpy()
    os.makedirs(out, exist_ok=True)
    np.savez_compressed(os.path.join(out, 'bench_eval_outputs.npz'), **dump)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
