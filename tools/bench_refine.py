"""KVNET's refinement configurations on one GPU, alternating in one job: the default DPV R-Net, the depth-upsampled DPV
R-Net (if_upsample_d=True, refined DPVs of 4D planes), the guided filter (refineNet_name='DGF') and no refinement
(if_refined=False).

Workloads (tests/cases.py 'c23_640x480_d64_v4_stream30', 640x480, D=64, V=4):
  - c2: one first-window forward (no prior);
  - c3: the stream through test_utils.test_KVNet.test (R_net=True, or R_net=False without refinement): D-Net + K-Net +
    the configuration's refinement + propagation per frame.
Reports frames/s per configuration (median of the rounds, CUDA events, profiler off); the guided-filter entry point's time
at 640x480 (CUDA events over many calls) and its bandwidth from the bytes its passes move (computed from the shapes); and
the card's name and power limit.
usage: bench_refine.py [rounds=3] [frames=12] [out=FILE.json]
"""
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralrgbd_b200 import arch, convops, synth                     # noqa: E402
from neuralrgbd_b200.models.KVNET import KVNET                       # noqa: E402
from neuralrgbd_b200.test_utils import test_KVNet as TK              # noqa: E402
from oracle import planesweep_oracle as O                            # noqa: E402
from tests import cases                                              # noqa: E402

NAME = 'c23_640x480_d64_v4_stream30'
CONFIGS = {'DPV': dict(if_refined=True, refineNet_name='DPV'),
           'DPV_up': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True),
           'DGF': dict(if_refined=True, refineNet_name='DGF'), 'none': dict(if_refined=False)}
dev = torch.device('cuda:0')


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def setup():
    c = cases.big_case(NAME)
    cam = cases.big_cam(O.make_cam_intrinsics, c)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']), intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    models = {}
    for name, kw in CONFIGS.items():
        sd = arch.synth_state_dict(cases.BIG_CFG[NAME]['wseed'], 64, c['D'], 2, 64,
                                   refine={'DGF': 'DGF', 'none': None}.get(name, 'DPV'), upsample_d=name == 'DPV_up')
        with contextlib.redirect_stdout(io.StringIO()):
            m = KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                      d_upsample_ratio_KV_net=None, t_win_r=2, **kw)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        models[name] = m.to(dev)
    fr = [{'img': torch.from_numpy(f[None]).to(dev)} for f in c['frames']]
    return c, cam, models, fr


def first_window(c, m, n):
    ref_f, src_f, poses = cases.window(c, 2)
    ref, src, P = (torch.from_numpy(a).to(dev) for a in (ref_f, src_f, poses))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        m(ref, src, P, torch.zeros(1), cam_intrinsics=[None])
        torch.cuda.synchronize()
        a.record()
        for _ in range(n):
            m(ref, src, P, torch.zeros(1), cam_intrinsics=[None])
        b.record()
    torch.cuda.synchronize()
    return n / (a.elapsed_time(b) / 1e3)


def stream(c, cam, m, fr, n, refined):
    r = c['t_win_r']
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    bv = None
    for k in range(n + 1):
        if k == 1:
            torch.cuda.synchronize()
            a.record()
        idx = r + k
        poses, nb = synth.window_rel_poses(c['exts'], idx, r)
        _, bv = TK.test(m, c['d'], [cam], r, [fr[idx]], [[fr[i] for i in nb]], torch.from_numpy(poses[None]).to(dev), bv,
                        R_net=refined)
    b.record()
    torch.cuda.synchronize()
    return n / (a.elapsed_time(b) / 1e3)


def gf_kernel(H=480, W=640, iters=200):
    rng = np.random.RandomState(0)
    dmap = torch.from_numpy((2.5 + rng.rand(H // 4, W // 4)).astype(np.float32)).to(dev)
    img = torch.from_numpy(rng.standard_normal((3, H, W)).astype(np.float32)).to(dev)
    w0, b0 = torch.randn(64, 3, 1, 1, device=dev) * 0.2, torch.randn(64, device=dev) * 0.1
    w1, b1 = torch.randn(1, 64, 1, 1, device=dev), torch.randn(1, device=dev) * 0.1
    for _ in range(10):
        convops.guided_filter_refine(dmap, img, w0, b0, w1, b1)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        convops.guided_filter_refine(dmap, img, w0, b0, w1, b1)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    HW, hw = H * W, H * W // 16
    # prep: dmap + rgb in, x and y out; each scan pass reads its source planes twice (segment totals, then the prefix walk)
    # and writes prefix, reads prefix, writes diff per output plane: column pass to [x | y | x*y | x*x] (5 source planes:
    # the products formed from x and y while loading), row pass over those 4, column pass to [A | b] (each from the 4 box
    # planes), row pass over those 2; output: 2 box planes + x in, 1 out
    floats = (hw + 3 * HW + 2 * HW) + (2 * 5 + 3 * 4) * HW + (2 + 3) * 4 * HW + (2 * 8 + 3 * 2) * HW + (2 + 3) * 2 * HW + 4 * HW
    return {'ms': ms, 'bytes': 4.0 * floats, 'GB_per_s': 4.0 * floats / (ms * 1e-3) / 1e9, 'shape': [H, W]}


def main():
    args = dict(a.split('=', 1) for a in sys.argv[1:])
    rounds = int(args.get('rounds', 3)); nfr = int(args.get('frames', 12))
    out_path = args.get('out')
    res = {'card': card(), 'workload': NAME, 'frames_per_round_c3': nfr}
    c, cam, models, fr = setup()
    assert nfr + 2 * c['t_win_r'] + 1 < len(fr)
    c2 = {k: [] for k in CONFIGS}
    c3 = {k: [] for k in CONFIGS}
    for name, m in models.items():                          # warm every configuration's shapes and graphs
        first_window(c, m, 2); stream(c, cam, m, fr, 2, name != 'none')
    for _ in range(rounds):
        for name, m in models.items():
            c2[name].append(first_window(c, m, 20))
            c3[name].append(stream(c, cam, m, fr, nfr, name != 'none'))
    res['c2_frames_per_s'] = {k: statistics.median(v) for k, v in c2.items()}
    res['c3_frames_per_s'] = {k: statistics.median(v) for k, v in c3.items()}
    res['c2_rounds'] = c2
    res['c3_rounds'] = c3
    res['guided_filter'] = gf_kernel()
    res['card_after'] = card()
    print(json.dumps(res))
    if out_path:
        with open(out_path, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
