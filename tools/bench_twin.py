"""KVNET at temporal window radii 1, 2 and 3 (V = 2, 4, 6 source views) on one GPU, alternating in one job.

Workloads (the frames and camera of tests/cases.py 'c23_640x480_d64_v4_stream30', 640x480, D=64, weights from
arch.synth_state_dict(..., t_win_r=r)):
  - c2: one first-window forward (no prior);
  - c3: the stream through test_utils.test_KVNet.test (R_net=True): D-Net + K-Net + R-Net + propagation per frame.
The plane sweep and the K-Net input volume scale with V; the feature CNN's batch is V + 1 frames; the convolutions after
K-Net's first layer do not depend on V.
Reports frames/s per radius (median of the rounds, CUDA events, profiler off) and the card's name and power limit.
usage: bench_twin.py [rounds=3] [frames=12] [out=FILE.json]
"""
import contextlib
import io
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralrgbd_b200 import arch, synth                              # noqa: E402
from neuralrgbd_b200.models.KVNET import KVNET                       # noqa: E402
from neuralrgbd_b200.test_utils import test_KVNet as TK              # noqa: E402
from oracle import planesweep_oracle as O                            # noqa: E402
from tests import cases                                              # noqa: E402
from tools.bench_refine import card                                  # noqa: E402

NAME = 'c23_640x480_d64_v4_stream30'
RADII = [1, 2, 3]
dev = torch.device('cuda:0')


def setup():
    c = cases.big_case(NAME)
    cam = cases.big_cam(O.make_cam_intrinsics, c)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']), intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    models = {}
    for r in RADII:
        sd = arch.synth_state_dict(cases.BIG_CFG[NAME]['wseed'], 64, c['D'], r, 64)
        with contextlib.redirect_stdout(io.StringIO()):
            m = KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                      d_upsample_ratio_KV_net=None, t_win_r=r)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        models[r] = m.to(dev)
    fr = [{'img': torch.from_numpy(f[None]).to(dev)} for f in c['frames']]
    return c, cam, models, fr


def first_window(c, r, m, n):
    ref_f, src_f, poses = cases.window(dict(c, t_win_r=r), r)
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


def stream(c, cam, r, m, fr, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    bv = None
    for k in range(n + 1):
        if k == 1:
            torch.cuda.synchronize()
            a.record()
        idx = r + k
        poses, nb = synth.window_rel_poses(c['exts'], idx, r)
        _, bv = TK.test(m, c['d'], [cam], r, [fr[idx]], [[fr[i] for i in nb]], torch.from_numpy(poses[None]).to(dev), bv,
                        R_net=True)
    b.record()
    torch.cuda.synchronize()
    return n / (a.elapsed_time(b) / 1e3)


def main():
    args = dict(a.split('=', 1) for a in sys.argv[1:])
    rounds = int(args.get('rounds', 3)); nfr = int(args.get('frames', 12))
    out_path = args.get('out')
    res = {'card': card(), 'workload': NAME, 'frames_per_round_c3': nfr, 'radii': RADII}
    c, cam, models, fr = setup()
    assert nfr + 2 * max(RADII) + 1 < len(fr)
    c2 = {r: [] for r in RADII}
    c3 = {r: [] for r in RADII}
    for r, m in models.items():                              # warm every radius's shapes and graphs
        first_window(c, r, m, 2); stream(c, cam, r, m, fr, 2)
    for _ in range(rounds):
        for r, m in models.items():
            c2[r].append(first_window(c, r, m, 20))
            c3[r].append(stream(c, cam, r, m, fr, nfr))
    res['c2_frames_per_s'] = {'r%d' % k: statistics.median(v) for k, v in c2.items()}
    res['c3_frames_per_s'] = {'r%d' % k: statistics.median(v) for k, v in c3.items()}
    res['c2_rounds'] = {'r%d' % k: v for k, v in c2.items()}
    res['c3_rounds'] = {'r%d' % k: v for k, v in c3.items()}
    res['card_after'] = card()
    print(json.dumps(res))
    if out_path:
        with open(out_path, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
