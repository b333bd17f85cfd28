"""conv_math 'f16x3' against 'f16' on one GPU, alternating in one job.

Workloads (the frames and camera of tests/cases.py 'c23_640x480_d64_v4_stream30', 640x480, D=64, V=4):
  - c2: one first-window forward (no prior);
  - c3: the stream through test_utils.test_KVNet.test (R_net=True): D-Net + K-Net + R-Net + propagation per frame.
Reports frames/s per mode (median of the rounds, CUDA events, profiler off), then per-shape convolution times of one eager
steady frame per mode (the engine's per-launch CUDA events, as bench.py's layer table; one line per convolution shape:
layer2-4 and lastconv at 120x160, the K-Net 3-D convolutions, the 480x640 R-Net convolutions, ...), and the card's name and
power limit before and after.
usage: bench_f16.py [rounds=3] [frames=12] [out=FILE.json]
"""
import contextlib
import ctypes
import io
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralrgbd_b200 import _lib, arch                               # noqa: E402
from neuralrgbd_b200.models.KVNET import KVNET                       # noqa: E402
from oracle import planesweep_oracle as O                            # noqa: E402
from tests import cases                                              # noqa: E402
from tools.bench_refine import card                                  # noqa: E402
from tools.bench_twin import first_window, stream                    # noqa: E402

NAME = 'c23_640x480_d64_v4_stream30'
MODES = ['f16x3', 'f16']
dev = torch.device('cuda:0')


def setup():
    c = cases.big_case(NAME)
    cam = cases.big_cam(O.make_cam_intrinsics, c)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']), intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    sd = arch.synth_state_dict(cases.BIG_CFG[NAME]['wseed'], 64, c['D'], 2, 64)
    models = {}
    for mode in MODES:
        with contextlib.redirect_stdout(io.StringIO()):
            m = KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                      d_upsample_ratio_KV_net=None, t_win_r=2)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        m = m.to(dev)
        m.conv_math = mode
        models[mode] = m
    fr = [{'img': torch.from_numpy(f[None]).to(dev)} for f in c['frames']]
    return c, cam, models, fr


def layer_table(c, cam, m, fr):
    """Per-shape convolution time (us) of one eager steady frame with K-Net and R-Net."""
    L = _lib.lib()
    ent = next(iter(m._engines.values()))
    h = ent['h']
    ms, wk, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
    _lib.check(L.nrgbd_kvnet_set_option(h, b'profile', 1))
    L.nrgbd_kvnet_profile_read(h, 0, ctypes.byref(ms), ctypes.byref(wk), ctypes.byref(n))    # clear
    stream(c, cam, 2, m, fr, 1)                               # prior-less first window + one steady frame
    L.nrgbd_kvnet_profile_read(h, 1, ctypes.byref(ms), ctypes.byref(wk), ctypes.byref(n))
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(L.nrgbd_kvnet_profile_table(h, 0, buf, len(buf)))
    L.nrgbd_kvnet_profile_read(h, 0, ctypes.byref(ms), ctypes.byref(wk), ctypes.byref(n))    # clear
    _lib.check(L.nrgbd_kvnet_set_option(h, b'profile', 0))
    rows = {}
    for ln in buf.value.decode().splitlines():
        tag, cnt, t, work = ln.split(';')
        rows[tag] = {'launches': int(cnt), 'us': float(t) * 1e3, 'tflops': float(work) / (float(t) * 1e-3) / 1e12}
    return rows


def main():
    args = dict(a.split('=', 1) for a in sys.argv[1:])
    rounds = int(args.get('rounds', 3)); nfr = int(args.get('frames', 12))
    out_path = args.get('out')
    res = {'card': card(), 'workload': NAME, 'frames_per_round_c3': nfr, 'modes': MODES}
    c, cam, models, fr = setup()
    c2 = {k: [] for k in MODES}
    c3 = {k: [] for k in MODES}
    for mode, m in models.items():                           # warm every mode's shapes and graphs
        first_window(c, 2, m, 2); stream(c, cam, 2, m, fr, 2)
    for _ in range(rounds):
        for mode, m in models.items():
            c2[mode].append(first_window(c, 2, m, 20))
            c3[mode].append(stream(c, cam, 2, m, fr, nfr))
    res['c2_frames_per_s'] = {k: statistics.median(v) for k, v in c2.items()}
    res['c3_frames_per_s'] = {k: statistics.median(v) for k, v in c3.items()}
    res['c2_rounds'] = c2
    res['c3_rounds'] = c3
    tabs = {mode: layer_table(c, cam, m, fr) for mode, m in models.items()}
    res['layers_us'] = {tag: {mode: tabs[mode].get(tag, {}).get('us') for mode in MODES} for tag in sorted(tabs['f16x3'])}
    res['layers_launches'] = {tag: tabs['f16x3'][tag]['launches'] for tag in sorted(tabs['f16x3'])}
    L = _lib.lib()
    res['workspace_bytes'] = {mode: L.nrgbd_kvnet_workspace_bytes(next(iter(m._engines.values()))['h']) for mode, m in models.items()}
    res['card_after'] = card()
    print(json.dumps(res))
    if out_path:
        with open(out_path, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
