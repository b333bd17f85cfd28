"""Times the f-5 backward kernels (CUDA events, median of rounds) and reports the bytes each must move, computed from
the shapes, and the bandwidth that implies. Records the card's name and power limit in the same run.

    python tools/bench_grad.py [iters=50] [rounds=5] [out=PATH]

Workloads (the 640x480 stream, 64 planes):
  * warp: the K-Net image warp, V = 4 views of C = 3 channels, at quarter resolution (120x160, what KVNET warps) and at
    image resolution (480x640);
  * resample: the DPV propagation (padding log(1/D), clamp [-1000, 0]) at quarter and image resolution;
  * regression: the expected depth of a quarter-resolution log-DPV.
Bytes: the upstream gradient read once, the gradient written twice (zeroed, then the scatter's lines written back),
inputs re-read by the backward (the volume for the clamp mask, BV for the exp) and the rays. Atomic traffic that stays
in L2 is not counted.
"""
import ctypes
import json
import math
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neuralrgbd_b200 import _lib, camera, synth                     # noqa: E402
from neuralrgbd_b200._lib import ptr                                 # noqa: E402
from neuralrgbd_b200.warping import homography as H                  # noqa: E402
from tests import cases                                              # noqa: E402
from tools.bench_refine import card                                  # noqa: E402

F = ctypes.c_float


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


def warp(h, w, D=64, V=4, C=3):
    L = _lib.lib()
    cam = cases.cam_for(camera.make_cam_intrinsics, w, h)
    K, rays = H._cam_tensors(cam, torch.device('cuda'))
    rng = np.random.RandomState(1)
    poses = cases._poses(rng, V)
    R = torch.from_numpy(np.ascontiguousarray(poses[:, :3, :3])).cuda()
    t = torch.from_numpy(np.ascontiguousarray(poses[:, :3, 3])).cuda()
    dpl = H._planes(synth.d_candidates(D), torch.device('cuda'))
    go = torch.randn((V, C, D, h * w), device='cuda')
    ws = torch.empty(L.nrgbd_sweep_workspace_floats(V), device='cuda')
    g = torch.empty((V, C, h * w), device='cuda')
    cx, cy = float(cam['intrinsic_M'][0, 2]), float(cam['intrinsic_M'][1, 2])
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    fn = lambda: L.nrgbd_warp_to_volume_backward(ptr(go), C, V, D, h, w, ptr(K), ptr(R), ptr(t), ptr(rays), ptr(dpl),   # noqa: E731
                                                 F(cx), F(cy), ptr(ws), ptr(g), st)
    return fn, 4 * (V * C * D * h * w + 2 * V * C * h * w + 3 * h * w)


def resample(h, w, D=64):
    L = _lib.lib()
    cam = cases.cam_for(camera.make_cam_intrinsics, w, h)
    _, rays = H._cam_tensors(cam, torch.device('cuda'))
    d = synth.d_candidates(D)
    d_pts, tan_hh, tan_hv, z_half, z_radius = H.resample_params(cam, d)
    dp = H.planes_tensor(d_pts, torch.device('cuda'))
    rng = np.random.RandomState(2)
    exts = synth.camera_track(rng, 2)
    E = torch.from_numpy(np.linalg.inv(exts[1].dot(np.linalg.inv(exts[0]))).astype(np.float32)).cuda()
    vol = torch.log_softmax(torch.randn((D, h * w), device='cuda'), 0).contiguous()
    go = torch.randn((D, h * w), device='cuda')
    g = torch.empty((D, h * w), device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    fn = lambda: L.nrgbd_resample_dpv_backward(ptr(vol), h * w, 1, ptr(E), ptr(rays), ptr(dp), D, h, w, F(tan_hh), F(tan_hv),   # noqa: E731
                                               F(z_half), F(z_radius), F(math.log(1.0 / D)), 1, F(-1000.0), F(0.0),
                                               ptr(go), h * w, 1, ptr(g), st)
    return fn, 4 * (4 * D * h * w + 3 * h * w)


def regression(h, w, D=64):
    L = _lib.lib()
    dpl = H._planes(synth.d_candidates(D), torch.device('cuda'))
    bv = torch.log_softmax(torch.randn((D, h * w), device='cuda'), 0).contiguous()
    go = torch.randn((h * w,), device='cuda')
    g = torch.empty((D, h * w), device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    fn = lambda: L.nrgbd_depth_regression_backward(ptr(go), ptr(bv), h * w, D, h * w, 1, ptr(dpl), 1, ptr(g), st)   # noqa: E731
    return fn, 4 * (h * w + 2 * D * h * w)


def main():
    args = dict(a.split('=', 1) for a in sys.argv[1:])
    iters, rounds = int(args.get('iters', 50)), int(args.get('rounds', 5))
    res = {'card': card(), 'iters': iters, 'rounds': rounds, 'kernels': {}}
    work = {'warp_v4_c3_d64_120x160': lambda: warp(120, 160), 'warp_v4_c3_d64_480x640': lambda: warp(480, 640),
            'resample_clamp_d64_120x160': lambda: resample(120, 160), 'resample_clamp_d64_480x640': lambda: resample(480, 640),
            'regression_log_d64_120x160': lambda: regression(120, 160)}
    for name, make in work.items():
        fn, nbytes = make()
        med, ts = _time(lambda: _lib.check(fn()), iters, rounds)
        res['kernels'][name] = {'us': med, 'rounds_us': ts, 'bytes': nbytes, 'GB_per_s': nbytes / (med * 1e-6) / 1e9}
    res['card_after'] = card()
    print(json.dumps(res))
    if args.get('out'):
        with open(args['out'], 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
