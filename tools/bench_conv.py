"""Conv micro-benchmark at the real layer shapes of the 640x480 workload: fp32 FFMA implicit GEMM
(nrgbd_conv_nhwc) vs wgmma 3xTF32 (nrgbd_conv_nhwc_tc, split time reported separately).
CUDA events, 256 MiB L2 flush between iterations. Development aid.

    python tools/bench_conv.py abflags [only=<name part>] [rounds=N] [out=<file.json>]
times the split-fp16 convolution (nrgbd_conv_nhwc_h2) at each shape with all schedule features on (flags 0) and with
each one switched off (8: 16 x 8 tile only, 32: one tile per CTA, 40: both), the arms
alternating round by round, and writes the medians to the JSON file `out` (default: bench_conv_ab.json)."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuralrgbd_b200 import _lib, convops        # noqa: E402
from neuralrgbd_b200._lib import ptr, check      # noqa: E402

dev = torch.device('cuda:0')
L = _lib.dev_lib()
st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)     # noqa: E731
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts))


SHAPES = [  # name, N, D, H, W, Cin, Cout, k(kd), stride, pad, dil
    ('layer1 32->32 @1/2', 5, 1, 240, 320, 32, 32, 3, 1, 1, 1),
    ('layer2 64->64 @1/4', 5, 1, 120, 160, 64, 64, 3, 1, 1, 1),
    ('layer3 128->128 @1/4', 5, 1, 120, 160, 128, 128, 3, 1, 1, 1),
    ('layer4 128->128 dil2', 5, 1, 120, 160, 128, 128, 3, 1, 2, 2),
    ('lastconv 320->128', 5, 1, 120, 160, 320, 128, 3, 1, 1, 1),
    ('rnet conv0 128->128', 1, 1, 120, 160, 128, 128, 3, 1, 1, 1),
    ('rnet conv1 96->96 @1/2', 1, 1, 240, 320, 96, 96, 3, 1, 1, 1),
    ('rnet conv2_2 64->64 @1', 1, 1, 480, 640, 64, 64, 3, 1, 1, 1),
    ('knet 64->64 3d (D=64)', 1, 64, 120, 160, 64, 64, 3, 1, 1, 1),
    ('rnet conv2 67->67 @1', 1, 1, 480, 640, 67, 67, 3, 1, 1, 1),
    ('rnet conv0 320->320 (D=256) @1/4 1080p', 1, 1, 270, 480, 320, 320, 3, 1, 1, 1),
]


def main():
    out = []
    for a in sys.argv[1:]:
        if a.startswith('h2flags='):
            L.nrgbd_dev_conv_h2_set_flags(int(a[8:]))
    only = [a[5:] for a in sys.argv[1:] if a.startswith('only=')]
    for name, N, D, H, W, Cin, Cout, k, s, p, d in SHAPES:
        if only and not any(o in name for o in only):
            continue
        kd = 3 if D > 1 else 1
        Cs = convops.pad_to(Cin, 32)
        x = torch.randn((N, D, H, W, Cs), device=dev)
        w = torch.randn((Cout, Cin) + ((kd,) if D > 1 else ()) + (k, k), device=dev) / np.sqrt(Cin * k * k * kd)
        wp = convops.pack_weight(w)
        wh, wl = convops.pack_weight_tc(w)
        Ho = (H + 2 * p - d * (k - 1) - 1) // s + 1; Wo = (W + 2 * p - d * (k - 1) - 1) // s + 1
        Cso = convops.pad4(Cout)
        y = torch.zeros((N, D, Ho, Wo, Cso), device=dev)
        y2 = torch.zeros_like(y)
        stats = torch.zeros((2, Cout), device=dev, dtype=torch.float64)
        xh = torch.empty_like(x); xl = torch.empty_like(x)
        flops = 2.0 * N * D * Ho * Wo * Cout * Cin * k * k * kd

        def simt():
            check(L.nrgbd_conv_nhwc(ptr(x), N, D, H, W, convops.pad4(Cin), Cs, ptr(wp), None, Cout, convops.pad4(Cout), kd, k, k, s, p, d,
                                    ptr(y), Ho, Wo, Cso, 0, 0, ctypes.c_void_p(stats.data_ptr()), st()))

        def split():
            check(L.nrgbd_split_tf32(ptr(x), x.numel(), ptr(xh), ptr(xl), st()))

        def tc():
            check(L.nrgbd_conv_nhwc_tc(ptr(xh), ptr(xl), N, D, H, W, Cs, Cs, ptr(wh), ptr(wl), None, Cout, convops.pad_to(Cout, 16), kd, k, k,
                                       s, p, d, ptr(y2), Ho, Wo, Cso, 0, 0, ctypes.c_void_p(stats.data_ptr()), st()))
        def tc2():
            check(L.nrgbd_conv_nhwc_tc2(ptr(x), N, D, H, W, Cs, Cs, ptr(wh), ptr(wl), None, Cout, convops.pad_to(Cout, 16), kd, k, k,
                                        s, p, d, ptr(y3), Ho, Wo, Cso, 0, 0, ctypes.c_void_p(stats.data_ptr()), st()))
        y3 = torch.zeros_like(y)
        y4 = torch.zeros_like(y)
        wp2, cin_p2, cout_p2, bn2 = convops.pack_weight_h2(w)
        ph = torch.empty(x.shape, device=dev, dtype=torch.float16); pl = torch.empty_like(ph)

        def split_h2():
            check(L.nrgbd_split_f16_pair(ptr(x), x.numel(), ptr(ph), ptr(pl), st()))

        def h2():
            check(L.nrgbd_conv_nhwc_h2(ptr(ph), ptr(pl), N, D, H, W, cin_p2, Cs, ptr(wp2), None, Cout, cout_p2, bn2, kd, k, k, s, p, d,
                                       ptr(y4), Ho, Wo, Cso, 0, 0, ctypes.c_void_p(stats.data_ptr()), st()))
        quick = 'quick' in sys.argv
        def safe(fn, iters=10):
            try:
                return timeit(fn, iters)
            except _lib.NrgbdError:
                return float('nan')
        if 'abflags' in sys.argv:
            arms = (0, 8, 32, 40)
            rounds = int(next((a[7:] for a in sys.argv if a.startswith('rounds=')), 5))
            ts = {a: [] for a in arms}
            for _ in range(rounds):
                for a in arms:
                    L.nrgbd_dev_conv_h2_set_flags(a)
                    ts[a].append(timeit(h2, 5))
            L.nrgbd_dev_conv_h2_set_flags(0)
            med = {a: float(np.median(v)) for a, v in ts.items()}
            rec = dict(layer=name, gflop=flops / 1e9, us={str(a): med[a] for a in arms},
                       tflops={str(a): flops / med[a] / 1e6 for a in arms},
                       spread={str(a): float((max(v) - min(v)) / np.median(v)) for a, v in ts.items()},
                       gain_vs_off={str(a): med[a] / med[0] - 1.0 for a in arms[1:]})
            out.append(rec)
            print(json.dumps(rec), flush=True)
            continue
        if 'h2only' in sys.argv:
            t_h2 = safe(h2)
            print(json.dumps(dict(layer=name, h2_us=t_h2, h2_tflops=flops / t_h2 / 1e6)), flush=True)
            continue
        t_simt = safe(simt, 3 if quick else 10); t_split = safe(split); t_tc = safe(tc, 3 if quick else 10); t_tc2 = safe(tc2)
        t_split_h2 = safe(split_h2); t_h2 = safe(h2)
        err = float((y - y2).abs().max() / y.abs().max())
        rec = dict(layer=name, gflop=flops / 1e9, simt_us=t_simt, simt_tflops=flops / t_simt / 1e6, split_us=t_split, tc_us=t_tc,
                   tc_tflops=flops / t_tc / 1e6, tc_vs_simt_relerr=err, tc2_us=t_tc2,
                   tc2_tflops=flops / t_tc2 / 1e6, tc2_vs_simt_relerr=float((y - y3).abs().max() / y.abs().max()),
                   h2_us=t_h2, h2_split_us=t_split_h2, h2_tflops=flops / t_h2 / 1e6,
                   h2_vs_simt_relerr=float((y - y4).abs().max() / y.abs().max()))
        out.append(rec)
        print(json.dumps(rec), flush=True)
    if 'abflags' in sys.argv:
        path = next((a[4:] for a in sys.argv[1:] if a.startswith('out=')), 'bench_conv_ab.json')
        with open(path, 'w') as f:
            json.dump(out, f, indent=1)
        return
    os.makedirs('gpurun_out', exist_ok=True)
    json.dump(out, open('gpurun_out/bench_conv.json', 'w'), indent=1)


if __name__ == '__main__':
    main()
