"""Golden fixtures of conv_math='f16' (single fp16 products): the UNMODIFIED reference with its convolutions' operands rounded.

Run in the build container only (needs /root/reference; CPU torch, the 4-line .cuda() shim of SURVEY 8c):
    python tests/golden/make_golden_f16.py

For every case of tests/cases_f16.py the reference's own test() (test_utils/test_KVNet.py:19-67) runs three times:
  - 'f16':  forward pre-hooks on every Conv2d / Conv3d / ConvTranspose2d the engine runs on tensor cores (all but the
            3-input-channel first layer) replace the input and the weight by x.half().float() for that call;
  - 'tf32': the same hooks with a 10-bit round-to-nearest significand (the reference's default GPU arithmetic, cuDNN TF32);
  - 'fp32': no hooks.
Stored ('f16/<case>/step<k>/<arith>/...', arith f16 and fp32): strided samples (SUB_LIMIT values) of the outputs the step
adds, full-array statistics of all four outputs and a strided expected depth; 'f16/hooked_layers' lists the hooked weights.
PINNING_f16.json holds, per step and output, on full arrays:
  - 'oracle_vs_f16': tests/oracle_f16.py (numpy, the same rounding) against the f16-emulated reference - the floor F;
  - 'f16_vs_fp32', 'tf32_vs_fp32': the emulated references against the plain one;
as probability, log-DPV, expected depth (mm) and argmax-flip deviations (cases_f16.deviations). Free-running steps feed
each arithmetic its own propagated prior, and the oracle the f16-emulated reference's prior of that step.
The npz is written with fixed member timestamps and no timings go to the JSON, so a re-run rewrites both byte for byte.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_eval as GE                        # noqa: E402  (the .cuda() shim, the reference on sys.path)
from make_golden_twin import save_npz                # noqa: E402

import models.KVNET as m_kvnet                       # noqa: E402  (reference)
import mutils.misc as m_misc                         # noqa: E402  (reference)

from oracle import planesweep_oracle as O            # noqa: E402
from tests import cases                              # noqa: E402
from tests import cases_f16 as CF                    # noqa: E402
from tests import oracle_f16 as OF                   # noqa: E402

T = torch.from_numpy
ROUND = {'f16': lambda t: t.half().float(),
         'tf32': lambda t: T(CF.round_tf32(t.detach().numpy())),
         'fp32': None}


def hook(model, rnd):
    """Rounds the operands of every tensor-core convolution of `model`; returns (handles, hooked weight names)."""
    handles, names = [], []
    for n, m in model.named_modules():
        if isinstance(m, (torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.ConvTranspose2d)) and m.in_channels != 3:
            names.append(n + '.weight')

            def pre(mod, inp):
                mod._w_full = mod.weight.data
                mod.weight.data = rnd(mod._w_full)
                return (rnd(inp[0]),) + tuple(inp[1:])

            def post(mod, inp, out):
                mod.weight.data = mod._w_full

            handles += [m.register_forward_pre_hook(pre), m.register_forward_hook(post)]
    return handles, sorted(names)


def run(c, camt, arith):
    """The case's steps in one arithmetic -> (per-step (inputs, prior, full outputs), hooked names)."""
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=camt, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                              d_upsample_ratio_KV_net=None, t_win_r=c['t_win_r'], if_refined=True)
    model.load_state_dict({k: T(v) for k, v in CF.state_dict(c).items()}, strict=True)
    model.train(CF.MODE[c['name']] == 'train')
    handles, names = hook(model, ROUND[arith]) if ROUND[arith] else ([], [])
    rec_model = GE.Recorder(torch.nn.DataParallel(model))      # DataParallel as test_KVNet.py:163 (no GPUs: falls through)
    steps, prior = [], None
    for k in range(c['n_steps']):
        if k and c['name'] not in CF.FREE_RUNNING:
            prior = CF.reseed_prior(c['name'], k)
        inputs, full, nxt = GE.step(rec_model, c, camt, c['t_win_r'] + k, prior if k else None)
        steps.append((inputs, prior if k else None, full))
        prior = nxt
    for h in handles:
        h.remove()
    return steps, names


def main():
    out, pin = {}, {'torch': torch.__version__, 'numpy': np.__version__, 'threads': torch.get_num_threads(), 'cases': {}}
    for name in CF.F16_CASES:
        c = CF.f16_case(name)
        cam = CF.cam(O.make_cam_intrinsics, c)
        camt = GE.cam_torch(cam)
        res = {}
        for arith in ('f16', 'tf32', 'fp32'):
            res[arith], names = run(c, camt, arith)
            if arith == 'f16':
                out['f16/hooked_layers'] = np.array(names)
        sd = CF.state_dict(c)
        for k in range(c['n_steps']):
            kk = 'f16/%s/step%d' % (name, k)
            for arith in ('f16', 'fp32'):
                full = res[arith][k][2]
                for nm, a in zip(CF.NAMES4, full):
                    if nm in CF.STORED[k == 0]:
                        out['%s/%s/%s' % (kk, arith, nm)] = cases.subsample_to(a, CF.SUB_LIMIT)
                    out['%s/%s/%s_stats' % (kk, arith, nm)] = cases.stats(np.exp(a.astype(np.float64)))
                dep = m_misc.depth_val_regression(T(full[3]), c['d'], BV_log=True).numpy()
                out['%s/%s/depth' % (kk, arith)] = cases.subsample_to(dep, CF.DEPTH_LIMIT)
            (ref_f, src_f, poses), prior, full16 = res['f16'][k]
            o = OF.kvnet_forward(sd, ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=prior,
                                 training=CF.MODE[name] == 'train')
            rec = {'oracle_vs_f16': {nm: CF.deviations(b, a, c['d']) for nm, a, b in zip(CF.NAMES4, full16, o)}}
            for arith in ('f16', 'tf32'):
                rec[arith + '_vs_fp32'] = {nm: CF.deviations(a, b, c['d'])
                                           for nm, a, b in zip(CF.NAMES4, res[arith][k][2], res['fp32'][k][2])}
            pin['cases'][kk] = rec
            print(kk, json.dumps(rec), flush=True)
    npz = os.path.join(HERE, 'f16_outputs.npz')
    save_npz(npz, out)
    with open(os.path.join(HERE, 'PINNING_f16.json'), 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote f16_outputs.npz %.2f MB' % (os.path.getsize(npz) / 1e6))


if __name__ == '__main__':
    main()
