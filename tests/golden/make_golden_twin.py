"""Golden fixtures of KVNET at temporal window radii 1 and 3 (V = 2 and 6 source views), from the UNMODIFIED reference.

Run in the build container only (needs /root/reference; CPU torch, the 4-line .cuda() shim of SURVEY 8c):
    python tests/golden/make_golden_twin.py

Cases (tests/cases_twin.py; frames, poses and weights from synth / arch.synth_state_dict(..., t_win_r=r)), all driven
through the reference's own test() (test_utils/test_KVNet.py:19-67):
  - r1_256_d16, r3_256_d16: 256x256, D = 16, first window + 2 steady steps, in train mode and in .eval();
  - r1_640x480_d64: 640x480, D = 64, first window + 1 steady step, train mode.
Every steady step is re-seeded with a train-mode prior of the reference that the repository already holds
(cases_twin.prior). Eval mode first warms the reference's running statistics with make_golden_eval.py's recipe (cumulative
average over train-mode steps of a differently seeded video) and stores them ('twin/eval/<case>/rs/<state_dict name>').
Stored per step, as make_golden_eval.py does: strided samples (SUB_LIMIT values) of the outputs that step adds,
full-array statistics of all four outputs and a strided expected depth. Also stored: the reference's state_dict (key,
shape) list of KVNET(t_win_r=r) for r = 1..4 ('twin/sd/r<r>/...').
The deviations of the numpy oracle (tests/oracle_eval.py, train or eval mode) from the reference go to PINNING_twin.json.
The npz is written with fixed member timestamps and no timings go to the JSON, so a re-run rewrites both byte for byte.
"""
import contextlib
import io
import json
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_eval as GE                        # noqa: E402  (the .cuda() shim, the reference on sys.path, warm-up recipe)

import models.KVNET as m_kvnet                       # noqa: E402  (reference)
import mutils.misc as m_misc                         # noqa: E402  (reference)

from oracle import planesweep_oracle as O            # noqa: E402
from tests import cases                              # noqa: E402
from tests import cases_twin as CT                   # noqa: E402
from tests import oracle_eval as E                   # noqa: E402

T = torch.from_numpy


def save_npz(path, arrays):
    """np.savez_compressed with a fixed member order and timestamp."""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def build(c, camt, r):
    with contextlib.redirect_stdout(io.StringIO()):
        return m_kvnet.KVNET(feature_dim=64, cam_intrinsics=camt, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                             d_upsample_ratio_KV_net=None, t_win_r=r, if_refined=True)


def state_dict_lists():
    c = CT.twin_case('r1_256_d16')
    camt = GE.cam_torch(CT.twin_cam(O.make_cam_intrinsics, c))
    out = {}
    for r in (1, 2, 3, 4):
        sd = build(c, camt, r).state_dict()
        out['twin/sd/r%d/keys' % r] = np.array(list(sd.keys()))
        out['twin/sd/r%d/shapes' % r] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
    return out


def record(rec_model, c, camt, cam, name, mode, sd_np, out, pin):
    """The case's steps through the reference's test() in the model's current mode; stores outputs, pins the oracle."""
    for k in range(c['n_steps']):
        prior = CT.prior(name, k) if k else None
        (ref_f, src_f, poses), full, _ = GE.step(rec_model, c, camt, c['t_win_r'] + k, prior)
        kk = 'twin/%s/%s/step%d' % (mode, name, k)
        if k == 0:
            assert np.array_equal(full[0], full[1]) and np.array_equal(full[2], full[3])     # KVNET.py:138-143
        for nm, a in zip(GE.NAMES4, full):
            if nm in GE.STORED[k == 0]:
                out['%s/%s' % (kk, nm)] = GE.sub(a)
            out['%s/%s_stats' % (kk, nm)] = cases.stats(np.exp(a.astype(np.float64)))
        dep = m_misc.depth_val_regression(T(full[3]), c['d'], BV_log=True).numpy()
        out[kk + '/depth'] = cases.subsample_to(dep, GE.DEPTH_LIMIT)
        o = E.kvnet_forward(sd_np, ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=prior, training=mode == 'train')
        rec = {}
        for nm, a, b in zip(GE.NAMES4, full, o):
            rec['oracle_' + nm + '_prob'] = GE.dev(np.exp(a), np.exp(b))
            rec['oracle_' + nm + '_prob_sub'] = GE.dev(np.exp(GE.sub(a)), np.exp(GE.sub(b)))
        rec['oracle_depth_mm'] = 1000 * GE.dev(dep, O.depth_val_regression(o[3], c['d']))
        pin[kk] = rec
        print(kk, json.dumps(rec), flush=True)


def run_case(name):
    c = CT.twin_case(name)
    cam = CT.twin_cam(O.make_cam_intrinsics, c)
    camt = GE.cam_torch(cam)
    model = build(c, camt, c['t_win_r'])
    model.load_state_dict({k: T(np.asarray(v)) for k, v in c['sd'].items()}, strict=True)
    rec_model = GE.Recorder(torch.nn.DataParallel(model))      # DataParallel as test_KVNet.py:163 (no GPUs: falls through)
    out, pin = {}, {}
    model.train()
    record(rec_model, c, camt, cam, name, 'train', {k: np.asarray(v) for k, v in c['sd'].items()}, out, pin)
    if name not in CT.EVAL_CASES:
        return out, pin
    # ---- make_golden_eval.py's warm-up of the running statistics, then .eval() -------------------------------------
    bns = GE.tracked_bns(model)
    assert len(bns) == 13, len(bns)
    for m in bns:
        m.reset_running_stats()
        m.momentum = None
    w = GE.warm_case(c)
    prior = None
    for k in range(GE.WARM_STEPS):
        _, _, prior = GE.step(rec_model, w, camt, c['t_win_r'] + k, prior)
    for m in bns:
        m.momentum = 0.1
    model.eval()
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        if k.endswith(('running_mean', 'running_var', 'num_batches_tracked')):
            out['twin/eval/%s/rs/%s' % (name, k)] = v.numpy()
    sd_np = {k: np.asarray(v) for k, v in c['sd'].items()}
    sd_np.update({k: v.numpy() for k, v in sd.items() if k.endswith(('running_mean', 'running_var'))})
    record(rec_model, c, camt, cam, name, 'eval', sd_np, out, pin)
    after = model.state_dict()
    assert all(torch.equal(sd[k], after[k]) for k in sd)
    return out, pin


def main():
    out = state_dict_lists()
    pin = {'torch': torch.__version__, 'numpy': np.__version__, 'threads': torch.get_num_threads(), 'cases': {}}
    for name in CT.TWIN_CASES:
        o, p = run_case(name)
        out.update(o)
        pin['cases'].update(p)
    npz = os.path.join(HERE, 'twin_outputs.npz')
    save_npz(npz, out)
    with open(os.path.join(HERE, 'PINNING_twin.json'), 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote twin_outputs.npz %.2f MB' % (os.path.getsize(npz) / 1e6))


if __name__ == '__main__':
    main()
