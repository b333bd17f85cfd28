"""Golden fixtures of KVNET in .eval() (running-statistics BatchNorm), from the UNMODIFIED reference.

Run in the build container only (needs /root/reference; CPU torch, the 4-line .cuda() shim of SURVEY 8c):
    python tests/golden/make_golden_eval.py [case ...]

Running statistics. He-init buffers (mean 0, var 1) would leave eval mode almost untested, so every case first warms
the reference's own buffers: all 13 tracked BatchNorm layers are reset and switched to momentum=None (cumulative
average), the reference's test() (test_utils/test_KVNet.py:19-67) is run in train mode over WARM_STEPS steps of a
DIFFERENT seeded video (the first step updates the feature CNN's downsample layers only, the steady steps K-Net as
well), then momentum=0.1 is restored and the model is put in .eval(). The warmed buffers are stored in the fixture
('<key>/rs/<state_dict name>'); the tests load them into the engine's model.

Cases, all driven through the reference's own test() (inputs regenerated from tests/cases.py seeds):
  - kvnet_256_d16: first window + 2 steady K-Net steps;
  - c23_640x480_d64_v4_stream30 (C2/C3): first window + 1 steady step.
Every steady step is re-seeded with the reference's TRAIN-mode prior of the step before, which the repository already holds
in full (reference_outputs.npz, configs_priors_<case>.npz): any valid prior serves as the K-Net input, and no prior has to
be stored again. Stored per step: strided samples (SUB_LIMIT values per array) of the outputs that step adds - the first
window's BV_cur and refined DPV (its filtered outputs are the same arrays), a steady step's filtered DPV and its refinement -
plus full-array statistics of all four outputs and a strided expected depth.
The eval oracle (tests/oracle_eval.py), fed the same priors, is compared with the reference; the deviations go to
PINNING_eval.json (the fp32-vs-fp32 floor the GPU gates are set against). The script also checks that the
reference's state_dict is unchanged by the eval forwards.
"""
import contextlib
import io
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, '/root/reference/code')
warnings.filterwarnings('ignore')

torch.Tensor.cuda = lambda s, *a, **k: s
torch.nn.Module.cuda = lambda s, *a, **k: s
torch.cuda.current_device = lambda: 0
torch.Tensor.get_device = lambda s: 0

import models.KVNET as m_kvnet                       # noqa: E402  (reference)
import test_utils.test_KVNet as ref_test             # noqa: E402  (reference)
import mutils.misc as m_misc                         # noqa: E402  (reference)

from neuralrgbd_b200 import synth                    # noqa: E402
from oracle import planesweep_oracle as O            # noqa: E402
from tests import cases                              # noqa: E402
from tests import oracle_eval as E                   # noqa: E402

T = torch.from_numpy
NAMES4 = ['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV']
WARM_STEPS = 4          # 1 first window + 3 steady steps
WARM_SEED = 1000        # the warm-up video is seeded apart from every test video
SUB_LIMIT = 8000        # values per stored output array (strided, see cases.subsample_to)
DEPTH_LIMIT = 2000
STORED = {True: ('BV_cur', 'dmap_cur_refined'), False: ('DPV', 'dmap_refined')}    # first window: / steady step:


def sub(a):
    return cases.subsample_to(a, SUB_LIMIT)


def reseed_prior(name, step):
    """The reference's train-mode prior after `step` - 1, as committed by make_golden.py / make_golden_configs.py."""
    if name in cases.KVNET_CASES:
        return np.load(os.path.join(HERE, 'reference_outputs.npz'))['kvnet/%s/step%d/BV_predict_next_full' % (name, step - 1)]
    assert step == 1
    return np.load(os.path.join(HERE, 'configs_priors_%s.npz' % name))['cfg/%s/step0/BV_predict_next_full' % name]


def case(name):
    if name in cases.KVNET_CASES:
        c = cases.kvnet_case(name)
        c['n_steps'] = 3
        c['cam'] = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
        return c
    c = cases.big_case(name)
    c['cam'] = cases.big_cam(O.make_cam_intrinsics, c)
    c['n_steps'] = 2
    return c


def warm_case(c):
    """The same camera / planes / weights on a different seeded video."""
    w = dict(c)
    nf = WARM_STEPS + 2 * c['t_win_r']
    w['frames'], rng = synth.video(WARM_SEED + c['H'] + c['W'], nf, c['H'], c['W'])
    w['exts'] = synth.camera_track(rng, nf)
    return w


def cam_torch(cam):
    c = dict(cam)
    c['unit_ray_array_2D'] = T(cam['unit_ray_array_2D'])
    c['intrinsic_M_cuda'] = T(cam['intrinsic_M_cuda'])
    return c


def dev(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.nanmax(np.abs(a - b))) if a.size else 0.0


class Recorder(torch.nn.Module):
    """Passes the call through to the reference model and keeps what it returned."""

    def __init__(self, model):
        super().__init__()
        self.model = model
        self.last = None

    def forward(self, **kw):
        self.last = self.model(**kw)
        return self.last


def step(rec_model, c, camt, idx, prior):
    ref_f, src_f, poses = cases.window(c, idx)
    Ref_Dats = [{'img': T(ref_f)}]
    Src_Dats = [[{'img': T(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
    _, bv_next = ref_test.test(rec_model, c['d'], [camt], c['t_win_r'], Ref_Dats, Src_Dats, T(poses),
                               None if prior is None else T(prior), R_net=False)
    return (ref_f, src_f, poses), [a.numpy() for a in rec_model.last], bv_next.numpy()


def tracked_bns(model):
    return [m for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm) and m.track_running_stats]


def run_case(name):
    c = case(name)
    cam = c['cam']; camt = cam_torch(cam)
    r = c['t_win_r']
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=camt, d_candi=c['d'], sigma_soft_max=c['sigma'],
                              KVNet_feature_dim=64, d_upsample_ratio_KV_net=None, t_win_r=r, if_refined=True)
    model.load_state_dict({k: T(np.asarray(v)) for k, v in c['sd'].items()})
    rec_model = Recorder(torch.nn.DataParallel(model))      # DataParallel as test_KVNet.py:163 (no GPUs: falls through)
    key = 'eval/%s' % name
    out, pin = {}, {}

    # ---- warm the running statistics (train mode, cumulative average) --------------------------------------------
    bns = tracked_bns(model)
    assert len(bns) == 13, len(bns)
    for m in bns:
        m.reset_running_stats()
        m.momentum = None
    model.train()
    w = warm_case(c)
    prior = None
    for k in range(WARM_STEPS):
        _, _, prior = step(rec_model, w, camt, r + k, prior)
    for m in bns:
        m.momentum = 0.1
    model.eval()
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        if k.endswith(('running_mean', 'running_var', 'num_batches_tracked')):
            out['%s/rs/%s' % (key, k)] = v.numpy()
    sd_np = dict(c['sd'])
    sd_np.update({k: v.numpy() for k, v in sd.items() if k.endswith(('running_mean', 'running_var'))})

    # ---- eval-mode outputs ---------------------------------------------------------------------------------------
    for k in range(c['n_steps']):
        t0 = time.time()
        prior = reseed_prior(name, k) if k else None
        (ref_f, src_f, poses), full, _ = step(rec_model, c, camt, r + k, prior)
        kk = '%s/step%d' % (key, k)
        rec = {}
        if k == 0:
            assert np.array_equal(full[0], full[1]) and np.array_equal(full[2], full[3])     # KVNET.py:138-143
        for nm, a in zip(NAMES4, full):
            if nm in STORED[k == 0]:
                out['%s/%s' % (kk, nm)] = sub(a)
            out['%s/%s_stats' % (kk, nm)] = cases.stats(np.exp(a.astype(np.float64)))
        dep = m_misc.depth_val_regression(T(full[3]), c['d'], BV_log=True).numpy()
        out[kk + '/depth'] = cases.subsample_to(dep, DEPTH_LIMIT)
        rec['seconds_reference'] = time.time() - t0
        to = time.time()
        o = E.kvnet_forward(sd_np, ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=prior, training=False)
        for nm, a, b in zip(NAMES4, full, o):
            rec['oracle_' + nm + '_prob'] = dev(np.exp(a), np.exp(b))
            rec['oracle_' + nm + '_prob_sub'] = dev(np.exp(sub(a)), np.exp(sub(b)))
        rec['oracle_depth_mm'] = 1000 * dev(dep, O.depth_val_regression(o[3], c['d']))
        rec['seconds_oracle'] = time.time() - to
        pin[kk] = rec
        print(kk, json.dumps(rec), flush=True)
    after = model.state_dict()
    changed = [k for k in sd if not torch.equal(sd[k], after[k])]
    assert not changed, changed
    pin[key + '/state_dict_unchanged'] = True
    return out, pin


def main():
    names = sys.argv[1:] or ['kvnet_256_d16', 'c23_640x480_d64_v4_stream30']
    npz = os.path.join(HERE, 'eval_outputs.npz')
    path = os.path.join(HERE, 'PINNING_eval.json')
    pin = {'torch': torch.__version__, 'numpy': np.__version__, 'threads': torch.get_num_threads(), 'cases': {}}
    out = {}
    if os.path.exists(path):
        pin['cases'] = json.load(open(path)).get('cases', {})
    if os.path.exists(npz):
        out = dict(np.load(npz))
    for name in names:
        o, p = run_case(name)
        out = {k: v for k, v in out.items() if not k.startswith('eval/%s/' % name)}
        out.update(o)
        pin['cases'].update(p)
        np.savez_compressed(npz, **out)
        with open(path, 'w') as f:
            json.dump(pin, f, indent=1, sort_keys=True)
    print('wrote eval_outputs.npz %.2f MB' % (os.path.getsize(npz) / 1e6))


if __name__ == '__main__':
    main()
