"""Golden fixtures of KVNET's other refinement configurations, from the UNMODIFIED reference.

Run in the build container only (needs /root/reference; CPU torch, the 4-line .cuda() shim of SURVEY 8c):
    python tests/golden/make_golden_refine.py [case ...]

Configurations: refineNet_name='DGF' (guided-filter depth refinement, models/Refine.py:583-641), if_refined=False, and the
depth-upsampled DPV R-Net (refineNet_name='DPV', if_upsample_d=True, Refine.py:44-48: refined DPVs of 4D planes).
  - state_dict: the reference's (key, shape) list of every configuration, including the default and the depth-upsampled DPV
    R-Net ('refine/sd/<config>'), so the mirror's module tree can be checked without the reference.
  - guided filter alone: RefineNet_DGF.forward on seeded inputs (tests/oracle_refine.py:gf_case) - ragged sizes, a textured
    guide, a guide that is flat over whole regions - stored in full ('refine/gf/<case>').
  - KVNET through the reference's own test() (train mode, as make_golden.py): kvnet_256_d16, first window + 2 steady steps;
    c23_640x480_d64_v4_stream30, first window + 1 steady step. Every steady step is re-seeded with the reference's prior of
    the step before that the repository already holds (reference_outputs.npz, configs_priors_<case>.npz), as
    make_golden_eval.py does. The shared weights are the case's; the DGF weights come from
    arch.synth_state_dict(..., refine='DGF') / (..., upsample_d=True). Stored per step: strided samples (SUB_LIMIT values) of
    the low-resolution DPV (once: it does not depend on the
    refinement), of the DGF depth maps and of the 4D-plane refined DPVs, plus full-array statistics, and the
    expected depth of the refined DPV over the loaders' dup4_candi (np.linspace(d.min(), d.max(), 4D), scanNet.py:327).
The deviations of tests/oracle_refine.py from the reference go to PINNING_refine.json:
  - oracle_dgf_m: the oracle's guided filter fed the reference's own low-resolution DPV (the filter alone);
  - oracle_fwd_dgf_m: the oracle's guided filter fed the numpy oracle's forward (tests/oracle_eval.py, train mode), i.e.
    the fp32-vs-fp32 deviation a faithful DPV carries into the ill-conditioned filter. The GPU gates are multiples of it;
  - oracle_up_prob / oracle_up_depth_mm: the numpy oracle's forward (whose R-Net takes its widths from the weights) against
    the reference's 4D-plane refined DPV, in probability and in expected depth over dup4_candi.
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
import models.Refine as m_refine                     # noqa: E402  (reference)
import test_utils.test_KVNet as ref_test             # noqa: E402  (reference)

from neuralrgbd_b200 import arch                     # noqa: E402
from oracle import planesweep_oracle as O            # noqa: E402
from tests import cases                              # noqa: E402
from tests import oracle_eval as E                   # noqa: E402
from tests import oracle_refine as R                 # noqa: E402

T = torch.from_numpy
SUB_LIMIT = 8000
CONFIGS = {'none': dict(if_refined=False), 'DGF': dict(if_refined=True, refineNet_name='DGF'),
           'DPV_up': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True)}
SD_CONFIGS = {'DPV': dict(if_refined=True, refineNet_name='DPV'), 'DPV_upsample_d': dict(if_refined=True, refineNet_name='DPV',
                                                                                       if_upsample_d=True),
              'DGF': dict(if_refined=True, refineNet_name='DGF'), 'none': dict(if_refined=False),
              'none_DGF': dict(if_refined=False, refineNet_name='DGF')}
STEPS = {'kvnet_256_d16': 3, 'c23_640x480_d64_v4_stream30': 2}


def sub(a):
    return cases.subsample_to(a, SUB_LIMIT)


def dev(a, b):
    return float(np.max(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))))


def case(name):
    if name in cases.KVNET_CASES:
        c = cases.kvnet_case(name)
        c['cam'] = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
        c['wseed'] = 5
    else:
        c = cases.big_case(name)
        c['cam'] = cases.big_cam(O.make_cam_intrinsics, c)
        c['wseed'] = cases.BIG_CFG[name]['wseed']
    return c


def reseed_prior(name, step):
    if name in cases.KVNET_CASES:
        return np.load(os.path.join(HERE, 'reference_outputs.npz'))['kvnet/%s/step%d/BV_predict_next_full' % (name, step - 1)]
    assert step == 1
    return np.load(os.path.join(HERE, 'configs_priors_%s.npz' % name))['cfg/%s/step0/BV_predict_next_full' % name]


def cam_torch(cam):
    return dict(cam, unit_ray_array_2D=T(cam['unit_ray_array_2D']), intrinsic_M_cuda=T(cam['intrinsic_M_cuda']))


class Recorder(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model
        self.last = None

    def forward(self, **kw):
        self.last = self.model(**kw)
        return self.last


def build(c, camt, cfg):
    with contextlib.redirect_stdout(io.StringIO()):
        return m_kvnet.KVNET(feature_dim=64, cam_intrinsics=camt, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                             d_upsample_ratio_KV_net=None, t_win_r=c['t_win_r'], **cfg)


def state_dict_lists():
    c = cases.kvnet_case('kvnet_256_d16')
    camt = cam_torch(cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4))
    out = {}
    for nm, cfg in SD_CONFIGS.items():
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            m = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=camt, d_candi=c['d'], sigma_soft_max=10.0, KVNet_feature_dim=64,
                              d_upsample_ratio_KV_net=None, t_win_r=2, **cfg)
        sd = m.state_dict()
        out['refine/sd/%s/keys' % nm] = np.array(list(sd.keys()))
        out['refine/sd/%s/shapes' % nm] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
        out['refine/sd/%s/printed' % nm] = np.array([ln for ln in buf.getvalue().splitlines() if ln.startswith(('KV-Net', 'with R-net', '\trefinement'))])
    return out


def gf_cases():
    out, pin = {}, {}
    for name in R.GF_CASES:
        g = R.gf_case(name)
        net = m_refine.RefineNet_DGF(3)
        net.load_state_dict({k[len('r_net.'):]: T(v) for k, v in g['sd'].items()})
        with torch.no_grad():
            y = net(T(g['dmap'][None, None]), T(g['img'][None]))[0, 0].numpy()
        out['refine/gf/%s/out' % name] = y
        o = R.dgf_refine(g['dmap'], g['img'], g['sd'])
        pin['gf/%s' % name] = {'oracle_m': dev(o, y), 'oracle_bitexact': bool(np.array_equal(o, y))}
        print('gf', name, pin['gf/%s' % name], flush=True)
    return out, pin


def run_case(name):
    c = case(name)
    camt = cam_torch(c['cam'])
    sd_all = {k: np.asarray(v) for k, v in c['sd'].items() if not k.startswith('r_net.')}
    dgf_sd = {k: v for k, v in arch.synth_state_dict(c['wseed'], 64, c['D'], c['t_win_r'], 64, refine='DGF').items()
              if k.startswith('r_net.')}
    up_sd = {k: v for k, v in arch.synth_state_dict(c['wseed'], 64, c['D'], c['t_win_r'], 64, upsample_d=True).items()
             if k.startswith('r_net.')}
    dup4 = np.linspace(c['d'].min(), c['d'].max(), 4 * len(c['d']))
    out, pin = {}, {}
    for cfg_name, cfg in CONFIGS.items():
        model = build(c, camt, cfg)
        sd = dict(sd_all, **{'DGF': dgf_sd, 'DPV_up': up_sd}.get(cfg_name, {}))
        model.load_state_dict({k: T(v) for k, v in sd.items()}, strict=True)
        rec = Recorder(torch.nn.DataParallel(model))
        key = 'refine/%s/%s' % (cfg_name, name)
        for k in range(STEPS[name]):
            t0 = time.time()
            prior = reseed_prior(name, k) if k else None
            ref_f, src_f, poses = cases.window(c, c['t_win_r'] + k)
            Ref_Dats = [{'img': T(ref_f)}]
            Src_Dats = [[{'img': T(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
            ref_test.test(rec, c['d'], [camt], c['t_win_r'], Ref_Dats, Src_Dats, T(poses), None if prior is None else T(prior),
                          R_net=cfg_name != 'none')
            full = rec.last
            kk = '%s/step%d' % (key, k)
            row = {'seconds_reference': time.time() - t0}
            lowres = full[2] if k == 0 else full[3]
            if cfg_name == 'none':          # the low-resolution DPV does not depend on the refinement: stored once
                out[kk + '/DPV'] = sub(lowres.numpy())
                out[kk + '/DPV_stats'] = cases.stats(np.exp(lowres.numpy().astype(np.float64)))
            else:
                assert np.array_equal(sub(lowres.numpy()), out['refine/none/%s/step%d/DPV' % (name, k)])
            if cfg_name == 'none':
                assert full[0] == -1 and full[1] == -1
            elif cfg_name == 'DPV_up':
                ref = (full[0] if k == 0 else full[1]).numpy()
                assert ref.shape == (1, 4 * c['D'], c['H'], c['W']), ref.shape
                out[kk + '/dpv_up'] = sub(ref[0])
                out[kk + '/dpv_up_stats'] = cases.stats(np.exp(ref.astype(np.float64)))
                dep = O.depth_val_regression(ref, dup4)[0]
                out[kk + '/depth_dup4'] = sub(dep)
                t1 = time.time()
                fwd = E.kvnet_forward(sd, ref_f, src_f, poses, c['cam'], c['d'], c['sigma'], BV_predict=prior, training=True)
                of = fwd[0] if k == 0 else fwd[1]
                row['oracle_up_prob'] = dev(np.exp(of), np.exp(ref))
                row['oracle_up_prob_sub'] = dev(np.exp(sub(of[0])), np.exp(sub(ref[0])))
                row['oracle_up_depth_mm'] = 1000 * dev(O.depth_val_regression(of, dup4)[0], dep)
                row['seconds_oracle'] = time.time() - t1
            else:
                ref = (full[0] if k == 0 else full[1]).numpy()
                assert ref.shape == (1, 1, c['H'], c['W']), ref.shape
                out[kk + '/dmap'] = sub(ref[0, 0])
                out[kk + '/dmap_stats'] = cases.stats(ref[0, 0])
                if k:
                    out[kk + '/dmap_cur'] = sub(full[0].numpy()[0, 0])
                o = R.kvnet_dgf_output(lowres.numpy()[0], ref_f[0], c['d'], sd)
                row['oracle_dgf_m'] = dev(o, ref[0, 0])
                t1 = time.time()
                fwd = E.kvnet_forward(c['sd'], ref_f, src_f, poses, c['cam'], c['d'], c['sigma'], BV_predict=prior, training=True)
                of = R.kvnet_dgf_output(fwd[2 if k == 0 else 3][0], ref_f[0], c['d'], sd)
                row['oracle_fwd_dgf_m'] = dev(of, ref[0, 0])
                row['oracle_fwd_dgf_m_sub'] = dev(sub(of), sub(ref[0, 0]))
                row['seconds_oracle'] = time.time() - t1
            pin[kk] = row
            print(kk, json.dumps(row), flush=True)
    return out, pin


def main():
    names = sys.argv[1:] or ['kvnet_256_d16', 'c23_640x480_d64_v4_stream30']
    npz = os.path.join(HERE, 'refine_outputs.npz')
    path = os.path.join(HERE, 'PINNING_refine.json')
    pin = {'torch': torch.__version__, 'numpy': np.__version__, 'threads': torch.get_num_threads(), 'cases': {}}
    out = {}
    if os.path.exists(path):
        pin['cases'] = json.load(open(path)).get('cases', {})
    if os.path.exists(npz):
        out = dict(np.load(npz))
    out.update(state_dict_lists())
    o, p = gf_cases()
    out.update(o); pin['cases'].update(p)
    for name in names:
        o, p = run_case(name)
        out = {k: v for k, v in out.items() if not any(k.startswith('refine/%s/%s/' % (cf, name)) for cf in CONFIGS)}
        out.update(o)
        pin['cases'].update(p)
        np.savez_compressed(npz, **out)
        with open(path, 'w') as f:
            json.dump(pin, f, indent=1, sort_keys=True)
    np.savez_compressed(npz, **out)
    with open(path, 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=True)
    print('wrote refine_outputs.npz %.2f MB' % (os.path.getsize(npz) / 1e6))


if __name__ == '__main__':
    main()
