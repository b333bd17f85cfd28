"""The reference's OWN inference step (test_utils/test_KVNet.py:test of an unmodified checkout) on the engine with
conv_math='f16': install_as_reference_modules(), construct models.KVNET.KVNET(t_win_r=1) by keyword, nn.DataParallel, .cuda(),
load the weights of tests/cases_f16.py's r1_256_d16, set conv_math on the module, then run its first window and its
re-seeded steady step. Prints one JSON line with the deviations of the filtered DPV from the f16-emulated reference
(tests/golden/make_golden_f16.py). Run as a subprocess by tests/test_gpu_f16.py (keeps the reference's top-level module
names out of the test process).
usage: dropin_f16_driver.py REF_CODE"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ref_code = sys.argv[1]
    import neuralrgbd_b200
    neuralrgbd_b200.install_as_reference_modules(ref_code)
    import models.KVNET as m_kvnet                     # reference module; KVNET re-pointed to the engine-backed class
    import test_utils.test_KVNet as ref_step           # the reference's file, unmodified
    from oracle import planesweep_oracle as O
    from tests import cases, cases_f16 as CF
    assert ref_step.__file__.startswith(os.path.abspath(ref_code)), ref_step.__file__
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'f16_outputs.npz'))
    name = 'r1_256_d16'
    c = CF.f16_case(name)
    r = c['t_win_r']
    cam = CF.cam(O.make_cam_intrinsics, c)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']),
               intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'],
                              KVNet_feature_dim=64, d_upsample_ratio_KV_net=None, t_win_r=r, if_refined=True)
    model = torch.nn.DataParallel(model)
    model.cuda()
    model.module.load_state_dict({k: torch.from_numpy(v) for k, v in CF.state_dict(c).items()}, strict=True)
    model.module.conv_math = 'f16'
    out = {'class': type(model.module).__module__, 'conv_math': model.module.conv_math, 'steps': []}
    for step in range(c['n_steps']):
        bv = torch.from_numpy(CF.reseed_prior(name, step)).cuda() if step else None
        ref_f, src_f, poses = cases.window(c, r + step)
        Ref_Dats = [{'img': torch.from_numpy(ref_f)}]
        Src_Dats = [[{'img': torch.from_numpy(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
        kv, bv_next = ref_step.test(model, c['d'], [cam], r, Ref_Dats, Src_Dats, torch.from_numpy(poses).cuda(), bv, R_net=False)
        key = 'f16/%s/step%d/f16/%s' % (name, step, 'DPV' if step else 'BV_cur')     # first window: DPV is BV_cur
        out['steps'].append({'DPV': float(np.abs(np.exp(cases.subsample_to(kv.cpu().numpy(), CF.SUB_LIMIT)) - np.exp(gold[key])).max()),
                             'prior_finite': bool(torch.isfinite(bv_next).all())})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
