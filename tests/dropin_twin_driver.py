"""The reference's OWN inference step (test_utils/test_KVNet.py:test of an unmodified checkout) on the engine at a temporal
window radius other than 2: install_as_reference_modules(), construct models.KVNET.KVNET(t_win_r=r) by keyword,
nn.DataParallel, .cuda(), load the case's weights, then stream the case's 3 frames (first window and two steady steps, each
steady step fed the reference's train-mode prior as tests/golden/make_golden_twin.py recorded it). Prints one JSON line with
the deviations of the filtered DPV from the fixtures. Run as a subprocess by tests/test_gpu_twin.py (keeps the reference's
top-level module names out of the test process).
usage: dropin_twin_driver.py REF_CODE CASE"""
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
    ref_code, name = sys.argv[1], sys.argv[2]
    import neuralrgbd_b200
    neuralrgbd_b200.install_as_reference_modules(ref_code)
    import models.KVNET as m_kvnet                     # reference module; KVNET re-pointed to the engine-backed class
    import test_utils.test_KVNet as ref_step           # the reference's file, unmodified
    from oracle import planesweep_oracle as O
    from tests import cases, cases_twin as CT
    assert ref_step.__file__.startswith(os.path.abspath(ref_code)), ref_step.__file__
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'twin_outputs.npz'))
    c = CT.twin_case(name)
    r = c['t_win_r']
    cam = CT.twin_cam(O.make_cam_intrinsics, c)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']),
               intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'],
                              KVNet_feature_dim=64, d_upsample_ratio_KV_net=None, t_win_r=r, if_refined=True)
    model = torch.nn.DataParallel(model)
    model.cuda()
    model.module.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in c['sd'].items()}, strict=True)
    out = {'class': type(model.module).__module__, 't_win_r': r, 'steps': []}
    for step in range(c['n_steps']):
        bv = torch.from_numpy(CT.prior(name, step)).cuda() if step else None
        ref_f, src_f, poses = cases.window(c, r + step)
        Ref_Dats = [{'img': torch.from_numpy(ref_f)}]
        Src_Dats = [[{'img': torch.from_numpy(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
        kv, bv_next = ref_step.test(model, c['d'], [cam], r, Ref_Dats, Src_Dats, torch.from_numpy(poses).cuda(), bv, R_net=False)
        key = 'twin/train/%s/step%d/%s' % (name, step, 'DPV' if step else 'BV_cur')     # first window: DPV is BV_cur
        out['steps'].append({'DPV': float(np.abs(np.exp(cases.subsample_to(kv.cpu().numpy(), 8000)) - np.exp(gold[key])).max()),
                             'V': int(src_f.shape[1]), 'prior_finite': bool(torch.isfinite(bv_next).all())})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
