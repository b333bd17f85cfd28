"""The reference's OWN inference step (test_utils/test_KVNet.py:test of an unmodified checkout) on the engine with
refineNet_name='DGF' (R_net=True: test() returns the refined depth map), the depth-upsampled DPV R-Net (if_upsample_d=True,
R_net=True: the refined log-DPV of 4D planes) or if_refined=False (R_net=False: the filtered DPV):
install_as_reference_modules(), construct models.KVNET.KVNET by keyword, nn.DataParallel, .cuda(), load the case's weights,
then run the first window and two steady steps re-seeded with the reference's priors, as tests/golden/make_golden_refine.py
recorded them. Prints one JSON line with the deviations from refine_outputs.npz. Run as a subprocess by tests/test_gpu_refine.py.
    python tests/dropin_refine_driver.py REF_CODE DGF|DPV_up|none [eval]"""
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
    ref_code, cfg = sys.argv[1], sys.argv[2]
    name = 'kvnet_256_d16'
    import neuralrgbd_b200
    neuralrgbd_b200.install_as_reference_modules(ref_code)
    import models.KVNET as m_kvnet                     # reference module; KVNET re-pointed to the engine-backed class
    import test_utils.test_KVNet as ref_step           # the reference's file, unmodified
    from neuralrgbd_b200 import arch
    from oracle import planesweep_oracle as O
    from tests import cases
    assert ref_step.__file__.startswith(os.path.abspath(ref_code)), ref_step.__file__
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'refine_outputs.npz'))
    ref_gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_outputs.npz'))
    c = cases.kvnet_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']),
               intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    kw = {'DGF': dict(if_refined=True, refineNet_name='DGF'), 'none': dict(if_refined=False),
          'DPV_up': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True)}[cfg]
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'],
                              KVNet_feature_dim=64, d_upsample_ratio_KV_net=None, t_win_r=2, **kw)
    model = torch.nn.DataParallel(model)
    model.cuda()
    sd = {k: v for k, v in c['sd'].items() if not k.startswith('r_net.')}
    if cfg != 'none':
        rn = arch.synth_state_dict(5, 64, c['D'], 2, 64, refine='DGF' if cfg == 'DGF' else 'DPV', upsample_d=cfg == 'DPV_up')
        sd.update({k: v for k, v in rn.items() if k.startswith('r_net.')})
    model.module.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    if len(sys.argv) > 3 and sys.argv[3] == 'eval':
        model.eval()
    out = {'class': type(model.module).__module__, 'steps': []}
    for step in range(3):
        bv = torch.from_numpy(ref_gold['kvnet/%s/step%d/BV_predict_next_full' % (name, step - 1)]).cuda() if step else None
        ref_f, src_f, poses = cases.window(c, 2 + step)
        Ref_Dats = [{'img': torch.from_numpy(ref_f)}]
        Src_Dats = [[{'img': torch.from_numpy(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
        res, bv_next = ref_step.test(model, c['d'], [cam], 2, Ref_Dats, Src_Dats, torch.from_numpy(poses).cuda(), bv,
                                     R_net=cfg != 'none')
        key = 'refine/%s/%s/step%d' % (cfg, name, step)
        row = {'shape': list(res.shape), 'finite': bool(torch.isfinite(res).all()) and bool(torch.isfinite(bv_next).all())}
        if cfg == 'DPV_up':
            row['DPV'] = float(np.abs(np.exp(cases.subsample_to(res.cpu().numpy()[0], 8000)) - np.exp(gold[key + '/dpv_up'])).max())
        elif cfg == 'DGF':
            row['dmap_m'] = float(np.abs(cases.subsample_to(res.cpu().numpy()[0, 0], 8000) - gold[key + '/dmap']).max())
        else:
            row['DPV'] = float(np.abs(np.exp(cases.subsample_to(res.cpu().numpy(), 8000)) - np.exp(gold[key + '/DPV'])).max())
        out['steps'].append(row)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
