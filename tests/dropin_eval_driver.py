"""The reference's OWN inference step (test_utils/test_KVNet.py:test of an unmodified checkout) on the engine with the model in
.eval(): install_as_reference_modules(), construct models.KVNET.KVNET by keyword, nn.DataParallel, .cuda(), load the weights
and the warmed running statistics of tests/golden/eval_outputs.npz, .eval(), then run the first window and two steady
steps, each steady step fed the reference's train-mode prior as the fixture was recorded. Prints one JSON line with the
deviations of the filtered DPV from the eval fixtures. Run as a subprocess by
tests/test_gpu_eval.py (keeps the reference's top-level module names out of the test process)."""
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
    name = 'kvnet_256_d16'
    import neuralrgbd_b200
    neuralrgbd_b200.install_as_reference_modules(ref_code)
    import models.KVNET as m_kvnet                     # reference module; KVNET re-pointed to the engine-backed class
    import test_utils.test_KVNet as ref_step           # the reference's file, unmodified
    from oracle import planesweep_oracle as O
    from tests import cases
    assert ref_step.__file__.startswith(os.path.abspath(ref_code)), ref_step.__file__
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_outputs.npz'))
    ref_gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_outputs.npz'))
    c = cases.kvnet_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']),
               intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'],
                              KVNet_feature_dim=64, d_upsample_ratio_KV_net=None, t_win_r=2, if_refined=True)
    model = torch.nn.DataParallel(model)
    model.cuda()
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in c['sd'].items()}
    pre = 'eval/%s/rs/' % name
    sd.update({k[len(pre):]: torch.from_numpy(np.asarray(gold[k])) for k in gold.files if k.startswith(pre)})
    model.module.load_state_dict(sd)
    model.eval()
    out = {'class': type(model.module).__module__, 'training': model.module.training, 'steps': []}
    for step in range(3):
        bv = torch.from_numpy(ref_gold['kvnet/%s/step%d/BV_predict_next_full' % (name, step - 1)]).cuda() if step else None
        ref_f, src_f, poses = cases.window(c, 2 + step)
        Ref_Dats = [{'img': torch.from_numpy(ref_f)}]
        Src_Dats = [[{'img': torch.from_numpy(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
        kv, _ = ref_step.test(model, c['d'], [cam], 2, Ref_Dats, Src_Dats, torch.from_numpy(poses).cuda(), bv, R_net=False)
        key = 'eval/%s/step%d/%s' % (name, step, 'DPV' if step else 'BV_cur')     # first window: DPV is BV_cur
        out['steps'].append({'DPV': float(np.abs(np.exp(cases.subsample_to(kv.cpu().numpy(), 8000)) - np.exp(gold[key])).max())})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
