"""Parameter gradients of the reference's OWN models.KVNET.KVNET (refineNet_name='DGF', unmodified copy of the reference)
under train_utils/train_KVNet.py's L1 loss (:126-145), variance terms included, with and without the mirrors, now
including models.GF.guided_filter.GuidedFilter.

A first window, then the prior propagated from the detached K-Net DPV by resample_vol_cuda + clamp (:155-168), then one
steady step, as tests/stats_kvnet_driver.py runs them ('full' loss at the reference's weight_var = 0.001). cuDNN and
matmul TF32 are off. Three runs on one set of weights and inputs:
  A, B  a KVNET built from the reference's own modules (B - A is the run-to-run floor of cuDNN's backward);
  P     a second KVNET built while models.GF.guided_filter.GuidedFilter is the neuralrgbd_b200 mirror (Refine.py looks
        DGF.GuidedFilter up when it constructs RefineNet_DGF), with the same state dict, run with
        warping.homography.{est_swp_volume_v4, warp_img_feats_v3, warp_img_feats_mgpu, resample_vol_cuda} and
        mutils.misc.{depth_val_regression, depth_var} set to the mirrors; every patch is restored afterwards.
Prints one JSON line: the losses, per parameter max |P - A|, max |B - A| and max |A|, whether P's r_net.dgf is the
mirror (and how often it ran) and whether both state_dict key lists agree.
Run as a subprocess by tests/test_gpu_gf.py.
    python tests/gf_kvnet_driver.py REF_CODE"""
import contextlib
import io
import json
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MIRRORED = {'warping.homography': ['est_swp_volume_v4', 'warp_img_feats_v3', 'warp_img_feats_mgpu', 'resample_vol_cuda'],
            'mutils.misc': ['depth_val_regression', 'depth_var'],
            'models.GF.guided_filter': ['GuidedFilter']}
WEIGHT_VAR = 0.001          # train_utils/train_KVNet.py:26, train_KVNet.py:127


@contextlib.contextmanager
def mirrors(on):
    import importlib
    saved = []
    if on:
        for mod, names in MIRRORED.items():
            ref = importlib.import_module(mod)
            mine = importlib.import_module('neuralrgbd_b200.' + mod)
            for n in names:
                saved.append((ref, n, getattr(ref, n)))
                setattr(ref, n, getattr(mine, n))
    try:
        yield
    finally:
        for ref, n, f in saved:
            setattr(ref, n, f)


def main():
    ref_code = sys.argv[1]
    sys.path.insert(1, ref_code)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    import models.KVNET as m_kvnet                     # the reference's modules, not re-pointed
    import models.GF.guided_filter as m_gf
    import warping.homography as wh
    import mutils.misc as m_misc
    from neuralrgbd_b200 import arch
    from neuralrgbd_b200.models.GF import guided_filter as mirror_gf
    from oracle import planesweep_oracle as O
    from tests import cases
    assert m_kvnet.__file__.startswith(os.path.abspath(ref_code)), m_kvnet.__file__
    c = cases.kvnet_case('kvnet_256_d16')
    d = c['d']
    cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']).cuda(),
               intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']).cuda())
    sd = {k: v for k, v in c['sd'].items() if not k.startswith('r_net.')}
    rn = arch.synth_state_dict(5, 64, c['D'], 2, 64, refine='DGF')
    sd.update({k: v for k, v in rn.items() if k.startswith('r_net.')})

    def build():
        with contextlib.redirect_stdout(io.StringIO()):
            m = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=d, sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                              d_upsample_ratio_KV_net=None, t_win_r=2, if_refined=True, refineNet_name='DGF')
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        return m.cuda().train()
    model_ref = build()
    with mirrors(True):
        model_mir = build()
    calls = []
    model_mir.r_net.dgf.register_forward_hook(lambda *a: calls.append(1))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    win = [cases.window(c, 2 + s) for s in range(2)]
    depth_ref = torch.full((1, 1, c['H'], c['W']), 2.0, device='cuda')
    depth_ref[..., : c['H'] // 8, :] = 0.0                             # pixels without ground truth
    mask = (depth_ref > 0.).type_as(depth_ref)

    def var_term(dpv):
        return torch.mean(m_misc.depth_var(dpv, m_misc.depth_val_regression(dpv, d, BV_log=True), d))

    def run(model, on):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(0)
        with mirrors(on):
            ref_f, src_f, poses = win[0]
            dcr0, _, d_dpv0, kv_dpv0 = model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam], BV_predict=None)
            l1_0, var_0 = F.l1_loss(dcr0 * mask, depth_ref * mask), var_term(d_dpv0)
            rel = T(poses)[0, 2].inverse()
            bv_pred = wh.resample_vol_cuda(src_vol=kv_dpv0.detach(), rel_extM=rel, cam_intrinsic=cam, d_candi=d,
                                           padding_value=math.log(1. / float(len(d)))).clamp(max=0, min=-1000.).unsqueeze(0)
            ref_f, src_f, poses = win[1]
            dcr1, dr1, d_dpv1, kv_dpv1 = model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam],
                                               BV_predict=bv_pred)
            l1_1 = F.l1_loss(dcr1 * mask, depth_ref * mask) + F.l1_loss(dr1 * mask, depth_ref * mask)
            var_1 = var_term(kv_dpv1) + var_term(d_dpv1)
            loss = (l1_0 + WEIGHT_VAR * var_0) + (l1_1 + WEIGHT_VAR * var_1)
            loss.backward()
        torch.cuda.synchronize()
        return float(loss), {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    la, A = run(model_ref, False)
    lb, B = run(model_ref, False)
    lp, P = run(model_mir, True)
    out = {'loss': [la, lb, lp], 'params': {}, 'missing': sorted(set(A) ^ set(P)),
           'n_params': len(list(model_ref.parameters())), 'dgf_calls': len(calls),
           'dgf_is_mirror': type(model_mir.r_net.dgf) is mirror_gf.GuidedFilter,
           'reference_dgf': type(model_ref.r_net.dgf) is m_gf.GuidedFilter,
           'same_state_dict_keys': list(model_mir.state_dict()) == list(model_ref.state_dict())}
    for n in sorted(A):
        if n in P:
            out['params'][n] = {'dev': float((P[n] - A[n]).abs().max()), 'floor': float((B[n] - A[n]).abs().max()),
                                'max': float(A[n].abs().max())}
    out['restored'] = bool(m_misc.depth_var.__module__ == 'mutils.misc' and wh.resample_vol_cuda.__module__ == 'warping.homography'
                           and m_gf.GuidedFilter.__module__ == 'models.GF.guided_filter')
    print(json.dumps(out))


if __name__ == '__main__':
    main()
