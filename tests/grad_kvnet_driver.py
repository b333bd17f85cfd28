"""Parameter gradients of the reference's OWN models.KVNET.KVNET (refineNet_name='DGF', unmodified copy of the reference)
on the GPU, with and without the mirrors: a first window, the prior propagated by resample_vol_cuda (+ the clamp of
test_utils/test_KVNet.py:54-59), one steady step, and an L1 loss on both refined depth maps. cuDNN and matmul TF32 are
off. Three runs on one model and one set of inputs:
  A, B  the reference's own warping.homography / mutils.misc (B gives the run-to-run floor of cuDNN's backward);
  P     warping.homography.{est_swp_volume_v4, warp_img_feats_v3, warp_img_feats_mgpu, resample_vol_cuda} and
        mutils.misc.depth_val_regression set to the neuralrgbd_b200 mirrors for the run, restored afterwards;
  Q     as P, but depth_val_regression returns a tensor without grad_fn, as the mirror did before it had a backward.
Prints one JSON line: per parameter max |P - A|, max |B - A| and max |A|, and the parameters Q gives a gradient.
Run as a subprocess by tests/test_gpu_grad.py.
    python tests/grad_kvnet_driver.py REF_CODE"""
import contextlib
import io
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MIRRORED = {'warping.homography': ['est_swp_volume_v4', 'warp_img_feats_v3', 'warp_img_feats_mgpu', 'resample_vol_cuda'],
            'mutils.misc': ['depth_val_regression']}


@contextlib.contextmanager
def mirrors(on, regression_grad=True):
    import importlib
    saved = []
    if on:
        for mod, names in MIRRORED.items():
            ref = importlib.import_module(mod)
            mine = importlib.import_module('neuralrgbd_b200.' + mod)
            for n in names:
                saved.append((ref, n, getattr(ref, n)))
                setattr(ref, n, getattr(mine, n))
        if not regression_grad:
            ref, mine = importlib.import_module('mutils.misc'), importlib.import_module('neuralrgbd_b200.mutils.misc')
            ref.depth_val_regression = lambda bv, *a, **k: mine.depth_val_regression(bv.detach(), *a, **k)
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
    import models.KVNET as m_kvnet                     # the reference's module, not re-pointed
    import warping.homography as wh
    from neuralrgbd_b200 import arch
    from oracle import planesweep_oracle as O
    from tests import cases
    assert m_kvnet.__file__.startswith(os.path.abspath(ref_code)), m_kvnet.__file__
    name = 'kvnet_256_d16'
    c = cases.kvnet_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    cam = dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']).cuda(),
               intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']).cuda())
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                              d_upsample_ratio_KV_net=None, t_win_r=2, if_refined=True, refineNet_name='DGF')
    sd = {k: v for k, v in c['sd'].items() if not k.startswith('r_net.')}
    rn = arch.synth_state_dict(5, 64, c['D'], 2, 64, refine='DGF')
    sd.update({k: v for k, v in rn.items() if k.startswith('r_net.')})
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    model.cuda().train()
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    win = [cases.window(c, 2 + s) for s in range(2)]
    target = torch.full((1, 1, c['H'], c['W']), 2.0, device='cuda')

    def run(on, regression_grad=True):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(0)
        with mirrors(on, regression_grad):
            ref_f, src_f, poses = win[0]
            d0, _, _, dpv0 = model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam], BV_predict=None)
            rel = T(poses)[0, 2].inverse()
            bv_pred = wh.resample_vol_cuda(src_vol=dpv0, rel_extM=rel, cam_intrinsic=cam, d_candi=c['d'],
                                           padding_value=math.log(1. / float(len(c['d'])))).clamp(max=0, min=-1000.).unsqueeze(0)
            ref_f, src_f, poses = win[1]
            _, d1, _, _ = model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam], BV_predict=bv_pred)
            loss = (d0 - target).abs().mean() + (d1 - target).abs().mean()
            loss.backward()
        torch.cuda.synchronize()
        return float(loss), {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    la, A = run(False)
    lb, B = run(False)
    lp, P = run(True)
    _, Q = run(True, regression_grad=False)
    out = {'loss': [la, lb, lp], 'params': {}, 'missing': sorted(set(A) ^ set(P)), 'with_grad_without_f5': sorted(Q),
           'restored': bool(wh.resample_vol_cuda.__module__ == 'warping.homography')}
    for n in sorted(A):
        if n not in P:
            continue
        out['params'][n] = {'dev': float((P[n] - A[n]).abs().max()), 'floor': float((B[n] - A[n]).abs().max()),
                            'max': float(A[n].abs().max())}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
