"""Runs the reference (an unmodified copy of its code/ directory) for the tests and prints one JSON line. It runs as a
subprocess (tests/harness.py: run_reference_driver), which keeps the reference's top-level module names (models, warping,
mutils, ...) out of the test process.

reference_driver.py REF_CODE step SCENARIO [ARGS]
  The reference's OWN inference step (test_utils/test_KVNet.py:test) on the engine after
  neuralrgbd_b200.install_as_reference_modules(), built the way test_KVNet.py:159-168 builds it: models.KVNET.KVNET by
  keyword, nn.DataParallel, .cuda(), load_state_dict; then test() on each window. Prints the outputs' deviations from the
  committed fixtures.
    kvnet              kvnet_256_d16, free-running: each step is fed the prior the one before returned (test_KVNet.py:
                       224-236); test() with R_net=True and R_net=False, the launch count       (test_gpu_dropin.py)
    eval               kvnet_256_d16 in .eval() with the running statistics of eval_outputs.npz  (test_gpu_eval.py)
    f16                r1_256_d16 with conv_math='f16', against the f16-emulated reference        (test_gpu_f16.py)
    twin NAME          a cases_twin case (t_win_r 1 or 3)                                         (test_gpu_twin.py)
    refine CFG [MODE]  CFG: DGF (refineNet_name='DGF', refined depth map), DPV_up (if_upsample_d=True, refined log-DPV of
                       4D planes) or none (if_refined=False, filtered DPV); MODE: train or eval  (test_gpu_refine.py)
  All but kvnet re-seed each steady step with the reference's train-mode prior, as their fixtures were recorded.

reference_driver.py REF_CODE grad SCENARIO
  Parameter gradients of the reference's OWN models.KVNET.KVNET (refineNet_name='DGF', nothing re-pointed) on the GPU,
  cuDNN and matmul TF32 off: a first window, the prior propagated by resample_vol_cuda + the clamp of
  test_utils/test_KVNet.py:54-59, one steady step, then a loss. Runs on one set of weights and inputs:
    A, B  the reference's own warping.homography / mutils.misc (B - A is the run-to-run floor of cuDNN's backward);
    P     the scenario's functions set to the neuralrgbd_b200 mirrors for the run, restored afterwards.
  Prints the losses and, per parameter, max |P - A|, max |B - A| and max |A|.
    geometry  est_swp_volume_v4, warp_img_feats_v3 / _mgpu, resample_vol_cuda and depth_val_regression mirrored; the prior
              from the K-Net DPV with its graph; L1 of both refined depth maps against a constant. A fourth run Q is P
              with depth_val_regression returning a tensor without grad_fn, as the mirror did before it had a backward:
              the parameters Q gives a gradient                                                  (test_gpu_grad.py)
    stats     also depth_var; the prior from the detached K-Net DPV; train_utils/train_KVNet.py's masked L1 loss with
              its variance terms (:126-168), 'full' at weight_var = 0.001 and 'var_only'       (test_gpu_stats.py)
    gf        also models.GF.guided_filter.GuidedFilter; stats' 'full' loss. P runs a second KVNET built while the
              GuidedFilter patch is active (Refine.py looks DGF.GuidedFilter up when it constructs RefineNet_DGF)
                                                                                                 (test_gpu_gf.py)
"""
import argparse
import contextlib
import importlib
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

from oracle import planesweep_oracle as O      # noqa: E402
from tests import cases, harness          # noqa: E402


# ---- step ------------------------------------------------------------------------------------------------------------
def _sub(limit):
    return lambda a: cases.subsample_to(a, limit)


def _dev(a, g, sub):
    """max |exp(a) - exp(g)| over the fixture's samples of log-DPV tensor a."""
    return float(np.abs(np.exp(sub(a.cpu().numpy())) - np.exp(g)).max())


def _filtered_dpv(gold, key, sub, extra=()):
    """Scores test(R_net=False): its filtered DPV against gold[key % step + '/DPV'] (a first window's is BV_cur), with the
    source view count ('V') and whether the prior it returns is finite ('prior_finite') when `extra` names them."""
    def score(step, res, src_f):
        kv, bv_next = res[0]
        row = {'DPV': _dev(kv, gold['%s/%s' % (key % step, 'DPV' if step else 'BV_cur')], sub)}
        if 'V' in extra:
            row['V'] = int(src_f.shape[1])
        if 'prior_finite' in extra:
            row['prior_finite'] = bool(torch.isfinite(bv_next).all())
        return row
    return score


def _kvnet_case(name):
    c = cases.kvnet_case(name)
    return c, cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)


def scenario_kvnet():
    name = 'kvnet_256_d16'
    c, cam = _kvnet_case(name)
    gold = harness.golden('reference_outputs.npz')

    def score(step, res, src_f):
        (dmap, bv_next), (kv, bv_next2) = res
        key = 'kvnet/%s/step%d' % (name, step)
        return {'dmap_refined': _dev(dmap, gold[key + '/dmap_refined'], cases.subsample),
                'DPV': _dev(kv, gold[key + '/DPV'], cases.subsample),
                'prior_next': _dev(bv_next, gold[key + '/BV_predict_next'], cases.subsample),
                'deterministic': bool(torch.equal(bv_next, bv_next2))}

    def report(model):
        from neuralrgbd_b200 import _lib
        return {'launches': int(_lib.lib().nrgbd_launch_count())}
    return dict(c=c, cam=cam, sd=c['sd'], n_steps=len(c['frames']) - 4, prior=None, r_net=(True, False), score=score,
                report=report)


def scenario_eval():
    name = 'kvnet_256_d16'
    c, cam = _kvnet_case(name)
    gold = harness.golden('eval_outputs.npz')
    sd = dict(c['sd'])
    pre = 'eval/%s/rs/' % name
    sd.update({k[len(pre):]: np.asarray(gold[k]) for k in gold.files if k.startswith(pre)})
    return dict(c=c, cam=cam, sd=sd, eval=True, n_steps=3, prior=lambda step: harness.reference_prior(name, step),
                r_net=(False,), score=_filtered_dpv(gold, 'eval/%s/step%%d' % name, _sub(8000)),
                report=lambda model: {'training': model.module.training})


def scenario_f16():
    from tests import cases_f16 as CF
    name = 'r1_256_d16'
    c = CF.f16_case(name)
    return dict(c=c, cam=CF.cam(O.make_cam_intrinsics, c), sd=CF.state_dict(c), conv_math='f16', n_steps=c['n_steps'],
                prior=lambda step: CF.reseed_prior(name, step), r_net=(False,),
                score=_filtered_dpv(harness.golden('f16_outputs.npz'), 'f16/%s/step%%d/f16' % name, _sub(CF.SUB_LIMIT),
                                    ('prior_finite',)),
                report=lambda model: {'conv_math': model.module.conv_math})


def scenario_twin(name):
    from tests import cases_twin as CT
    c = CT.twin_case(name)
    return dict(c=c, cam=CT.twin_cam(O.make_cam_intrinsics, c), sd=c['sd'], n_steps=c['n_steps'],
                prior=lambda step: CT.prior(name, step), r_net=(False,),
                score=_filtered_dpv(harness.golden('twin_outputs.npz'), 'twin/train/%s/step%%d' % name, _sub(8000),
                                    ('V', 'prior_finite')),
                report=lambda model: {'t_win_r': c['t_win_r']})


def scenario_refine(cfg, mode='train'):
    from neuralrgbd_b200 import arch
    assert mode in ('train', 'eval'), mode
    name = 'kvnet_256_d16'
    c, cam = _kvnet_case(name)
    gold = harness.golden('refine_outputs.npz')
    kw = {'DGF': dict(if_refined=True, refineNet_name='DGF'), 'none': dict(if_refined=False),
          'DPV_up': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True)}[cfg]
    sd = {k: v for k, v in c['sd'].items() if not k.startswith('r_net.')}
    if cfg != 'none':
        rn = arch.synth_state_dict(5, 64, c['D'], 2, 64, refine='DGF' if cfg == 'DGF' else 'DPV', upsample_d=cfg == 'DPV_up')
        sd.update({k: v for k, v in rn.items() if k.startswith('r_net.')})

    def score(step, res, src_f):
        r, bv_next = res[0]
        key = 'refine/%s/%s/step%d' % (cfg, name, step)
        row = {'shape': list(r.shape), 'finite': bool(torch.isfinite(r).all()) and bool(torch.isfinite(bv_next).all())}
        if cfg == 'DPV_up':
            row['DPV'] = _dev(r[0], gold[key + '/dpv_up'], _sub(8000))
        elif cfg == 'DGF':
            row['dmap_m'] = float(np.abs(cases.subsample_to(r.cpu().numpy()[0, 0], 8000) - gold[key + '/dmap']).max())
        else:
            row['DPV'] = _dev(r, gold[key + '/DPV'], _sub(8000))
        return row
    return dict(c=c, cam=cam, sd=sd, kw=kw, eval=mode == 'eval', n_steps=3, prior=lambda step: harness.reference_prior(name, step),
                r_net=(cfg != 'none',), score=score, report=lambda model: {})


STEP_SCENARIOS = {'kvnet': scenario_kvnet, 'eval': scenario_eval, 'f16': scenario_f16, 'twin': scenario_twin,
                  'refine': scenario_refine}


def step(ref_code, scenario, args):
    import neuralrgbd_b200
    neuralrgbd_b200.install_as_reference_modules(ref_code)
    import models.KVNET as m_kvnet                     # reference module; KVNET re-pointed to the engine-backed class
    import test_utils.test_KVNet as ref_step           # the reference's file, unmodified
    assert ref_step.__file__.startswith(os.path.abspath(ref_code)), ref_step.__file__
    s = STEP_SCENARIOS[scenario](*args)
    c, r = s['c'], s['c']['t_win_r']
    cam = harness.cam_tensors(s['cam'])
    with contextlib.redirect_stdout(io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                              d_upsample_ratio_KV_net=None, t_win_r=r, **s.get('kw', dict(if_refined=True)))   # test_KVNet.py:159-162
    model = torch.nn.DataParallel(model)               # :163
    model.cuda()                                       # :164
    model.module.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in s['sd'].items()}, strict=True)
    if s.get('conv_math'):
        model.module.conv_math = s['conv_math']
    model.train(not s.get('eval', False))
    out = {'class': type(model.module).__module__, 'steps': []}
    bv = None
    for k in range(s['n_steps']):
        if k and s['prior']:
            bv = torch.from_numpy(s['prior'](k)).cuda()
        ref_f, src_f, poses = cases.window(c, r + k)
        Ref_Dats = [{'img': torch.from_numpy(ref_f)}]
        Src_Dats = [[{'img': torch.from_numpy(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
        poses_t = torch.from_numpy(poses).cuda()
        res = [ref_step.test(model, c['d'], [cam], r, Ref_Dats, Src_Dats, poses_t, bv, R_net=rn) for rn in s['r_net']]
        out['steps'].append(s['score'](k, res, src_f))
        bv = res[0][1]                                 # free-running unless the scenario re-seeds the next step
    out.update(s['report'](model))
    return out


# ---- grad ------------------------------------------------------------------------------------------------------------
GEOMETRY = {'warping.homography': ['est_swp_volume_v4', 'warp_img_feats_v3', 'warp_img_feats_mgpu', 'resample_vol_cuda'],
            'mutils.misc': ['depth_val_regression']}
STATS = dict(GEOMETRY, **{'mutils.misc': ['depth_val_regression', 'depth_var']})
GF = dict(STATS, **{'models.GF.guided_filter': ['GuidedFilter']})
GRAD_SCENARIOS = ['geometry', 'stats', 'gf']
WEIGHT_VAR = 0.001          # train_utils/train_KVNet.py:26, train_KVNet.py:127


@contextlib.contextmanager
def mirrors(names, regression_grad=True):
    """The reference's `names` ({module: [attribute]}) set to the neuralrgbd_b200 mirrors inside the block; without
    regression_grad, depth_val_regression detaches its input."""
    saved = []
    for mod, attrs in names.items():
        ref, mine = importlib.import_module(mod), importlib.import_module('neuralrgbd_b200.' + mod)
        for n in attrs:
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


def restored(names):
    """Whether every patched name is the reference's own again."""
    return all(getattr(importlib.import_module(mod), n).__module__ == mod for mod, attrs in names.items() for n in attrs)


def grad(ref_code, scenario):
    sys.path.insert(1, ref_code)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    import models.KVNET as m_kvnet                     # the reference's modules, not re-pointed
    import warping.homography as wh
    import mutils.misc as m_misc
    from neuralrgbd_b200 import arch
    assert m_kvnet.__file__.startswith(os.path.abspath(ref_code)), m_kvnet.__file__
    c = cases.kvnet_case('kvnet_256_d16')
    d = c['d']
    cam = harness.cam_tensors(cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4), 'cuda')
    sd = {k: v for k, v in c['sd'].items() if not k.startswith('r_net.')}
    rn = arch.synth_state_dict(5, 64, c['D'], 2, 64, refine='DGF')
    sd.update({k: v for k, v in rn.items() if k.startswith('r_net.')})

    def build():
        with contextlib.redirect_stdout(io.StringIO()):
            m = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=d, sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                              d_upsample_ratio_KV_net=None, t_win_r=2, if_refined=True, refineNet_name='DGF')
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        return m.cuda().train()

    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    win = [cases.window(c, 2 + s) for s in range(2)]
    depth_ref = torch.full((1, 1, c['H'], c['W']), 2.0, device='cuda')
    if scenario != 'geometry':
        depth_ref[..., : c['H'] // 8, :] = 0.0                         # pixels without ground truth
    mask = (depth_ref > 0.).type_as(depth_ref)

    def windows(model):
        """Outputs of the first window and of the steady step fed its propagated prior."""
        ref_f, src_f, poses = win[0]
        out0 = model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam], BV_predict=None)
        dpv0 = out0[3] if scenario == 'geometry' else out0[3].detach()
        rel = T(poses)[0, 2].inverse()
        bv_pred = wh.resample_vol_cuda(src_vol=dpv0, rel_extM=rel, cam_intrinsic=cam, d_candi=d,
                                       padding_value=math.log(1. / float(len(d)))).clamp(max=0, min=-1000.).unsqueeze(0)
        ref_f, src_f, poses = win[1]
        return out0, model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam], BV_predict=bv_pred)

    def l1_loss(out0, out1):
        return (out0[0] - depth_ref).abs().mean() + (out1[1] - depth_ref).abs().mean()

    def var_term(dpv):
        return torch.mean(m_misc.depth_var(dpv, m_misc.depth_val_regression(dpv, d, BV_log=True), d))

    def train_loss(part):
        """train_KVNet.py's L1 branch: window 0 L1(dmap_cur_refined) + weight_var * var(d_dpv), window 1
        L1(dmap_cur_refined) + L1(dmap_refined) + weight_var * (var(kv_dpv) + var(d_dpv)); 'var_only' the variance terms."""
        def loss(out0, out1):
            l1_0, var_0 = F.l1_loss(out0[0] * mask, depth_ref * mask), var_term(out0[2])
            l1_1 = F.l1_loss(out1[0] * mask, depth_ref * mask) + F.l1_loss(out1[1] * mask, depth_ref * mask)
            var_1 = var_term(out1[3]) + var_term(out1[2])
            if part == 'full':
                return (l1_0 + WEIGHT_VAR * var_0) + (l1_1 + WEIGHT_VAR * var_1)
            return var_0 + var_1
        return loss

    def run(model, names, loss_fn, regression_grad=True):
        model.zero_grad(set_to_none=True)
        torch.manual_seed(0)
        with mirrors(names, regression_grad):
            loss = loss_fn(*windows(model))
            loss.backward()
        torch.cuda.synchronize()
        return float(loss), {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    def abp(model_ref, model_mir, names, loss_fn):
        (la, A), (lb, B), (lp, P) = run(model_ref, {}, loss_fn), run(model_ref, {}, loss_fn), run(model_mir, names, loss_fn)
        rec = {'loss': [la, lb, lp], 'params': {}, 'missing': sorted(set(A) ^ set(P))}
        for n in sorted(A):
            if n in P:
                rec['params'][n] = {'dev': float((P[n] - A[n]).abs().max()), 'floor': float((B[n] - A[n]).abs().max()),
                                    'max': float(A[n].abs().max())}
        return rec

    if scenario == 'geometry':
        model = build()
        out = abp(model, model, GEOMETRY, l1_loss)
        _, Q = run(model, GEOMETRY, l1_loss, regression_grad=False)
        out['with_grad_without_f5'] = sorted(Q)
        out['restored'] = restored(GEOMETRY)
    elif scenario == 'stats':
        model = build()
        out = {part: abp(model, model, STATS, train_loss(part)) for part in ('full', 'var_only')}
        out['restored'] = restored(STATS)
    else:
        import models.GF.guided_filter as m_gf
        from neuralrgbd_b200.models.GF import guided_filter as mirror_gf
        model_ref = build()
        with mirrors(GF):
            model_mir = build()
        calls = []
        model_mir.r_net.dgf.register_forward_hook(lambda *a: calls.append(1))
        out = abp(model_ref, model_mir, GF, train_loss('full'))
        out.update({'n_params': len(list(model_ref.parameters())), 'dgf_calls': len(calls),
                    'dgf_is_mirror': type(model_mir.r_net.dgf) is mirror_gf.GuidedFilter,
                    'reference_dgf': type(model_ref.r_net.dgf) is m_gf.GuidedFilter,
                    'same_state_dict_keys': list(model_mir.state_dict()) == list(model_ref.state_dict()),
                    'restored': restored(GF)})
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument('ref_code', help="the reference's code/ directory")
    sub = p.add_subparsers(dest='cmd', required=True)
    ps = sub.add_parser('step', help="the reference's test() on the engine: kvnet | eval | f16 | twin NAME | refine CFG [MODE]")
    ps.add_argument('scenario', choices=list(STEP_SCENARIOS))
    ps.add_argument('args', nargs='*')
    pg = sub.add_parser('grad', help="parameter gradients of the reference's KVNET with and without the mirrors: %s"
                        % ' | '.join(GRAD_SCENARIOS))
    pg.add_argument('scenario', choices=GRAD_SCENARIOS)
    a = p.parse_args()
    out = step(a.ref_code, a.scenario, a.args) if a.cmd == 'step' else grad(a.ref_code, a.scenario)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
