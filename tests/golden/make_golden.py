"""Writes the golden fixtures: runs the UNMODIFIED reference (CPU torch) on the seeded inputs of tests/cases*.py, stores
its outputs under tests/golden/ and the numpy oracle's measured deviations from them in tests/golden/PINNING_*.json, the
records that pin the oracle and the fp32-vs-fp32 floors the GPU gates are set against.

    python tests/golden/make_golden.py [--ref DIR] FIXTURE [CASE ...]

FIXTURE is a name of FIXTURES (each function's docstring says what its fixture holds) or `all`, which runs every fixture in
dependency order: eval, refine, twin, f16 and drift read what reference and configs wrote. The reference's code/ directory
is the one tests/harness.py:run_reference_driver runs (oracle/fetch_reference.py:code_dir), or DIR. It hard-codes .cuda();
on a CPU-only machine cpu_shim() (SURVEY.md §8(c)) turns those calls into no-ops. Inputs are regenerated from seeds; only
reference OUTPUTS are stored (large ones strided, plus full-array statistics).
"""
import argparse
import contextlib
import importlib
import io
import json
import os
import sys
import tempfile
import time
import types
import warnings
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from neuralrgbd_b200 import arch, synth              # noqa: E402
from oracle import fetch_reference                   # noqa: E402
from oracle import kvnet_oracle as N                 # noqa: E402
from oracle import planesweep_oracle as O            # noqa: E402
from tests import cases, harness                     # noqa: E402
from tests.harness import NAMES4                     # noqa: E402

T = torch.from_numpy
REF_CODE = None         # --ref: the reference's code/ directory; None: fetch_reference.code_dir()
STORED = {True: ('BV_cur', 'dmap_cur_refined'), False: ('DPV', 'dmap_refined')}    # first window: / steady step:
DEPTH_LIMIT = 2000      # strided expected-depth values per step (eval, twin, f16)
WARM_STEPS = 4          # running-statistics warm-up: 1 first window + 3 steady steps
WARM_SEED = 1000        # the warm-up video is seeded apart from every test video


# ---- the reference -----------------------------------------------------------------------------------------------------
def cpu_shim():
    """The reference's hard-coded .cuda() / device queries as no-ops, for a CPU-only torch."""
    torch.Tensor.cuda = lambda s, *a, **k: s
    torch.nn.Module.cuda = lambda s, *a, **k: s
    torch.cuda.current_device = lambda: 0
    torch.Tensor.get_device = lambda s: 0


def reference(*names):
    """The reference's modules `names`, imported from its code/ directory with cpu_shim() applied."""
    code = os.path.realpath(REF_CODE or fetch_reference.code_dir())
    assert os.path.isdir(code), 'no copy of the reference: oracle/_ref is made by __graft_entry__.build() (or pass --ref)'
    if code not in sys.path:
        sys.path.insert(0, code)
    cpu_shim()
    mods = [importlib.import_module(n) for n in names]
    for m in mods:
        assert os.path.realpath(m.__file__).startswith(code + os.sep), (m.__name__, m.__file__, code)
    return mods


# ---- small helpers -----------------------------------------------------------------------------------------------------
def dev(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.nanmax(np.abs(a - b))) if a.size else 0.0


def new_pin(*keys):
    """An empty pin recording the versions ('torch', 'numpy') and CPU thread count ('threads') named by `keys`."""
    now = {'torch': torch.__version__, 'numpy': np.__version__, 'threads': torch.get_num_threads()}
    return dict({k: now[k] for k in keys}, cases={})


def save_npz(name, arrays, fixed=False):
    """tests/golden/<name>: np.savez_compressed in insertion order, or with `fixed` sorted members and a fixed timestamp."""
    path = os.path.join(HERE, name)
    if not fixed:
        np.savez_compressed(path, **arrays)
    else:
        with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
            for k in sorted(arrays):
                buf = io.BytesIO()
                np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
                info = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
                info.compress_type = zipfile.ZIP_DEFLATED
                zf.writestr(info, buf.getvalue())
    print('wrote %s %.2f MB, %d arrays' % (name, os.path.getsize(path) / 1e6, len(arrays)), flush=True)


def save_pin(name, pin, newline=False, sort_keys=True):
    """tests/golden/<name> as indented JSON (`newline`: with a trailing newline)."""
    with open(os.path.join(HERE, name), 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=sort_keys)
        if newline:
            f.write('\n')


def load_existing(pin, pin_name, npz_name=None):
    """Merge targets of a partial run: the committed pin's cases into `pin`; -> the committed npz's arrays ({} without)."""
    path = os.path.join(HERE, pin_name)
    if os.path.exists(path):
        pin['cases'] = json.load(open(path)).get('cases', {})
    npz = os.path.join(HERE, npz_name or '')
    return dict(np.load(npz)) if npz_name and os.path.exists(npz) else {}


def record(out, pin, key, ref, orc, sub, suffix=''):
    """Stores reference array `ref` as sub(ref) under key + suffix with its cases.summary under key + '/stats', and pins
    the oracle's `orc` deviation from the full array."""
    ref = np.asarray(ref)
    out[key + suffix] = sub(ref)
    out[key + '/stats'] = cases.summary(ref)
    pin['cases'][key] = {'maxabs_oracle': float(np.abs(np.asarray(orc, np.float64) - ref).max()),
                         'max_ref': float(np.abs(ref).max()), 'shape': list(ref.shape)}
    print(key, pin['cases'][key], flush=True)


# ---- KVNET recipes -----------------------------------------------------------------------------------------------------
class Recorder(torch.nn.Module):
    """Passes the call through to the reference model and keeps what it returned (test() discards some of it)."""

    def __init__(self, model):
        super().__init__()
        self.model = model
        self.last = None

    def forward(self, **kw):
        self.last = self.model(**kw)
        return self.last


def build_kvnet(c, camt, sd=None, printout=None, **kw):
    """The reference's models.KVNET.KVNET for case `c`, built by keyword as test_KVNet.py:159-168 does (t_win_r=c['t_win_r'],
    if_refined=True unless `kw` says otherwise) with its printout sent to `printout` (default: dropped); `sd` (name ->
    array) is loaded when given."""
    m_kvnet, = reference('models.KVNET')
    kw = dict(dict(t_win_r=c['t_win_r'], if_refined=True), **kw)
    with contextlib.redirect_stdout(printout or io.StringIO()):
        model = m_kvnet.KVNET(feature_dim=64, cam_intrinsics=camt, d_candi=c['d'], sigma_soft_max=c['sigma'],
                              KVNet_feature_dim=64, d_upsample_ratio_KV_net=None, **kw)
    if sd is not None:
        model.load_state_dict({k: T(np.asarray(v)) for k, v in sd.items()})
    return model


def dp_recorder(model):
    """Recorder(DataParallel(model)): DataParallel as test_KVNet.py:163 (no GPUs: it falls through)."""
    return Recorder(torch.nn.DataParallel(model))


def test_step(model, c, camt, idx, prior, R_net=False):
    """The reference's own test() (test_utils/test_KVNet.py:19-67) on window `idx` of case `c`, `prior` a log-DPV (array or
    tensor) or None -> ((ref_f, src_f, poses), what test() returned)."""
    ref_test, = reference('test_utils.test_KVNet')
    ref_f, src_f, poses = cases.window(c, idx)
    Ref_Dats = [{'img': T(ref_f)}]
    Src_Dats = [[{'img': T(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
    prior = T(prior) if isinstance(prior, np.ndarray) else prior
    return (ref_f, src_f, poses), ref_test.test(model, c['d'], [camt], c['t_win_r'], Ref_Dats, Src_Dats, T(poses), prior,
                                                R_net=R_net)


def recorded_step(rec, c, camt, idx, prior):
    """test_step(R_net=False) through a Recorder -> (inputs, KVNET.forward's four outputs, the propagated prior), numpy."""
    inputs, (_, bv_next) = test_step(rec, c, camt, idx, prior)
    return inputs, [a.numpy() for a in rec.last], bv_next.numpy()


def stream_case(name):
    """kvnet_256_d16 (first window + 2 steady steps) or a BIG case (first window + 1 steady step) with its camera and the
    seed of its weights."""
    if name in cases.KVNET_CASES:
        c = cases.kvnet_case(name)
        c.update(cam=cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4), n_steps=3, wseed=5)
    else:
        c = cases.big_case(name)
        c.update(cam=cases.big_cam(O.make_cam_intrinsics, c), n_steps=2, wseed=cases.BIG_CFG[name]['wseed'])
    return c


def warm_running_stats(model, rec, c, camt, out, key):
    """Warms the reference's own running statistics and puts the model in .eval(). He-init buffers (mean 0, var 1) would
    leave eval mode almost untested, so all 13 tracked BatchNorm layers are reset and switched to momentum=None (cumulative
    average), test() runs in train mode over WARM_STEPS steps of a DIFFERENT seeded video (the first step updates the
    feature CNN's downsample layers only, the steady steps K-Net as well), then momentum=0.1 is restored. The warmed
    buffers are stored as '<key>/rs/<state_dict name>'. -> (the state_dict after warming, the weights with the warmed
    statistics as arrays)."""
    bns = [m for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm) and m.track_running_stats]
    assert len(bns) == 13, len(bns)
    for m in bns:
        m.reset_running_stats()
        m.momentum = None
    model.train()
    w = dict(c)                 # the same camera / planes / weights on a different seeded video
    nf = WARM_STEPS + 2 * c['t_win_r']
    w['frames'], rng = synth.video(WARM_SEED + c['H'] + c['W'], nf, c['H'], c['W'])
    w['exts'] = synth.camera_track(rng, nf)
    prior = None
    for k in range(WARM_STEPS):
        _, _, prior = recorded_step(rec, w, camt, c['t_win_r'] + k, prior)
    for m in bns:
        m.momentum = 0.1
    model.eval()
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        if k.endswith(('running_mean', 'running_var', 'num_batches_tracked')):
            out['%s/rs/%s' % (key, k)] = v.numpy()
    sd_np = {k: np.asarray(v) for k, v in c['sd'].items()}
    sd_np.update({k: v.numpy() for k, v in sd.items() if k.endswith(('running_mean', 'running_var'))})
    return sd, sd_np


def store_step(out, kk, full, d, first, sub_limit):
    """A step's storage: strided samples (sub_limit values) of the outputs the step adds - the first window's BV_cur and
    dmap_cur_refined (its filtered outputs are the same arrays, KVNET.py:138-143), a steady step's filtered DPV and
    dmap_refined - full-array statistics of all four probabilities and a strided expected depth. -> the full depth."""
    m_misc, = reference('mutils.misc')
    if first:
        assert np.array_equal(full[0], full[1]) and np.array_equal(full[2], full[3])
    for nm, a in zip(NAMES4, full):
        if nm in STORED[first]:
            out['%s/%s' % (kk, nm)] = cases.subsample_to(a, sub_limit)
        out['%s/%s_stats' % (kk, nm)] = cases.stats(np.exp(a.astype(np.float64)))
    dep = m_misc.depth_val_regression(T(full[3]), d, BV_log=True).numpy()
    out[kk + '/depth'] = cases.subsample_to(dep, DEPTH_LIMIT)
    return dep


def record_steps(rec, c, camt, key, sd_np, training, prior_of, out, pin, timed=False):
    """eval and twin: the case's steps through test() in the model's current mode, each steady step re-seeded with the
    reference's train-mode prior of case `prior_of` (harness.reference_prior); stores each step (store_step, 8000 values)
    and pins the numpy oracle in the same mode, fed the same prior, under '<key>/step<k>'."""
    for k in range(c['n_steps']):
        t0 = time.time()
        prior = harness.reference_prior(prior_of, k) if k else None
        (ref_f, src_f, poses), full, _ = recorded_step(rec, c, camt, c['t_win_r'] + k, prior)
        kk = '%s/step%d' % (key, k)
        dep = store_step(out, kk, full, c['d'], k == 0, 8000)
        row = {'seconds_reference': time.time() - t0}
        to = time.time()
        o = N.kvnet_forward(sd_np, ref_f, src_f, poses, c['cam'], c['d'], c['sigma'], BV_predict=prior, training=training)
        for nm, a, b in zip(NAMES4, full, o):
            row['oracle_' + nm + '_prob'] = dev(np.exp(a), np.exp(b))
            row['oracle_' + nm + '_prob_sub'] = dev(np.exp(cases.subsample_to(a, 8000)), np.exp(cases.subsample_to(b, 8000)))
        row['oracle_depth_mm'] = 1000 * dev(dep, O.depth_val_regression(o[3], c['d']))
        row['seconds_oracle'] = time.time() - to
        if not timed:
            del row['seconds_reference'], row['seconds_oracle']
        pin[kk] = row
        print(kk, json.dumps(row), flush=True)


def assert_unchanged(model, sd):
    after = model.state_dict()
    changed = [k for k in sd if not torch.equal(sd[k], after[k])]
    assert not changed, changed


# ---- fixtures ----------------------------------------------------------------------------------------------------------
def fixture_reference():
    """reference_outputs.npz / PINNING.json: the plane sweep (a1-a3), the image warp (a7, and the mgpu entry,
    homography.py:183-232, which must give the same numbers), resample_vol_cuda (a12), depth regression (a11) and the full
    KVNET.forward with the unmodified test() streaming (a4-a10), free-running on cases.KVNET_CASES, plus the NaN-prior
    branch (KVNET.py:142), which must equal the first window. The oracle runs on the same inputs (fed the REFERENCE's prior
    at every step, so each step's deviation is its own); its deviations go to PINNING.json."""
    wh, m_misc = reference('warping.homography', 'mutils.misc')
    pin = new_pin('torch', 'numpy')
    out = {}
    for name in cases.SWEEP_CASES:
        c = cases.sweep_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
        ref = wh.est_swp_volume_v4(T(c['ref']), T(c['src']), c['d'], T(c['R']), T(c['t']), harness.cam_tensors(cam),
                                   c['sigma'], feat_dist=c['feat_dist']).numpy()
        orc = O.est_swp_volume_v4(c['ref'], c['src'], c['d'], c['R'], c['t'], cam, c['sigma'], c['feat_dist'])
        bv_r = torch.log_softmax(-T(ref), 1).numpy(); bv_o = O.d_net_dpv_from_cost(orc)
        out['sweep/%s/cost' % name] = cases.subsample(ref)
        out['sweep/%s/cost_stats' % name] = cases.stats(ref)
        pin['cases']['sweep/' + name] = {'cost_maxabs': dev(ref, orc), 'cost_max': float(ref.max()),
                                         'logdpv_maxabs': dev(bv_r, bv_o),
                                         'prob_maxabs': dev(np.exp(bv_r), np.exp(bv_o))}
        print(name, pin['cases']['sweep/' + name])

    for name in cases.WARP_CASES:
        c = cases.warp_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
        ref = wh.warp_img_feats_v3([T(i) for i in c['imgs']], c['d'], [T(r) for r in c['R']],
                                   [T(t) for t in c['t']], harness.cam_tensors(cam))
        ref = np.stack([r.numpy() for r in ref])
        orc = np.stack(O.warp_img_feats_v3(c['imgs'], c['d'], c['R'], c['t'], cam))
        mg = wh.warp_img_feats_mgpu([T(i) for i in c['imgs']], c['d'], [T(r) for r in c['R']],
                                    [T(t) for t in c['t']], T(cam['intrinsic_M_cuda'])[None],
                                    T(cam['unit_ray_array_2D'])[None])
        mg = np.stack([r.numpy() for r in mg])
        out['warp/%s/vol' % name] = cases.subsample(ref)
        out['warp/%s/vol_stats' % name] = cases.stats(ref)
        pin['cases']['warp/' + name] = {'maxabs': dev(ref, orc), 'mgpu_vs_v3': dev(ref, mg)}
        print(name, pin['cases']['warp/' + name])

    for name in cases.RESAMPLE_CASES:
        c = cases.resample_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
        ref = wh.resample_vol_cuda(T(c['vol']), T(c['rel']), harness.cam_tensors(cam), c['d'], d_candi_new=c['d_new'],
                                   padding_value=c['pad']).numpy()
        orc = O.resample_vol_cuda(c['vol'], c['rel'], cam, c['d'], d_candi_new=c['d_new'], padding_value=c['pad'])
        out['resample/%s/vol' % name] = cases.subsample(ref)
        out['resample/%s/vol_stats' % name] = cases.stats(ref)
        pin['cases']['resample/' + name] = {'maxabs': dev(ref, orc),
                                            'nonidentity_vs_input': dev(ref, c['vol'][0])}
        print(name, pin['cases']['resample/' + name])

    c = cases.resample_case('resample_pose_d32')
    ref = m_misc.depth_val_regression(T(c['vol']), c['d'], BV_log=True).numpy()
    orc = O.depth_val_regression(c['vol'], c['d'])
    out['regress/resample_pose_d32/depth'] = ref
    pin['cases']['regress/resample_pose_d32'] = {'maxabs_m': dev(ref, orc)}
    print('regress', pin['cases']['regress/resample_pose_d32'])

    for name in cases.KVNET_CASES:
        c = cases.kvnet_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
        camt = harness.cam_tensors(cam)
        model = torch.nn.DataParallel(build_kvnet(c, camt, c['sd']))
        bv_pred = None; bv_pred_o = None
        n_steps = len(c['frames']) - 4
        for step in range(n_steps):
            ref_f, src_f, poses = cases.window(c, 2 + step)
            # the refined outputs too: a direct call beside test(R_net=False), which returns (kv_dpv, BVs_predict)
            with torch.no_grad():
                full = model(ref_frame=T(ref_f), src_frames=T(src_f), src_cam_poses=T(poses),
                             BatchIdx=torch.zeros(1), cam_intrinsics=[camt], BV_predict=bv_pred)
            _, (kv_dpv, bv_next) = test_step(model, c, camt, 2 + step, bv_pred)
            o = N.kvnet_forward(c['sd'], ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=bv_pred_o)
            rel_t = T(poses)[0, 2].inverse().numpy()
            bv_next_o = O.propagate_dpv(o[3], rel_t, cam, c['d'])
            key = 'kvnet/%s/step%d' % (name, step)
            rec = {}
            for nm, a, b in zip(NAMES4, full, o):
                a = a.numpy()
                out['%s/%s' % (key, nm)] = cases.subsample(a)
                out['%s/%s_stats' % (key, nm)] = cases.stats(a)
                rec[nm + '_log'] = dev(a, b); rec[nm + '_prob'] = dev(np.exp(a), np.exp(b))
                rec[nm + '_min'] = float(a.min())
            dep_r = m_misc.depth_val_regression(full[3], c['d'], BV_log=True).numpy()
            dep_o = O.depth_val_regression(o[3], c['d'])
            rec['depth_mm'] = 1000 * dev(dep_r, dep_o)
            out[key + '/rel_inv'] = rel_t
            out[key + '/BV_predict_next'] = cases.subsample(bv_next.numpy())
            out[key + '/BV_predict_next_stats'] = cases.stats(bv_next.numpy())
            if step < n_steps - 1:      # the next step's prior, in full, so tests can feed the reference's prior
                out[key + '/BV_predict_next_full'] = bv_next.numpy()
            rec['kv_dpv_eq_full'] = dev(kv_dpv.numpy(), full[3].numpy())
            rec['BV_predict_next_log'] = dev(bv_next.numpy(), bv_next_o)
            pin['cases'][key] = rec
            print(key, rec)
            bv_pred = bv_next
            bv_pred_o = bv_next.numpy()
        ref_f, src_f, poses = cases.window(c, 2)
        nanp = torch.full((1, c['D'], c['H'] // 4, c['W'] // 4), float('nan'))
        with torch.no_grad():
            full = model(ref_frame=T(ref_f), src_frames=T(src_f), src_cam_poses=T(poses),
                         BatchIdx=torch.zeros(1), cam_intrinsics=[camt], BV_predict=nanp)
        pin['cases']['kvnet/%s/nan_prior_eq_first' % name] = dev(
            cases.subsample(full[3].numpy()), out['kvnet/%s/step0/DPV' % name])

    save_npz('reference_outputs.npz', out)
    save_pin('PINNING.json', pin)


def fixture_configs(*names):
    """configs_<case>.npz, configs_priors_<case>.npz / PINNING_configs.json: the BASELINE.json configurations
    (cases.BIG_CASES, or `names`, merged into the pin) at their real sizes. The reference's own streaming step is driven
    FREE-RUNNING over the whole frame list: step k receives the prior the reference itself propagated at step k-1.
    Stored per step: strided samples + full-array statistics of the outputs, the expected depth of the filtered DPV and
    the propagated prior (strided); the full prior after step 0 goes to configs_priors_<case>.npz so that one steady step
    can also be tested re-seeded. The numpy oracle runs on step 0 and step 1 (fed the reference's prior); its deviation,
    the fp32-vs-fp32 noise floor AT THESE SHAPES, goes to PINNING_configs.json."""
    m_misc, = reference('mutils.misc')
    pin = new_pin('torch', 'numpy', 'threads')
    load_existing(pin, 'PINNING_configs.json')
    for name in names or cases.BIG_CASES:
        c = cases.big_case(name)
        cam = cases.big_cam(O.make_cam_intrinsics, c)
        camt = harness.cam_tensors(cam)
        r = c['t_win_r']
        rec_model = dp_recorder(build_kvnet(c, camt, c['sd']))
        out, priors = {}, {}
        bv_pred = None
        for step in range(c['n_steps']):
            t0 = time.time()
            (ref_f, src_f, poses), (kv_dpv, bv_next) = test_step(rec_model, c, camt, r + step, bv_pred)
            full = [a.numpy() for a in rec_model.last]
            key = 'cfg/%s/step%d' % (name, step)
            rec = {'seconds_reference': None}
            thin = step >= cases.BIG_FULL_STEPS
            for nm, a in zip(NAMES4, full):
                if thin and nm in ('dmap_cur_refined', 'BV_cur'):
                    continue
                out['%s/%s' % (key, nm)] = cases.subsample_to(a, 30000) if thin else cases.subsample(a)
                out['%s/%s_stats' % (key, nm)] = cases.stats(np.exp(a.astype(np.float64)))
                rec[nm + '_min'] = float(a.min())
            dep = m_misc.depth_val_regression(T(full[3]), c['d'], BV_log=True).numpy()
            out[key + '/depth'] = cases.subsample_to(dep, 5000)
            out[key + '/BV_predict_next'] = cases.subsample_to(bv_next.numpy(), 30000)
            rec['kv_dpv_eq_forward'] = dev(kv_dpv.numpy(), full[3])
            if step == 0:
                priors['cfg/%s/step0/BV_predict_next_full' % name] = bv_next.numpy()
            if step < 2:
                to = time.time()
                o = N.kvnet_forward(c['sd'], ref_f, src_f, poses, cam, c['d'], c['sigma'],
                                    BV_predict=None if bv_pred is None else bv_pred.numpy())
                for nm, a, b in zip(NAMES4, full, o):
                    rec['oracle_' + nm + '_prob'] = dev(np.exp(a), np.exp(b))
                    rec['oracle_' + nm + '_log'] = dev(a, b)
                rec['oracle_depth_mm'] = 1000 * dev(dep, O.depth_val_regression(o[3], c['d']))
                rec['oracle_argmax_flips'] = int((full[3].argmax(1) != o[3].argmax(1)).sum())
                rel_t = T(poses)[0, r].inverse().numpy()
                rec['oracle_BV_predict_next_prob'] = dev(np.exp(bv_next.numpy()),
                                                         np.exp(O.propagate_dpv(o[3], rel_t, cam, c['d'])))
                rec['seconds_oracle'] = time.time() - to
                t0 += rec['seconds_oracle']
            rec['seconds_reference'] = time.time() - t0
            pin['cases'][key] = rec
            print(key, json.dumps(rec), flush=True)
            bv_pred = bv_next
        save_npz('configs_%s.npz' % name, out)
        save_npz('configs_priors_%s.npz' % name, priors)
        save_pin('PINNING_configs.json', pin)


def fixture_eval(*names):
    """eval_outputs.npz / PINNING_eval.json: KVNET in .eval() (running-statistics BatchNorm), for kvnet_256_d16 (first
    window + 2 steady steps) and c23_640x480_d64_v4_stream30 (first window + 1 steady step), or `names`, merged into the
    existing files. The running statistics are warmed first (warm_running_stats, stored as 'eval/<case>/rs/...'); every
    steady step is re-seeded with the reference's TRAIN-mode prior of the step before, which the repository already holds
    in full (any valid prior serves as the K-Net input). Stored per step as store_step does (8000 values per array). The
    eval-mode oracle, fed the same priors, is pinned in PINNING_eval.json (the fp32-vs-fp32 floor the GPU gates are set
    against). The reference's state_dict must be unchanged by the eval forwards."""
    pin = new_pin('torch', 'numpy', 'threads')
    out = load_existing(pin, 'PINNING_eval.json', 'eval_outputs.npz')
    for name in names or ['kvnet_256_d16', 'c23_640x480_d64_v4_stream30']:
        c = stream_case(name)
        camt = harness.cam_tensors(c['cam'])
        model = build_kvnet(c, camt, c['sd'])
        rec = dp_recorder(model)
        key = 'eval/%s' % name
        o, p = {}, {}
        sd, sd_np = warm_running_stats(model, rec, c, camt, o, key)
        record_steps(rec, c, camt, key, sd_np, False, name, o, p, timed=True)
        assert_unchanged(model, sd)
        p[key + '/state_dict_unchanged'] = True
        out = {k: v for k, v in out.items() if not k.startswith(key + '/')}
        out.update(o)
        pin['cases'].update(p)
        save_npz('eval_outputs.npz', out)
        save_pin('PINNING_eval.json', pin)


def fixture_refine(*names):
    """refine_outputs.npz / PINNING_refine.json: KVNET's other refinement configurations - refineNet_name='DGF'
    (guided-filter depth refinement, models/Refine.py:583-641), if_refined=False, and the depth-upsampled DPV R-Net
    (refineNet_name='DPV', if_upsample_d=True, Refine.py:44-48: refined DPVs of 4D planes).
      - state_dict: the reference's (key, shape) list of every configuration, including the default and the
        depth-upsampled DPV R-Net ('refine/sd/<config>'), so the mirror's module tree can be checked without the reference.
      - guided filter alone: RefineNet_DGF.forward on seeded inputs (tests/oracle_refine.py:gf_case) - ragged sizes, a
        textured guide, a guide that is flat over whole regions - stored in full ('refine/gf/<case>').
      - KVNET through the reference's own test() in train mode on stream_case's cases (or `names`, merged into the
        existing files), every steady step re-seeded with the reference's prior of the step before. The shared weights are
        the case's; the DGF weights come from arch.synth_state_dict(..., refine='DGF') / (..., upsample_d=True). Stored
        per step: strided samples (8000 values) of the low-resolution DPV (once: it does not depend on the refinement),
        of the DGF depth maps and of the 4D-plane refined DPVs, plus full-array statistics, and the expected depth of the
        refined DPV over the loaders' dup4_candi (np.linspace(d.min(), d.max(), 4D), scanNet.py:327).
    The deviations of tests/oracle_refine.py from the reference go to PINNING_refine.json:
      - oracle_dgf_m: the oracle's guided filter fed the reference's own low-resolution DPV (the filter alone);
      - oracle_fwd_dgf_m: the oracle's guided filter fed the numpy oracle's forward (oracle/kvnet_oracle.py, train mode),
        i.e. the fp32-vs-fp32 deviation a faithful DPV carries into the ill-conditioned filter. The GPU gates are
        multiples of it;
      - oracle_up_prob / oracle_up_depth_mm: the numpy oracle's forward (whose R-Net takes its widths from the weights)
        against the reference's 4D-plane refined DPV, in probability and in expected depth over dup4_candi."""
    from tests import oracle_refine as R
    m_refine, = reference('models.Refine')
    configs = {'none': dict(if_refined=False), 'DGF': dict(if_refined=True, refineNet_name='DGF'),
               'DPV_up': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True)}
    sd_configs = {'DPV': dict(if_refined=True, refineNet_name='DPV'),
                  'DPV_upsample_d': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True),
                  'DGF': dict(if_refined=True, refineNet_name='DGF'), 'none': dict(if_refined=False),
                  'none_DGF': dict(if_refined=False, refineNet_name='DGF')}

    def sub(a):
        return cases.subsample_to(a, 8000)

    pin = new_pin('torch', 'numpy', 'threads')
    out = load_existing(pin, 'PINNING_refine.json', 'refine_outputs.npz')
    c = cases.kvnet_case('kvnet_256_d16')
    camt = harness.cam_tensors(cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4))
    for nm, cfg in sd_configs.items():
        buf = io.StringIO()
        sd = build_kvnet(c, camt, printout=buf, **cfg).state_dict()
        out['refine/sd/%s/keys' % nm] = np.array(list(sd.keys()))
        out['refine/sd/%s/shapes' % nm] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
        out['refine/sd/%s/printed' % nm] = np.array([ln for ln in buf.getvalue().splitlines()
                                                     if ln.startswith(('KV-Net', 'with R-net', '\trefinement'))])

    for name in R.GF_CASES:
        g = R.gf_case(name)
        net = m_refine.RefineNet_DGF(3)
        net.load_state_dict({k[len('r_net.'):]: T(v) for k, v in g['sd'].items()})
        with torch.no_grad():
            y = net(T(g['dmap'][None, None]), T(g['img'][None]))[0, 0].numpy()
        out['refine/gf/%s/out' % name] = y
        o = R.dgf_refine(g['dmap'], g['img'], g['sd'])
        pin['cases']['gf/%s' % name] = {'oracle_m': dev(o, y), 'oracle_bitexact': bool(np.array_equal(o, y))}
        print('gf', name, pin['cases']['gf/%s' % name], flush=True)

    for name in names or ['kvnet_256_d16', 'c23_640x480_d64_v4_stream30']:
        c = stream_case(name)
        camt = harness.cam_tensors(c['cam'])
        sd_all = {k: np.asarray(v) for k, v in c['sd'].items() if not k.startswith('r_net.')}
        r_net_sd = {cfg: {k: v for k, v in arch.synth_state_dict(c['wseed'], 64, c['D'], c['t_win_r'], 64, **kw).items()
                          if k.startswith('r_net.')}
                    for cfg, kw in (('DGF', dict(refine='DGF')), ('DPV_up', dict(upsample_d=True)))}
        dup4 = np.linspace(c['d'].min(), c['d'].max(), 4 * len(c['d']))
        o_name, p_name = {}, {}
        for cfg_name, cfg in configs.items():
            sd = dict(sd_all, **r_net_sd.get(cfg_name, {}))
            rec = dp_recorder(build_kvnet(c, camt, sd, **cfg))
            key = 'refine/%s/%s' % (cfg_name, name)
            for k in range(c['n_steps']):
                t0 = time.time()
                prior = harness.reference_prior(name, k) if k else None
                (ref_f, src_f, poses), _ = test_step(rec, c, camt, c['t_win_r'] + k, prior, R_net=cfg_name != 'none')
                full = rec.last
                kk = '%s/step%d' % (key, k)
                row = {'seconds_reference': time.time() - t0}
                lowres = full[2] if k == 0 else full[3]
                if cfg_name == 'none':          # the low-resolution DPV does not depend on the refinement: stored once
                    o_name[kk + '/DPV'] = sub(lowres.numpy())
                    o_name[kk + '/DPV_stats'] = cases.stats(np.exp(lowres.numpy().astype(np.float64)))
                else:
                    assert np.array_equal(sub(lowres.numpy()), o_name['refine/none/%s/step%d/DPV' % (name, k)])
                if cfg_name == 'none':
                    assert full[0] == -1 and full[1] == -1
                elif cfg_name == 'DPV_up':
                    ref = (full[0] if k == 0 else full[1]).numpy()
                    assert ref.shape == (1, 4 * c['D'], c['H'], c['W']), ref.shape
                    o_name[kk + '/dpv_up'] = sub(ref[0])
                    o_name[kk + '/dpv_up_stats'] = cases.stats(np.exp(ref.astype(np.float64)))
                    dep = O.depth_val_regression(ref, dup4)[0]
                    o_name[kk + '/depth_dup4'] = sub(dep)
                    t1 = time.time()
                    fwd = N.kvnet_forward(sd, ref_f, src_f, poses, c['cam'], c['d'], c['sigma'], BV_predict=prior)
                    of = fwd[0] if k == 0 else fwd[1]
                    row['oracle_up_prob'] = dev(np.exp(of), np.exp(ref))
                    row['oracle_up_prob_sub'] = dev(np.exp(sub(of[0])), np.exp(sub(ref[0])))
                    row['oracle_up_depth_mm'] = 1000 * dev(O.depth_val_regression(of, dup4)[0], dep)
                    row['seconds_oracle'] = time.time() - t1
                else:
                    ref = (full[0] if k == 0 else full[1]).numpy()
                    assert ref.shape == (1, 1, c['H'], c['W']), ref.shape
                    o_name[kk + '/dmap'] = sub(ref[0, 0])
                    o_name[kk + '/dmap_stats'] = cases.stats(ref[0, 0])
                    if k:
                        o_name[kk + '/dmap_cur'] = sub(full[0].numpy()[0, 0])
                    o = R.kvnet_dgf_output(lowres.numpy()[0], ref_f[0], c['d'], sd)
                    row['oracle_dgf_m'] = dev(o, ref[0, 0])
                    t1 = time.time()
                    fwd = N.kvnet_forward(c['sd'], ref_f, src_f, poses, c['cam'], c['d'], c['sigma'], BV_predict=prior)
                    of = R.kvnet_dgf_output(fwd[2 if k == 0 else 3][0], ref_f[0], c['d'], sd)
                    row['oracle_fwd_dgf_m'] = dev(of, ref[0, 0])
                    row['oracle_fwd_dgf_m_sub'] = dev(sub(of), sub(ref[0, 0]))
                    row['seconds_oracle'] = time.time() - t1
                p_name[kk] = row
                print(kk, json.dumps(row), flush=True)
        out = {k: v for k, v in out.items() if not any(k.startswith('refine/%s/%s/' % (cf, name)) for cf in configs)}
        # 'none' runs first (the other configurations check their DPV against its), but is stored after 'DGF'
        out.update(sorted(o_name.items(), key=lambda kv: ('DGF', 'none', 'DPV_up').index(kv[0].split('/')[1])))
        pin['cases'].update(p_name)
        save_npz('refine_outputs.npz', out)
        save_pin('PINNING_refine.json', pin)


def fixture_twin():
    """twin_outputs.npz / PINNING_twin.json: KVNET at temporal window radii 1 and 3 (V = 2 and 6 source views), on the
    cases of tests/cases_twin.py (frames, poses and weights from synth / arch.synth_state_dict(..., t_win_r=r)), all driven
    through the reference's own test():
      - r1_256_d16, r3_256_d16: 256x256, D = 16, first window + 2 steady steps, in train mode and in .eval();
      - r1_640x480_d64: 640x480, D = 64, first window + 1 steady step, train mode.
    Every steady step is re-seeded with a train-mode prior of the reference that the repository already holds
    (cases_twin.prior). Eval mode first warms the reference's running statistics as the eval fixture does and stores them
    ('twin/eval/<case>/rs/<state_dict name>'). Stored per step as store_step does (8000 values per array). Also stored:
    the reference's state_dict (key, shape) list of KVNET(t_win_r=r) for r = 1..4 ('twin/sd/r<r>/...'). The deviations of
    the numpy oracle (train or eval mode) from the reference go to PINNING_twin.json. The npz is written with fixed member
    timestamps and no timings go to the JSON, so a re-run rewrites both byte for byte."""
    from tests import cases_twin as CT
    out = {}
    c = CT.twin_case('r1_256_d16')
    camt = harness.cam_tensors(CT.twin_cam(O.make_cam_intrinsics, c))
    for r in (1, 2, 3, 4):
        sd = build_kvnet(c, camt, t_win_r=r).state_dict()
        out['twin/sd/r%d/keys' % r] = np.array(list(sd.keys()))
        out['twin/sd/r%d/shapes' % r] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
    pin = new_pin('torch', 'numpy', 'threads')
    for name in CT.TWIN_CASES:
        c = CT.twin_case(name)
        c['cam'] = CT.twin_cam(O.make_cam_intrinsics, c)
        camt = harness.cam_tensors(c['cam'])
        model = build_kvnet(c, camt, c['sd'])
        rec = dp_recorder(model)
        model.train()
        prior_of = CT.TWIN_CFG[name]['prior_of']
        record_steps(rec, c, camt, 'twin/train/%s' % name, c['sd'], True, prior_of, out, pin['cases'])
        if name not in CT.EVAL_CASES:
            continue
        sd, sd_np = warm_running_stats(model, rec, c, camt, out, 'twin/eval/%s' % name)
        record_steps(rec, c, camt, 'twin/eval/%s' % name, sd_np, False, prior_of, out, pin['cases'])
        assert_unchanged(model, sd)
    save_npz('twin_outputs.npz', out, fixed=True)
    save_pin('PINNING_twin.json', pin, newline=True)


def fixture_f16():
    """f16_outputs.npz / PINNING_f16.json: conv_math='f16' (single fp16 products), the reference with its convolutions'
    operands rounded. For every case of tests/cases_f16.py the reference's own test() runs three times:
      - 'f16':  forward pre-hooks on every Conv2d / Conv3d / ConvTranspose2d the engine runs on tensor cores (all but the
                3-input-channel first layer) replace the input and the weight by x.half().float() for that call;
      - 'tf32': the same hooks with a 10-bit round-to-nearest significand (the reference's default GPU arithmetic, cuDNN
                TF32);
      - 'fp32': no hooks.
    Stored ('f16/<case>/step<k>/<arith>/...', arith f16 and fp32) as store_step does (cases_f16.SUB_LIMIT values per
    array); 'f16/hooked_layers' lists the hooked weights. PINNING_f16.json holds, per step and output, on full arrays:
      - 'oracle_vs_f16': tests/oracle_f16.py (numpy, the same rounding) against the f16-emulated reference - the floor F;
      - 'f16_vs_fp32', 'tf32_vs_fp32': the emulated references against the plain one;
    as probability, log-DPV, expected depth (mm) and argmax-flip deviations (cases_f16.deviations). Free-running steps
    feed each arithmetic its own propagated prior, and the oracle the f16-emulated reference's prior of that step.
    The npz is written with fixed member timestamps and no timings go to the JSON, so a re-run rewrites both byte for
    byte."""
    from tests import cases_f16 as CF
    from tests import oracle_f16 as OF
    rounding = {'f16': lambda t: t.half().float(), 'tf32': lambda t: T(CF.round_tf32(t.detach().numpy())), 'fp32': None}

    def hook(model, rnd):
        """Rounds the operands of every tensor-core convolution of `model`; returns (handles, hooked weight names)."""
        handles, names = [], []
        for n, m in model.named_modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.ConvTranspose2d)) and m.in_channels != 3:
                names.append(n + '.weight')

                def pre(mod, inp):
                    mod._w_full = mod.weight.data
                    mod.weight.data = rnd(mod._w_full)
                    return (rnd(inp[0]),) + tuple(inp[1:])

                def post(mod, inp, out):
                    mod.weight.data = mod._w_full

                handles += [m.register_forward_pre_hook(pre), m.register_forward_hook(post)]
        return handles, sorted(names)

    def run(c, camt, arith):
        """The case's steps in one arithmetic -> (per-step (inputs, prior, full outputs), hooked names)."""
        model = build_kvnet(c, camt, CF.state_dict(c))
        model.train(CF.MODE[c['name']] == 'train')
        handles, names = hook(model, rounding[arith]) if rounding[arith] else ([], [])
        rec = dp_recorder(model)
        steps, prior = [], None
        for k in range(c['n_steps']):
            if k and c['name'] not in CF.FREE_RUNNING:
                prior = CF.reseed_prior(c['name'], k)
            inputs, full, nxt = recorded_step(rec, c, camt, c['t_win_r'] + k, prior if k else None)
            steps.append((inputs, prior if k else None, full))
            prior = nxt
        for h in handles:
            h.remove()
        return steps, names

    out, pin = {}, new_pin('torch', 'numpy', 'threads')
    for name in CF.F16_CASES:
        c = CF.f16_case(name)
        cam = CF.cam(O.make_cam_intrinsics, c)
        camt = harness.cam_tensors(cam)
        res = {}
        for arith in ('f16', 'tf32', 'fp32'):
            res[arith], names = run(c, camt, arith)
            if arith == 'f16':
                out['f16/hooked_layers'] = np.array(names)
        sd = CF.state_dict(c)
        for k in range(c['n_steps']):
            kk = 'f16/%s/step%d' % (name, k)
            for arith in ('f16', 'fp32'):
                store_step(out, '%s/%s' % (kk, arith), res[arith][k][2], c['d'], k == 0, CF.SUB_LIMIT)
            (ref_f, src_f, poses), prior, full16 = res['f16'][k]
            o = OF.kvnet_forward(sd, ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=prior,
                                 training=CF.MODE[name] == 'train')
            rec = {'oracle_vs_f16': {nm: CF.deviations(b, a, c['d']) for nm, a, b in zip(NAMES4, full16, o)}}
            for arith in ('f16', 'tf32'):
                rec[arith + '_vs_fp32'] = {nm: CF.deviations(a, b, c['d'])
                                           for nm, a, b in zip(NAMES4, res[arith][k][2], res['fp32'][k][2])}
            pin['cases'][kk] = rec
            print(kk, json.dumps(rec), flush=True)
    save_npz('f16_outputs.npz', out, fixed=True)
    save_pin('PINNING_f16.json', pin, newline=True)


def fixture_drift(name='c23_640x480_d64_v4_stream30', n_steps=None):
    """PINNING_drift_<case>.json: how fast two fp32 implementations of the K-Net recursion drift apart (the floor for the
    free-running GPU gates); needs no reference. The numpy oracle runs FREE-RUNNING over the whole stream of a BIG case (or
    its first `n_steps` steps), feeding its own propagated prior exactly like the engine in tests/test_gpu_configs.py, and
    every step is compared with the committed outputs of the live reference (configs_<case>.npz), which was also
    free-running. Both are fp32; they differ only in summation order. The per-step deviations (probability of the filtered
    DPV / refined DPV / next prior, expected depth in mm) are the measured growth of rounding noise through the
    recursion, which no fp32 implementation can stay below."""
    gold = np.load(os.path.join(HERE, 'configs_%s.npz' % name))
    c = cases.big_case(name)
    cam = cases.big_cam(O.make_cam_intrinsics, c)
    r = c['t_win_r']
    rows = []
    prior = None
    for step in range(min(c['n_steps'], int(n_steps) if n_steps else 10 ** 9)):
        t0 = time.time()
        ref_f, src_f, poses = cases.window(c, r + step)
        o = N.kvnet_forward(c['sd'], ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=prior)
        rel = T(poses)[0, r].inverse().numpy()          # the same fp32 inverse the drivers use
        prior = O.propagate_dpv(o[3], rel, cam, c['d'])
        key = 'cfg/%s/step%d' % (name, step)
        thin = step >= cases.BIG_FULL_STEPS
        row = {'step': step}
        for nm, a in zip(NAMES4, o):
            k = '%s/%s' % (key, nm)
            if k in gold.files:
                row[nm + '_prob'] = dev(np.exp(cases.subsample_to(a, 30000) if thin else cases.subsample(a)), np.exp(gold[k]))
        row['depth_mm'] = 1000 * dev(cases.subsample_to(O.depth_val_regression(o[3], c['d']), 5000), gold[key + '/depth'])
        row['prior_next_prob'] = dev(np.exp(cases.subsample_to(prior, 30000)), np.exp(gold[key + '/BV_predict_next']))
        row['seconds'] = time.time() - t0
        rows.append(row)
        print(json.dumps(row), flush=True)
        save_pin('PINNING_drift_%s.json' % name, {'case': name, 'what': 'numpy oracle free-running vs live reference '
                                                  'free-running (both fp32)', 'steps': rows}, sort_keys=False)


def fixture_backward():
    """sweep_backward.npz / PINNING_backward.json: torch autograd through the reference's est_swp_volume_v4 - what
    train_utils/train_KVNet.py:149-153 differentiates - on cases.sweep_case inputs with a seeded upstream gradient
    (cases.sweep_grad): d loss / d feat_img_ref and d loss / d feat_img_src, and the oracle's deviation from them."""
    wh, = reference('warping.homography')
    out, pin = {}, new_pin('torch', 'numpy')
    for name in cases.SWEEP_BACKWARD_CASES:
        c = cases.sweep_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
        ref = T(c['ref']).clone().requires_grad_(True)
        src = T(c['src']).clone().requires_grad_(True)
        cost = wh.est_swp_volume_v4(ref, src, c['d'], T(c['R']), T(c['t']), harness.cam_tensors(cam), c['sigma'],
                                    feat_dist=c['feat_dist'])
        g = cases.sweep_grad(name, cost.shape)
        cost.backward(T(g))
        g_ref, g_src = ref.grad.numpy(), src.grad.numpy()
        out[name + '/g_ref'] = g_ref
        out[name + '/g_src'] = g_src
        o_ref, o_src = O.est_swp_volume_v4_backward(g, c['ref'], c['src'], c['d'], c['R'], c['t'], cam, c['sigma'],
                                                    c['feat_dist'])
        pin['cases'][name] = {
            'g_ref_maxabs': float(np.abs(o_ref - g_ref).max()), 'g_ref_max': float(np.abs(g_ref).max()),
            'g_src_maxabs': float(np.abs(o_src - g_src).max()), 'g_src_max': float(np.abs(g_src).max()),
        }
        print(name, pin['cases'][name])
    save_npz('sweep_backward.npz', out)
    save_pin('PINNING_backward.json', pin)


def fixture_camera():
    """camera_outputs.npz (a14): the reference's OWN intrinsics recipe and ray table. A ScanNet-style `_info.txt` is
    written for each calibration of cases.CAMERA_CASES and read by mdataloader/scanNet.py:read_IntM_from_txt (:204-272,
    which calls warping/View.py:32-62 normalised_pixel_to_ray_array); what it returned (hfov, vfov, focal_length,
    intrinsic_M, intrinsic_M_cuda, unit_ray_array_2D) is stored. tests/test_oracle_camera.py holds neuralrgbd_b200.camera
    and oracle.make_cam_intrinsics - the function every other fixture's inputs are built with - to these values bit for
    bit."""
    ref_scannet, = reference('mdataloader.scanNet')
    out = {}
    for name, c in cases.CAMERA_CASES.items():
        m = [c['fx'], 0, c['cx'], 0, 0, c['fy'], c['cy'], 0, 0, 0, 1, 0, 0, 0, 0, 1]
        info = '\n'.join([         # the 8 lines read_IntM_from_txt parses (SensReader's _info.txt layout)
            'm_versionNumber = 4', 'm_sensorName = synthetic', 'm_colorWidth = %d' % c['width'],
            'm_colorHeight = %d' % c['height'], 'm_depthWidth = %d' % c['width'], 'm_depthHeight = %d' % c['height'],
            'm_depthShift = 1000', 'm_calibrationColorIntrinsic = ' + ' '.join(repr(float(v)) for v in m)]) + '\n'
        with tempfile.NamedTemporaryFile('w', suffix='_info.txt', delete=False) as f:
            f.write(info)
            path = f.name
        cam = ref_scannet.read_IntM_from_txt(path, out_size=c['out_size'])
        os.unlink(path)
        out[name + '/scalars'] = np.array([cam['hfov'], cam['vfov'], cam['focal_length']], np.float64)
        out[name + '/intrinsic_M'] = np.asarray(cam['intrinsic_M'], np.float64)
        out[name + '/intrinsic_M_cuda'] = cam['intrinsic_M_cuda'].numpy()
        out[name + '/unit_ray_array_2D'] = cam['unit_ray_array_2D'].numpy()
        ura = np.asarray(cam['unit_ray_array'], np.float64)
        out[name + '/unit_ray_array_stats'] = np.array([ura.sum(), np.square(ura).sum(), ura[0, 0, 0], ura[-1, -1, 1]])
        print(name, out[name + '/scalars'])
    save_npz('camera_outputs.npz', out)


def fixture_export():
    """export_outputs.npz / PINNING_export.json: the output stage, the reference's export_res_img on cases.export_case
    inputs: its d_*.pgm / conf_*.pgm bytes and its float maps, and the oracle's deviations from them. matplotlib is not
    installed here; export_res.py imports it only to write preview PNGs, so a stub module with a no-op imsave stands in
    for it (the .pgm files, which are what is pinned, are written by PIL)."""
    from oracle import export_oracle as E
    mpl = types.ModuleType('matplotlib'); mpl.use = lambda *a, **k: None
    plt = types.ModuleType('matplotlib.pyplot'); plt.imsave = lambda *a, **k: None
    mpl.pyplot = plt
    sys.modules.setdefault('matplotlib', mpl); sys.modules.setdefault('matplotlib.pyplot', plt)
    ref_export, = reference('test_utils.export_res')
    out, pin = {}, new_pin('torch', 'numpy')
    for name in cases.EXPORT_CASES:
        bv, d_candi, img = cases.export_case(name)
        with tempfile.TemporaryDirectory() as tmp:
            ref_export.export_res_img({'img': T(img)}, T(bv), d_candi, tmp, 7)
            d_bytes = open(os.path.join(tmp, 'd_00007.pgm'), 'rb').read()
            c_bytes = open(os.path.join(tmp, 'conf_00007.pgm'), 'rb').read()
        D, H, W = bv.shape[1:]
        vol = torch.ones(1, D, H, W)
        for i in range(D):
            vol[0, i] = vol[0, i] * d_candi[i]
        dmap = ref_export.depth_regression(vol, T(bv)).astype(np.float32)
        conf = torch.exp(torch.max(T(bv), dim=1)[0]).squeeze().numpy()
        out[name + '/d_pgm'] = np.frombuffer(d_bytes, np.uint8)
        out[name + '/conf_pgm'] = np.frombuffer(c_bytes, np.uint8)
        out[name + '/dmap'] = dmap
        out[name + '/conf'] = conf
        od, oc, od16, oc16 = E.export_maps(bv[0], d_candi)
        hdr = b'P5\n%d %d\n65535\n' % (W, H)
        assert d_bytes.startswith(hdr) and c_bytes.startswith(hdr), 'unexpected PGM header from PIL'
        rd16 = np.frombuffer(d_bytes[len(hdr):], '>u2').reshape(H, W).astype(np.int64)
        rc16 = np.frombuffer(c_bytes[len(hdr):], '>u2').reshape(H, W).astype(np.int64)
        pin['cases'][name] = {
            'dmap_max_rel': float(np.max(np.abs(od - dmap) / np.maximum(np.abs(dmap), 1e-6))),
            'conf_max_rel': float(np.max(np.abs(oc - conf) / np.maximum(conf, 1e-6))),
            'dmap_u16_max_lsb': int(np.max(np.abs(od16.astype(np.int64) - rd16))),
            'conf_u16_max_lsb': int(np.max(np.abs(oc16.astype(np.int64) - rc16))),
            'dmap_u16_mismatch_frac': float(np.mean(od16.astype(np.int64) != rd16)),
            'pgm_bytes_equal_given_same_u16': bool(E.pgm16_bytes(rd16.astype(np.uint16)) == d_bytes),
        }
    save_npz('export_outputs.npz', out)
    save_pin('PINNING_export.json', pin)
    print(json.dumps(pin, indent=1))


def fixture_gf():
    """gf_outputs.npz / PINNING_gf.json: the reference's models/GF GuidedFilter and BoxFilter, forward and torch autograd,
    on the seeded cases of tests/cases_gf.py: GuidedFilter's output and the gradients of x and y, BoxFilter(r)'s output on
    y and its gradient, each recorded (record) against tests/oracle_gf.py. Both files are written with fixed member order
    and timestamps, so a re-run reproduces them."""
    from tests import cases_gf as CG
    from tests import oracle_gf as OG
    gf, box = reference('models.GF.guided_filter', 'models.GF.box_filter')
    torch.set_num_threads(8)
    out, pin = {}, new_pin('torch', 'numpy')
    for name in CG.CASES:
        c = CG.case(name)
        x, y = T(c['x']).clone().requires_grad_(True), T(c['y']).clone().requires_grad_(True)
        o = gf.GuidedFilter(c['r'], c['eps'])(x, y)
        o.backward(T(c['g']))
        key = 'gf/' + name
        record(out, pin, key + '/out', o.detach().numpy(), OG.guided_filter(c['x'], c['y'], c['r'], c['eps']), CG.sub)
        gx, gy = OG.guided_filter_backward(c['g'], c['x'], c['y'], c['r'], c['eps'])
        record(out, pin, key + '/g_x', x.grad.numpy(), gx, CG.sub)
        record(out, pin, key + '/g_y', y.grad.numpy(), gy, CG.sub)

        yb = T(c['y']).clone().requires_grad_(True)
        ob = box.BoxFilter(c['r'])(yb)
        ob.backward(T(c['g_box']))
        key = 'box/' + name
        record(out, pin, key + '/out', ob.detach().numpy(), OG.box_filter(c['y'], c['r']), CG.sub)
        record(out, pin, key + '/g_x', yb.grad.numpy(), OG.box_filter_backward(c['g_box'], c['r']), CG.sub)
    save_npz('gf_outputs.npz', out, fixed=True)
    save_pin('PINNING_gf.json', pin, newline=True)


def fixture_grad():
    """grad_outputs.npz / PINNING_grad.json: torch autograd through the reference's warp_img_feats_v3 (list and tensor
    forms), resample_vol_cuda (+ the clamp of test_utils/test_KVNet.py:58-59) and mutils.misc.depth_val_regression, on the
    seeded cases of tests/cases_grad.py: each gradient recorded (record, as '<case>/g') against tests/oracle_grad.py.
    Both files are written with fixed member order and timestamps, so a re-run reproduces them."""
    from tests import cases_grad as CG
    from tests import oracle_grad as OG
    wh, m_misc = reference('warping.homography', 'mutils.misc')
    torch.set_num_threads(8)
    out, pin = {}, new_pin('torch', 'numpy')
    for name in CG.WARP_CASES:
        c = CG.warp_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
        camt = harness.cam_tensors(cam)
        if c['tensor']:
            img = T(c['imgs']).clone().requires_grad_(True)
            res = wh.warp_img_feats_v3(img, c['d'], T(c['R']), T(c['t']), camt)
            (res * T(c['grads'])).sum().backward()
            g = img.grad.numpy()
            o = OG.warp_img_feats_backward([c['grads']], c['d'], [c['R']], [c['t']], cam, c['h'], c['w'])[0]
        else:
            imgs = [T(i).clone().requires_grad_(True) for i in c['imgs']]
            res = wh.warp_img_feats_v3(imgs, c['d'], [T(r) for r in c['R']], [T(t) for t in c['t']], camt)
            sum((r * T(gv)).sum() for r, gv in zip(res, c['grads'])).backward()
            g = np.concatenate([i.grad.numpy() for i in imgs])
            o = np.concatenate(OG.warp_img_feats_backward(c['grads'], c['d'], c['R'], c['t'], cam, c['h'], c['w']))
        del res
        record(out, pin, 'warp/' + name, g, o, CG.sub, '/g')

    for name in CG.RESAMPLE_CASES:
        c = CG.resample_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
        vol = T(c['vol']).clone().requires_grad_(True)
        res = wh.resample_vol_cuda(vol, T(c['rel']), harness.cam_tensors(cam), c['d'], c['d_new'], padding_value=c['pad'])
        if c['clamp'] is not None:
            res = res.clamp(min=c['clamp'][0], max=c['clamp'][1])
        res.backward(T(c['grad']))
        o = OG.resample_vol_cuda_backward(c['grad'], c['vol'], c['rel'], cam, c['d'], c['d_new'], c['pad'], c['clamp'])
        record(out, pin, 'resample/' + name, vol.grad.numpy(), o, CG.sub, '/g')

    for name in CG.REGRESSION_CASES:
        c = CG.regression_case(name)
        bv = T(c['bv']).clone().requires_grad_(True)
        m_misc.depth_val_regression(bv, c['d'], BV_log=c['log']).backward(T(c['grad']))
        o = OG.depth_val_regression_backward(c['grad'], c['bv'], c['d'], c['log'])
        record(out, pin, 'regression/' + name, bv.grad.numpy(), o, CG.sub, '/g')
    save_npz('grad_outputs.npz', out, fixed=True)
    save_pin('PINNING_grad.json', pin, newline=True)


def fixture_lba():
    """lba_outputs.npz / PINNING_lba.json: the LBA depth-map back-warp (SURVEY 8 f-3), the reference's back_warp_th_Rt /
    back_warp_th_Rt_msrc (warping/homography.py:479-574), with the single-view warp differentiated w.r.t. R, t and the
    image by torch autograd - what ICP/opt_pose_numerical.py does - and the oracle's deviations."""
    wh, = reference('warping.homography')
    out, pin = {}, new_pin('torch')
    for name in cases.LBA_CASES:
        c = cases.lba_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
        camt = harness.cam_tensors(cam)
        multi = wh.back_warp_th_Rt_msrc(T(c['imgs']), T(c['dmap']), T(c['Rs']), T(c['ts']), camt).numpy()
        R = T(c['Rs'][0]).clone().requires_grad_(True); t = T(c['ts'][0]).clone().requires_grad_(True)
        img = T(c['imgs'][:1]).clone().requires_grad_(True)
        single = wh.back_warp_th_Rt(img, T(c['dmap']), R, t, camt)
        g = np.random.RandomState(7).standard_normal(tuple(single.shape)).astype(np.float32)
        single.backward(T(g))
        out[name + '/warp_msrc'] = multi
        out[name + '/grad_out'] = g
        out[name + '/g_R'] = R.grad.numpy(); out[name + '/g_t'] = t.grad.numpy(); out[name + '/g_img'] = img.grad.numpy()
        o_multi = O.back_warp_th_Rt_msrc(c['imgs'], c['dmap'], c['Rs'], c['ts'], cam)
        gR, gt, gi = O.back_warp_th_Rt_backward(g, c['imgs'][:1], c['dmap'], c['Rs'][0], c['ts'][0], cam)
        pin['cases'][name] = {'warp_maxabs': float(np.abs(o_multi - multi).max()),
                              'single_equals_msrc_view0': float(np.abs(single.detach().numpy() - multi[:1]).max()),
                              'g_R_rel': float(np.abs(gR - out[name + '/g_R']).max() / np.abs(out[name + '/g_R']).max()),
                              'g_t_rel': float(np.abs(gt - out[name + '/g_t']).max() / np.abs(out[name + '/g_t']).max()),
                              'g_img_maxabs': float(np.abs(gi - out[name + '/g_img']).max())}
    save_npz('lba_outputs.npz', out)
    save_pin('PINNING_lba.json', pin)
    print(json.dumps(pin, indent=1))


def fixture_lba_opt():
    """lba_opt_outputs.npz / PINNING_lba_opt.json: the LBA pose optimiser (ICP/opt_pose_numerical.py local_BA_direct /
    local_BA_direct_parallel) on the scenes of tests/cases_lba_opt.py:lba_opt_case. Per case: the returned poses, the
    printed lines, Rotation2UnitQ / UnitQ2Rotation of the initial poses and, for every Adam step (torch.optim.Adam.step is
    wrapped here, and only while this fixture runs), the parameters, gradients and Adam state before and after it and the
    L1 loss the iteration evaluated (nn.L1Loss.forward is wrapped too); and the oracle's deviations from the reference."""
    from oracle import lba_opt_oracle as LO
    from tests import cases_lba_opt as LC
    ref_opt, ref_misc = reference('ICP.opt_pose_numerical', 'mutils.misc')
    steps_rec, losses = [], []
    adam_step, l1_forward = torch.optim.Adam.step, torch.nn.L1Loss.forward

    def snap(self, *a, **k):
        ps = [p for g in self.param_groups for p in g['params']]
        st = [self.state.get(p, {}) for p in ps]
        rec = {'p': [p.detach().clone().numpy() for p in ps], 'g': [p.grad.clone().numpy() for p in ps],
               'm': [s['exp_avg'].clone().numpy() if 'exp_avg' in s else np.zeros(tuple(p.shape), np.float32)
                     for p, s in zip(ps, st)],
               'v': [s['exp_avg_sq'].clone().numpy() if 'exp_avg_sq' in s else np.zeros(tuple(p.shape), np.float32)
                     for p, s in zip(ps, st)],
               'lr': self.param_groups[0]['lr']}
        out = adam_step(self, *a, **k)
        rec['p1'] = [p.detach().clone().numpy() for p in ps]
        rec['m1'] = [self.state[p]['exp_avg'].clone().numpy() for p in ps]
        rec['v1'] = [self.state[p]['exp_avg_sq'].clone().numpy() for p in ps]
        steps_rec.append(rec)
        return out

    def loss(self, a, b):
        out = l1_forward(self, a, b)
        losses.append(float(out.detach()))
        return out

    def run_reference(c):
        del steps_rec[:], losses[:]
        fn = ref_opt.local_BA_direct_parallel if c['entry'] == 'parallel' else ref_opt.local_BA_direct
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            poses = fn(T(c['ref']), [T(s) for s in c['srcs']], T(c['dmap']), T(c['conf']),
                       [harness.cam_tensors(k) for k in c['cams']], c['dw_scales'], list(c['poses_init']), c['max_iter'],
                       c['step'], c['opt_vars'])
        return np.stack([p.numpy() for p in poses]), buf.getvalue().splitlines()

    def per_step(c):
        """Steps as arrays [S, V, 3] for 't' / 'u' (whichever Adam updates), loss [S, V] (serial) or [S, 1] (parallel)."""
        V, S = len(c['srcs']), 3 * c['max_iter']
        names = {(0, 1): ['t'], (0, 0): ['t'], (1, 1): ['t', 'u'], (1, 0): ['u']}[tuple(c['opt_vars'])]
        out = {}
        serial = c['entry'] == 'serial'
        for j, nm in enumerate(names):
            for key in ('p', 'g', 'm', 'v', 'p1', 'm1', 'v1'):
                a = np.stack([np.asarray(r[key][j], np.float32).reshape(-1, 3) for r in steps_rec])   # [V*S or S, 1 or V, 3]
                out['%s/%s' % (key, nm)] = a.reshape(V, S, 3).transpose(1, 0, 2) if serial else a
        out['lr'] = np.array([r['lr'] for r in steps_rec][:S])
        la = np.asarray(losses, np.float32)
        out['loss'] = la.reshape(V, S).T if serial else la.reshape(S, 1)
        return out

    def one_step_deviation(c, steps):
        """The oracle's iteration started from every recorded reference state: its gradients (relative to the largest
        reference gradient) and the parameters after its Adam step, against the reference's."""
        levels = LO.pyramid(c['ref'], c['srcs'], c['dmap'], c['conf'], c['dw_scales'])
        init = [LO.init_state(p) for p in c['poses_init']]
        names = [nm for nm in ('t', 'u') if 'g/' + nm in steps]
        S = steps['g/' + names[0]].shape[0]
        d = {}
        for nm in names:
            d['grad_%s_rel' % nm] = 0.0
            d['step_%s_maxabs' % nm] = 0.0
        for k in range(S):
            states = []
            for v, x0 in enumerate(init):
                x = dict(x0)
                for nm in names:
                    x[nm] = steps['p/' + nm][k][v]
                x['R'] = LO.unitq_to_rotation(x['u'])
                states.append(x)
            _, g_u, g_t = LO.gradients(levels[k // c['max_iter']], states, c['cams'][k // c['max_iter']],
                                       c['entry'] == 'parallel')
            for nm, g in (('t', g_t), ('u', g_u)):
                if nm not in names:
                    continue
                g_ref = steps['g/' + nm][k]
                d['grad_%s_rel' % nm] = max(d['grad_%s_rel' % nm], float(np.abs(g - g_ref).max() / np.abs(g_ref).max()))
                p1, _, _ = LO.adam_step(steps['p/' + nm][k], g, steps['m/' + nm][k], steps['v/' + nm][k], k + 1,
                                        c['step'] / 2 ** (k // c['max_iter']))
                d['step_%s_maxabs' % nm] = max(d['step_%s_maxabs' % nm], float(np.abs(p1 - steps['p1/' + nm][k]).max()))
        return d

    out, pin = {}, new_pin('torch')
    torch.optim.Adam.step, torch.nn.L1Loss.forward = snap, loss
    try:
        for name in LC.LBA_OPT_CASES:
            c = LC.lba_opt_case(name)
            poses, lines = run_reference(c)
            steps = per_step(c)
            out[name + '/poses'] = poses
            out[name + '/printed'] = np.array(lines)
            for k, a in steps.items():
                out[name + '/' + k] = a
            init_u = np.stack([ref_misc.Rotation2UnitQ(T(np.ascontiguousarray(p[:3, :3]))).numpy() for p in c['poses_init']])
            out[name + '/init_u'] = init_u
            out[name + '/init_R'] = np.stack([ref_misc.UnitQ2Rotation(T(u)).numpy() for u in init_u])
            rec = []
            o_poses = np.stack(LO.local_ba(c['ref'], c['srcs'], c['dmap'], c['conf'], c['cams'], c['dw_scales'],
                                           c['poses_init'], c['max_iter'], c['step'], c['opt_vars'], c['entry'] == 'parallel',
                                           record=rec))
            d = {'final_pose_maxabs': float(np.abs(o_poses - poses).max()),
                 'init_pose_error': float(np.abs(c['poses_init'] - c['poses_true']).max()),
                 'final_pose_error_reference': float(np.abs(poses - c['poses_true']).max())}
            d.update(one_step_deviation(c, steps))
            pin['cases'][name] = d
            print(name, json.dumps(d), flush=True)
    finally:
        torch.optim.Adam.step, torch.nn.L1Loss.forward = adam_step, l1_forward
    save_npz('lba_opt_outputs.npz', out)
    save_pin('PINNING_lba_opt.json', pin)


def fixture_preprocess():
    """preprocess_outputs.npz / PINNING_preprocess.json: the input stage, the reference's own transform
    (mdataloader.m_preprocess.get_transform, i.e. torchvision ToTensor + Normalize) applied after PIL's NEAREST resize,
    exactly as mdataloader/scanNet.py:368-369,438 do, and the oracle's deviations (expected: 0)."""
    import PIL
    import PIL.Image
    import torchvision
    from oracle import preprocess_oracle as P
    ref_pre, = reference('mdataloader.m_preprocess')
    out = {}
    pin = {'pillow': PIL.__version__, 'torchvision': torchvision.__version__, 'torch': torch.__version__, 'cases': {}}
    tf = ref_pre.get_transform()
    for name in cases.PREPROCESS_CASES:
        img, size = cases.preprocess_case(name)
        pil = PIL.Image.fromarray(img)
        if size is not None:
            pil = pil.resize(size, PIL.Image.NEAREST)              # scanNet.py:369
        ref = tf(pil).unsqueeze_(0).numpy()                        # scanNet.py:438, :446 ('img': img.unsqueeze_(0))
        out[name] = ref
        mine = P.preprocess(img, size)
        pin['cases'][name] = {'bit_identical': bool(np.array_equal(mine, ref)), 'maxabs': float(np.abs(mine - ref).max())}
    save_npz('preprocess_outputs.npz', out)
    save_pin('PINNING_preprocess.json', pin)
    print(json.dumps(pin, indent=1))


def fixture_stats():
    """stats_outputs.npz / PINNING_stats.json: the reference's mutils.misc.depth_var and dpv_statistics, forward and torch
    autograd, on the seeded cases of tests/cases_stats.py: each output and gradient recorded (record) against
    tests/oracle_stats.py, and the plane indices torch.max / torch.min select inside dpv_statistics (misc.py:600-603) as
    uint8, in full for the tie case. Both files are written with fixed member order and timestamps, so a re-run
    reproduces them."""
    from tests import cases_stats as CS
    from tests import oracle_stats as OS
    m_misc, = reference('mutils.misc')
    full_index = ('prior_pad_120x160_d64',)     # the tie case keeps every index, its border pixels included
    torch.set_num_threads(8)
    out, pin = {}, new_pin('torch', 'numpy')
    for name in CS.CASES:
        c = CS.case(name)
        bv0, d, log = c['bv'], c['d'], c['log']
        # depth_var with the expected depth as its mean, as train_utils/train_KVNet.py:137-138 calls it
        mean0 = c['mean']
        bv, mean = T(bv0).clone().requires_grad_(True), T(mean0).clone().requires_grad_(True)
        var = m_misc.depth_var(bv, mean, d, BV_log=log, d_sigma=c['sigma'])
        var.backward(T(c['g_var']))
        key = 'var/' + name
        record(out, pin, key + '/out', var.detach().numpy(), OS.depth_var(bv0, mean0, d, log, c['sigma']), CS.sub)
        g_bv, g_mu = OS.depth_var_backward(c['g_var'], bv0, mean0, d, log, c['sigma'])
        record(out, pin, key + '/g_bv', bv.grad.numpy(), g_bv, CS.sub)
        record(out, pin, key + '/g_mean', mean.grad.numpy(), g_mu.reshape(mean0.shape), CS.sub)

        # dpv_statistics, differentiated through every channel (the variance's mean included)
        bv = T(bv0).clone().requires_grad_(True)
        feats = m_misc.dpv_statistics(bv, d, c['stats'], BV_log=log)
        feats.backward(T(c['g_stats']))
        of, parts = OS.dpv_statistics(bv0, d, c['stats'], log)
        key = 'stats/' + name
        record(out, pin, key + '/out', feats.detach().numpy(), of, CS.sub)
        record(out, pin, key + '/g_bv', bv.grad.numpy(), OS.dpv_statistics_backward(c['g_stats'], bv0, d, parts, log), CS.sub)
        # the planes the reference's max / min pick (misc.py:600-603 compute them and drop them)
        p = torch.exp(T(bv0)) if log else T(bv0)
        for kind, fn in (('argmax', torch.max), ('argmin', torch.min if log else torch.max)):
            idx = fn(p, dim=1)[1].numpy()
            out[key + '/' + kind] = idx.astype(np.uint8) if name in full_index else CS.sub(idx).astype(np.uint8)
            orc = OS.extreme(bv0, log, kind == 'argmin' and log)[1]
            pin['cases'][key + '/' + kind] = {'mismatch_oracle': int((orc != idx).sum()), 'shape': list(idx.shape)}
            print(key + '/' + kind, pin['cases'][key + '/' + kind], flush=True)
    save_npz('stats_outputs.npz', out, fixed=True)
    save_pin('PINNING_stats.json', pin, newline=True)


FIXTURES = {     # in dependency order
    'reference': fixture_reference, 'configs': fixture_configs, 'eval': fixture_eval, 'refine': fixture_refine,
    'twin': fixture_twin, 'f16': fixture_f16, 'drift': fixture_drift, 'backward': fixture_backward,
    'camera': fixture_camera, 'export': fixture_export, 'gf': fixture_gf, 'grad': fixture_grad, 'lba': fixture_lba,
    'lba_opt': fixture_lba_opt, 'preprocess': fixture_preprocess, 'stats': fixture_stats,
}


def main():
    global REF_CODE
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--ref', help="the reference's code/ directory (default: oracle/fetch_reference.py:code_dir())")
    ap.add_argument('fixture', choices=list(FIXTURES) + ['all'])
    ap.add_argument('cases', nargs='*', help='eval, refine, configs: the cases to (re)write; drift: [case] [n_steps]')
    args = ap.parse_args()
    REF_CODE = args.ref
    warnings.filterwarnings('ignore')
    if args.fixture == 'all':
        assert not args.cases, '`all` takes no cases'
        for fn in FIXTURES.values():
            fn()
    else:
        FIXTURES[args.fixture](*args.cases)


if __name__ == '__main__':
    main()
