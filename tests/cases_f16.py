"""Seeded cases of conv_math='f16' (numpy only): shared by tests/golden/make_golden_f16.py, which runs the unmodified
reference on them with its convolutions' operands rounded, and by the tests.

Arithmetic emulated on the reference (forward pre-hooks on the convolution modules):
  - 'f16':  input and weight of every convolution the engine runs on tensor cores replaced by RN_f16(.) (x.half().float());
  - 'tf32': the same layers with a 10-bit round-to-nearest significand (TF32), standing in for the reference's default GPU
            arithmetic (cuDNN with allow_tf32);
  - 'fp32': no hook.
The engine runs every convolution on tensor cores except the feature CNN's first layer, whose input has 3 channels.

Cases (steps: 0 = first window):
  - c2_640x480_d64: the C2/C3 frame, V = 4, D = 64: first window + one steady step re-seeded with the reference's
    train-mode prior (configs_priors_c23_640x480_d64_v4_stream30.npz);
  - stream_256_d16: 256x256, D = 16, 6 frames free-running in train mode (each step fed the arithmetic's own propagated
    prior);
  - eval_256_d16: kvnet_256_d16 in .eval() with the running statistics make_golden_eval.py warmed (eval_outputs.npz):
    first window + one steady step re-seeded with the train-mode prior of reference_outputs.npz;
  - r1_256_d16: t_win_r = 1 (V = 2), train mode: first window + one re-seeded steady step.
"""
import os

import numpy as np

from neuralrgbd_b200 import arch, synth
from tests import cases
from tests import cases_twin as CT

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
F16_CASES = ['c2_640x480_d64', 'stream_256_d16', 'eval_256_d16', 'r1_256_d16']
MODE = {'c2_640x480_d64': 'train', 'stream_256_d16': 'train', 'eval_256_d16': 'eval', 'r1_256_d16': 'train'}
FREE_RUNNING = {'stream_256_d16'}
SUB_LIMIT = 4000          # values per stored output array (strided, cases.subsample_to)
DEPTH_LIMIT = 2000
STORED = {True: ('BV_cur', 'dmap_cur_refined'), False: ('DPV', 'dmap_refined')}    # first window: / steady step:
NAMES4 = ['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV']


def f16_case(name):
    """-> dict(frames, exts, sd, d, H, W, D, sigma, t_win_r, n_steps, cam_args) for cases.window."""
    if name == 'c2_640x480_d64':
        c = cases.big_case('c23_640x480_d64_v4_stream30')
        c['n_steps'] = 2
    elif name == 'stream_256_d16':
        frames, rng = synth.video(81, 10, 256, 256)
        c = dict(frames=frames, exts=synth.camera_track(rng, 10), sd=arch.synth_state_dict(5, 64, 16, 2, 64),
                 d=synth.d_candidates(16), H=256, W=256, D=16, sigma=10.0, t_win_r=2, n_steps=6)
    elif name == 'eval_256_d16':
        c = cases.kvnet_case('kvnet_256_d16')
        c['n_steps'] = 2
    else:
        c = CT.twin_case('r1_256_d16')
        c['n_steps'] = 2
    c['name'] = name
    return c


def cam(make_cam, c):
    if c['name'] == 'c2_640x480_d64':
        return cases.big_cam(make_cam, c)
    return cases.cam_for(make_cam, c['W'] // 4, c['H'] // 4)


def running_stats():
    """The running statistics make_golden_eval.py warmed for kvnet_256_d16 (state_dict name -> array)."""
    g = np.load(os.path.join(GOLDEN, 'eval_outputs.npz'))
    pre = 'eval/kvnet_256_d16/rs/'
    return {k[len(pre):]: np.asarray(g[k]) for k in g.files if k.startswith(pre)}


def state_dict(c):
    sd = {k: np.asarray(v) for k, v in c['sd'].items()}
    if MODE[c['name']] == 'eval':
        sd.update(running_stats())
    return sd


def reseed_prior(name, step):
    """The reference's train-mode prior of a re-seeded steady step (step 1 of the non-streaming cases)."""
    assert step == 1 and name not in FREE_RUNNING
    if name == 'c2_640x480_d64':
        return np.load(os.path.join(GOLDEN, 'configs_priors_c23_640x480_d64_v4_stream30.npz'))[
            'cfg/c23_640x480_d64_v4_stream30/step0/BV_predict_next_full']
    if name == 'eval_256_d16':
        return np.load(os.path.join(GOLDEN, 'reference_outputs.npz'))['kvnet/kvnet_256_d16/step0/BV_predict_next_full']
    return CT.prior('r1_256_d16', 1)


def tc_layers(specs):
    """Names of the convolution weights the engine runs on tensor cores, from arch.kvnet_param_specs: every convolution
    weight (4-D / 5-D) except the 3-input-channel first layer of the feature CNN."""
    out = []
    for n, s, kind in specs:
        if len(s) < 4 or not n.endswith('.weight') or n.startswith('d_net.'):
            continue
        cin = s[0] if '.trans_conv' in n else s[1]
        if cin != 3:
            out.append(n)
    return sorted(out)


def round_tf32(a):
    """float32 -> the nearest value with a 10-bit significand (round to nearest even), numpy."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    r = (u + np.uint32(0xFFF) + ((u >> np.uint32(13)) & np.uint32(1))) & np.uint32(0xFFFFE000)
    return r.view(np.float32)


def deviations(a, b, d):
    """Deviation of log-DPV a from log-DPV b ([1, D, H, W]): probability, log-DPV (finite entries), expected depth (mm) and
    the fraction of pixels whose most likely plane differs."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    pa, pb = np.exp(a), np.exp(b)
    fin = np.isfinite(a) & np.isfinite(b)
    da = (pa * np.asarray(d, np.float64).reshape(1, -1, 1, 1)).sum(1)
    db = (pb * np.asarray(d, np.float64).reshape(1, -1, 1, 1)).sum(1)
    return {'prob': float(np.max(np.abs(pa - pb))), 'log': float(np.max(np.abs(a - b)[fin])) if fin.any() else 0.0,
            'depth_mm': 1000.0 * float(np.max(np.abs(da - db))), 'argmax_flips': float(np.mean(a.argmax(1) != b.argmax(1)))}
