"""Seeded KVNET cases at temporal window radii other than 2 (numpy only).

KVNET(t_win_r=r) reads V = 2r source views per reference frame, and K-Net's first layer takes 3(2r + 1) + 1 = 3V + 4
channels: 10 at r = 1, 22 at r = 3 (16 at the default r = 2, 28 at r = 4). Shared by tests/golden/make_golden_twin.py (which
runs the unmodified reference on them) and the tests. Every input is regenerated from its seed.

Steady steps are re-seeded with a train-mode prior of the reference that the repository already holds at the same
(D, h, w): the r = 2 case of the same frame size (reference_outputs.npz, configs_priors_<case>.npz). A prior is a
[1, D, h, w] log-DPV and does not depend on the window radius, so any valid one serves as K-Net's input.
"""
from neuralrgbd_b200 import arch, synth
from tests import cases, harness

TWIN_CFG = {
    'r1_256_d16': dict(seed=71, H=256, W=256, D=16, t_win_r=1, wseed=5, n_steps=3, prior_of='kvnet_256_d16'),
    'r3_256_d16': dict(seed=73, H=256, W=256, D=16, t_win_r=3, wseed=5, n_steps=3, prior_of='kvnet_256_d16'),
    # the BASELINE frame size and plane count (configs[1] / [2]) at the smallest radius
    'r1_640x480_d64': dict(seed=75, H=480, W=640, D=64, t_win_r=1, wseed=7, n_steps=2,
                           prior_of='c23_640x480_d64_v4_stream30'),
}
TWIN_CASES = list(TWIN_CFG)
EVAL_CASES = ['r1_256_d16', 'r3_256_d16']      # also recorded in .eval()


def twin_case(name):
    """-> dict(frames, exts, sd, d, H, W, D, sigma, t_win_r, n_steps) for cases.window; frames t_win_r + k, k < n_steps,
    are the reference frames of the recorded steps."""
    cfg = TWIN_CFG[name]
    r = cfg['t_win_r']
    nf = cfg['n_steps'] + 2 * r
    frames, rng = synth.video(cfg['seed'], nf, cfg['H'], cfg['W'])
    exts = synth.camera_track(rng, nf)
    sd = arch.synth_state_dict(cfg['wseed'], 64, cfg['D'], r, 64)
    return dict(frames=frames, exts=exts, sd=sd, d=synth.d_candidates(cfg['D']), H=cfg['H'], W=cfg['W'], D=cfg['D'],
                sigma=10.0, t_win_r=r, n_steps=cfg['n_steps'], wseed=cfg['wseed'])


def twin_cam(make_cam, c):
    """The 7-Scenes pinhole (cases.FX, ...) at the case's quarter resolution."""
    return cases.cam_for(make_cam, c['W'] // 4, c['H'] // 4)


def prior(name, step):
    """The reference's train-mode prior that re-seeds steady step `step` >= 1 of case `name`."""
    return harness.reference_prior(TWIN_CFG[name]['prior_of'], step)
