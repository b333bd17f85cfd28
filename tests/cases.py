"""Seeded input builders for the parity cases (numpy only).

Shared by tests/golden/make_golden.py (which runs the LIVE reference on them in the
build container and commits its outputs) and by the tests (which run the oracle and
the CUDA path on the same inputs).  Every input is regenerated from its seed, so the
fixtures hold reference OUTPUTS only.
"""
import math
import numpy as np

from neuralrgbd_b200 import synth, arch

FX = FY = 585.0          # DSO/cam_info_7scenes.mat: 640x480, fx=fy=585, cx=320, cy=240
CX, CY = 320.0, 240.0


def cam_for(make_cam, w, h):
    return make_cam(FX, FY, CX, CY, [w, h])


def _feat_pair(rng, C, h, w, V, mix=0.7):
    ref = synth.smooth_image(rng, C, h, w)
    src = np.stack([mix * ref + (1 - mix) * synth.smooth_image(rng, C, h, w) for _ in range(V)])
    return ref[None], src[None]


def _poses(rng, V, step_t=0.03, step_rot=0.7):
    """V relative poses E_src . E_ref^-1 around a reference in the middle of a track."""
    exts = synth.camera_track(rng, V + 1, step_t, step_rot)
    r = V // 2
    inv_ref = np.linalg.inv(exts[r])
    return np.stack([exts[i].dot(inv_ref) for i in range(V + 1) if i != r]).astype(np.float32)


def sweep_case(name):
    """-> dict(ref, src, d, R, t, w, h, sigma, feat_dist)."""
    cfg = {
        # BASELINE.json configs[0]: 320x256 ref + 1 source, 32 planes, C=67
        'c1_320x256_v1_d32_c67': dict(seed=11, h=256, w=320, C=67, V=1, D=32, dist='L2'),
        'c1_320x256_v1_d32_c3': dict(seed=12, h=256, w=320, C=3, V=1, D=32, dist='L2'),
        'small_v4_d32_c67_L2': dict(seed=13, h=64, w=80, C=67, V=4, D=32, dist='L2'),
        'small_v4_d32_c67_L1': dict(seed=13, h=64, w=80, C=67, V=4, D=32, dist='L1'),
        'bwd_v2_d8_c67_L2': dict(seed=17, h=40, w=56, C=67, V=2, D=8, dist='L2'),
        'bwd_v2_d8_c67_L1': dict(seed=17, h=40, w=56, C=67, V=2, D=8, dist='L1'),
        'ragged_v3_d7_c5': dict(seed=14, h=37, w=53, C=5, V=3, D=7, dist='L2'),
        # d_min = 0 plane (test_KVNet.py:58 default) and a camera moved *behind* the
        # reference so that P_z <= 0 for near planes (the +1e-10 path, homography.py:438)
        'dzero_behind_v2_d16_c8': dict(seed=15, h=48, w=64, C=8, V=2, D=16, dist='L2', d_min=0.0,
                                        d_max=2.0, step_t=0.6),
        'identity_v1_d8_c16': dict(seed=16, h=48, w=64, C=16, V=1, D=8, dist='L2', identity=True),
    }[name]
    rng = np.random.RandomState(cfg['seed'])
    ref, src = _feat_pair(rng, cfg['C'], cfg['h'], cfg['w'], cfg['V'])
    poses = _poses(rng, cfg['V'], cfg.get('step_t', 0.03))
    if cfg.get('identity'):
        poses = np.stack([np.eye(4, dtype=np.float32)] * cfg['V'])
        src = np.repeat(ref[:, None], cfg['V'], axis=1)
    if 'step_t' in cfg:       # push the source cameras along +z of the reference (points fall behind)
        poses[:, 2, 3] += np.float32(0.5)
    d = synth.d_candidates(cfg['D'], cfg.get('d_min', 0.1), cfg.get('d_max', 5.0))
    return dict(ref=ref, src=src, d=d, R=np.ascontiguousarray(poses[:, :3, :3]),
                t=np.ascontiguousarray(poses[:, :3, 3]), w=cfg['w'], h=cfg['h'], sigma=10.0,
                feat_dist=cfg['dist'])


# small enough for torch autograd through the reference's D x C x h x w intermediates on CPU
SWEEP_BACKWARD_CASES = ['bwd_v2_d8_c67_L2', 'bwd_v2_d8_c67_L1', 'ragged_v3_d7_c5', 'dzero_behind_v2_d16_c8']


def sweep_grad(name, shape):
    """Seeded upstream gradient d loss / d cost [1, D, h, w] (with a block of exact zeros: skipped planes)."""
    rng = np.random.RandomState(sum(name.encode()) % 10007)
    g = rng.standard_normal(shape).astype(np.float32)
    g[:, ::3, : shape[2] // 4] = 0.0
    return g


SWEEP_CASES = ['c1_320x256_v1_d32_c67', 'c1_320x256_v1_d32_c3', 'small_v4_d32_c67_L2',
               'small_v4_d32_c67_L1', 'ragged_v3_d7_c5', 'dzero_behind_v2_d16_c8', 'identity_v1_d8_c16']


def warp_case(name):
    cfg = {'warp_v4_d32': dict(seed=21, h=64, w=80, V=4, D=32),
           'warp_v2_d5_ragged': dict(seed=22, h=33, w=47, V=2, D=5)}[name]
    rng = np.random.RandomState(cfg['seed'])
    imgs = [synth.smooth_image(rng, 3, cfg['h'], cfg['w'])[None] for _ in range(cfg['V'])]
    poses = _poses(rng, cfg['V'])
    d = synth.d_candidates(cfg['D'])
    return dict(imgs=imgs, d=d, R=[np.ascontiguousarray(p[:3, :3]) for p in poses],
                t=[np.ascontiguousarray(p[:3, 3]) for p in poses], w=cfg['w'], h=cfg['h'])


WARP_CASES = ['warp_v4_d32', 'warp_v2_d5_ragged']


def resample_case(name):
    cfg = {'resample_pose_d32': dict(seed=31, h=64, w=80, D=32),
           'resample_identity_d16': dict(seed=32, h=48, w=64, D=16, identity=True),
           'resample_dnew_d16': dict(seed=33, h=48, w=64, D=16, d_new=True),
           'resample_bigmove_d12': dict(seed=34, h=40, w=56, D=12, step_t=0.5)}[name]
    rng = np.random.RandomState(cfg['seed'])
    D, h, w = cfg['D'], cfg['h'], cfg['w']
    logits = 3.0 * synth.smooth_image(rng, D, h, w)
    m = logits.max(axis=0, keepdims=True)
    vol = (logits - m - np.log(np.exp(logits - m).sum(axis=0, keepdims=True)))[None].astype(np.float32)
    exts = synth.camera_track(rng, 2, cfg.get('step_t', 0.03))
    rel = np.linalg.inv(exts[1].dot(np.linalg.inv(exts[0]))).astype(np.float32)
    if cfg.get('identity'):
        rel = np.eye(4, dtype=np.float32)
    d = synth.d_candidates(D)
    d_new = synth.d_candidates(D, 0.3, 4.0) if cfg.get('d_new') else None
    return dict(vol=vol, rel=rel, d=d, d_new=d_new, w=w, h=h, pad=math.log(1.0 / D))


RESAMPLE_CASES = ['resample_pose_d32', 'resample_identity_d16', 'resample_dnew_d16', 'resample_bigmove_d12']


def kvnet_case(name):
    """Full KVNET.forward / streaming cases. The CNN needs H/4, W/4 >= 64 (SPP
    AvgPool2d(64), psm_submodule.py:103) so 256x256 is the smallest legal frame."""
    cfg = {'kvnet_256_d16': dict(seed=41, H=256, W=256, D=16, n_frames=7, wseed=5),
           'kvnet_256x320_d8': dict(seed=42, H=256, W=320, D=8, n_frames=6, wseed=6)}[name]
    frames, rng = synth.video(cfg['seed'], cfg['n_frames'], cfg['H'], cfg['W'])
    exts = synth.camera_track(rng, cfg['n_frames'])
    sd = arch.synth_state_dict(cfg['wseed'], 64, cfg['D'], 2, 64)
    d = synth.d_candidates(cfg['D'])
    return dict(frames=frames, exts=exts, sd=sd, d=d, H=cfg['H'], W=cfg['W'], D=cfg['D'], sigma=10.0,
                t_win_r=2)


KVNET_CASES = ['kvnet_256_d16', 'kvnet_256x320_d8']


# ---- the BASELINE.json configurations at (or standing in for) their full sizes ----------------------------------
# Fixtures: tests/golden/make_golden.py configs (live reference, FREE-RUNNING: every step is fed the reference's own
# propagated prior; the engine under test feeds its own, so the comparison includes the drift of the recursion).
KITTI = dict(fx=721.5377, fy=721.5377, cx=624.0, cy=188.0)     # KITTI-like pinhole centred on the 1248x376 frame
BIG_CFG = {
    # configs[1] (first window = step 0) and configs[2] (30-frame stream, steps 1..29 steady state with K-Net)
    'c23_640x480_d64_v4_stream30': dict(seed=61, H=480, W=640, D=64, n_frames=34, wseed=7, t_win_r=2),
    # configs[3]: the reference CNN rejects 1242x375 (SURVEY 7), 1248x376 is the nearest legal frame; KITTI planes
    'c4_1248x376_d128_v4': dict(seed=63, H=376, W=1248, D=128, n_frames=6, wseed=8, t_win_r=2, d_min=1.0, d_max=60.0,
                                intr=KITTI),
    # configs[4] stand-in at the smallest legal frame: V=8 (K-Net 28 input channels), D=256 (R-Net 320 channels)
    'c5s_256x256_d256_v8': dict(seed=64, H=256, W=256, D=256, n_frames=10, wseed=9, t_win_r=4),
}
BIG_CASES = list(BIG_CFG)
# steps whose four outputs are stored at the normal sub-sampling; later steps store the filtered DPV + refined DPV thinner
BIG_FULL_STEPS = 4


def big_case(name, n_frames=None):
    cfg = BIG_CFG[name]
    nf = cfg['n_frames']
    frames, rng = synth.video(cfg['seed'], nf, cfg['H'], cfg['W'])
    exts = synth.camera_track(rng, nf)
    r = cfg['t_win_r']
    sd = arch.synth_state_dict(cfg['wseed'], 64, cfg['D'], r, 64)
    d = synth.d_candidates(cfg['D'], cfg.get('d_min', 0.1), cfg.get('d_max', 5.0))
    intr = cfg.get('intr', dict(fx=FX, fy=FY, cx=CX, cy=CY))
    return dict(frames=frames, exts=exts, sd=sd, d=d, H=cfg['H'], W=cfg['W'], D=cfg['D'], sigma=10.0, t_win_r=r,
                intr=intr, n_steps=nf - 2 * r)


def big_cam(make_cam, c):
    i = c['intr']
    return make_cam(i['fx'], i['fy'], i['cx'], i['cy'], [c['W'] // 4, c['H'] // 4])


def subsample_to(a, limit):
    """subsample() with an explicit size limit (strides up to 64)."""
    a = np.asarray(a)
    step = 1
    while a[..., ::step, ::step].size > limit and step < 64:
        step += 1
    return np.ascontiguousarray(a[..., ::step, ::step])


def window(case, ref_idx):
    """ref frame [1,3,H,W], src [1,V,3,H,W], poses [1,V,4,4] for the 5-frame window
    centred on ref_idx (mutils/misc.py:509-517)."""
    poses, idx = synth.window_rel_poses(case['exts'], ref_idx, case['t_win_r'])
    ref = case['frames'][ref_idx][None]
    src = np.stack([case['frames'][i] for i in idx])[None]
    return ref, src, poses[None]


def subsample(a, limit=60000):
    """Strided view (last two dims) keeping large reference outputs small in the
    fixtures; the stride is a pure function of the shape so tests can re-derive it."""
    a = np.asarray(a)
    step = 1
    while a.ndim >= 2 and a[..., ::step, ::step].size > limit and step < 16:
        step += 1
    return np.ascontiguousarray(a[..., ::step, ::step])


def stats(a):
    a = np.asarray(a, np.float64)
    fin = np.isfinite(a)
    return np.array([a[fin].sum(), np.square(a[fin]).sum(), float(fin.sum())], np.float64)


def summary(a):
    """Full-array statistics stored beside a strided sample: sum, sum of squares, finite count, max |a| (finite values)."""
    a = np.asarray(a, np.float64)
    fin = np.isfinite(a)
    return np.concatenate([stats(a), [float(np.abs(a[fin]).max()) if fin.any() else 0.0]])


# ---- output stage (SURVEY 8 f-2): a refined log-DPV, its plane depths and the (normalised) reference image --------
def export_case(name):
    """-> bv [1, D, H, W] float32 log-probabilities, d_candi float64 [D], img [1, 3, H, W] float32."""
    cfg = {'export_48x64_d16': dict(D=16, H=48, W=64, lo=0.1, hi=5.0, sharp=3.0, seed=31),
           'export_ragged_37x53_d64': dict(D=64, H=37, W=53, lo=0.1, hi=5.0, sharp=6.0, seed=32),
           'export_kitti_d128': dict(D=128, H=24, W=80, lo=1.0, hi=60.0, sharp=2.0, seed=33)}[name]
    rng = np.random.RandomState(cfg['seed'])
    z = (rng.standard_normal((1, cfg['D'], cfg['H'], cfg['W'])) * cfg['sharp']).astype(np.float32)
    z = z - z.max(axis=1, keepdims=True)
    bv = (z - np.log(np.exp(z.astype(np.float64)).sum(axis=1, keepdims=True))).astype(np.float32)
    d_candi = np.linspace(cfg['lo'], cfg['hi'], cfg['D'])
    img = rng.standard_normal((1, 3, cfg['H'], cfg['W'])).astype(np.float32)
    return bv, d_candi, img


EXPORT_CASES = ['export_48x64_d16', 'export_ragged_37x53_d64', 'export_kitti_d128']


# ---- input stage (SURVEY 8 f-4): decoded uint8 frames and target sizes (W, H) ------------------------------------
def preprocess_case(name):
    cfg = {'pre_down_97x131_to_64x48': dict(Hs=97, Ws=131, size=(64, 48), seed=41),
           'pre_up_37x53_to_80x64': dict(Hs=37, Ws=53, size=(80, 64), seed=42),
           'pre_same_48x64': dict(Hs=48, Ws=64, size=None, seed=43),
           'pre_odd_100x100_to_77x33': dict(Hs=100, Ws=100, size=(77, 33), seed=44)}[name]
    rng = np.random.RandomState(cfg['seed'])
    img = rng.randint(0, 256, (cfg['Hs'], cfg['Ws'], 3)).astype(np.uint8)
    img[0, 0] = (0, 0, 0); img[-1, -1] = (255, 255, 255)
    return img, cfg['size']


PREPROCESS_CASES = ['pre_down_97x131_to_64x48', 'pre_up_37x53_to_80x64', 'pre_same_48x64', 'pre_odd_100x100_to_77x33']


# ---- f-3 (oracle pinned ahead of the kernels): depth-map back-warp of the local bundle adjustment ------------------
def lba_case(name):
    """-> imgs [N,C,h,w], dmap [h,w], Rs [N,3,3], ts [N,3], w, h."""
    cfg = {'lba_v1_c5_37x53': dict(N=1, C=5, h=37, w=53, seed=51, step_t=0.05),
           'lba_v3_c3_48x64': dict(N=3, C=3, h=48, w=64, seed=52, step_t=0.08)}[name]
    rng = np.random.RandomState(cfg['seed'])
    imgs = rng.standard_normal((cfg['N'], cfg['C'], cfg['h'], cfg['w'])).astype(np.float32)
    dmap = (0.8 + 2.5 * rng.rand(cfg['h'], cfg['w'])).astype(np.float32)
    poses = _poses(rng, cfg['N'], step_t=cfg['step_t'])
    return dict(imgs=imgs, dmap=dmap, Rs=np.ascontiguousarray(poses[:, :3, :3]), ts=np.ascontiguousarray(poses[:, :3, 3]),
                w=cfg['w'], h=cfg['h'])


LBA_CASES = ['lba_v1_c5_37x53', 'lba_v3_c3_48x64']


# ---- a14: calibrations pushed through the reference's intrinsics recipe (tests/golden/make_golden.py camera) -------
CAMERA_CASES = {
    '7scenes_to_160x120': dict(width=640, height=480, fx=585.0, fy=585.0, cx=320.0, cy=240.0, out_size=[160, 120]),
    'scannet_to_96x64': dict(width=1296, height=968, fx=1170.187988, fy=1170.187988, cx=647.75, cy=483.75, out_size=[96, 64]),
    'kitti_to_312x94': dict(width=1248, height=376, fx=721.5377, fy=721.5377, cx=624.0, cy=188.0, out_size=[312, 94]),
    'offcentre_ragged_53x37': dict(width=640, height=480, fx=600.0, fy=590.0, cx=300.0, cy=250.0, out_size=[53, 37]),
}
