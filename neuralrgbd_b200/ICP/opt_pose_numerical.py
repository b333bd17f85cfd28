"""ICP/opt_pose_numerical.py mirror: the local bundle adjustment's pose optimiser on the device (csrc/lba_opt.cu).

local_BA_direct and local_BA_direct_parallel keep the reference's signature, printed lines, exceptions and return value (a
list of CPU float32 4x4 tensors). Each call uploads its frames once, builds the avg-pool pyramid on the device and enqueues
all 3 x max_iter Adam iterations on the input device's current stream (one fused kernel each); the final poses and the
per-iteration losses come back in one device-to-host copy at the end.

local_BA_direct optimises every view on its own (its own Adam, mean over 3 H W): the views are independent, so they share
the launches of one call; results and print order are those of the reference's view-by-view loop.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .._lib import check, ptr
from ..warping.homography import _cam_tensors

f32 = np.float32
STATE = 40                         # NRGBD_LBA_STATE_FLOATS
_U, _T, _R = 0, 3, 6               # NRGBD_LBA_U / _T / _R
OPT_R, OPT_T = 1, 2


# ---- host conversion of the initial poses: mutils/misc.py Rotation2UnitQ / UnitQ2Rotation, each torch op rounded in fp32 ----
def _rotation_to_unitq(R):
    R = np.asarray(R, f32)
    q = np.zeros(4, f32)
    with np.errstate(divide='ignore', invalid='ignore'):
        tr = [f32(f32(f32(R[0, 0] + R[1, 1]) + R[2, 2]) + f32(1)), f32(f32(f32(R[0, 0] - R[1, 1]) - R[2, 2]) + f32(1)),
              f32(f32(f32(R[1, 1] - R[0, 0]) - R[2, 2]) + f32(1)), f32(f32(f32(R[2, 2] - R[0, 0]) - R[1, 1]) + f32(1))]
        if tr[0] > 0:
            q[3] = f32(.5 * np.sqrt(float(tr[0])))
            s = f32(f32(f32(1) / q[3]) * f32(.25))
            q[0] = s * f32(R[2, 1] - R[1, 2]); q[1] = s * f32(R[0, 2] - R[2, 0]); q[2] = s * f32(R[1, 0] - R[0, 1])
        elif tr[1] > 0:
            q[0] = f32(.5 * np.sqrt(float(tr[1])))
            s = f32(f32(f32(1) / q[0]) * f32(.25))
            q[1] = s * f32(R[1, 0] + R[0, 1]); q[2] = s * f32(R[0, 2] + R[2, 0]); q[3] = s * f32(R[2, 1] + R[1, 2])
        elif tr[2] > 0:                       # the reference's third and fourth branches divide by quat[0] (still 0)
            q[1] = f32(.5 * np.sqrt(float(tr[2])))
            s = f32(f32(f32(1) / q[0]) * f32(.25))
            q[0] = s * f32(R[1, 0] + R[0, 1]); q[2] = s * f32(R[1, 2] + R[2, 1]); q[3] = s * f32(R[0, 2] - R[2, 0])
        elif tr[3] > 0:
            q[2] = f32(.5 * np.sqrt(float(tr[3])))
            s = f32(f32(f32(1) / q[0]) * f32(.25))
            q[0] = s * f32(R[2, 0] + R[0, 2]); q[1] = s * f32(R[2, 1] + R[1, 2]); q[3] = s * f32(R[1, 0] - R[0, 1])
        k = f32(f32(f32(f32(1) - q[2]) / f32(q[2] + f32(1))) + f32(1))          # quat_to_unitQ
        return np.array([f32(q[3] * k) * f32(.5), f32(q[0] * k) * f32(.5), f32(q[1] * k) * f32(.5)], f32)


def _unitq_to_rotation(u):
    x, y, z = (f32(v) for v in u)
    a2 = f32(f32(f32(x * x) + f32(y * y)) + f32(z * z))
    den = f32(a2 + f32(1))
    qw, qx, qy, qz = f32(f32(x * f32(2)) / den), f32(f32(y * f32(2)) / den), f32(f32(z * f32(2)) / den), f32(f32(f32(1) - a2) / den)
    s2 = f32(f32(f32(1) / f32(f32(f32(f32(qw * qw) + f32(qx * qx)) + f32(qy * qy)) + f32(qz * qz))) * f32(2))
    xx, yy, zz = f32(qx * qx), f32(qy * qy), f32(qz * qz)
    return np.array([[f32(1) - f32(s2 * f32(yy + zz)), f32(f32(qx * qy) - f32(qw * qz)) * f32(2), f32(f32(qx * qz) + f32(qw * qy)) * f32(2)],
                     [f32(f32(qx * qy) + f32(qw * qz)) * f32(2), f32(1) - f32(s2 * f32(xx + zz)), f32(f32(qy * qz) - f32(qw * qx)) * f32(2)],
                     [f32(f32(qx * qz) - f32(qw * qy)) * f32(2), f32(f32(qy * qz) + f32(qw * qx)) * f32(2), f32(1) - f32(s2 * f32(xx + yy))]], f32)


def initial_state(rel_pose_inits):
    """[V, 40] float32 optimiser state: u = Rotation2UnitQ(R), t, R = UnitQ2Rotation(u), zero Adam moments."""
    st = np.zeros((len(rel_pose_inits), STATE), f32)
    for v, pose in enumerate(rel_pose_inits):
        P = np.asarray(pose, f32)
        u = _rotation_to_unitq(P[:3, :3])
        st[v, _U:_U + 3] = u
        st[v, _T:_T + 3] = P[:3, 3]
        st[v, _R:_R + 9] = _unitq_to_rotation(u).reshape(9)
    return st


def _mode(opt_vars):
    if opt_vars[0] != 1:
        return OPT_T
    if opt_vars[1] == 0:
        return OPT_R
    if opt_vars[1] == 1:
        return OPT_R | OPT_T
    raise Exception('undefined optmization variable option')


def _run(ref_frame, src_frames, dmap_ref, conf_map_ref, cams_intrin, dw_scales, rel_pose_inits, max_iter, step, mode, parallel):
    """-> (state [V, 40] float32, losses [levels, max_iter, V] float64 sums of |residual|, level sizes)."""
    L = _lib.lib()
    dev = ref_frame.device if ref_frame.is_cuda else torch.device('cuda', torch.cuda.current_device())
    V = len(rel_pose_inits)
    H, W = ref_frame.shape[-2:]
    with torch.cuda.device(dev):
        # one upload: [ref (3), conf, dmap, sources (3 V)] planes at full resolution
        planes = torch.cat([ref_frame.reshape(3, H, W), conf_map_ref.reshape(1, H, W), dmap_ref.reshape(1, H, W)]
                           + [s.reshape(3, H, W) for s in src_frames], 0).to(device=dev, dtype=torch.float32).contiguous()
        n_lv, n_st = len(dw_scales), V * STATE // 2
        rec = torch.empty(n_lv * max_iter * V + n_st, device=dev, dtype=torch.float64)    # losses, then the state: one read-back
        state = rec[n_lv * max_iter * V:].view(torch.float32)
        state.copy_(torch.from_numpy(initial_state(rel_pose_inits).reshape(-1)))
        sizes = [(H // d, W // d) if d > 1 else (H, W) for d in dw_scales]
        ws = torch.empty(max(L.nrgbd_lba_pose_opt_workspace_bytes(V, h, w) for h, w in sizes), device=dev, dtype=torch.uint8)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        for s, (dw, (h, w)) in enumerate(zip(dw_scales, sizes)):
            lv = planes
            if dw > 1:
                lv = torch.empty((planes.shape[0], h, w), device=dev, dtype=torch.float32)
                check(L.nrgbd_lba_avgpool(ptr(planes), planes.shape[0], H, W, int(dw), ptr(lv), stream))
            K, rays = _cam_tensors(cams_intrin[s], dev)
            assert rays.shape[1] == h * w, 'cams_intrin[%d] does not match the %dx%d pyramid level' % (s, w, h)
            check(L.nrgbd_lba_pose_opt_scale(ptr(lv[0:3]), ptr(lv[3]), ptr(lv[4]), ptr(lv[5:]), ptr(K), ptr(rays), V, h, w, mode,
                                             1.0 / ((V if parallel else 1) * 3 * h * w), float(step / (2 ** s)), s * max_iter, max_iter,
                                             ptr(state), ctypes.c_void_p(rec.data_ptr() + 8 * s * max_iter * V),
                                             ctypes.c_void_p(ws.data_ptr()), stream))
        host = rec.cpu().numpy()
    losses = host[:n_lv * max_iter * V].reshape(n_lv, max_iter, V)
    return host[n_lv * max_iter * V:].view(f32).reshape(V, STATE), losses, sizes


def _print_level(s, max_iter, l0, l1):
    print('opt_pose(): scale=%d, iter %d/%d, d_loss = %f' % (s, max_iter, max_iter, (l1 - l0) * 100))


def _poses(state):
    out = []
    for row in state:
        P = torch.eye(4)
        P[:3, 3] = torch.from_numpy(row[_T:_T + 3].copy())
        P[:3, :3] = torch.from_numpy(row[_R:_R + 9].reshape(3, 3).copy())
        out.append(P)
    return out


def _check_inputs(ref_frame, src_frames, dmap_ref, conf_map_ref):
    assert isinstance(ref_frame, torch.Tensor) and isinstance(src_frames[0], torch.Tensor) \
        and isinstance(dmap_ref, torch.Tensor) and isinstance(conf_map_ref, torch.Tensor)


def local_BA_direct_parallel(ref_frame, src_frames, dmap_ref, conf_map_ref, cams_intrin, dw_scales, rel_pose_inits, max_iter, step,
                             opt_vars):
    '''
    optimize the poses for src frames at the same time (ICP/opt_pose_numerical.py:306-356): one Adam over all views, the L1
    loss averaged over all of them. Returns the list of optimised 4x4 relative poses (CPU float32 tensors).
    '''
    _check_inputs(ref_frame, src_frames, dmap_ref, conf_map_ref)
    assert len(src_frames) > 1 and sum(int(s.shape[0]) for s in src_frames) > 1       # should have more than one src view
    mode = _mode(opt_vars)
    state, losses, sizes = _run(ref_frame, src_frames, dmap_ref, conf_map_ref, cams_intrin, dw_scales, rel_pose_inits, max_iter, step,
                                mode, True)
    V = len(rel_pose_inits)
    for s, (h, w) in enumerate(sizes):
        if max_iter > 0:
            n = V * 3 * h * w
            _print_level(s, max_iter, f32(losses[s, 0].sum() / n), f32(losses[s, -1].sum() / n))
    return _poses(state)


def local_BA_direct(ref_frame, src_frames, dmap_ref, conf_map_ref, cams_intrin, dw_scales, rel_pose_inits, max_iter, step, opt_vars):
    '''
    ICP/opt_pose_numerical.py:358-417: every source view optimised on its own (its own Adam, its own mean L1 loss).
    ref_frame, src_frames[i], dmap_ref, conf_map_ref: NCHW; cams_intrin[s]: intrinsics of level s; dw_scales e.g. [4, 2, 1];
    rel_pose_inits: 4x4 arrays (src -> ref); opt_vars = [opt_r, opt_t]. Returns the list of optimised 4x4 poses.
    '''
    _check_inputs(ref_frame, src_frames, dmap_ref, conf_map_ref)
    mode = _mode(opt_vars)
    V = len(rel_pose_inits)
    if V == 0:
        return []
    state, losses, sizes = _run(ref_frame, src_frames[:V], dmap_ref, conf_map_ref, cams_intrin, dw_scales, rel_pose_inits, max_iter, step,
                                mode, False)
    for v in range(V):
        for s, (h, w) in enumerate(sizes):
            if max_iter > 0:
                n = 3 * h * w
                _print_level(s, max_iter, f32(losses[s, 0, v] / n), f32(losses[s, -1, v] / n))
    return _poses(state)
