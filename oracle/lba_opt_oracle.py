"""numpy float32 restatement of the LBA pose optimiser, ICP/opt_pose_numerical.py:28-417 (local_BA_direct and
local_BA_direct_parallel), reusing the back-warp and its gradients of planesweep_oracle.

Pyramid: F.avg_pool2d(x, dw) for dw > 1. Parameters per source view: t = init_pose[:3, 3] and the unit-quaternion rotation
u = Rotation2UnitQ(init_pose[:3, :3]); the warp always uses R = UnitQ2Rotation(u). One iteration: w = back_warp(src, dmap,
R, t), mask = (w != 0), loss = mean |w mask conf - ref mask conf|, its gradient through grid_sample to R, t and from R
through quaternion2Rotation (as written, s = 1 / |q|^2 included) and unitQ_to_quat to u, then torch.optim.Adam.
local_BA_direct optimises each view on its own (mean over 3 H W); local_BA_direct_parallel all views at once (mean over
V 3 H W). Adam's state carries across the levels; level s runs at lr = step / 2^s.
"""
import math

import numpy as np

from oracle import planesweep_oracle as O

f32 = np.float32


# ---- pose parameterisation (mutils/misc.py:295-502), each torch op rounded in fp32 ---------------------------------------
def rotation_to_unitq(R):
    """Rotation2Quaternion (TUM x, y, z, w; branches 3 and 4 as written: they divide by quat[0] = 0) then quat_to_unitQ."""
    R = np.asarray(R, f32)
    q = np.zeros(4, f32)
    with np.errstate(divide='ignore', invalid='ignore'):
        def s_of(qi):                                              # s = 1 / 4 / q_i  ->  reciprocal(q_i) * 0.25
            return f32(f32(f32(1) / qi) * f32(0.25))
        if f32(f32(f32(R[0, 0] + R[1, 1]) + R[2, 2]) + f32(1)) > 0:
            q[3] = f32(.5 * math.sqrt(float(f32(f32(R[0, 0] + R[1, 1]) + R[2, 2]) + f32(1))))
            s = s_of(q[3])
            q[0] = s * f32(R[2, 1] - R[1, 2]); q[1] = s * f32(R[0, 2] - R[2, 0]); q[2] = s * f32(R[1, 0] - R[0, 1])
        elif f32(f32(f32(R[0, 0] - R[1, 1]) - R[2, 2]) + f32(1)) > 0:
            q[0] = f32(.5 * math.sqrt(float(f32(f32(R[0, 0] - R[1, 1]) - R[2, 2]) + f32(1))))
            s = s_of(q[0])
            q[1] = s * f32(R[1, 0] + R[0, 1]); q[2] = s * f32(R[0, 2] + R[2, 0]); q[3] = s * f32(R[2, 1] + R[1, 2])
        elif f32(f32(f32(R[1, 1] - R[0, 0]) - R[2, 2]) + f32(1)) > 0:
            q[1] = f32(.5 * math.sqrt(float(f32(f32(R[1, 1] - R[0, 0]) - R[2, 2]) + f32(1))))
            s = s_of(q[0])
            q[0] = s * f32(R[1, 0] + R[0, 1]); q[2] = s * f32(R[1, 2] + R[2, 1]); q[3] = s * f32(R[0, 2] - R[2, 0])
        elif f32(f32(f32(R[2, 2] - R[0, 0]) - R[1, 1]) + f32(1)) > 0:
            q[2] = f32(.5 * math.sqrt(float(f32(f32(R[2, 2] - R[0, 0]) - R[1, 1]) + f32(1))))
            s = s_of(q[0])
            q[0] = s * f32(R[2, 0] + R[0, 2]); q[1] = s * f32(R[2, 1] + R[1, 2]); q[3] = s * f32(R[1, 0] - R[0, 1])
        # quat_to_unitQ: q1, q2, q3, q0 = quat[0], quat[1], quat[2], quat[3]; alpha2 = (1 - q3) / (1 + q3)
        a2 = f32(f32(f32(1) - q[2]) / f32(q[2] + f32(1)))
        k = f32(a2 + f32(1))
        return np.array([f32(q[3] * k) * f32(.5), f32(q[0] * k) * f32(.5), f32(q[1] * k) * f32(.5)], f32)


def unitq_to_quat(u):
    x, y, z = (f32(v) for v in u)
    a2 = f32(f32(f32(x * x) + f32(y * y)) + f32(z * z))
    den = f32(a2 + f32(1))
    return np.array([f32(f32(y * f32(2)) / den), f32(f32(z * f32(2)) / den), f32(f32(f32(1) - a2) / den), f32(f32(x * f32(2)) / den)], f32)


def quat_to_rotation(q):
    x, y, z, w = (f32(v) for v in q)
    n = f32(f32(f32(f32(w * w) + f32(x * x)) + f32(y * y)) + f32(z * z))
    s2 = f32(f32(f32(1) / n) * f32(2))
    xx, yy, zz = f32(x * x), f32(y * y), f32(z * z)
    R = np.zeros((3, 3), f32)
    R[0, 0] = f32(1) - f32(s2 * f32(yy + zz)); R[1, 1] = f32(1) - f32(s2 * f32(xx + zz)); R[2, 2] = f32(1) - f32(s2 * f32(xx + yy))
    R[0, 1] = f32(f32(x * y) - f32(w * z)) * f32(2); R[1, 0] = f32(f32(x * y) + f32(w * z)) * f32(2)
    R[0, 2] = f32(f32(x * z) + f32(w * y)) * f32(2); R[2, 0] = f32(f32(x * z) - f32(w * y)) * f32(2)
    R[1, 2] = f32(f32(y * z) - f32(w * x)) * f32(2); R[2, 1] = f32(f32(y * z) + f32(w * x)) * f32(2)
    return R


def unitq_to_rotation(u):
    """UnitQ2Rotation."""
    return quat_to_rotation(unitq_to_quat(u))


def unitq_grad(u, gR):
    """dL/du for dL/dR [3,3] (float64): quaternion2Rotation as written, then unitQ_to_quat (autograd's chain)."""
    x, y, z = (float(v) for v in u)
    G = np.asarray(gR, np.float64).reshape(9)
    a2 = x * x + y * y + z * z; D = 1.0 + a2
    qw, qx, qy, qz = 2 * x / D, 2 * y / D, 2 * z / D, (1 - a2) / D
    s = 1.0 / (qw * qw + qx * qx + qy * qy + qz * qz)
    A = G[0] * (qy * qy + qz * qz) + G[4] * (qx * qx + qz * qz) + G[8] * (qx * qx + qy * qy)
    dA = (2 * qx * (G[4] + G[8]), 2 * qy * (G[0] + G[8]), 2 * qz * (G[0] + G[4]))
    ds = [-2 * q * s * s for q in (qx, qy, qz, qw)]                    # d s / d q
    gq = [-2 * (ds[i] * A + s * (dA[i] if i < 3 else 0.0)) for i in range(4)]
    gq[0] += 2 * (qy * (G[1] + G[3]) + qz * (G[2] + G[6]) + qw * (G[7] - G[5]))
    gq[1] += 2 * (qx * (G[1] + G[3]) + qz * (G[5] + G[7]) + qw * (G[2] - G[6]))
    gq[2] += 2 * (qx * (G[2] + G[6]) + qy * (G[5] + G[7]) + qw * (G[3] - G[1]))
    gq[3] += 2 * (qz * (G[3] - G[1]) + qy * (G[2] - G[6]) + qx * (G[7] - G[5]))
    gqx, gqy, gqz, gqw = gq
    c = 4 * (gqw * x + gqx * y + gqy * z + gqz) / (D * D)
    return np.array([2 * gqw / D - x * c, 2 * gqx / D - y * c, 2 * gqy / D - z * c])


# ---- torch.optim.Adam(lr, betas=(.9, .999)), eps 1e-8: the fp32 op order of torch 2.11's CPU step -----------------------
def adam_step(p, g, m, v, step, lr):
    """exp_avg.lerp_(g, 1 - b1) (an FMA on the CPU), exp_avg_sq.mul_(b2).addcmul_(g, g, 1 - b2) (an FMA), bias corrections as
    Python doubles, denom = sqrt(v) / sqrt(bc2) + eps, p.addcdiv_(m, denom, -lr / bc1). Returns new (p, m, v)."""
    p, g, m, v = (np.asarray(a, f32) for a in (p, g, m, v))
    m = O._fma(f32(1 - .9), (g - m).astype(f32), m)
    v = O._fma((f32(1 - .999) * g).astype(f32), g, (v * f32(.999)).astype(f32))
    bc1 = 1 - .9 ** float(step); bc2 = 1 - .999 ** float(step)
    den = ((np.sqrt(v) / f32(bc2 ** 0.5)).astype(f32) + f32(1e-8)).astype(f32)
    p = (p + ((f32(-(lr / bc1)) * m).astype(f32) / den).astype(f32)).astype(f32)
    return p, m, v


def avg_pool(x, k):
    """F.avg_pool2d(x, k) on [..., H, W]: fp32 sum over the window (rows, then columns), divided by k * k."""
    x = np.asarray(x, f32)
    if k <= 1:
        return x
    H, W = x.shape[-2] // k, x.shape[-1] // k
    acc = np.zeros(x.shape[:-2] + (H, W), f32)
    for dy in range(k):
        for dx in range(k):
            acc = (acc + x[..., dy:dy + H * k:k, dx:dx + W * k:k]).astype(f32)
    return (acc / f32(k * k)).astype(f32)


# ---- one iteration and the two entry points ------------------------------------------------------------------------------
def iteration(ref, conf, dmap, src, R, t, cam, loss_scale):
    """One view at one level: (sum |residual| (float64), dL/dR [3,3], dL/dt [3]) with dL = loss_scale * d sum |residual|."""
    w = O.back_warp_th_Rt(src, dmap, R, t, cam)
    mask = (w != 0).astype(f32)
    cf = np.asarray(conf, f32).reshape(1, 1, *w.shape[2:])
    r = ((w * mask).astype(f32) * cf).astype(f32) - ((np.asarray(ref, f32) * mask).astype(f32) * cf).astype(f32)
    g = ((np.sign(r) * f32(loss_scale)).astype(f32) * cf).astype(f32) * mask
    gR, gt, _ = O.back_warp_th_Rt_backward(g, src, dmap, R, t, cam)
    return float(np.abs(r.astype(np.float64)).sum()), gR, gt


def init_state(pose):
    pose = np.asarray(pose, f32)
    u = rotation_to_unitq(pose[:3, :3])
    z = np.zeros(3, f32)
    return dict(u=u, t=pose[:3, 3].copy(), R=unitq_to_rotation(u), m_u=z.copy(), v_u=z.copy(), m_t=z.copy(), v_t=z.copy())


def pyramid(ref_frame, src_frames, dmap_ref, conf_map_ref, dw_scales):
    """Per level: (ref [1,3,h,w], srcs [V] x [1,3,h,w], dmap [h,w], conf [h,w]) as downsample_img gives them."""
    return [(avg_pool(ref_frame, dw), [avg_pool(f, dw) for f in src_frames], avg_pool(dmap_ref, dw)[0, 0], avg_pool(conf_map_ref, dw)[0, 0])
            for dw in dw_scales]


def gradients(level, states, cam, parallel):
    """One iteration's evaluation for every view: (loss sums [V], dL/du [V,3] float32, dL/dt [V,3] float32)."""
    ref, srcs, dm, cf = level
    V = len(states)
    scale = 1.0 / ((V if parallel else 1) * 3 * dm.size)
    out = [iteration(ref, cf, dm, srcs[v], x['R'], x['t'], cam, scale) for v, x in enumerate(states)]
    g_u = np.stack([unitq_grad(x['u'], o[1]).astype(f32) for x, o in zip(states, out)])
    return np.array([o[0] for o in out]), g_u, np.stack([o[2] for o in out]).astype(f32)


def local_ba(ref_frame, src_frames, dmap_ref, conf_map_ref, cams_intrin, dw_scales, rel_pose_inits, max_iter, step, opt_vars,
             parallel, record=None):
    """local_BA_direct(_parallel) -> list of V float32 4x4 poses. `record` (a list) receives one dict per (level, iteration):
    the state before the step, the gradients and each view's sum |residual|."""
    opt_R = opt_vars[0] == 1
    if opt_R and opt_vars[1] not in (0, 1):
        raise Exception('undefined optmization variable option')
    upd_u, upd_t = opt_R, (not opt_R) or opt_vars[1] == 1
    st = [init_state(p) for p in rel_pose_inits]
    step_no = 0
    for s, level in enumerate(pyramid(ref_frame, src_frames, dmap_ref, conf_map_ref, dw_scales)):
        lr = step / (2 ** s)
        for it in range(max_iter):
            step_no += 1
            before = [{k: a.copy() for k, a in x.items()} for x in st]
            lsum, g_u, g_t = gradients(level, st, cams_intrin[s], parallel)
            for v, x in enumerate(st):
                if upd_u:
                    x['u'], x['m_u'], x['v_u'] = adam_step(x['u'], g_u[v], x['m_u'], x['v_u'], step_no, lr)
                    x['R'] = unitq_to_rotation(x['u'])
                if upd_t:
                    x['t'], x['m_t'], x['v_t'] = adam_step(x['t'], g_t[v], x['m_t'], x['v_t'], step_no, lr)
            if record is not None:
                record.append({'level': s, 'iter': it, 'state': before, 'loss_sum': lsum, 'g_u': g_u, 'g_t': g_t})
    out = []
    for x in st:
        P = np.eye(4, dtype=f32); P[:3, :3] = x['R']; P[:3, 3] = x['t']
        out.append(P)
    return out
