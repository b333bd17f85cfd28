"""Drop-in mirror of the reference's `models.KVNET.KVNET` (models/KVNET.py:28-185).

Same constructor / forward signatures, attribute names and state_dict keys (so
kvnet_scannet.tar / kvnet_kitti.tar load, with or without the DataParallel 'module.'
prefix), same return tuple. forward() does no math in Python: it hands the frame to the
native engine (include/nrgbd.h nrgbd_kvnet_*), which runs D-Net -> R-Net -> (K-Net -> R-Net)
as hand-written sm_90a kernels on the current CUDA stream. No CPU path.

Refinement (KVNET.py:80-85, 126-136, 175-180): refineNet_name='DPV' (default) refines the DPV to image size, with
4D planes when if_upsample_d=True (Refine.py:44-48; regress it with 4D candidates, e.g. the loaders' dup4_candi);
'DGF' refines the expected depth with the guided filter of Refine.py:583-641 ([1,1,H,W] depth maps); if_refined=False
runs no R-Net at all and returns -1 for both refined outputs.
"""
import ctypes
import math

import numpy as np
import torch
import torch.nn as nn

from .. import _lib, arch
from .._lib import ptr, check
from ..mutils import misc as m_misc


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference's module tree / parameter names."""


def _register(root, name, tensor, is_buffer):
    parts = name.split('.')
    node = root
    for p in parts[:-1]:
        if p not in node._modules:
            node.add_module(p, _Node())
        node = node._modules[p]
    if is_buffer:
        node.register_buffer(parts[-1], tensor)
    else:
        node.register_parameter(parts[-1], nn.Parameter(tensor))


def _init_tensor(name, shape, kind, gen):
    """Reference initialisation: He-normal convs (basic.py:28-40, Refine.py:109-116), BN weight 1 /
    bias 0, bilinear transposed-conv kernels (Refine.py:121-132), PyTorch-default conv biases."""
    if kind in ('conv2d', 'conv3d'):
        n = int(np.prod(shape[2:])) * shape[0]
        return torch.randn(shape, generator=gen) * math.sqrt(2. / n)
    if kind == 'convT2d':
        k = shape[2]; factor = (k + 1) // 2
        center = factor - 1 if k % 2 == 1 else factor - .5
        og = np.ogrid[:k, :k]
        bil = (1 - abs(og[0] - center) / factor) * (1 - abs(og[1] - center) / factor)
        return torch.from_numpy(np.broadcast_to(bil, shape).copy()).float()
    if kind == 'bn_w':
        return torch.ones(shape)
    if kind in ('bn_b', 'bn_rm'):
        return torch.zeros(shape)
    if kind == 'bn_rv':
        return torch.ones(shape)
    if kind == 'bn_nb':
        return torch.zeros(shape, dtype=torch.long)
    if kind == 'bias':
        return (torch.rand(shape, generator=gen) - 0.5) * 0.1
    raise ValueError(kind)


class KVNET(nn.Module):
    r'''
    The full KV-Net pipeline on the H100 engine:
    * D-Net (feature extraction + plane sweep + BV_cur estimation)
    * R-Net DPV refinement / up-sampling
    * KV-Net Bayesian update against the propagated DPV
    '''

    def __init__(self, feature_dim, cam_intrinsics, d_candi, sigma_soft_max,
                 KVNet_feature_dim, d_upsample_ratio_KV_net,
                 if_refined=True, refineNet_name='DPV',
                 t_win_r=2, refine_channel=3, if_upsample_d=False):
        super(KVNET, self).__init__()
        if if_refined and refineNet_name not in ('DPV', 'DGF'):
            raise NotImplementedError("refineNet_name must be 'DPV' or 'DGF' (models/KVNET.py:81-85); got %r" % (refineNet_name,))
        if d_upsample_ratio_KV_net is not None:
            raise NotImplementedError('d_upsample_ratio_KV_net is not implemented: for a ratio other than 1 the reference '
                                      'itself fails with a shape error where K-Net\'s gain is added to BV_predict '
                                      '(models/KVNET.py:172)')
        self.t_win_r = t_win_r
        self.feature_dim = feature_dim
        self.KVNet_feature_dim = KVNet_feature_dim
        self.sigma_soft_max = sigma_soft_max
        self.d_upsample_ratio_KV_net = d_upsample_ratio_KV_net
        self.d_candi = d_candi
        self.if_refined = if_refined
        self.refineNet_name = refineNet_name
        self.if_upsample_d = if_upsample_d
        self.refine_channel = refine_channel
        self._refine = refineNet_name if if_refined else None     # 'DPV', 'DGF' or None
        self._upsample_d = bool(if_refined and refineNet_name == 'DPV' and if_upsample_d)   # refined DPVs of 4D planes
        self.cam_intrinsics = cam_intrinsics          # captured at construction: used by D-Net (KVNET.py:64-67)
        self.feat_dist = 'L2'                         # basic.py:146 default, never overridden by KVNET
        # convolution arithmetic: 'f16x3' (default; wgmma on split-fp16 operand pairs, 22-bit products, fp32 accumulate -
        # the fastest AND the closest to the reference of the tensor paths), 'tf32x3' (wgmma 3xTF32), 'fp32' (exact CUDA-core FFMA),
        # 'f16' (opt-in throughput mode: one fp16 product per MAC, fp32 accumulate - the operand precision of a TF32 GPU run,
        # not the 1e-4 envelope of the other modes; INTEGRATION.md)
        self.conv_math = 'f16x3'

        D = len(d_candi)
        gen = torch.Generator().manual_seed(0)
        specs = arch.kvnet_param_specs(feature_dim, D, t_win_r, KVNet_feature_dim, self._refine, self._upsample_d)
        self._specs = [(n, s, k) for n, s, k in specs if not n.startswith('d_net.feature_extraction.')]
        for name, shape, kind in self._specs:
            _register(self, name, _init_tensor(name, tuple(shape), kind, gen), kind in ('bn_rm', 'bn_rv', 'bn_nb'))
        # the extractor object is registered under both parents (KVNET.py:63-67): same tensors, two names
        self.add_module('d_net', _Node())
        self.d_net.add_module('feature_extraction', self.feature_extractor)
        # reference order of state_dict(): feature_extractor, d_net, kv_net, r_net
        for k in ('kv_net', 'r_net'):
            if k in self._modules:
                self._modules[k] = self._modules.pop(k)
        self._engines = {}
        self.register_state_dict_pre_hook(KVNET._flush_batches_tracked)
        print('KV-Net initialization:')
        print('with R-net: %r' % (self.if_refined))
        if self.if_refined:
            print('\trefinement name: %s' % (self.refineNet_name))

    # ------------------------------------------------------------------ engine plumbing
    def _engine(self, H, W, V, device):
        key = (device.index, H, W, V)
        ent = self._engines.get(key)
        if ent is None:
            L = _lib.lib()
            hnd = ctypes.c_void_p()
            check(L.nrgbd_kvnet_create(H, W, len(self.d_candi), V, int(self.feature_dim), int(self.KVNet_feature_dim),
                                       ctypes.c_float(float(self.sigma_soft_max)), 0 if self.feat_dist == 'L2' else 1,
                                       ctypes.byref(hnd)))
            d32 = np.ascontiguousarray(np.asarray(self.d_candi).astype(np.float32))
            check(L.nrgbd_kvnet_set_planes(hnd, d32.ctypes.data_as(ctypes.c_void_p), len(d32)))
            ent = {'h': hnd, 'params': {}, 'cams': [None, None], 'keep': {}, 'conv_math': None, 'bn_eval': False, 'refine': 0,
                   'upsample_d': False}
            self._engines[key] = ent
        return ent

    def _resolve(self, name):
        """Tensor registered under the dotted state_dict name, found by walking attributes: works on the module
        itself and on an nn.DataParallel replica (replicate() re-attaches the broadcast copies as plain tensor
        attributes, so a replica's named_parameters() is empty)."""
        node = self
        for part in name.split('.'):
            node = getattr(node, part)
        return node

    def _param_list(self):
        """(name, tensor) for every float parameter / buffer the engine needs, cached per module object
        (a DataParallel replica is a new object each forward and rebuilds it)."""
        cache = self.__dict__.get('_plist')
        if cache is None or cache[0] != id(self):
            cache = (id(self), [(name, self._resolve(name)) for name, shape, kind in self._specs if kind != 'bn_nb'])
            self.__dict__['_plist'] = cache
        return cache[1]

    def _sync_params(self, ent, device):
        L = _lib.lib()
        seen = ent['params']
        # a DataParallel replica holds fresh broadcast copies every forward: the caching allocator may hand back an
        # address the engine has seen (same data_ptr, version 0) with new contents, so replicas always re-register
        replica = bool(getattr(self, '_is_replica', False))
        for name, t in self._param_list():
            tag = (t.data_ptr(), t._version)
            if replica or seen.get(name) != tag:
                if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
                    raise _lib.NrgbdError('parameter %s must be a contiguous float32 tensor on %s (call .cuda())' % (name, device))
                check(L.nrgbd_kvnet_set_param(ent['h'], name.encode(), ctypes.c_void_p(t.data_ptr()), t.numel(), 1))
                seen[name] = tag

    def _flush_batches_tracked(self, *args, **kwargs):
        """BatchNorm's num_batches_tracked side effect (training mode) is applied lazily: one counter per
        forward on the host, materialised into the 15 buffers when the state_dict is read."""
        n_all = self.__dict__.get('_nb_pending', 0)          # every forward: the feature-CNN BatchNorms
        n_kv = self.__dict__.get('_nb_pending_kv', 0)        # forwards that ran K-Net (valid prior): kv_net BatchNorm3d
        if n_all or n_kv:
            for name, _, kind in self._specs:
                if kind == 'bn_nb':
                    n = n_kv if name.startswith('kv_net.') else n_all
                    if n:
                        self.get_buffer(name).add_(n)
            self.__dict__['_nb_pending'] = 0
            self.__dict__['_nb_pending_kv'] = 0

    def _set_camera(self, ent, slot, cam=None, IntM=None, rays=None):
        L = _lib.lib()
        if cam is not None:
            # keyed by CONTENT of the small members (K, principal point, fovs) and identity + version of the ray
            # table: an in-place edit of the dict, or another trajectory's dict at a recycled id(), is seen
            rays_t = torch.as_tensor(cam['unit_ray_array_2D'])
            K = np.ascontiguousarray(torch.as_tensor(cam['intrinsic_M_cuda']).detach().cpu().numpy().astype(np.float32))
            cx, cy = float(cam['intrinsic_M'][0, 2]), float(cam['intrinsic_M'][1, 2])
            hf, vf = float(cam.get('hfov', 0.)), float(cam.get('vfov', 0.))
            tag = (id(cam), K.tobytes(), cx, cy, hf, vf, rays_t.data_ptr(), rays_t._version, tuple(rays_t.shape))
            if ent['cams'][slot] == tag:
                return
            R = np.ascontiguousarray(rays_t.detach().cpu().numpy().astype(np.float32))
            ent['keep'][slot] = cam
        else:
            # scattered tensors are re-allocated every forward and the allocator recycles addresses: key by content
            # (K and a checksum of the ray table, one small device->host read)
            sig = torch.cat([IntM.detach().reshape(-1)[:9].float(), rays.detach().float().sum().reshape(1),
                             rays.detach().float().abs().max().reshape(1)]).cpu().numpy()
            tag = (sig.tobytes(), tuple(rays.shape))
            if ent['cams'][slot] == tag:
                return
            K = np.ascontiguousarray(sig[:9].reshape(3, 3).astype(np.float32))
            R = np.ascontiguousarray(rays.detach().reshape(3, -1).cpu().numpy().astype(np.float32))
            cx, cy = float(K[0, 2]), float(K[1, 2])
            hf = math.degrees(math.atan(cx / K[0, 0]) * 2); vf = math.degrees(math.atan(cy / K[1, 1]) * 2)
        check(L.nrgbd_kvnet_set_camera(ent['h'], slot, K.ctypes.data_as(ctypes.c_void_p),
                                       R.ctypes.data_as(ctypes.c_void_p), ctypes.c_float(cx), ctypes.c_float(cy), hf, vf))
        ent['cams'][slot] = tag

    # ------------------------------------------------------------------ forward
    def forward(self, ref_frame, src_frames, src_cam_poses, BatchIdx, cam_intrinsics=None, BV_predict=None, mGPU=False,
                IntMs=None, unit_ray_Ms_2D=None, return_depth=False):
        r'''
        Inputs (as models/KVNET.py:93-112):
        ref_frame - NCHW format tensor on GPU, N = 1
        src_frames - NVCHW: V - # of source views, N = 1
        src_cam_poses - N x V x4 x4 - relative cam poses, N = 1
        BatchIdx - e.g. for 4 gpus: [0,1,2,3], used for indexing list input for multi-gpu training
        cam_intrinsics - list of cam_intrinsics dict.
        BV_predict - NDHW tensor, the predicted BV, from the last reference frame, N=1

        Outputs: dmap_cur_refined, dmap_kv_refined, BV_cur, BV_KV. The refined entries are log-DPVs at image size
        ('DPV'; 4D planes with if_upsample_d), depth maps 1 x 1 x H x W ('DGF'), or -1 (if_refined=False).
        '''
        if self._refine == 'DGF':
            # RefineNet_DGF.forward's input checks (Refine.py:627-628), as the reference meets them in its first R-Net call
            assert ref_frame.dim() == 4, 'input format is wrong'
            assert self.refine_channel == ref_frame.shape[1]
        if not ref_frame.is_cuda:
            raise _lib.NrgbdError('neuralrgbd_b200.KVNET has no CPU path: inputs must be CUDA tensors')
        if isinstance(BV_predict, torch.Tensor):
            if m_misc.valid_dpv(BV_predict):
                assert BV_predict.shape[0] == 1
        assert src_frames.shape[0] == 1, 'dim0 of src_frames should be 0'      # basic.py:240
        L = _lib.lib()
        dev = ref_frame.device
        with torch.cuda.device(dev):
            _, _, H, W = ref_frame.shape
            V = src_frames.shape[1]
            D = len(self.d_candi)
            ent = self._engine(H, W, V, dev)
            self._sync_params(ent, dev)
            if ent['conv_math'] != self.conv_math:
                modes = {'fp32': 0, 'tf32x3': 1, 'f16x3': 2, 'f16': 3}
                if self.conv_math not in modes:
                    raise ValueError("conv_math must be 'fp32', 'tf32x3', 'f16x3' or 'f16'")
                check(L.nrgbd_kvnet_set_option(ent['h'], b'conv_math', modes[self.conv_math]))
                ent['conv_math'] = self.conv_math
            # .eval(): the 13 BatchNorm layers with running statistics (K-Net's BatchNorm3d, the feature CNN's downsample
            # BatchNorm2d) normalise with them and nothing is updated; the others keep batch statistics, as in PyTorch
            refine = {'DPV': 0, 'DGF': 1, None: 2}[self._refine]
            if ent['refine'] != refine:
                check(L.nrgbd_kvnet_set_option(ent['h'], b'refine', refine))
                ent['refine'] = refine
            if ent['upsample_d'] != self._upsample_d:
                check(L.nrgbd_kvnet_set_option(ent['h'], b'refine_upsample_d', int(self._upsample_d)))
                ent['upsample_d'] = self._upsample_d
            bn_eval = not self.training
            if ent['bn_eval'] != bn_eval:
                check(L.nrgbd_kvnet_set_option(ent['h'], b'bn_eval', int(bn_eval)))
                ent['bn_eval'] = bn_eval
            self._set_camera(ent, 0, cam=self.cam_intrinsics)
            prior = None
            if isinstance(BV_predict, torch.Tensor) and m_misc.valid_dpv(BV_predict):
                prior = BV_predict[0].to(device=dev, dtype=torch.float32).contiguous()
                if mGPU:
                    self._set_camera(ent, 1, IntM=IntMs, rays=unit_ray_Ms_2D)
                else:
                    self._set_camera(ent, 1, cam=cam_intrinsics[int(BatchIdx)])
            frames = torch.cat((src_frames[0], ref_frame), dim=0).float().contiguous()
            poses = src_cam_poses[0].to(device=dev, dtype=torch.float32).contiguous()
            h, w = H // 4, W // 4
            Dr = {'DPV': 4 * D if self._upsample_d else D, 'DGF': 1, None: 0}[self._refine]     # planes of a refined output
            dmap_cur = torch.empty((1, Dr, H, W), device=dev, dtype=torch.float32) if Dr else None
            bv_cur = torch.empty((1, D, h, w), device=dev, dtype=torch.float32)
            dmap_kv = dpv = None
            if prior is not None:
                dmap_kv = torch.empty((1, Dr, H, W), device=dev, dtype=torch.float32) if Dr else None
                dpv = torch.empty((1, D, h, w), device=dev, dtype=torch.float32)
            depth = conf = None
            if return_depth:
                depth = torch.empty((1, h, w), device=dev, dtype=torch.float32)
                conf = torch.empty((1, h, w), device=dev, dtype=torch.float32)
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            check(L.nrgbd_kvnet_forward(ent['h'], ptr(frames), ptr(poses), ptr(prior), ptr(dmap_cur), ptr(dmap_kv),
                                        ptr(bv_cur), ptr(dpv), ptr(depth), ptr(conf), st))
            # BatchNorm's num_batches_tracked side effect (train mode only), applied lazily; a replica shares the counters' owner
            owner = self.__dict__.get('_owner_ref', None)
            owner = owner() if owner is not None else self
            if owner is not None and self.training:
                owner.__dict__['_nb_pending'] = owner.__dict__.get('_nb_pending', 0) + 1
                if prior is not None:
                    owner.__dict__['_nb_pending_kv'] = owner.__dict__.get('_nb_pending_kv', 0) + 1
        if self._refine is None:
            dmap_cur = dmap_kv = -1                         # KVNET.py:136, 182
        if prior is None:
            out = (dmap_cur, dmap_cur, bv_cur, bv_cur)     # KVNET.py:138-143
        else:
            out = (dmap_cur, dmap_kv, bv_cur, dpv)
        return out + (depth, conf) if return_depth else out

    def propagate(self, kv_dpv, rel_pose_inv):
        """BV_predict for the next frame (test_utils/test_KVNet.py:46-59) through the engine:
        clamp(resample_vol_cuda(kv_dpv, rel_pose_inv, padding=log(1/D)), -1000, 0) -> [1,D,h,w]."""
        L = _lib.lib()
        dev = kv_dpv.device
        with torch.cuda.device(dev):
            _, D, h, w = kv_dpv.shape
            ent = None
            for (di, H, W, V), e in self._engines.items():
                if di == dev.index and H // 4 == h and W // 4 == w:
                    ent = e
            if ent is None:
                raise _lib.NrgbdError('propagate() needs a forward() at this resolution first')
            if ent['cams'][1] is None:
                self._set_camera(ent, 1, cam=self.cam_intrinsics)
            src = kv_dpv[0].float().contiguous()
            E = rel_pose_inv.to(device=dev, dtype=torch.float32).contiguous()
            out = torch.empty((1, D, h, w), device=dev, dtype=torch.float32)
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            check(L.nrgbd_kvnet_propagate(ent['h'], ptr(src), ptr(E), ptr(out), st))
        return out

    def _replicate_for_data_parallel(self):
        """nn.DataParallel replica: shares the engine table with its owner (engines are keyed by device, one per
        GPU) but never owns the native handles - only the module that created the table destroys them."""
        import weakref
        replica = super()._replicate_for_data_parallel()
        replica.__dict__['_owner_ref'] = self.__dict__.get('_owner_ref') or weakref.ref(self)
        replica.__dict__.pop('_plist', None)
        return replica

    def __del__(self):
        if self.__dict__.get('_is_replica', False) or self.__dict__.get('_owner_ref') is not None:
            return                      # handles belong to the owner module
        try:
            L = _lib.lib()
            engines = self.__dict__.get('_engines') or {}
            for ent in list(engines.values()):
                L.nrgbd_kvnet_destroy(ent['h'])
            engines.clear()
        except Exception:
            pass
