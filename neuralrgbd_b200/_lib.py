"""ctypes binding of libnrgbd.so (include/nrgbd.h). Fails loudly when the library is missing:
there is no CPU or PyTorch fallback for any entry point."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libnrgbd.so')

c_int, c_float, c_ll, c_vp = ctypes.c_int, ctypes.c_float, ctypes.c_longlong, ctypes.c_void_p

# name -> (restype, argtypes); mirrors include/nrgbd.h one to one.
SIGNATURES = {
    'nrgbd_abi_version': (c_int, []),
    'nrgbd_last_error': (ctypes.c_char_p, []),
    'nrgbd_launch_count': (c_ll, []),
    'nrgbd_reset_launch_count': (None, []),
    'nrgbd_sweep_channel_split': (None, [c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    'nrgbd_pack_features': (c_int, [c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    'nrgbd_transpose2d': (c_int, [c_vp, c_int, c_int, c_vp, c_vp]),
    'nrgbd_sweep_workspace_floats': (c_int, [c_int]),
    'nrgbd_plane_sweep_cost_packed': (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int,
                                              c_vp, c_vp, c_vp, c_vp, c_vp, c_float, c_float, c_float, c_int,
                                              c_vp, c_vp, c_vp]),
    'nrgbd_plane_sweep_dpv_packed': (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int,
                                             c_vp, c_vp, c_vp, c_vp, c_vp, c_float, c_float, c_float, c_int,
                                             c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_warp_to_volume': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp,
                                     c_vp, c_vp, c_float, c_float, c_vp, c_vp, c_vp]),
    'nrgbd_knet_input_volume': (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                        c_vp, c_vp, c_vp, c_float, c_float, c_vp, c_vp, c_vp]),
    'nrgbd_knet_input_volume_pair': (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                             c_vp, c_vp, c_vp, c_float, c_float, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_resample_dpv': (c_int, [c_vp, c_ll, c_ll, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_float, c_float,
                                   c_float, c_float, c_float, c_int, c_float, c_float, c_vp, c_ll, c_ll, c_vp]),
    'nrgbd_dpv_normalize': (c_int, [c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_float, c_int, c_int, c_vp, c_ll, c_ll,
                                    c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_depth_regression': (c_int, [c_vp, c_int, c_int, c_ll, c_ll, c_vp, c_int, c_vp, c_vp, c_vp]),
    'nrgbd_exp': (c_int, [c_vp, c_ll, c_vp, c_vp]),
    'nrgbd_pack_conv_weight': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    'nrgbd_conv_nhwc': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int, c_int, c_int,
                                c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp,
                                c_vp]),
    'nrgbd_conv_transpose2d_k4s2_nhwc': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int, c_int,
                                                 c_vp, c_int, c_int, c_int, c_vp]),
    'nrgbd_conv_tc_supported': (c_int, [c_int, c_int]),
    'nrgbd_split_tf32': (c_int, [c_vp, c_ll, c_vp, c_vp, c_vp]),
    'nrgbd_pack_conv_weight_tc': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    'nrgbd_conv_nhwc_tc': (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_int,
                                   c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp,
                                   c_vp]),
    'nrgbd_conv_transpose2d_k4s2_nhwc_tc': (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int,
                                                    c_int, c_vp, c_int, c_int, c_int, c_vp]),
    'nrgbd_conv_tc2_supported': (c_int, [c_int, c_int]),
    'nrgbd_conv_nhwc_tc2': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_int,
                                    c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp,
                                    c_vp]),
    'nrgbd_conv_nhwc_tc2_bn_in': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_int,
                                          c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp,
                                          c_vp, c_vp]),
    'nrgbd_conv_transpose2d_k4s2_nhwc_tc2': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int,
                                                     c_int, c_vp, c_int, c_int, c_int, c_vp]),
    'nrgbd_conv_h2_plan': (c_int, [c_int, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    'nrgbd_split_f16_pair': (c_int, [c_vp, c_ll, c_vp, c_vp, c_vp]),
    'nrgbd_pack_conv_weight_h2': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    'nrgbd_conv_nhwc_h2': (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int, c_int, c_int,
                                   c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp,
                                   c_vp]),
    'nrgbd_conv_nhwc_h2_pair': (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int, c_int, c_int,
                                        c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp]),
    'nrgbd_conv_transpose2d_k4s2_nhwc_h2': (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int, c_int,
                                                    c_int, c_vp, c_int, c_int, c_int, c_vp]),
    'nrgbd_bn_finalize': (c_int, [c_vp, c_int, ctypes.c_double, c_vp, c_vp, c_float, c_vp, c_vp, c_vp, c_vp,
                                  c_float, c_vp]),
    'nrgbd_bn_apply_stats': (c_int, [c_vp, c_vp, ctypes.c_double, c_vp, c_vp, c_float, c_vp, c_vp, c_float, c_vp, c_int, c_ll,
                                     c_int, c_int, c_vp, c_vp]),
    'nrgbd_tap_gather_sum': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_vp, c_vp]),
    'nrgbd_bn_apply_stats_pair': (c_int, [c_vp, c_vp, ctypes.c_double, c_vp, c_vp, c_float, c_vp, c_vp, c_float, c_vp, c_vp, c_vp, c_int,
                                          c_ll, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_bn_apply': (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_ll, c_int, c_int, c_vp, c_vp]),
    'nrgbd_nchw_to_nhwc': (c_int, [c_vp, c_int, c_int, c_ll, c_vp, c_int, c_int, c_vp]),
    'nrgbd_nhwc_to_nchw': (c_int, [c_vp, c_int, c_int, c_ll, c_int, c_int, c_vp, c_vp]),
    'nrgbd_avgpool_nhwc': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_vp]),
    'nrgbd_upsample_bilinear_ac_nhwc': (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                                c_int, c_vp]),
    'nrgbd_copy_channels': (c_int, [c_vp, c_ll, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_vp]),
    'nrgbd_plane_sweep_backward_packed': (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp,
                                                  c_vp, c_vp, c_float, c_float, c_float, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_unpack_features': (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    'nrgbd_lba_back_warp': (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    'nrgbd_lba_back_warp_backward': (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp,
                                             c_vp]),
    'nrgbd_preprocess_rgb_u8': (c_int, [c_vp, c_int, c_int, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_export_depth_conf': (c_int, [c_vp, c_vp, c_int, c_ll, c_float, c_float, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_write_pgm16': (c_int, [ctypes.c_char_p, c_vp, c_int, c_int]),
    'nrgbd_kvnet_create': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int, ctypes.POINTER(c_vp)]),
    'nrgbd_kvnet_destroy': (c_int, [c_vp]),
    'nrgbd_kvnet_set_param': (c_int, [c_vp, ctypes.c_char_p, c_vp, c_ll, c_int]),
    'nrgbd_kvnet_set_camera': (c_int, [c_vp, c_int, c_vp, c_vp, c_float, c_float, ctypes.c_double, ctypes.c_double]),
    'nrgbd_kvnet_set_planes': (c_int, [c_vp, c_vp, c_int]),
    'nrgbd_kvnet_set_option': (c_int, [c_vp, ctypes.c_char_p, c_int]),
    'nrgbd_kvnet_workspace_bytes': (c_ll, [c_vp]),
    'nrgbd_kvnet_profile_read': (c_int, [c_vp, c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                         ctypes.POINTER(c_ll)]),
    'nrgbd_kvnet_profile_table': (c_int, [c_vp, c_int, ctypes.c_char_p, c_ll]),
    'nrgbd_kvnet_forward': (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'nrgbd_kvnet_propagate': (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp]),
}

# include/nrgbd_dev.h: development probes / A-B knobs. Bound only by dev_lib() (tools/, kernel-variant tests), never by the
# product modules.
DEV_SIGNATURES = {
    'nrgbd_dev_set_bn_unroll': (None, [c_int]),
    'nrgbd_dev_set_bn_blocks_per_sm': (None, [c_int]),
    'nrgbd_dev_conv_h2_set_flags': (None, [c_int]),
    'nrgbd_dev_conv_h2_set_smem_cap_kb': (None, [c_int]),
}


class BnInput(ctypes.Structure):
    """include/nrgbd.h: nrgbd_bn_input."""
    _fields_ = [('stats', c_vp), ('count', ctypes.c_double), ('gamma', c_vp), ('beta', c_vp), ('running_mean', c_vp),
                ('running_var', c_vp), ('eps', c_float), ('momentum', c_float), ('relu', c_int), ('C', c_int)]


_lib = None


class NrgbdError(RuntimeError):
    pass


def lib():
    """Load libnrgbd.so once. Raises if it has not been built (python -m neuralrgbd_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NrgbdError('libnrgbd.so not found at %s: build it with `python -m neuralrgbd_b200.build` '
                             '(there is no fallback path)' % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)      # AttributeError if the library does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def dev_lib():
    """The library with the development entry points of include/nrgbd_dev.h bound as well (tools and variant tests only)."""
    L = lib()
    if not getattr(L, '_nrgbd_dev_bound', False):
        for name, (res, args) in DEV_SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        L._nrgbd_dev_bound = True
    return L


def check(rc):
    if rc != 0:
        msg = lib().nrgbd_last_error()
        raise NrgbdError('nrgbd error %d: %s' % (rc, msg.decode() if msg else ''))


def ptr(t):
    """Device pointer of a CUDA float32 contiguous tensor (or None)."""
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), 'nrgbd entry points take contiguous CUDA tensors'
    return ctypes.c_void_p(t.data_ptr())
