"""neuralrgbd_b200: H100-native plane-sweep depth-probability-volume engine behind the
NVlabs/neuralrgbd call surface (`models.KVNET.KVNET`, `warping.homography.*`, `mutils.misc`).

`install_as_reference_modules()` puts the engine behind the reference's own import names so that an
unmodified reference checkout (its `code/` directory) runs on it: the reference's modules stay the
modules that are imported - only the hot-path symbols SURVEY 8(a) lists are re-pointed to the mirrors.
"""
import importlib
import os
import sys
import types

# reference module -> (mirror module, symbols that are re-pointed)
_PATCHES = (
    ('warping.homography', 'neuralrgbd_b200.warping.homography',
     ('est_swp_volume_v4', 'warp_img_feats_v3', 'warp_img_feats_mgpu', 'resample_vol_cuda', 'get_rel_extrinsicM',
      'back_warp_th_Rt', 'back_warp_th_Rt_msrc')),
    ('mutils.misc', 'neuralrgbd_b200.mutils.misc', ('depth_val_regression', 'valid_dpv')),
    ('models.KVNET', 'neuralrgbd_b200.models.KVNET', ('KVNET',)),
)


def install_as_reference_modules(reference_code_dir=None):
    """Route the reference's hot path through libnrgbd.

    reference_code_dir: the `code/` directory of an NVlabs/neuralrgbd checkout (e.g. $NRGBD_REFERENCE_CODE). It is put on
    sys.path and the reference's OWN modules are imported; then the mirrored functions / classes are set as
    attributes on them (`warping.homography.est_swp_volume_v4`, `warp_img_feats_v3`, `warp_img_feats_mgpu`,
    `resample_vol_cuda`, `mutils.misc.depth_val_regression`, `models.KVNET.KVNET`, ...). Everything else the reference
    modules define (`warping.View`, `mutils.misc.get_entries_list_dict`, `m_makedir`, `save_ScenePathInfo`, the
    data loaders' imports) keeps working, because the packages are not replaced.  The unmodified
    `test_utils/test_KVNet.py:test` looks both `warp_homo.resample_vol_cuda` and `model_KV(...)` up at call time,
    so it runs on the engine as is.

    Without a reference checkout (reference_code_dir=None and `warping` not importable) the mirrors themselves are
    registered under the reference's names - enough for code that only needs the mirrored symbols.

    Returns a namespace with the three patched (or registered) modules and `patched`: {module: [symbols]}.
    """
    if reference_code_dir is not None:
        reference_code_dir = os.path.abspath(reference_code_dir)
        if not os.path.isdir(os.path.join(reference_code_dir, 'warping')):
            raise FileNotFoundError('%s is not the code/ directory of a neuralrgbd checkout' % reference_code_dir)
        if reference_code_dir not in sys.path:
            sys.path.insert(0, reference_code_dir)
    mods, patched = {}, {}
    for ref_name, mirror_name, symbols in _PATCHES:
        mirror = importlib.import_module(mirror_name)
        ref_mod = sys.modules.get(ref_name)
        if ref_mod is None or (getattr(ref_mod, '__name__', '') or '').startswith('neuralrgbd_b200'):
            try:
                sys.modules.pop(ref_name, None)
                ref_mod = importlib.import_module(ref_name)
                if (getattr(ref_mod, '__file__', '') or '').startswith(os.path.dirname(os.path.abspath(__file__))):
                    raise ImportError('resolved to the mirror package')
            except Exception:
                if reference_code_dir is not None:
                    raise
                ref_mod = None
        if ref_mod is None:
            # no reference on the path: register the mirror (and its package) under the reference's names
            pkg_name = ref_name.split('.')[0]
            if pkg_name not in sys.modules:
                sys.modules[pkg_name] = importlib.import_module('neuralrgbd_b200.' + pkg_name)
            sys.modules[ref_name] = mirror
            mods[ref_name] = mirror
            patched[ref_name] = list(symbols)
            continue
        for s in symbols:
            if not hasattr(ref_mod, '_nrgbd_original_' + s):
                setattr(ref_mod, '_nrgbd_original_' + s, getattr(ref_mod, s, None))
            setattr(ref_mod, s, getattr(mirror, s))
        mods[ref_name] = ref_mod
        patched[ref_name] = list(symbols)
    return types.SimpleNamespace(homography=mods['warping.homography'], misc=mods['mutils.misc'],
                                 KVNET=mods['models.KVNET'], patched=patched)


def uninstall_reference_patches():
    """Undo install_as_reference_modules() on the reference's modules (used by the tests)."""
    for ref_name, _, symbols in _PATCHES:
        m = sys.modules.get(ref_name)
        if m is None:
            continue
        if (getattr(m, '__name__', '') or '').startswith('neuralrgbd_b200'):
            sys.modules.pop(ref_name, None)
            continue
        for s in symbols:
            orig = getattr(m, '_nrgbd_original_' + s, None)
            if orig is not None:
                setattr(m, s, orig)
                delattr(m, '_nrgbd_original_' + s)
