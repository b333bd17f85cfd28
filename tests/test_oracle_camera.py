"""a14: the host-side camera recipe against the reference's own (CPU only).

tests/golden/camera_outputs.npz holds what the UNMODIFIED mdataloader/scanNet.py:read_IntM_from_txt (:204-272)
+ warping/View.py:32-62 returned for the calibrations of tests/cases.py:CAMERA_CASES. Both
neuralrgbd_b200.camera.make_cam_intrinsics (product: the dict handed to the engine) and
oracle.planesweep_oracle.make_cam_intrinsics (the function every other fixture's inputs are built with) must
reproduce it BIT FOR BIT - same float64 expressions, same float32 casts.
"""
import numpy as np
import pytest

from neuralrgbd_b200 import camera
from oracle import planesweep_oracle as O
from tests import cases, harness


gold = harness.golden_fixture('camera_outputs.npz')


def _np(x):
    return x.numpy() if hasattr(x, 'numpy') else np.asarray(x)


@pytest.mark.parametrize('impl', ['product', 'oracle'])
@pytest.mark.parametrize('name', list(cases.CAMERA_CASES))
def test_camera_recipe_bit_identical_to_reference(gold, name, impl):
    c = cases.CAMERA_CASES[name]
    if impl == 'product':
        cam = camera.make_cam_intrinsics(c['fx'], c['fy'], c['cx'], c['cy'], c['out_size'], full_width=c['width'])
    else:
        cam = O.make_cam_intrinsics(c['fx'], c['fy'], c['cx'], c['cy'], c['out_size'])
    sc = gold[name + '/scalars']
    assert cam['hfov'] == sc[0] and cam['vfov'] == sc[1]
    if impl == 'product' or 2.0 * c['cx'] == c['width']:          # the oracle assumes a centred principal point for this one
        assert cam['focal_length'] == sc[2]
    assert np.array_equal(np.asarray(cam['intrinsic_M'], np.float64), gold[name + '/intrinsic_M'])
    assert np.array_equal(_np(cam['intrinsic_M_cuda']), gold[name + '/intrinsic_M_cuda'])
    r2 = _np(cam['unit_ray_array_2D'])
    assert r2.dtype == np.float32 and np.array_equal(r2, gold[name + '/unit_ray_array_2D'])
    ura = np.asarray(cam['unit_ray_array'], np.float64)
    st = gold[name + '/unit_ray_array_stats']
    assert ura.shape == (c['out_size'][1], c['out_size'][0], 3)
    assert ura[0, 0, 0] == st[2] and ura[-1, -1, 1] == st[3]
    assert abs(ura.sum() - st[0]) <= 1e-9 * max(1.0, abs(st[0]))


def test_fixture_generators_use_the_pinned_recipe():
    """cases.cam_for / cases.big_cam feed every sweep / KVNET fixture: same function object as the one pinned above."""
    cam = cases.cam_for(O.make_cam_intrinsics, 160, 120)
    ref = O.make_cam_intrinsics(cases.FX, cases.FY, cases.CX, cases.CY, [160, 120])
    assert np.array_equal(cam['unit_ray_array_2D'], ref['unit_ray_array_2D'])
