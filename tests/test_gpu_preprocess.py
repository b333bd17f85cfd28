"""f-4 on the device: resize + normalise kernel bit-exact against the oracle / the reference transform, and the
resident sliding window."""
import numpy as np
import pytest
import torch

from oracle import preprocess_oracle as P
from tests import cases, harness

pytestmark = pytest.mark.gpu


gold = harness.golden_fixture('preprocess_outputs.npz')


@pytest.mark.parametrize('name', cases.PREPROCESS_CASES)
def test_device_transform_bit_exact(gold, name):
    from neuralrgbd_b200.mdataloader import m_preprocess as M
    img, size = cases.preprocess_case(name)
    out = M.device_transform(img, size)
    assert out.is_cuda and tuple(out.shape) == gold[name].shape
    assert np.array_equal(out.cpu().numpy(), gold[name])                 # reference transform, bit for bit
    assert np.array_equal(out.cpu().numpy(), P.preprocess(img, size))
    # a device-resident uint8 frame and the get_transform() callable give the same tensor
    out2 = M.get_transform(size)(torch.from_numpy(img).cuda())
    assert torch.equal(out, out2)


def test_full_size_scannet_frame_and_window():
    """1296x968 raw ScanNet frame -> 640x480 (the metric shape): bit-exact against the oracle; FrameWindow keeps
    2*t_win_r+1 frames resident and hands out the reference's (ref, src) split."""
    from neuralrgbd_b200.mdataloader import m_preprocess as M
    rng = np.random.RandomState(3)
    frames = [rng.randint(0, 256, (968, 1296, 3)).astype(np.uint8) for _ in range(6)]
    want = [P.preprocess(f, (640, 480)) for f in frames]
    win = M.FrameWindow(t_win_r=2, img_size=(640, 480))
    full = [win.push(f, extM=np.eye(4) * i) for i, f in enumerate(frames)]
    assert full == [False, False, False, False, True, True]
    ref, src = win.window()                      # frames 1..5, reference = frame 3
    assert tuple(ref.shape) == (1, 3, 480, 640) and tuple(src.shape) == (1, 4, 3, 480, 640)
    assert np.array_equal(ref.cpu().numpy(), want[3])
    for k, i in enumerate((1, 2, 4, 5)):
        assert np.array_equal(src[0, k].cpu().numpy(), want[i][0])
    dicts = win.frame_dicts()
    assert len(dicts) == 5 and dicts[2]['extM'][0, 0] == 3
    # value range of a normalised image: ((0..255)/255 - mean)/std
    lo = (0 - 0.485) / 0.229; hi = (1 - 0.406) / 0.225
    assert float(ref.min()) >= lo - 1e-5 and float(ref.max()) <= hi + 1e-5


def test_input_stage_has_no_cpu_path():
    from neuralrgbd_b200 import _lib
    from neuralrgbd_b200.mdataloader import m_preprocess as M
    with pytest.raises(_lib.NrgbdError):
        M.device_transform(np.zeros((4, 4, 3), np.uint8), None, device='cpu')
