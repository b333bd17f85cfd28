"""Output stage on the device (SURVEY 8 f-2): nrgbd_export_depth_conf and the export_res mirror against the oracle,
the live-reference fixtures, and size-independent properties at the metric shape."""
import os

import numpy as np
import pytest
import torch

from oracle import export_oracle as E
from tests import cases, harness
from tests.test_oracle_export import parse_pgm16

pytestmark = pytest.mark.gpu


gold = harness.golden_fixture('export_outputs.npz')


@pytest.mark.parametrize('name', cases.EXPORT_CASES)
def test_export_kernel_vs_oracle_and_reference(gold, name):
    from neuralrgbd_b200.test_utils import export_res as X
    bv, d_candi, _ = cases.export_case(name)
    maps = X.depth_conf_maps(torch.from_numpy(bv).cuda(), d_candi)
    dmap, conf = maps['dmap'].cpu().numpy(), maps['conf'].cpu().numpy()
    d16 = maps['dmap_u16'].cpu().numpy().view(np.uint16).astype(np.int64)
    c16 = maps['conf_u16'].cpu().numpy().view(np.uint16).astype(np.int64)
    od, oc, od16, oc16 = E.export_maps(bv[0], d_candi)
    # same summation order as the oracle: only expf (device) vs np.exp separates them
    assert np.max(np.abs(dmap - od) / np.abs(od)) <= 1e-6
    assert np.max(np.abs(conf - oc) / oc) <= 1e-6
    assert np.abs(d16 - od16.astype(np.int64)).max() <= 1 and np.abs(c16 - oc16.astype(np.int64)).max() <= 1
    # against what the unmodified reference wrote: <= 1 LSB (1 mm of depth, 0.001 of confidence), equal almost everywhere
    for mine, key in ((d16, '/d_pgm'), (c16, '/conf_pgm')):
        diff = np.abs(mine - parse_pgm16(gold[name + key]))
        assert diff.max() <= 1 and np.mean(diff != 0) <= 0.01
    assert np.max(np.abs(dmap - gold[name + '/dmap']) / np.abs(gold[name + '/dmap'])) <= 2e-6


@pytest.mark.parametrize('name', cases.EXPORT_CASES[:2])
def test_export_res_img_writes_reference_files(gold, name, tmp_path):
    """Same call as test_utils/export_res.py:43 export_res_img; files parse to the reference's samples (+-1 LSB)."""
    from neuralrgbd_b200.test_utils import export_res as X
    bv, d_candi, img = cases.export_case(name)
    X.export_res_img({'img': torch.from_numpy(img).cuda()}, torch.from_numpy(bv).cuda(), d_candi, str(tmp_path), 7)
    for fn, key in (('d_00007.pgm', '/d_pgm'), ('conf_00007.pgm', '/conf_pgm')):
        mine = open(os.path.join(str(tmp_path), fn), 'rb').read()
        ref = bytes(gold[name + key])
        assert len(mine) == len(ref) and mine[:20] == ref[:20]
        diff = np.abs(parse_pgm16(mine) - parse_pgm16(ref))
        assert diff.max() <= 1 and np.mean(diff != 0) <= 0.01
    # depth_regression keeps the reference's (volume, BV) signature
    D, H, W = bv.shape[1:]
    vol = torch.ones(1, D, H, W, device='cuda') * torch.from_numpy(d_candi.astype(np.float32)).cuda().view(1, D, 1, 1)
    dm = X.depth_regression(vol, torch.from_numpy(bv).cuda())
    assert np.max(np.abs(dm - gold[name + '/dmap']) / np.abs(gold[name + '/dmap'])) <= 2e-6


def test_export_full_size_properties():
    """640x480x64 (BASELINE metric shape): bounds, agreement with depth_val_regression, one-hot and uniform DPVs."""
    from neuralrgbd_b200.mutils import misc
    from neuralrgbd_b200.test_utils import export_res as X
    D, H, W = 64, 480, 640
    d_candi = np.linspace(0.1, 5.0, D)
    g = torch.Generator(device='cuda').manual_seed(3)
    bv = torch.log_softmax(torch.randn((1, D, H, W), device='cuda', generator=g) * 4, dim=1)
    m = X.depth_conf_maps(bv, d_candi)
    dmap, conf = m['dmap'], m['conf']
    assert float(dmap.min()) >= 0.1 - 1e-5 and float(dmap.max()) <= 5.0 + 1e-5
    assert float(conf.min()) >= 1.0 / D - 1e-6 and float(conf.max()) <= 1.0 + 1e-6
    ref = misc.depth_val_regression(bv, d_candi, BV_log=True)
    assert float((ref.reshape(H, W) - dmap).abs().max()) <= 2e-6 * 5.0
    d16 = m['dmap_u16'].cpu().numpy().view(np.uint16).astype(np.int64)
    assert np.abs(d16 - np.floor(dmap.cpu().numpy().astype(np.float32) * np.float32(1000))).max() == 0
    # one-hot DPV: depth is exactly the plane, confidence 1 -> 1000
    k = torch.randint(0, D, (H, W), device='cuda', generator=g)
    hot = torch.full((1, D, H, W), -1e4, device='cuda')
    hot.scatter_(1, k.view(1, 1, H, W), 0.0)
    mh = X.depth_conf_maps(hot, d_candi)
    want = torch.from_numpy(d_candi.astype(np.float32)).cuda()[k]
    assert float((mh['dmap'] - want).abs().max()) == 0.0
    assert int(mh['conf_u16'].cpu().numpy().view(np.uint16).min()) == 1000
    # uniform DPV: mean plane depth, confidence 1/D
    uni = torch.full((1, D, H, W), float(np.log(1.0 / D)), device='cuda')
    mu = X.depth_conf_maps(uni, d_candi)
    assert abs(float(mu['dmap'][0, 0]) - float(d_candi.mean())) <= 1e-5
    assert int(mu['conf_u16'][0, 0].cpu().numpy().view(np.uint16)) == int(np.float32(np.exp(np.float32(np.log(1.0 / D)))) * np.float32(1000))


def test_export_res_refineNet_products(tmp_path):
    """export_res.py:77-160 mirror: .mat contents, 16-bit depth PNG, cv2 (BGR) byte order of rgb_*.png, KeyError on a frame dict
    without 'img_path' (the reference indexes it), previews only with matplotlib."""
    import scipy.io as sio
    import PIL.Image as image
    from neuralrgbd_b200.test_utils import export_res as X
    bv, d_candi, img = cases.export_case('export_48x64_d16')
    ref_dat = {'img': torch.from_numpy(img), 'img_path': 'scene0000/frame-000010.color.jpg'}
    dmap, conf = X.export_res_refineNet(ref_dat, torch.from_numpy(bv).cuda(), d_candi, str(tmp_path), 7, output_pngs=True, save_mat=True,
                                        output_dmap_ref=False)
    od, oc, od16, _ = E.export_maps(bv[0], d_candi)
    assert np.max(np.abs(dmap - od) / np.abs(od)) <= 1e-6 and np.max(np.abs(conf - oc) / oc) <= 1e-6
    m = sio.loadmat(str(tmp_path / 'depth_00007.mat'))
    assert np.array_equal(m['dmap'], dmap) and np.array_equal(m['confMap'], conf) and m['img_path'][0] == ref_dat['img_path']
    d_png = np.array(image.open(str(tmp_path / 'output_pngs' / 'd_00007.png')))
    assert np.abs(d_png.astype(np.int64) - od16.astype(np.int64)).max() <= 1
    rgb = np.array(image.open(str(tmp_path / 'output_pngs' / 'rgb_00007.png')))
    want = (X._un_normalize(img[0].transpose(1, 2, 0)) * 255).astype(np.uint8)
    assert np.array_equal(rgb[:, :, ::-1], want)                       # decoded R channel = the array's B channel, as cv2.imwrite leaves it
    try:
        import matplotlib      # noqa: F401
        assert (tmp_path / 'res_00007.png').exists() and (tmp_path / 'conf.png').exists()
    except ImportError:
        assert not (tmp_path / 'res_00007.png').exists()
    with pytest.raises(KeyError):
        X.export_res_refineNet({'img': torch.from_numpy(img)}, torch.from_numpy(bv).cuda(), d_candi, str(tmp_path), 8, output_dmap_ref=False)
