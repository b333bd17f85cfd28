"""Output stage (SURVEY 8 f-2): the oracle against the live-reference fixtures, and the host-side PGM writer of the
C ABI against the reference's own files (no GPU needed: nrgbd_write_pgm16 is host-only)."""
import ctypes
import os

import numpy as np
import pytest

from neuralrgbd_b200 import _lib
from oracle import export_oracle as E
from tests import cases, harness


gold = harness.golden_fixture('export_outputs.npz')


def parse_pgm16(b):
    b = bytes(b)
    assert b[:3] == b'P5\n'
    w, h = [int(t) for t in b[3:b.index(b'\n', 3)].split()]
    hdr = b'P5\n%d %d\n65535\n' % (w, h)
    assert b.startswith(hdr)
    return np.frombuffer(b[len(hdr):], '>u2').reshape(h, w).astype(np.int64)


@pytest.mark.parametrize('name', cases.EXPORT_CASES)
def test_oracle_matches_reference_export(gold, name):
    bv, d_candi, _ = cases.export_case(name)
    dmap, conf, d16, c16 = E.export_maps(bv[0], d_candi)
    # float maps: torch's vectorised exp / reduction order vs plain loops -> a few ulp
    assert np.max(np.abs(dmap - gold[name + '/dmap']) / np.abs(gold[name + '/dmap'])) <= 2e-6
    assert np.max(np.abs(conf - gold[name + '/conf']) / gold[name + '/conf']) <= 1e-6
    # uint16 maps (what the reference writes, depth in mm): within one LSB, and equal almost everywhere
    for mine, key in ((d16, '/d_pgm'), (c16, '/conf_pgm')):
        ref = parse_pgm16(gold[name + key])
        diff = np.abs(mine.astype(np.int64) - ref)
        assert diff.max() <= 1 and np.mean(diff != 0) <= 0.01


@pytest.mark.parametrize('name', cases.EXPORT_CASES)
def test_pgm_writer_is_byte_identical_to_reference_files(gold, name, tmp_path):
    """Feed the reference's own uint16 samples through the oracle's and the C ABI's writer: same bytes as PIL wrote."""
    for key in ('/d_pgm', '/conf_pgm'):
        ref_bytes = bytes(gold[name + key])
        im = parse_pgm16(ref_bytes).astype(np.uint16)
        assert E.pgm16_bytes(im) == ref_bytes
        path = str(tmp_path / 'x.pgm')
        L = _lib.lib()
        im = np.ascontiguousarray(im)
        assert L.nrgbd_write_pgm16(os.fsencode(path), ctypes.c_void_p(im.ctypes.data), im.shape[1], im.shape[0]) == 0
        assert open(path, 'rb').read() == ref_bytes


def test_pgm_writer_error_codes(tmp_path):
    L = _lib.lib()
    im = np.zeros((2, 3), np.uint16)
    assert L.nrgbd_write_pgm16(os.fsencode(str(tmp_path / 'no' / 'such' / 'dir.pgm')), ctypes.c_void_p(im.ctypes.data), 3, 2) == -5
    assert b'cannot open' in L.nrgbd_last_error()
    assert L.nrgbd_write_pgm16(None, ctypes.c_void_p(im.ctypes.data), 3, 2) == -1
    assert L.nrgbd_write_pgm16(os.fsencode(str(tmp_path / 'a.pgm')), ctypes.c_void_p(im.ctypes.data), 0, 2) == -1
