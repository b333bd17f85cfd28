"""f-4: the input-stage oracle (PIL NEAREST + ToTensor + Normalize restated) is bit-identical to the reference transform."""
import numpy as np
import pytest

from oracle import preprocess_oracle as P
from tests import cases, harness


gold = harness.golden_fixture('preprocess_outputs.npz')


@pytest.mark.parametrize('name', cases.PREPROCESS_CASES)
def test_oracle_bit_identical_to_reference_transform(gold, name):
    img, size = cases.preprocess_case(name)
    out = P.preprocess(img, size)
    assert out.dtype == np.float32 and out.shape == gold[name].shape
    assert np.array_equal(out, gold[name])


def test_host_index_table_matches_oracle():
    from neuralrgbd_b200.mdataloader import m_preprocess as M
    for n_out, n_in in ((480, 968), (640, 1296), (33, 100), (77, 100), (5, 7), (64, 64), (80, 53)):
        assert np.array_equal(M.nearest_index(n_out, n_in).astype(np.int64), P.nearest_index(n_out, n_in))
