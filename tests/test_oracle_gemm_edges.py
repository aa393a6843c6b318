"""CPU checks of the GEMM edge cases (tests/gemm_edge_cases.py) that tests/test_gpu_gemm_edges.py runs on the device: every builder's oracle
output holds the edge the case is named for (the builders assert it), and the torch restatement the device tests use as their reference
gives the oracle's bits on every case, NaN positions included."""
import numpy as np
import pytest

from tests import gemm_edge_cases as edges


@pytest.mark.parametrize("name", edges.CASE_NAMES)
def test_case_holds_its_edge_and_restatement_matches_oracle(name):
    c = edges.build(name)
    assert c.name == name
    M, N = c.out.shape
    assert c.aq.shape[0] == M and c.wt.w8.shape == (N, c.aq.shape[1])
    assert edges.same_bits(edges.restated_out(c), c.out)


def test_same_bits_compares_nan_positions_only():
    a = np.array([1.0, np.nan, -0.0], np.float16)
    b = a.copy()
    b.view(np.uint16)[1] = 0x7E01  # another NaN payload
    assert edges.same_bits(a, b)
    assert not edges.same_bits(a, np.array([1.0, np.nan, 0.0], np.float16))   # -0 vs +0
    assert not edges.same_bits(a, np.array([np.nan, np.nan, -0.0], np.float16))
