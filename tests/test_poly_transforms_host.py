"""The oracle of the polynomial transforms (oracle_dense/capi.cpp orcd_poly_*) against Python integers (tests/pyref.py):
k sequential top and bottom binds, split and new_padded, on the CPU.  The GPU tests compare against both."""
import numpy as np
import pytest

import dense_poly_cases as dc
import poly_transform_cases as pt


@pytest.mark.parametrize("nv", [1, 2, 5, 9])
def test_binds_match_python_integers(nv):
    rng = np.random.default_rng(40 + nv)
    Z, r = dc.random_full(rng, 1 << nv), dc.random_full(rng, nv)
    for k in range(1, nv + 1):
        for top in (True, False):
            assert (pt.bind(Z, r[:k], top) == pt.py_bind(Z, r[:k], top)).all(), (k, top)


def test_split_and_padding():
    rng = np.random.default_rng(3)
    Z = dc.random_full(rng, 64)
    for idx in (1, 4, 32):
        lo, hi = pt.split(Z, idx)
        assert (lo == Z[:idx]).all() and (hi == Z[idx:2 * idx]).all()
    for n, want in ((0, 1), (1, 1), (3, 4), (5, 8), (64, 64)):
        got = pt.new_padded(Z[:n])
        assert got.shape == (want, 4) and (got[:n] == Z[:n]).all() and not got[n:].any()
