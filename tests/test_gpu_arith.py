"""The field and group primitives of the sm_90a build, one operation at a time, against plain Python integers
(arith_cases.py): Fr in Montgomery form, the loosely reduced Fq at the limb patterns and values near q and 2^256
where its carries and folds run, the Edwards group law on the 8-torsion and on several projective representatives
of each point, and the quad-lane forms of quad.cuh with eight different quads in every warp.

Each operation runs in both compilations of fq_mul the library uses (tests/kernel_harness/arith_default.cu: inlined,
arguments by reference; arith_msm.cu: out of line, by value, as in msm_kernels.cu and msm_large.cu).  A failure
names the operation, the variant, the element, its inputs in hex and the value received against the one wanted."""
import numpy as np
import pytest

import arith_cases as ac
import kernel_harness_lib as kh

pytestmark = pytest.mark.gpu

VARIANTS = {"default": 0, "msm": 1}


@pytest.fixture(scope="module")
def ids():
    return kh.op_ids(kh.lib().kh_arith_op_name)


def test_op_table_matches_the_cases(ids):
    assert set(ids) == set(ac.OPS)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", list(ac.OPS))
def test_device_op(ids, name, variant):
    def run(op, A, B, K):
        out = np.zeros_like(A)
        kh.call("kh_arith", VARIANTS[variant], ids[op], A.shape[0], A.ctypes.data, B.ctypes.data, K.ctypes.data,
                out.ctypes.data)
        return out

    ac.check_op(run, variant, name)
