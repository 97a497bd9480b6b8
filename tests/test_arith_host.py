"""The op table of tests/kernel_harness/arith_ops.cuh compiled with g++ from the headers and run on the host, on the
same edge grids and against the same plain-integer references as test_gpu_arith.py (arith_cases.py).  On the host
the carry chains are the emulated ones of fr.cuh and fr_mul / fr_inv take the 64-bit paths of the prover's
Fiat-Shamir glue.  The quad-lane operations use warp shuffles and are device only."""
import ctypes as C
import os
import subprocess

import pytest

import arith_cases as ac
import kernel_harness_lib as kh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WRAPPER = r'''
#include <cstddef>
#include "arith_ops.cuh"
extern "C" const char* kh_arith_op_name(int op) { return arith::op_name(op); }
extern "C" int kh_arith_host(int op, size_t n, const uint64_t* a, const uint64_t* b, const uint64_t* k, uint64_t* out) {
  if (!arith::op_name(op) || op >= arith::OP_quad_add) return -4;
  for (size_t i = 0; i < n; i++)
    arith::apply(op, (const uint32_t*)(a + 16 * i), (const uint32_t*)(b + 16 * i), k[i], (uint32_t*)(out + 16 * i));
  return 0;
}
'''


@pytest.fixture(scope="module")
def host_run(tmp_path_factory):
    d = tmp_path_factory.mktemp("arith_host")
    src, so = d / "arith_host.cpp", d / "libarith_host.so"
    src.write_text(WRAPPER)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wno-psabi", "-shared", "-fPIC",
                           "-I", os.path.join(ROOT, "tests", "kernel_harness"), str(src), "-o", str(so)])
    lib = C.CDLL(str(so))
    lib.kh_arith_op_name.argtypes = [C.c_int]
    lib.kh_arith_op_name.restype = C.c_char_p
    lib.kh_arith_host.argtypes = [C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    ids = kh.op_ids(lib.kh_arith_op_name)

    def run(name, A, B, K):
        import numpy as np

        out = np.zeros_like(A)
        rc = lib.kh_arith_host(ids[name], A.shape[0], A.ctypes.data, B.ctypes.data, K.ctypes.data, out.ctypes.data)
        assert rc == 0, "kh_arith_host(%s) returned %d" % (name, rc)
        return out

    run.ids = ids
    return run


def test_op_table_matches_the_cases(host_run):
    """every operation of arith_ops.cuh has a reference here, and the other way round"""
    assert set(host_run.ids) == set(ac.OPS)


@pytest.mark.parametrize("name", ac.THREAD_OPS)
def test_host_op(host_run, name):
    ac.check_op(host_run, "host", name)
