"""Seeded inputs of the polynomial transforms (binds of several variables, split, new_padded) and their oracle:
tests/golden/poly_transforms.json, tests/test_gpu_poly_transforms.py, tests/test_poly_transforms_host.py and
tools/poly_transform_bench.py.  The oracle entry points are oracle_dense/capi.cpp's orcd_poly_*."""
import ctypes as C
import hashlib

import numpy as np

import dense_poly_cases as dc
import oracle_dense_lib as od
import oracle_lib as ol
import pyref

# golden sizes, bind lengths and split points (len / SPLIT_DIV)
GOLDEN_NV = (22, 24)
GOLDEN_K = (1, 3, 8, 9, 12)
SPLIT_DIV = (2, 8)
PADDED_LEN = (1 << 22) + 1


def _lib():
    L = od.lib()
    L.orcd_poly_new_padded.restype = C.c_size_t
    return L


def bind(Z, r, top):
    """k sequential bound_poly_var_top / _bot calls of the oracle, r[0] first"""
    Z, r = np.ascontiguousarray(Z, dtype=np.uint64), np.ascontiguousarray(r, dtype=np.uint64).reshape(-1, 4)
    out = np.zeros((Z.shape[0] >> r.shape[0], 4), dtype=np.uint64)
    fn = _lib().orcd_poly_bind_top if top else _lib().orcd_poly_bind_bot
    fn(ol.P(Z), ol.sz(Z.shape[0]), ol.P(r), ol.sz(r.shape[0]), ol.P(out))
    return out


def split(Z, idx):
    Z = np.ascontiguousarray(Z, dtype=np.uint64)
    lo, hi = np.zeros((idx, 4), dtype=np.uint64), np.zeros((idx, 4), dtype=np.uint64)
    _lib().orcd_poly_split(ol.P(Z), ol.sz(Z.shape[0]), ol.sz(idx), ol.P(lo), ol.P(hi))
    return lo, hi


def new_padded(Z):
    Z = np.ascontiguousarray(Z, dtype=np.uint64).reshape(-1, 4)
    n = 1
    while n < Z.shape[0]:
        n <<= 1
    out = np.zeros((n, 4), dtype=np.uint64)
    assert _lib().orcd_poly_new_padded(ol.P(Z) if Z.shape[0] else None, ol.sz(Z.shape[0]), ol.P(out)) == n
    return out


# ---- the same in Python integers (tests/pyref.py): binds are linear, so Montgomery forms bind as integers mod l
def ints(a):
    return [int.from_bytes(np.ascontiguousarray(a[i]).tobytes(), "little") for i in range(a.shape[0])]


def py_bind(Z, r, top):
    """Z: Montgomery limbs (n, 4); r: Montgomery limbs (k, 4) -> Montgomery limbs of the k sequential binds"""
    z = ints(Z)
    for x in ol.fr_ints(r):
        z = pyref.bind_top(z, x) if top else pyref.bind_bot(z, x)
    return np.array([[(v >> (64 * j)) & (2**64 - 1) for j in range(4)] for v in z], dtype=np.uint64).reshape(-1, 4)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint64).tobytes()).hexdigest()


def golden_inputs(nv):
    """-> (Z (2^nv, 4) full width, r (12, 4))"""
    rng = np.random.default_rng(7000 + nv)
    return dc.random_full(rng, 1 << nv), dc.random_full(rng, max(GOLDEN_K))


def padded_input():
    return dc.random_full(np.random.default_rng(7100), PADDED_LEN)
