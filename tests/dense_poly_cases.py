"""Seeded inputs of the dense-polynomial cases at size (tests/golden/dense_poly.json, tests/test_gpu_dense_poly.py,
tools/dense_poly_bench.py).  Every array is derived from the case's seed with numpy and the oracle's u64 -> Fr
conversion, so the GPU machine regenerates exactly what the golden hashes were computed from."""
import numpy as np

import oracle_lib as ol

# name -> (num_vars, values, seed); values "full": uniform Montgomery limbs below 2^252 (canonical residues whose
# integer values are full width), "u16": integers below 2^16 (the polynomial commits through the 16-bit tables)
CASES = {
    "full_nv20": (20, "full", 2020), "u16_nv20": (20, "u16", 1620),
    "full_nv22": (22, "full", 2022), "u16_nv22": (22, "u16", 1622),
    "full_nv24": (24, "full", 2024), "u16_nv24": (24, "u16", 1624),
}
TRANSCRIPT_LABEL, TAPE_LABEL, COMMIT_LABEL = b"dense_poly_golden", b"proof", b"poly"


def fr_from_u64(v):
    v = np.ascontiguousarray(v, dtype=np.uint64)
    out = np.zeros((v.shape[0], 4), dtype=np.uint64)
    ol.lib().orc_fr_from_u64_batch(ol.P(v), ol.sz(v.shape[0]), ol.P(out))
    return out


def random_full(rng, n):
    """n canonical Montgomery residues: four uniform limbs, the top one below 2^60 (so below 2^252 < l)"""
    z = rng.integers(0, 2**64, size=(n, 4), dtype=np.uint64)
    z[:, 3] &= np.uint64(2**60 - 1)
    return z


def inputs(name):
    """-> (num_vars, Z (2^nv, 4), r (nv, 4), tape seed (4,))"""
    nv, values, seed = CASES[name]
    rng = np.random.default_rng(seed)
    n = 1 << nv
    Z = random_full(rng, n) if values == "full" else fr_from_u64(rng.integers(0, 1 << 16, size=n, dtype=np.uint64))
    r = random_full(rng, nv)
    tape_seed = random_full(rng, 1)[0]
    return nv, Z, r, tape_seed


def n_generators(nv):
    return (1 << (nv - nv // 2)) + 2
