"""Seeded inputs of the combined-opening tests (tests/test_combined_eval_host.py, tests/test_gpu_combined_eval.py,
tests/golden/combined_eval.json).  Every array is derived from a seed with numpy, so the GPU machine regenerates exactly
what the golden hashes were computed from."""
import numpy as np

import dense_poly_cases as dc

# name -> (number of components k, component num_vars, values, seed); values "full": uniform canonical residues, "u32":
# integers below 2^32.  The merged polynomial has nv + log2(next_pow2(k)) variables.  All of them are small enough for
# the CPU oracle, which the host tests run on the SMALL ones.
GOLDEN = {
    "k3_nv4_full": (3, 4, "full", 34), "k5_nv6_u32": (5, 6, "u32", 56), "k8_nv7_full": (8, 7, "full", 87),
    "k4_nv18_u32": (4, 18, "u32", 418), "k3_nv18_full": (3, 18, "full", 318),
}
SMALL = ("k3_nv4_full", "k5_nv6_u32", "k8_nv7_full")
TRANSCRIPT_LABEL, TAPE_LABEL = b"combined_eval_golden", b"proof"


def values(kind, n, rng):
    if kind == "full":
        return dc.random_full(rng, n)
    return dc.fr_from_u64(rng.integers(0, 1 << 32, size=n, dtype=np.uint64))


def golden_inputs(name):
    """-> (component num_vars, the k components (2^nv, 4), r (nv, 4), tape seed (4,))"""
    k, nv, kind, seed = GOLDEN[name]
    rng = np.random.default_rng(seed)
    comps = [values(kind, 1 << nv, rng) for _ in range(k)]
    r = dc.random_full(rng, nv)
    tape_seed = dc.random_full(rng, 1)[0]
    return nv, comps, r, tape_seed


def digest_input(evals, proof):
    """the bytes the golden SHA-256 covers: evals || proof"""
    return np.ascontiguousarray(evals, dtype=np.uint64).tobytes() + proof
