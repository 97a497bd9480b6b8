"""Seeded inputs of the grand-product tests over a caller's polynomials (tests/test_grand_product_host.py,
tests/test_gpu_grand_product.py, tests/golden/grand_product.json, tools/grand_product_bench.py).  Every array is derived
from a seed with numpy, so the GPU machine regenerates exactly what the golden hashes were computed from."""
import numpy as np

import dense_poly_cases as dc

# name -> (number of circuits, num_vars, seed); the small ones are reproduced by the CPU oracle in the host tests
GOLDEN = {
    "n3_nv6": (3, 6, 306), "n2_nv10": (2, 10, 210),
    "n2_nv20": (2, 20, 220), "n2_nv22": (2, 22, 222),
}
SMALL = ("n3_nv6", "n2_nv10")
TRANSCRIPT_LABEL = b"grand_product_golden"


def golden_inputs(name):
    """-> (num_vars, the n polynomials (2^nv, 4) of uniform canonical residues)"""
    n, nv, seed = GOLDEN[name]
    rng = np.random.default_rng(seed)
    return nv, [dc.random_full(rng, 1 << nv) for _ in range(n)]


def digest_input(res):
    """the bytes the golden SHA-256 covers: proof || products || rand || claims"""
    return res["proof"] + res["products"].tobytes() + res["r"].tobytes() + res["claims"].tobytes()
