"""Combining functions and seeded inputs of the sumcheck tests over a caller's polynomials (tests/test_sumcheck_host.py,
tests/test_gpu_sumcheck.py, tests/golden/sumcheck.json, tools/sumcheck_bench.py).  Every array is derived from a seed
with numpy and the oracle's conversions, so the GPU machine regenerates exactly what the golden hashes were computed
from.  A combining function is a plain Python function of a list of values: traced by lasso_b200.Comb, and called on
Python integers (mod l) for checks that depend on neither interpreter."""
import numpy as np

import dense_poly_cases as dc
import oracle_lib as ol

L = ol.L_FR


def spartan(v):  # eq(tau, x) * (A(x) * B(x) - C(x))
    return v[0] * (v[1] * v[2] - v[3])


def prod9(v):  # eq * prod_{i < 8} P_i: degree 9
    g = v[0]
    for x in v[1:]:
        g = g * x
    return g


# name -> (function, number of inputs); the golden cases use spartan and prod9
FUNCS = {
    "spartan": (spartan, 4),
    "prod9": (prod9, 9),
    "linear": (lambda v: v[0] + 3 * v[1] - 5, 2),
    "square": (lambda v: v[0] * v[0], 1),
    "consts": (lambda v: (v[0] - 7) * (v[1] + (L - 1)) * 11 + v[2], 3),
    "wide16": (lambda v: sum((i + 1) * v[i] for i in range(16)) * v[15] + v[0] * v[1] * v[2], 16),
    "deg16": (lambda v: prod9([v[i % 2] for i in range(16)]), 2),
}

# name -> (function, num_vars, seed)
GOLDEN = {
    "spartan_nv20": ("spartan", 20, 3020), "spartan_nv22": ("spartan", 22, 3022), "spartan_nv24": ("spartan", 24, 3024),
    "prod9_nv20": ("prod9", 20, 3920),
}
TRANSCRIPT_LABEL = b"sumcheck_golden"


def g_int(name, vals):
    """the combining function on Python integers, reduced mod l"""
    return FUNCS[name][0]([int(x) for x in vals]) % L


def eq_evals(tau):
    """EqPolynomial::new(tau).evals() from the oracle: (2^len(tau), 4) Montgomery limbs"""
    tau = np.ascontiguousarray(tau, dtype=np.uint64).reshape(-1, 4)
    out = np.zeros((1 << tau.shape[0], 4), dtype=np.uint64)
    ol.lib().orc_eq_evals(ol.P(tau), ol.sz(tau.shape[0]), ol.P(out))
    return out


def golden_inputs(name):
    """-> (function name, num_vars, tau (nv, 4), the k polynomials with polys[0] = eq(tau))"""
    fname, nv, seed = GOLDEN[name]
    rng = np.random.default_rng(seed)
    k = FUNCS[fname][1]
    tau = dc.random_full(rng, nv)
    return fname, nv, tau, [eq_evals(tau)] + [dc.random_full(rng, 1 << nv) for _ in range(k - 1)]
