"""Seeded inputs of the batched cubic sumcheck tests (tests/test_cubic_batched_host.py, tests/test_gpu_cubic_batched.py,
tests/golden/cubic_batched.json, tools/cubic_batched_bench.py), and the claim and eq table they need, computed with
Python integers in numpy object arrays.  Every array is derived from a seed with numpy, so the GPU machine regenerates
exactly what the golden hashes were computed from."""
import numpy as np

import dense_poly_cases as dc
import oracle_lib as ol

L = ol.L_FR
R_INV = pow(2**256, -1, L)

# name -> (n pairs, num_vars, seed, C kind, num_rounds)
GOLDEN = {
    "n2_nv20_eq": (2, 20, 2020, "eq", 20),
    "n8_nv20_partial": (8, 20, 8020, "random", 17),
    "n2_nv22_eq": (2, 22, 2022, "eq", 22),
}
TRANSCRIPT_LABEL = b"cubic_batched_golden"


def _raw(a):
    """(k, 4) limbs -> object array of the k integers they hold (Montgomery form, x R mod l)"""
    a = np.asarray(a, dtype=np.uint64).reshape(-1, 4)
    out = a[:, 0].astype(object)
    for i in range(1, 4):
        out = out + (a[:, i].astype(object) << (64 * i))
    return out


def _limbs(x):
    """object array of integers below 2^256 -> (k, 4) limbs"""
    x = np.asarray(x, dtype=object).reshape(-1)
    out = np.zeros((x.shape[0], 4), dtype=np.uint64)
    for i in range(4):
        out[:, i] = ((x >> (64 * i)) & (2**64 - 1)).astype(np.uint64)
    return out


def eq_table(tau):
    """EqPolynomial::new(tau).evals(), tau[0] the top variable -> (2^len(tau), 4) Montgomery limbs"""
    one = 2**256 % L  # 1 in Montgomery form
    ev = np.array([one], dtype=object)
    for t in _raw(tau):
        hi = ev * t % L * R_INV % L
        nxt = np.empty(2 * ev.shape[0], dtype=object)
        nxt[0::2] = (ev - hi) % L
        nxt[1::2] = hi
        ev = nxt
    return _limbs(ev)


def true_claim(A, B, C, coeffs):
    """sum_x C(x) sum_k coeffs[k] A_k(x) B_k(x) -> (4,) Montgomery limbs"""
    acc = np.zeros(C.shape[0], dtype=object)
    for a, b, k in zip(A, B, _raw(coeffs)):
        acc = (acc + _raw(a) * _raw(b) % L * k) % L
    # every product carries R^4 (four Montgomery factors): one R back is the Montgomery form, so divide by R^3
    s = int((acc * _raw(C) % L).sum()) % L
    return _limbs(np.array([s * pow(R_INV, 3, L) % L], dtype=object))[0]


def random_case(n, nv, seed, ckind="random", kinds=("full",)):
    """-> (A, B, C, coeffs): n pairs of (2^nv, 4) arrays, C = eq(tau) or random, uniform coefficients.  kinds cycles
    over the value kinds of the pairs: "full" uniform residues, "u32" integers below 2^32."""
    rng = np.random.default_rng(seed)
    size = 1 << nv

    def vals(kind):
        if kind == "u32":
            return dc.fr_from_u64(rng.integers(0, 1 << 32, size=size, dtype=np.uint64))
        return dc.random_full(rng, size)

    A = [vals(kinds[k % len(kinds)]) for k in range(n)]
    B = [vals(kinds[(k + 1) % len(kinds)]) for k in range(n)]
    C = eq_table(ol.rand_fr(rng, nv)) if ckind == "eq" else dc.random_full(rng, size)
    coeffs = ol.rand_fr(rng, n)
    return A, B, C, coeffs


def golden_inputs(name):
    """-> (A, B, C, coeffs, num_rounds) of a golden case"""
    n, nv, seed, ckind, rounds = GOLDEN[name]
    A, B, C, coeffs = random_case(n, nv, seed, ckind)
    return A, B, C, coeffs, rounds


def digest_input(proof, r, finals):
    """the bytes the golden SHA-256 covers: proof || r || finals"""
    return bytes(proof) + np.ascontiguousarray(r).tobytes() + np.ascontiguousarray(finals).tobytes()
