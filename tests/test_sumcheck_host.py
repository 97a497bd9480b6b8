"""Sumchecks over a caller's polynomials without a GPU: the oracle's SumcheckInstanceProof::prove_arbitrary against its
verifier and against a sumcheck restated here in Python integers, and lasso_comb_create's program rules at each
boundary, each rejected case next to an accepted one a step away."""
import numpy as np
import pytest

import oracle_dense_lib as od
import oracle_lib as ol
import oracle_sumcheck_lib as osc
import sumcheck_cases as sc

L = ol.L_FR
ERR_STRATEGY = 4


def _rand_polys(rng, k, nv):
    return [ol.rand_fr(rng, 1 << nv) for _ in range(k)]


def _bind_top(Z, r):
    """dense_mlpoly.rs:209-216 in Python integers"""
    h = len(Z) // 2
    return [(Z[i] + r * (Z[h + i] - Z[i])) % L for i in range(h)]


def _oracle(name, polys, num_rounds, degree, label=b"host"):
    import lasso_b200 as lb

    fn, k = sc.FUNCS[name]
    prog, consts, _ = lb.trace_combine_lookups(fn, k)
    t = od.Transcript(label)
    return osc.sumcheck_prove(polys, num_rounds, prog, consts, degree, t, round_evals=True)


CASES = [  # (function, num_vars, num_rounds, declared degree or None for the traced one)
    ("spartan", 5, 5, None), ("spartan", 6, 3, None), ("prod9", 4, 4, None), ("linear", 3, 3, None),
    ("linear", 4, 2, 4), ("square", 1, 1, None), ("consts", 5, 5, 6), ("wide16", 3, 3, None), ("deg16", 3, 3, None),
    ("deg16", 5, 1, None),
]


@pytest.mark.parametrize("name,nv,rounds,degree", CASES)
def test_oracle_round_trip(name, nv, rounds, degree):
    """prove -> verify; the verifier's final claim equals the sum of g over the unbound variables, computed in Python
    integers from the polynomials bound at r, and final_evals are element 0 of those"""
    import lasso_b200 as lb

    fn, k = sc.FUNCS[name]
    deg = degree or lb.trace_combine_lookups(fn, k)[2]
    rng = np.random.default_rng(100 * nv + rounds)
    polys = _rand_polys(rng, k, nv)
    got = _oracle(name, polys, rounds, deg)
    assert len(got["proof"]) == 8 + rounds * (8 + 32 * deg)
    v = od.Transcript(b"host")
    rc, e, r = osc.sumcheck_verify(got["proof"], got["claim"], rounds, deg, v)
    assert rc == 0
    assert np.array_equal(r, got["r"])
    Z = [ol.fr_ints(p) for p in polys]
    for rj in ol.fr_ints(r):
        Z = [_bind_top(z, rj) for z in Z]
    assert ol.fr_ints(got["final_evals"]) == [z[0] for z in Z]
    want = sum(sc.g_int(name, [z[i] for z in Z]) for i in range(len(Z[0]))) % L
    assert ol.fr_ints(e)[0] == want
    # the verifier decompresses each round with the running claim as its hint (unipoly.rs:98-109), so a wrong claim
    # shows in the final claim, which no longer matches g
    rc, e_bad, _ = osc.sumcheck_verify(got["proof"], ol.fr_array([ol.fr_ints(got["claim"])[0] + 1])[0], rounds, deg,
                                      od.Transcript(b"host"))
    assert rc == 0 and ol.fr_ints(e_bad)[0] != want


@pytest.mark.parametrize("name,nv", [("spartan", 4), ("prod9", 3), ("consts", 6), ("square", 2)])
def test_oracle_rounds_against_python(name, nv):
    """every round polynomial at 0..degree, restated: s_j(t) = sum_x g(P(r_0..r_{j-1}, t, x))"""
    import lasso_b200 as lb

    fn, k = sc.FUNCS[name]
    deg = lb.trace_combine_lookups(fn, k)[2]
    polys = _rand_polys(np.random.default_rng(nv), k, nv)
    got = _oracle(name, polys, nv, deg)
    Z = [ol.fr_ints(p) for p in polys]
    assert ol.fr_ints(got["claim"])[0] == sum(sc.g_int(name, [z[i] for z in Z]) for i in range(1 << nv)) % L
    for j, rj in enumerate(ol.fr_ints(got["r"])):
        h = len(Z[0]) // 2
        for t in range(deg + 1):
            s = sum(sc.g_int(name, [(z[i] + t * (z[h + i] - z[i])) for z in Z]) for i in range(h)) % L
            assert ol.fr_ints(got["round_evals"][j][t])[0] == s, (j, t)
        Z = [_bind_top(z, rj) for z in Z]


# ---- lasso_comb_create: every program rule at its boundary
def _create(n_inputs, prog, consts=None, degree=1):
    import lasso_b200 as lb

    consts = np.zeros((0, 4), dtype=np.uint64) if consts is None else consts
    try:
        lb.Comb.from_program(prog, consts, n_inputs, degree)
        return 0
    except lb.LassoError as e:
        return e.code


def _sum_program(n):
    """x_0 + x_1 + ... + x_{n-1} (n - 1 instructions; one ADDK 0 for n = 1)"""
    if n == 1:
        return [[4, 0, 0]], ol.fr_array([0])
    prog, acc = [[0, 0, 1]], n
    for i in range(2, n):
        prog.append([0, acc, i])
        acc = n + len(prog) - 1
    return prog, None


def test_comb_inputs():
    for n, ok in [(0, False), (1, True), (16, True), (17, False)]:
        prog, consts = _sum_program(max(n, 1))
        assert (_create(n, prog, consts) == 0) == ok, n


def test_comb_instruction_count():
    one = [[0, 0, 0]]
    assert _create(1, np.zeros((0, 3), dtype=np.int32)) == ERR_STRATEGY
    assert _create(1, one) == 0
    assert _create(1, one * 128) == 0
    assert _create(1, one * 129) == ERR_STRATEGY


def test_comb_constants():
    assert _create(1, [[4, 0, 63]], ol.fr_array(list(range(64)))) == 0
    assert _create(1, [[4, 0, 64]], ol.fr_array(list(range(65)))) == ERR_STRATEGY
    assert _create(1, [[4, 0, 0]], ol.fr_array([L - 1])) == 0
    not_canonical = ol.int_to_limbs(L).reshape(1, 4)  # the limbs of l itself: not a residue below l
    assert _create(1, [[4, 0, 0]], not_canonical) == ERR_STRATEGY
    assert _create(1, [[4, 0, 0]], ol.fr_array([1])) == 0
    assert _create(1, [[4, 0, 1]], ol.fr_array([1])) == ERR_STRATEGY  # constant index out of range


def test_comb_operands():
    # instruction 1 of a 2-input program may name slots 0..2
    assert _create(2, [[0, 0, 1], [0, 2, 2]]) == 0
    assert _create(2, [[0, 0, 1], [0, 3, 2]]) == ERR_STRATEGY
    assert _create(2, [[0, 0, 1], [0, 2, 3]]) == ERR_STRATEGY
    assert _create(2, [[0, 0, 1], [0, -1, 2]]) == ERR_STRATEGY
    assert _create(2, [[4, 0, 0]], ol.fr_array([1])) == 0
    assert _create(2, [[5, 0, 0]], ol.fr_array([1])) == ERR_STRATEGY  # unknown opcode
    assert _create(2, [[-1, 0, 0]]) == ERR_STRATEGY


def _live_program(m):
    """m values x_0 + x_0 kept live, then added up: m physical slots"""
    prog = [[0, 0, 0] for _ in range(m)]
    acc = 1
    for j in range(1, m):
        prog.append([0, acc if j > 1 else 1, 1 + j])
        acc = len(prog)
    return prog


def test_comb_live_values():
    assert _create(1, _live_program(16)) == 0
    assert _create(1, _live_program(17)) == ERR_STRATEGY


def test_comb_degree():
    sq = [[2, 0, 0]]  # x_0 * x_0: degree 2
    assert _create(1, sq, degree=1) == ERR_STRATEGY
    assert _create(1, sq, degree=2) == 0
    assert _create(1, [[0, 0, 0]], degree=0) == ERR_STRATEGY
    assert _create(1, [[0, 0, 0]], degree=1) == 0
    assert _create(1, [[0, 0, 0]], degree=16) == 0
    assert _create(1, [[0, 0, 0]], degree=17) == ERR_STRATEGY


def test_comb_traced_degree():
    import lasso_b200 as lb

    g = lb.Comb(sc.spartan, 4)
    assert g.degree == g.traced_degree == 3
    assert lb.Comb(sc.spartan, 4, degree=5).degree == 5
    with pytest.raises(lb.LassoError) as e:
        lb.Comb(sc.spartan, 4, degree=2)
    assert e.value.code == ERR_STRATEGY and "below the program's degree 3" in str(e.value)
