"""Caller-defined strategies on the CPU: the Python tracer of combine_lookups, and the oracle for caller-defined strategies
(explicit tables, maps, program and declared degree) against its built-in strategies."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

import custom_builtins as cb
import oracle_custom_lib as oc
import oracle_lib as ol

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "proofs.json")))
NGENS = 600

# the e2e_test.rs shapes (name, kind, C, log_m, log_r, lookups, same_index)
E2E = [
    ("prove_4d_lt", cb.LT, 4, 4, 0, 16, True),
    ("prove_4d_and", cb.AND, 4, 4, 0, 16, True),
    ("prove_3d_range", cb.RANGE_CHECK, 3, 8, 40, 16, False),
    ("xor_c3", cb.XOR, 3, 8, 0, 64, False),
    ("or_c2", cb.OR, 2, 8, 0, 32, False),
]


def _lb():
    import lasso_b200 as lb  # the tracer is pure Python: importing needs no GPU

    return lb


def make_inputs(C, log_m, n, seed, same):
    rng = np.random.default_rng(seed)
    col = rng.integers(0, 1 << log_m, size=(n, 1), dtype=np.uint64)
    idx = np.repeat(col, C, axis=1) if same else rng.integers(0, 1 << log_m, size=(n, C), dtype=np.uint64)
    s = 1 << max(0, (n - 1).bit_length())
    r = ol.rand_fr(rng, max(1, s.bit_length() - 1))
    return np.ascontiguousarray(idx), r, ol.rand_fr(rng, 1)[0], s


# ---------------------------------------------------------------- tracer
def test_tracer_xor_program():
    lb = _lb()
    S = cb.as_custom(None, cb.XOR, 4, 16)
    # Horner from the last memory: ((v3 * 2^8 + v2) * 2^8 + v1) * 2^8 + v0
    assert S.program.tolist() == [[3, 3, 0], [0, 4, 2], [3, 5, 0], [0, 6, 1], [3, 7, 0], [0, 8, 0]]
    assert ol.fr_ints(S.constants) == [256]
    assert S.degree == 1 and S.num_memories == 4 and S.num_subtables == 1 and S.sumcheck_poly_degree == 2
    assert S.memory_to_subtable.tolist() == [0] * 4 and S.memory_to_dimension.tolist() == [0, 1, 2, 3]
    assert lb.trace_combine_lookups(lambda v: v[0], 1)[0].tolist() == [[4, 0, 0]]  # g = v0: ADDK 0


def test_tracer_lt_program():
    S = cb.as_custom(None, cb.LT, 3, 8)
    # h = LT_2; h = LT_1 + EQ_1 h; h = LT_0 + EQ_0 h: 2 instructions per dimension
    assert S.program.tolist() == [[2, 3, 4], [0, 2, 6], [2, 1, 7], [0, 0, 8]]
    assert S.constants.shape == (0, 4)
    assert S.degree == 3 and S.num_memories == 6 and S.memory_to_subtable.tolist() == [0, 1] * 3
    assert S.memory_to_dimension.tolist() == [0, 0, 1, 1, 2, 2]


@pytest.mark.parametrize("kind,C,log_m,log_r,deg", [(cb.AND, 2, 8, 0, 1), (cb.OR, 1, 16, 0, 1), (cb.LT, 8, 16, 0, 8),
                                                     (cb.RANGE_CHECK, 4, 16, 40, 1)])
def test_tracer_builtin_degree(kind, C, log_m, log_r, deg):
    S = cb.as_custom(None, kind, C, log_m, log_r)
    assert S.degree == deg and S.g_poly_degree == deg


def test_tracer_constants_and_degree():
    lb = _lb()
    prog, K, deg = lb.trace_combine_lookups(lambda v: 3 - v[0] * v[1] * v[1] + (-5) * v[2] - 7, 3)
    assert deg == 3
    assert sorted(ol.fr_ints(K)) == sorted([x % ol.L_FR for x in (-1, 3, -5, -7)])
    # the program evaluated by the oracle's interpreter agrees with Python big-int arithmetic
    S = lb.CustomStrategy(None, 1, 2, [np.zeros(4)] * 3, lambda v: 3 - v[0] * v[1] * v[1] + (-5) * v[2] - 7, 3)
    x = [11, 2**200 + 5, 99]
    want = (3 - x[0] * x[1] * x[1] - 5 * x[2] - 7) % ol.L_FR
    assert ol.fr_ints(oc.combine_lookups(S, ol.fr_array(x))) == [want]


def test_tracer_rejects_low_degree_and_bad_descriptors():
    lb = _lb()
    g, _ = cb.builtin_g(cb.LT, 4, 8)
    with pytest.raises(lb.LassoError) as e:
        lb.CustomStrategy(None, 4, 8, cb.builtin_tables(cb.LT, 4, 8), g, 3)
    assert e.value.code == 4
    t = np.arange(16)
    for bad in (dict(tables=[t[:8]]), dict(tables=[t + 2**32]), dict(g=lambda v: 5), dict(mts=[0, 0], mtd=[0])):
        with pytest.raises(lb.LassoError):
            lb.CustomStrategy(None, 2, 4, bad.get("tables", [t]), bad.get("g", lambda v: v[0] + v[1]), 1,
                              bad.get("mts"), bad.get("mtd"))
    with pytest.raises(lb.LassoError):  # more than 16 memories
        lb.CustomStrategy(None, 16, 4, [t, t], lambda v: v[0], 1)


# ---------------------------------------------------------------- oracle: MLE parity
@pytest.mark.parametrize("kind,C,log_m,log_r", [(cb.AND, 2, 8, 0), (cb.OR, 2, 8, 0), (cb.XOR, 2, 6, 0),
                                                (cb.LT, 2, 8, 0), (cb.RANGE_CHECK, 3, 8, 20), (cb.RANGE_CHECK, 2, 5, 7)])
def test_dense_mle_matches_closed_form(kind, C, log_m, log_r):
    """the custom oracle's evaluate_subtable_mle (dense MLE, point[0] the MSB) equals the closed forms of and.rs, lt.rs,
    range_check.rs ... at random points, and at Boolean points equals the table"""
    S = _lb().CustomStrategy(None, C, log_m, cb.builtin_tables(kind, C, log_m, log_r), lambda v: v[0], 1)
    rng = np.random.default_rng(kind * 100 + log_m)
    for k in range(S.num_subtables):
        for trial in range(3):
            point = ol.rand_fr(rng, log_m)
            out = np.zeros(4, dtype=np.uint64)
            ol.lib().orc_evaluate_subtable_mle(kind, ol.sz(C), ol.sz(log_m), ol.sz(log_r), ol.sz(k), ol.P(point),
                                               ol.sz(log_m), ol.P(out))
            assert (oc.evaluate_subtable_mle(S, k, point) == out).all(), (k, trial)
        i = int(rng.integers(0, 1 << log_m))
        boolean = ol.fr_array([(i >> (log_m - 1 - b)) & 1 for b in range(log_m)])
        assert ol.fr_ints(oc.evaluate_subtable_mle(S, k, boolean)) == [int(S.tables[k][i])]


# ---------------------------------------------------------------- oracle: byte identity with the built-ins
@pytest.mark.parametrize("name,kind,C,log_m,log_r,n,same", E2E, ids=[c[0] for c in E2E])
def test_oracle_custom_builtin_identical_bytes(name, kind, C, log_m, log_r, n, same):
    idx, r, seed, s = make_inputs(C, log_m, n, len(name), same)
    S = cb.as_custom(None, kind, C, log_m, log_r)
    gens = ol.generators(NGENS)
    ref = ol.prove(kind, C, log_m, log_r, idx, r, gens, seed, flags=1)
    got = oc.prove(S, idx, r, gens, seed, flags=1)
    assert ref["rc"] == 0 and got["rc"] == 0
    assert got["commitment"] == ref["commitment"]
    assert got["proof"] == ref["proof"]
    assert (got["challenges"] == ref["challenges"]).all()


@pytest.mark.parametrize("case", GOLD["cases"], ids=[c["name"] for c in GOLD["cases"]])
def test_oracle_custom_reproduces_golden(case):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden import inputs

    idx, r, seed, s = inputs(case["C"], case["log_m"], case["lookups"], case["seed"], case["same_index"])
    S = cb.as_custom(None, case["kind"], case["C"], case["log_m"], case["log_r"])
    res = oc.prove(S, idx, r, ol.generators(NGENS), seed, flags=1)
    assert res["rc"] == 0
    assert hashlib.sha256(res["commitment"]).hexdigest() == case["commitment_sha256"]
    assert hashlib.sha256(res["proof"]).hexdigest() == case["proof_sha256"]
    assert len(res["challenges"]) == case["n_challenges"]


# ---------------------------------------------------------------- oracle: new tables
@pytest.mark.parametrize("name", sorted(cb.NEW_TABLES))
def test_oracle_verifies_new_tables(name):
    """the verifier accepts proofs over tables that are not built in, and rejects them with a tampered claimed
    evaluation (flags bit 1) or a tampered memory-checking evaluation (flags bit 2)"""
    S = cb.NEW_TABLES[name](None)
    idx, r, seed, s = make_inputs(S.C, S.log_m, 40, len(name), False)
    gens = ol.generators(NGENS)
    assert oc.prove(S, idx, r, gens, seed, flags=1)["rc"] == 0
    assert oc.prove(S, idx, r, gens, seed, flags=1 | 2)["rc"] == 1
    assert oc.prove(S, idx, r, gens, seed, flags=1 | 4)["rc"] == 1


def test_oracle_custom_round_matches_builtin_round():
    rng = np.random.default_rng(5)
    for kind, C, log_m, log_r in [(cb.XOR, 3, 8, 0), (cb.LT, 3, 4, 0), (cb.RANGE_CHECK, 3, 8, 20)]:
        S = cb.as_custom(None, kind, C, log_m, log_r)
        polys = np.stack([ol.rand_fr(rng, 8) for _ in range(S.num_memories + 1)])
        ref = np.zeros((S.sumcheck_poly_degree + 1, 4), dtype=np.uint64)
        ol.lib().orc_sumcheck_round_arbitrary(kind, ol.sz(C), ol.sz(log_m), ol.sz(log_r), ol.P(polys), ol.sz(8),
                                              ol.P(ref))
        assert (oc.sumcheck_round(S, polys) == ref).all()
