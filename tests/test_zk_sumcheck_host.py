"""Zero-knowledge sumchecks without a GPU: the oracle's DotProductProof and ZKSumcheckInstanceProof provers against its
verifiers (restated from subprotocols/dot_product.rs and subprotocols/sumcheck.rs:331-447).  Every field of a proof is
load-bearing: changing any one, the claim's commitment or the generators makes the verifier reject."""
import numpy as np
import pytest

import oracle_dense_lib as od
import oracle_lib as ol
import oracle_zk_lib as oz
import sumcheck_cases as sc

L = ol.L_FR
SEED = ol.fr_array([4242])[0]


def _stream(n):
    return ol.generators(n + 2, b"zk_gens")


def _prog(fn, k):
    import lasso_b200 as lb

    return lb.trace_combine_lookups(fn, k)


def _zk(fn, k, polys, rounds, degree, blind_claim, label=b"zk"):
    """oracle ZK proof -> (proof dict, gens_1, gens_n)"""
    prog, consts, _ = _prog(fn, k)
    gens_1, gens_n = oz.dot_gens(_stream(degree + 1), degree + 1)
    got = oz.zk_prove(polys, rounds, prog, consts, degree, blind_claim, gens_1, gens_n, od.Transcript(label),
                      od.RandomTape(b"tape", SEED))
    return got, gens_1, gens_n


def _verify(got, rounds, degree, gens_1, gens_n, proof=None, comm_claim=None, label=b"zk"):
    return oz.zk_verify(got["proof"] if proof is None else proof, got["comm_claim"] if comm_claim is None else comm_claim,
                        rounds, degree, gens_1, gens_n, od.Transcript(label))


CASES = [  # (function, num_vars, num_rounds)
    ("spartan", 1, 1), ("spartan", 5, 5), ("spartan", 6, 3), ("prod9", 4, 4), ("linear", 3, 3), ("square", 2, 1),
    ("consts", 5, 5), ("wide16", 3, 3), ("deg16", 3, 3), ("deg16", 5, 1), ("spartan", 12, 12), ("spartan", 12, 4),
]


@pytest.mark.parametrize("name,nv,rounds", CASES)
def test_round_trip(name, nv, rounds):
    """prove -> verify accepts, with the verifier's r; the last comm_eval commits to g(final_evals) with blind_eval when
    every variable is bound"""
    fn, k = sc.FUNCS[name]
    deg = _prog(fn, k)[2]
    rng = np.random.default_rng(nv * 31 + rounds)
    polys = [ol.rand_fr(rng, 1 << nv) for _ in range(k)]
    bc = ol.rand_fr(rng, 1)[0]
    got, g1, gn = _zk(fn, k, polys, rounds, deg, bc)
    assert len(got["proof"]) == 24 + rounds * (200 + 32 * (deg + 1))
    rc, e, r = _verify(got, rounds, deg, g1, gn)
    assert rc == 0 and np.array_equal(r, got["r"])
    Z = [ol.fr_ints(p) for p in polys]
    claim = sum(sc.g_int(name, [z[i] for z in Z]) for i in range(1 << nv)) % L
    assert ol.fr_ints(got["claim"]) == [claim]
    assert got["comm_claim"] == oz.commit(g1, got["claim"], bc)
    if rounds == nv:
        v = sc.g_int(name, ol.fr_ints(got["final_evals"]))
        assert e == oz.commit(g1, ol.fr_array([v]), got["blind_eval"])


@pytest.mark.parametrize("d", list(range(1, 17)))
def test_degrees(d):
    """x_0 x_1 x_0 .. (d factors) over 2 inputs, declared at its degree"""
    fn = (lambda v: sc.prod9([v[i % 2] for i in range(d)])) if d > 1 else (lambda v: v[0] + v[1])
    rng = np.random.default_rng(d)
    polys = [ol.rand_fr(rng, 1 << 3) for _ in range(2)]
    got, g1, gn = _zk(fn, 2, polys, 3, d, ol.rand_fr(rng, 1)[0])
    assert _verify(got, 3, d, g1, gn)[0] == 0


@pytest.mark.parametrize("k", [1, 2, 7, 16])
def test_inputs(k):
    fn = lambda v: sum((i + 1) * v[i] for i in range(k)) * v[k - 1] + v[0]  # noqa: E731
    rng = np.random.default_rng(50 + k)
    polys = [ol.rand_fr(rng, 1 << 4) for _ in range(k)]
    got, g1, gn = _zk(fn, k, polys, 4, 2, ol.rand_fr(rng, 1)[0])
    assert _verify(got, 4, 2, g1, gn)[0] == 0


def _fields(rounds, n):
    """byte offsets of every point and scalar of a ZKSumcheckInstanceProof of `rounds` rounds, n = degree + 1"""
    pts, frs = [], []
    at = 8
    for _ in range(2):
        pts += [at + 32 * j for j in range(rounds)]
        at += 32 * rounds + 8
    for _ in range(rounds):
        pts += [at, at + 32]
        at += 64 + 8
        frs += [at + 32 * i for i in range(n + 2)]
        at += 32 * (n + 2)
    return pts, frs


def test_every_field_is_checked():
    rng = np.random.default_rng(9)
    nv = 3
    polys = [ol.rand_fr(rng, 1 << nv) for _ in range(4)]
    got, g1, gn = _zk(sc.spartan, 4, polys, nv, 3, ol.rand_fr(rng, 1)[0])
    proof = got["proof"]
    other_pt = oz.commit(g1, ol.fr_array([7]), ol.fr_array([0])[0])
    other_fr = (12345).to_bytes(32, "little")
    pts, frs = _fields(nv, 4)
    assert len(pts) == 4 * nv and len(frs) == 6 * nv
    for off in pts:
        assert _verify(got, nv, 3, g1, gn, proof=proof[:off] + other_pt + proof[off + 32:])[0] == 1, off
    for off in frs:
        assert _verify(got, nv, 3, g1, gn, proof=proof[:off] + other_fr + proof[off + 32:])[0] == 1, off
    assert _verify(got, nv, 3, g1, gn, comm_claim=other_pt)[0] == 1
    wrong_g1 = (ol.generators(1, b"other")[0:1], g1[1])
    assert _verify(got, nv, 3, wrong_g1, gn)[0] == 1
    assert _verify(got, nv, 3, g1, gn)[0] == 0


def test_dot_product_proof():
    """accepted; a wrong y is rejected; every field is checked"""
    rng = np.random.default_rng(10)
    for n in (1, 2, 17):
        g1, gn = oz.dot_gens(_stream(n), n)
        x, a = ol.rand_fr(rng, n), ol.rand_fr(rng, n)
        bx, by = ol.rand_fr(rng, 2)
        y = ol.fr_array([sum(p * q for p, q in zip(ol.fr_ints(x), ol.fr_ints(a))) % L])[0]
        for yy, want in ((y, 0), (ol.fr_array([(ol.fr_ints(y)[0] + 1) % L])[0], 1)):
            proof, Cx, Cy = oz.dot_prove(g1, gn, od.Transcript(b"d"), od.RandomTape(b"t", SEED), x, bx, a, yy, by)
            assert len(proof) == 136 + 32 * n
            assert Cx == oz.commit(gn, x, bx) and Cy == oz.commit(g1, yy, by)
            assert oz.dot_verify(g1, gn, proof, a, Cx, Cy, od.Transcript(b"d")) == want
        proof, Cx, Cy = oz.dot_prove(g1, gn, od.Transcript(b"d"), od.RandomTape(b"t", SEED), x, bx, a, y, by)
        other_fr, other_pt = (12345).to_bytes(32, "little"), oz.commit(g1, ol.fr_array([7]), ol.fr_array([0])[0])
        for off, other in [(0, other_pt), (32, other_pt)] + [(72 + 32 * i, other_fr) for i in range(n + 2)]:
            bad = proof[:off] + other + proof[off + 32:]
            assert oz.dot_verify(g1, gn, bad, a, Cx, Cy, od.Transcript(b"d")) == 1, (n, off)
