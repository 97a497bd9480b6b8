"""CPU checks of the oracle's grand-product entry points (oracle_dense/) that tests/test_gpu_grand_product.py compares the
GPU with: the prove -> verify round trip for 1..32 circuits and num_vars 1..12, rejection of a tampered proof, product
or claim, the proof length formula of the C ABI, final claims equal to the polynomials at rand, the pointwise map, and
the small cases of tests/golden/grand_product.json."""
import hashlib
import json
import os

import numpy as np
import pytest

import dense_poly_cases as dc
import grand_product_cases as gc
import oracle_dense_lib as od
import oracle_grand_product_lib as ogp
import oracle_lib as ol

HERE = os.path.dirname(os.path.abspath(__file__))
L = ol.L_FR


def _round_trip(polys, label=b"gp"):
    nv = polys[0].shape[0].bit_length() - 1
    got = ogp.gp_prove(polys, od.Transcript(label))
    rc, claims, r = ogp.gp_verify(got["proof"], got["products"], nv, od.Transcript(label))
    assert rc == 0
    assert np.array_equal(r, got["r"]) and np.array_equal(claims, got["claims"])
    return nv, got


@pytest.mark.parametrize("n", list(range(1, 33)))
def test_round_trip_batch_sizes(n):
    rng = np.random.default_rng(n)
    _round_trip([dc.random_full(rng, 1 << 4) for _ in range(n)])


@pytest.mark.parametrize("nv", list(range(1, 13)))
def test_round_trip_num_vars(nv):
    rng = np.random.default_rng(50 + nv)
    polys = [dc.random_full(rng, 1 << nv) for _ in range(3)]
    _, got = _round_trip(polys)
    for p, prod in zip(polys, ol.fr_ints(got["products"])):  # evaluate(): the product of all evaluations
        want = 1
        for x in ol.fr_ints(p):
            want = want * x % L
        assert prod == want


def test_round_trip_32_circuits_at_12_vars():
    rng = np.random.default_rng(9)
    _round_trip([dc.random_full(rng, 1 << 12) for _ in range(32)])


def test_tampering_rejects():
    rng = np.random.default_rng(10)
    nv, n = 6, 3
    polys = [dc.random_full(rng, 1 << nv) for _ in range(n)]
    _, got = _round_trip(polys)
    proof, products = got["proof"], got["products"]
    for at in (8, 100, len(proof) // 2, len(proof) - 40):  # any changed byte: rejected or unparseable
        bad = bytearray(proof)
        bad[at] ^= 0x01
        assert ogp.gp_verify(bytes(bad), products, nv, od.Transcript(b"gp"))[0] != 0, at
    bad = products.copy()
    bad[1] = ol.fr_array([ol.fr_ints(products[1])[0] + 1])[0]
    assert ogp.gp_verify(proof, bad, nv, od.Transcript(b"gp"))[0] == 1
    # the last claim_prod_right plus one, re-encoded canonically: the layer's sumcheck no longer closes
    bad = bytearray(proof)
    x = int.from_bytes(bad[-32:], "little")
    bad[-32:] = ((x + 1) % L).to_bytes(32, "little")
    assert ogp.gp_verify(bytes(bad), products, nv, od.Transcript(b"gp"))[0] == 1
    # a claim the caller goes on to open: it no longer equals the polynomial at rand
    assert ol.fr_ints(od.evaluate(polys[0], got["r"]))[0] != (ol.fr_ints(got["claims"][0])[0] + 1) % L


@pytest.mark.parametrize("n,nv", [(1, 1), (2, 2), (5, 7), (32, 3)])
def test_proof_length_formula(n, nv):
    """8 + v (24 + 64 n) + 52 v (v - 1) bytes, the size include/lasso_b200.h states"""
    import lasso_b200 as lb

    rng = np.random.default_rng(n * 100 + nv)
    _, got = _round_trip([dc.random_full(rng, 1 << nv) for _ in range(n)])
    want = 8 + nv * (24 + 64 * n) + 52 * nv * (nv - 1)
    assert len(got["proof"]) == ogp.proof_len(n, nv) == lb.BatchedGrandProductArgument.proof_len(n, nv) == want


@pytest.mark.parametrize("nv", [1, 2, 8])
def test_claims_are_evaluations(nv):
    rng = np.random.default_rng(20 + nv)
    polys = [dc.random_full(rng, 1 << nv) for _ in range(4)]
    _, got = _round_trip(polys)
    for p, claim in zip(polys, got["claims"]):
        assert np.array_equal(od.evaluate(p, got["r"]), claim)


def test_comb_map():
    import lasso_b200 as lb

    rng = np.random.default_rng(30)
    polys = [dc.random_full(rng, 64) for _ in range(3)]
    prog, consts, _ = lb.trace_combine_lookups(lambda v: v[2] * 9 + v[1] * v[0] - 4, 3)
    out = ogp.comb_map(polys, prog, consts)
    a, b, c = (ol.fr_ints(p) for p in polys)
    assert ol.fr_ints(out) == [(z * 9 + y * x - 4) % L for x, y, z in zip(a, b, c)]


GOLDEN = json.load(open(os.path.join(HERE, "golden", "grand_product.json")))


@pytest.mark.parametrize("name", gc.SMALL)
def test_golden_small_cases(name):
    nv, polys = gc.golden_inputs(name)
    g = GOLDEN["cases"][name]
    t = od.Transcript(gc.TRANSCRIPT_LABEL)
    got = ogp.gp_prove(polys, t)
    assert len(got["proof"]) == g["proof_len"]
    assert hashlib.sha256(gc.digest_input(got)).hexdigest() == g["sha256"]
    assert t.challenge_scalar(b"after").tobytes().hex() == g["after_challenge_hex"]
    rc, _, _ = ogp.gp_verify(got["proof"], got["products"], nv, od.Transcript(gc.TRANSCRIPT_LABEL))
    assert rc == 0 and g["oracle_verifier"] == "accepted"


def test_golden_covers_the_sizes():
    assert {(c["n_circuits"], c["num_vars"]) for c in GOLDEN["cases"].values()} >= {(2, 20), (2, 22)}
    assert set(GOLDEN["cases"]) == set(gc.GOLDEN)
