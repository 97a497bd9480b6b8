"""CPU checks of the oracle's merge and CombinedTableEvalProof entry points (oracle_dense/) that
tests/test_gpu_combined_eval.py compares the GPU with: merge as concatenation plus zero padding, the prove -> verify round
trip for 1..32 claims, rejection of a changed eval, proof byte or point, the proof length formula of the C ABI, and the
small cases of tests/golden/combined_eval.json."""
import hashlib
import json
import os

import numpy as np
import pytest

import combined_eval_cases as cc
import dense_poly_cases as dc
import oracle_combined_eval_lib as oce
import oracle_dense_lib as od
import oracle_lib as ol

HERE = os.path.dirname(os.path.abspath(__file__))
L = ol.L_FR
SEED = ol.fr_array([7])[0]


def _setup(k, nv, seed):
    """k random components of nv variables, r, their evaluations at r, the merged polynomial, its generators and
    commitment"""
    rng = np.random.default_rng(seed)
    comps = [dc.random_full(rng, 1 << nv) for _ in range(k)]
    r = dc.random_full(rng, nv)
    evals = np.stack([od.evaluate(c, r) for c in comps])
    Z = oce.merge(comps)
    mv = Z.shape[0].bit_length() - 1
    stream = np.ascontiguousarray(ol.generators(dc.n_generators(mv)))
    return comps, r, evals, Z, mv, stream, od.commit(Z, stream)


@pytest.mark.parametrize("sizes", [[4], [4, 4, 4], [1, 2, 4, 8], [8, 1], [2, 2, 2, 2, 2], [16, 16]])
def test_merge_is_concatenation_and_padding(sizes):
    rng = np.random.default_rng(sum(sizes))
    comps = [dc.random_full(rng, n) for n in sizes]
    got = oce.merge(comps)
    flat = np.concatenate(comps)
    assert got.shape[0] == oce.next_pow2(flat.shape[0])
    assert np.array_equal(got[: flat.shape[0]], flat) and not got[flat.shape[0]:].any()


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 8, 17, 32])
@pytest.mark.parametrize("nv", [1, 3])
def test_round_trip(k, nv):
    _, r, evals, Z, mv, stream, comm = _setup(k, nv, 10 * k + nv)
    assert mv == nv + (oce.next_pow2(k).bit_length() - 1)
    proof = oce.prove(Z, evals, r, stream, od.Transcript(b"ce"), od.RandomTape(b"proof", SEED))
    assert oce.verify(stream, mv, comm, proof, evals, r, od.Transcript(b"ce")) == 0


def test_round_trip_no_point():
    """components of one evaluation each: r is empty and the opening point is the challenges alone"""
    _, r, evals, Z, mv, stream, comm = _setup(5, 0, 3)
    assert r.shape[0] == 0 and mv == 3
    proof = oce.prove(Z, evals, r, stream, od.Transcript(b"ce"), od.RandomTape(b"proof", SEED))
    assert oce.verify(stream, mv, comm, proof, evals, r, od.Transcript(b"ce")) == 0


def test_tampering_rejects():
    _, r, evals, Z, mv, stream, comm = _setup(5, 4, 99)
    proof = oce.prove(Z, evals, r, stream, od.Transcript(b"ce"), od.RandomTape(b"proof", SEED))
    assert oce.verify(stream, mv, comm, proof, evals, r, od.Transcript(b"ce")) == 0
    for i in (0, 4):  # one claim changed
        bad = evals.copy()
        bad[i] = ol.fr_array([(ol.fr_ints(evals[i])[0] + 1) % L])[0]
        assert oce.verify(stream, mv, comm, proof, bad, r, od.Transcript(b"ce")) == 1, i
    for at in (8, 40, len(proof) // 2, len(proof) - 40, len(proof) - 1):  # any changed byte: rejected or unparseable
        bad = bytearray(proof)
        bad[at] ^= 0x01
        assert oce.verify(stream, mv, comm, bytes(bad), evals, r, od.Transcript(b"ce")) != 0, at
    bad_r = r.copy()
    bad_r[2] = ol.fr_array([(ol.fr_ints(r[2])[0] + 1) % L])[0]
    assert oce.verify(stream, mv, comm, proof, evals, bad_r, od.Transcript(b"ce")) == 1
    # a proof made from a wrong claim is rejected against the true claims, and against its own
    wrong = evals.copy()
    wrong[1] = ol.fr_array([(ol.fr_ints(evals[1])[0] + 5) % L])[0]
    proof_w = oce.prove(Z, wrong, r, stream, od.Transcript(b"ce"), od.RandomTape(b"proof", SEED))
    assert oce.verify(stream, mv, comm, proof_w, evals, r, od.Transcript(b"ce")) == 1
    assert oce.verify(stream, mv, comm, proof_w, wrong, r, od.Transcript(b"ce")) == 1


@pytest.mark.parametrize("k,nv", [(1, 1), (2, 2), (3, 5), (17, 2), (4, 7)])
def test_proof_length_formula(k, nv):
    """2 (8 + 32 lg) + 128 bytes with lg = mv - mv // 2, the size include/lasso_b200.h states"""
    import lasso_b200 as lb

    _, r, evals, Z, mv, stream, _ = _setup(k, nv, k + 100 * nv)
    proof = oce.prove(Z, evals, r, stream, od.Transcript(b"ce"), od.RandomTape(b"proof", SEED))
    lg = mv - mv // 2
    assert len(proof) == oce.proof_len(mv) == lb.CombinedTableEvalProof.proof_len(mv) == 2 * (8 + 32 * lg) + 128


GOLDEN = json.load(open(os.path.join(HERE, "golden", "combined_eval.json")))


@pytest.mark.parametrize("name", cc.SMALL)
def test_golden_small_cases(name):
    nv, comps, r, seed = cc.golden_inputs(name)
    g = GOLDEN["cases"][name]
    Z = oce.merge(comps)
    mv = Z.shape[0].bit_length() - 1
    stream = np.ascontiguousarray(ol.generators(dc.n_generators(mv)))
    evals = np.stack([od.evaluate(c, r) for c in comps])
    t = od.Transcript(cc.TRANSCRIPT_LABEL)
    proof = oce.prove(Z, evals, r, stream, t, od.RandomTape(cc.TAPE_LABEL, seed))
    assert len(proof) == g["proof_len"] and mv == g["merged_num_vars"]
    assert hashlib.sha256(cc.digest_input(evals, proof)).hexdigest() == g["sha256"]
    assert t.challenge_scalar(b"after").tobytes().hex() == g["after_challenge_hex"]
    comm = od.commit(Z, stream)
    assert hashlib.sha256(comm).hexdigest() == g["commitment_sha256"]
    assert oce.verify(stream, mv, comm, proof, evals, r, od.Transcript(cc.TRANSCRIPT_LABEL)) == 0


def test_golden_covers_the_cases():
    assert set(GOLDEN["cases"]) == set(cc.GOLDEN)
    assert all(c["oracle_verifier"] == "accepted" for c in GOLDEN["cases"].values())
