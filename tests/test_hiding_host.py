"""Hiding commitments and openings of dense polynomials in the CPU oracle (oracle_dense/): the forms with blinds on h
that lasso_poly_commit_hiding / lasso_poly_eval_prove_hiding are compared against on the GPU.  Zero blinds give the
unblinded bytes, a blinded proof verifies against its own C_Zr and against nothing else, and the commitment draws
exactly random_vector("poly_blinds", L) from the tape."""
import numpy as np
import pytest

import dense_poly_cases as dc
import oracle_dense_lib as od
import oracle_hiding_lib as oh
import oracle_lib as ol

NVS = [1, 2, 5, 8]


def _case(nv, seed):
    rng = np.random.default_rng(seed)
    Z = dc.random_full(rng, 1 << nv)
    r = dc.random_full(rng, nv)
    tape_seed = dc.random_full(rng, 1)[0]
    stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
    return Z, r, tape_seed, stream, rng


@pytest.mark.parametrize("nv", NVS)
def test_zero_blinds_are_the_unblinded_bytes(nv):
    Z, r, tape_seed, stream, _ = _case(nv, nv)
    L = 1 << (nv // 2)
    comm, _ = oh.commit_hiding(Z, stream, blinds=np.zeros((L, 4), dtype=np.uint64))
    assert comm == od.commit(Z, stream)
    Zr = od.evaluate(Z, r)
    zero = np.zeros(4, dtype=np.uint64)
    t1, t2 = od.Transcript(b"zero"), od.Transcript(b"zero")
    want = od.prove(Z, r, Zr, stream, t1, od.RandomTape(b"proof", tape_seed))
    got = oh.prove_hiding(Z, r, Zr, stream, t2, od.RandomTape(b"proof", tape_seed),
                          blinds=np.zeros((L, 4), dtype=np.uint64), blind_Zr=zero)
    assert got == want
    assert np.array_equal(t1.challenge_scalar(b"after"), t2.challenge_scalar(b"after"))


@pytest.mark.parametrize("nv", NVS)
def test_blinded_proof_verifies_only_against_its_commitments(nv):
    Z, r, tape_seed, stream, rng = _case(nv, 100 + nv)
    comm, blinds = oh.commit_hiding(Z, stream, tape=od.RandomTape(b"commit", tape_seed))
    assert comm != od.commit(Z, stream)
    Zr = od.evaluate(Z, r)
    blind_Zr = dc.random_full(rng, 1)[0]

    def prove(bl, bz):
        t = od.Transcript(b"hiding")
        t.append_poly_commitment(b"poly", comm)
        return oh.prove_hiding(Z, r, Zr, stream, t, od.RandomTape(b"proof", tape_seed), blinds=bl, blind_Zr=bz)

    def verify(proof, czr=None, zr=None):
        t = od.Transcript(b"hiding")
        t.append_poly_commitment(b"poly", comm)
        if czr is not None:
            return oh.verify(stream, nv, comm, proof, r, czr, t)
        return od.verify(stream, nv, comm, proof, r, zr, t)

    proof, czr = prove(blinds, blind_Zr)
    assert verify(proof, czr=czr) == 0
    assert verify(proof, zr=Zr) == 1  # verify_plain assumes blind_Zr = 0: the blind is in effect
    other_czr = prove(blinds, dc.random_full(rng, 1)[0])[1]
    assert other_czr != czr and verify(proof, czr=other_czr) == 1
    # one row blind differs from the commitment's
    wrong = blinds.copy()
    wrong[-1] = ol.fr_array([ol.fr_ints([wrong[-1]])[0] + 1])[0]
    bad, bad_czr = prove(wrong, blind_Zr)
    assert bad_czr == czr and verify(bad, czr=bad_czr) == 1
    # without blinds the hiding commitment does not open either
    plain, plain_czr = prove(None, blind_Zr)
    assert verify(plain, czr=plain_czr) == 1


@pytest.mark.parametrize("nv", [0, 3, 9])
def test_commit_draws_poly_blinds(nv):
    Z, _, tape_seed, stream, _ = _case(nv, 200 + nv)
    L = 1 << (nv // 2)
    tape = od.RandomTape(b"commit", tape_seed)
    _, blinds = oh.commit_hiding(Z, stream, tape=tape)
    ref = od.RandomTape(b"commit", tape_seed)
    assert np.array_equal(blinds, ref.random_vector(b"poly_blinds", L))
    assert np.array_equal(tape.random_scalar(b"next"), ref.random_scalar(b"next"))
    # the blinds given back commit to the same bytes
    again, _ = oh.commit_hiding(Z, stream, tape=od.RandomTape(b"commit", tape_seed))
    assert again == oh.commit_hiding(Z, stream, blinds=blinds)[0]
