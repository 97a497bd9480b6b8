"""The host side of memory checking inside a caller's protocol, without a GPU: the oracle's standalone
MemoryCheckingProof (accepted by its verifier, equal to the tail of the lookup proof when (gamma, tau) are drawn as
surge.rs:188 draws them, a tampered element rejected) that the GPU tests compare with, and
lasso_b200.Transcript.append_combined_table_commitment against the oracle's transcript."""
import numpy as np
import pytest

import lasso_b200 as lb
from lasso_b200.api import LASSO_ERR_LENGTH, LASSO_ERR_VALUE
import oracle_compose_lib as ocl
import oracle_dense_lib as od
import oracle_lib as ol
import oracle_memory_check_lib as oml
from oracle_lib import L_FR


def _inputs(kind, C_, log_m, n, seed):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    s = 1 << (n - 1).bit_length()
    alpha = int(ol.lib().orc_num_memories(kind, ol.sz(C_), ol.sz(log_m), ol.sz(0)))
    stream = ol.generators(lb.gens_points_needed(C_, s, alpha, log_m))
    return rng, idx, s, alpha, stream


def _fr_bytes(x):
    return int(x % L_FR).to_bytes(32, "little")


def _with_fr(proof, at, delta=1):
    v = int.from_bytes(proof[at:at + 32], "little")
    return proof[:at] + _fr_bytes(v + delta) + proof[at + 32:]


CASES = [(lb.XOR, 2, 4, 6), (lb.LT, 2, 4, 8), (lb.AND, 3, 4, 5), (lb.OR, 2, 6, 9)]


@pytest.mark.parametrize("kind,C_,log_m,n", CASES)
def test_standalone_proof_is_accepted(kind, C_, log_m, n):
    rng, idx, s, alpha, stream = _inputs(kind, C_, log_m, n, n)
    gamma, tau = ol.rand_fr(rng, 2)
    seed = ol.rand_fr(rng, 1)[0]
    T = od.Transcript(b"memory check")
    proof, comm, derefs = oml.prove(kind, C_, log_m, 0, idx, gamma, tau, stream, T, od.RandomTape(b"proof", seed))
    log_s = s.bit_length() - 1
    gpa = lb.BatchedGrandProductArgument.proof_len
    dpl = lb.CombinedTableEvalProof.proof_len
    nv_l = (2 * C_ * s - 1).bit_length()
    nv_m = (C_ * (1 << log_m) - 1).bit_length()
    nv_d = (alpha * s - 1).bit_length()
    assert len(proof) == (4 * 32 * alpha + gpa(2 * alpha, log_m) + gpa(2 * alpha, log_s) + 32 * (3 * C_ + alpha)
                          + dpl(nv_l) + dpl(nv_m) + dpl(nv_d))
    V = od.Transcript(b"memory check")
    assert oml.verify(kind, C_, log_m, 0, stream, comm, derefs, proof, gamma, tau, V) == 0
    assert T.challenge_scalar(b"next").tolist() == V.challenge_scalar(b"next").tolist()
    # another (gamma, tau) is another multiset hash: the claims no longer match the hash layer
    assert oml.verify(kind, C_, log_m, 0, stream, comm, derefs, proof, tau, gamma, od.Transcript(b"memory check")) == 1


@pytest.mark.parametrize("kind,C_,log_m,n", CASES[:3])
def test_standalone_proof_is_the_tail_of_the_lookup_proof(kind, C_, log_m, n):
    rng, idx, s, alpha, stream = _inputs(kind, C_, log_m, n, 100 + n)
    r = ol.rand_fr(rng, s.bit_length() - 1)
    seed = ol.rand_fr(rng, 1)[0]
    T1, T2 = od.Transcript(b"example"), od.Transcript(b"example")
    full, _, _ = ocl.sparse_prove(kind, C_, log_m, 0, idx, r, stream, T1, od.RandomTape(b"proof", seed))
    zero = np.zeros(4, dtype=np.uint64)
    mc, _, _ = oml.prove(kind, C_, log_m, 0, idx, zero, zero, stream, T2, od.RandomTape(b"proof", seed), r=r)
    assert len(mc) < len(full) and full.endswith(mc)
    assert T1.challenge_scalar(b"next").tolist() == T2.challenge_scalar(b"next").tolist()


def test_tampered_element_is_rejected():
    kind, C_, log_m, n = lb.XOR, 2, 4, 6
    rng, idx, s, alpha, stream = _inputs(kind, C_, log_m, n, 3)
    gamma, tau = ol.rand_fr(rng, 2)
    proof, comm, derefs = oml.prove(kind, C_, log_m, 0, idx, gamma, tau, stream, od.Transcript(b"t"),
                                    od.RandomTape(b"proof", ol.rand_fr(rng, 1)[0]))
    gpa = lb.BatchedGrandProductArgument.proof_len
    hash_at = 4 * 32 * alpha + gpa(2 * alpha, log_m) + gpa(2 * alpha, s.bit_length() - 1)
    # a multiset claim, and the first hash-layer evaluation (eval_dim[0])
    for at in (0, 32, hash_at, hash_at + 32 * C_):
        bad = _with_fr(proof, at)
        assert oml.verify(kind, C_, log_m, 0, stream, comm, derefs, bad, gamma, tau, od.Transcript(b"t")) == 1, at
    assert oml.verify(kind, C_, log_m, 0, stream, comm, derefs, proof[:-1], gamma, tau, od.Transcript(b"t")) == 2


def _derefs():
    kind, C_, log_m, n = lb.XOR, 2, 4, 6
    rng, idx, s, alpha, stream = _inputs(kind, C_, log_m, n, 4)
    zero = np.zeros(4, dtype=np.uint64)
    return oml.prove(kind, C_, log_m, 0, idx, zero, zero, stream, od.Transcript(b"t"), od.RandomTape(b"p", zero))[2]


def test_append_combined_table_commitment_matches_oracle():
    """subtables/mod.rs:382-393: the begin / end subtable_evals_commitment messages around the PolyCommitment's"""
    derefs = _derefs()
    t, o = lb.Transcript(b"compose"), od.Transcript(b"compose")
    t.append_combined_table_commitment(derefs)
    o.append_message(b"subtable_evals_commitment", b"begin_subtable_evals_commitment")
    o.append_poly_commitment(b"comm_poly_row_col_ops_val", derefs)
    o.append_message(b"subtable_evals_commitment", b"end_subtable_evals_commitment")
    assert t.challenge_scalar(b"next").tolist() == o.challenge_scalar(b"next").tolist()
    other = lb.Transcript(b"compose")
    other.append_poly_commitment(b"comm_poly_row_col_ops_val", derefs)
    assert other.challenge_scalar(b"next").tolist() != o.challenge_scalar(b"next").tolist()


def _bad_point():
    probe = od.Transcript(b"probe")
    for y in range(2, 200):
        b = y.to_bytes(32, "little")
        if od.lib().orcd_transcript_append_point(probe.h, b"p", b) != 0:
            return b
    raise AssertionError("no undecompressable point below 200")


def test_append_combined_table_commitment_rejects():
    derefs = _derefs()
    bad = derefs[:8] + _bad_point() + derefs[40:]
    for data, code in ((derefs[:-1], LASSO_ERR_LENGTH), (derefs + b"\0", LASSO_ERR_LENGTH), (b"", LASSO_ERR_LENGTH),
                       (bad, LASSO_ERR_VALUE)):
        t, twin = lb.Transcript(b"c"), lb.Transcript(b"c")
        with pytest.raises(lb.LassoError) as e:
            t.append_combined_table_commitment(data)
        assert e.value.code == code
        assert t.challenge_scalar(b"next").tolist() == twin.challenge_scalar(b"next").tolist()
