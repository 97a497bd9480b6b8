"""The host side of lookups inside a caller's protocol, without a GPU: lasso_b200.Transcript.append_sparse_commitment
against the oracle's SparsePolynomialCommitment::append_to_transcript, its rejections, the argument checks of
SparsePolynomialEvaluationProof.prove, and the composed protocol in the oracle (commit to the lookup outputs v, absorb
the sparse commitment, draw r, prove on the transcript, open v at r at the proof's claimed evaluation) that the GPU
tests compare with."""
import numpy as np
import pytest

import compose_cases as cc
import lasso_b200 as lb
from lasso_b200.api import LASSO_ERR_LENGTH, LASSO_ERR_VALUE
import oracle_compose_lib as ocl
import oracle_dense_lib as od
import oracle_lib as ol

XOR, C_, LOG_M = 2, 2, 4


def _sparse(n=6, seed=0):
    """a small XOR proof's inputs and the oracle's commitment bytes -> (indices, stream, commitment)"""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, 1 << LOG_M, size=(n, C_), dtype=np.uint64)
    s = 1 << (n - 1).bit_length()
    stream = ol.generators(lb.gens_points_needed(C_, s, C_, LOG_M))
    r = ol.rand_fr(rng, s.bit_length() - 1)
    _, comm, _ = ocl.sparse_prove(XOR, C_, LOG_M, 0, idx, r, stream, od.Transcript(b"x"), od.RandomTape(b"t", ol.rand_fr(rng, 1)[0]))
    return idx, stream, comm


def _next(t):
    return t.challenge_scalar(b"next").tolist()


@pytest.mark.parametrize("n", [2, 6, 33])
def test_append_sparse_commitment_matches_oracle(n):
    _, _, comm = _sparse(n, seed=n)
    t, o = lb.Transcript(b"compose"), od.Transcript(b"compose")
    t.append_protocol_name(b"p")
    o.append_protocol_name(b"p")
    t.append_sparse_commitment(comm)
    assert ocl.append_sparse_commitment(o, comm) == 0
    assert _next(t) == _next(o)
    assert _next(t) != _next(lb.Transcript(b"compose"))


def _bad_point():
    """32 bytes whose y is canonical but (y^2 - 1) / (d y^2 + 1) is not a square: the oracle cannot decompress them"""
    o = od.Transcript(b"probe")
    for y in range(2, 200):
        b = y.to_bytes(32, "little")
        if od.lib().orcd_transcript_append_point(o.h, b"p", b, ) != 0:
            return b
    raise AssertionError("no undecompressable point below 200")


def _with_point(comm, k, point):
    b = bytearray(comm)
    b[8 + 32 * k: 8 + 32 * (k + 1)] = point
    return bytes(b)


def _cases():
    _, _, comm = _sparse(6, seed=1)
    n1 = int.from_bytes(comm[:8], "little")
    big = bytearray(comm)
    big[:8] = (n1 + 1).to_bytes(8, "little")
    huge = bytearray(comm)
    huge[:8] = (2**63).to_bytes(8, "little")
    yield "truncated", comm[:-1], LASSO_ERR_LENGTH
    yield "trailing", comm + b"\0", LASSO_ERR_LENGTH
    yield "empty", b"", LASSO_ERR_LENGTH
    yield "count+1", bytes(big), LASSO_ERR_LENGTH
    yield "count huge", bytes(huge), LASSO_ERR_LENGTH
    yield "bad point", _with_point(comm, 0, _bad_point()), LASSO_ERR_VALUE
    y_p = (2**255 - 19).to_bytes(32, "little")  # y = q: not canonical
    yield "y = q", _with_point(comm, 0, y_p), LASSO_ERR_VALUE


NAMES = ["truncated", "trailing", "empty", "count+1", "count huge", "bad point", "y = q"]


@pytest.mark.parametrize("name", NAMES)
def test_append_sparse_commitment_rejects(name):
    data, code = {c[0]: c[1:] for c in _cases()}[name]
    t, twin = lb.Transcript(b"compose"), lb.Transcript(b"compose")
    with pytest.raises(lb.LassoError) as e:
        t.append_sparse_commitment(data)
    assert e.value.code == code
    assert ocl.append_sparse_commitment(od.Transcript(b"x"), data) == 1  # the oracle cannot parse them either
    assert _next(t) == _next(twin)


def test_decompression_check_agrees_with_oracle():
    """every y below 300 with either sign: the library accepts exactly the points the oracle decompresses"""
    _, _, comm = _sparse(6, seed=2)
    o = od.Transcript(b"probe")
    for y in range(300):
        for sign in (0, 0x80):
            b = bytearray(y.to_bytes(32, "little"))
            b[31] |= sign
            ok = od.lib().orcd_transcript_append_point(o.h, b"p", bytes(b)) == 0
            t = lb.Transcript(b"c")
            try:
                t.append_sparse_commitment(_with_point(comm, 0, bytes(b)))
                got = True
            except lb.LassoError as e:
                assert e.code == LASSO_ERR_VALUE
                got = False
            assert got == ok, (y, sign)


def test_prove_argument_checks():
    """one handle without the other, or a handle with a label or seed, is refused before anything runs"""
    t, tape = lb.Transcript(b"t"), lb.RandomTape(b"p", np.zeros(4, dtype=np.uint64))
    S = lb.Strategy(lb.XOR, 2, 4)
    for kw in (dict(transcript=t), dict(random_tape=tape), dict(transcript=t, random_tape=tape, tape_seed=np.zeros(4)),
               dict(transcript=t, random_tape=tape, transcript_label=b"example"),
               dict(transcript=t, random_tape=tape, tape_label=b"proof")):
        with pytest.raises(lb.LassoError):
            lb.SparsePolynomialEvaluationProof.prove(None, S, None, np.zeros((1, 4), dtype=np.uint64), None, **kw)


def compose_oracle(kind, C_, log_m, log_r, idx, seed, prefix=b"Lasso composed", tamper_v=False, prove_prefix=None):
    """The composed protocol in the oracle, prover then verifier on fresh transcripts -> (sparse verdict, opening
    verdict).  prove_prefix: the prover runs the sparse proof on a transcript whose protocol name differs."""
    rng = np.random.default_rng(seed)
    n = idx.shape[0]
    s = 1 << (n - 1).bit_length()
    log_s = s.bit_length() - 1
    alpha = int(ol.lib().orc_num_memories(kind, ol.sz(C_), ol.sz(log_m), ol.sz(log_r)))
    stream = ol.generators(lb.gens_points_needed(C_, s, alpha, log_m))
    v_stream = ol.generators(lb.poly_gens_points_needed(log_s), b"gens_outputs")
    tape_seed = ol.rand_fr(rng, 1)[0]
    v = cc.outputs(kind, C_, log_m, log_r, cc.dim_usize(idx, s))
    if tamper_v:
        v = v.copy()
        v[int(rng.integers(0, s))] = ol.fr_array([12345])[0]
    comm_v = od.commit(v, v_stream)
    _, comm_sparse, _ = ocl.sparse_prove(kind, C_, log_m, log_r, idx, np.zeros((log_s, 4), dtype=np.uint64), stream,
                                        od.Transcript(b"scratch"), od.RandomTape(b"scratch", tape_seed))
    T, tape = od.Transcript(b"compose"), od.RandomTape(b"proof", tape_seed)
    T.append_protocol_name(prove_prefix or prefix)
    T.append_poly_commitment(b"outputs", comm_v)
    assert ocl.append_sparse_commitment(T, comm_sparse) == 0
    r = T.challenge_vector(b"r", log_s)
    proof, _, claim = ocl.sparse_prove(kind, C_, log_m, log_r, idx, r, stream, T, tape)
    opening, _ = od.prove(v, r, claim, v_stream, T, tape)
    V = od.Transcript(b"compose")
    V.append_protocol_name(prefix)
    V.append_poly_commitment(b"outputs", comm_v)
    assert ocl.append_sparse_commitment(V, comm_sparse) == 0
    rv = V.challenge_vector(b"r", log_s)
    ok_sparse = ocl.sparse_verify(kind, C_, log_m, log_r, stream, comm_sparse, proof, rv, V)
    deg = C_ + 1 if kind == lb.LT else 2
    zr = cc.claim_in_proof(proof, log_s, deg)
    ok_open = od.verify(v_stream, log_s, comm_v, opening, rv, zr, V)
    return ok_sparse, ok_open


@pytest.mark.parametrize("kind,C_,log_m,n", [(lb.XOR, 2, 4, 6), (lb.LT, 2, 4, 8), (lb.AND, 3, 4, 5)])
def test_composed_protocol_in_the_oracle(kind, C_, log_m, n):
    idx = np.random.default_rng(n).integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    assert compose_oracle(kind, C_, log_m, 0, idx, 7) == (0, 0)
    assert compose_oracle(kind, C_, log_m, 0, idx, 7, tamper_v=True)[1] == 1
    assert compose_oracle(kind, C_, log_m, 0, idx, 7, prove_prefix=b"another protocol")[0] == 1
