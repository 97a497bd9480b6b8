"""ctypes wrappers for the oracle's SparsePolynomialEvaluationProof on a caller-held transcript and tape (test
infrastructure only): the entry points oracle_dense/ and oracle_custom/ add for lookups inside a caller's protocol.
Transcripts and tapes are oracle_dense_lib objects; field elements are (..., 4) uint64 Montgomery limbs."""
import ctypes as C

import numpy as np

import oracle_custom_fr_lib as ocf
import oracle_custom_lib as oc
import oracle_dense_lib as od
from oracle_lib import P, sz


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _commitment_bytes(buf):
    """the serialised SparsePolynomialCommitment at the start of buf: two point vectors, then s, log_m, m"""
    at = 0
    for _ in range(2):
        at += 8 + 32 * int(np.frombuffer(buf[at:at + 8].tobytes(), dtype=np.uint64)[0])
    return buf[: at + 24].tobytes()


def append_sparse_commitment(transcript, commitment):
    """SparsePolynomialCommitment::append_to_transcript of lasso_commit-shaped bytes: 0 absorbed, 1 they do not parse"""
    return od.lib().orcd_sparse_append_commitment(transcript.h, bytes(commitment), sz(len(commitment)))


def sparse_prove(kind, C_, log_m, log_r, indices, r, stream, transcript, tape):
    """Densify -> commit -> SparsePolynomialEvaluationProof::prove for a built-in strategy on the oracle transcript and
    tape objects, advanced in place -> (proof bytes, commitment bytes, claimed evaluation)"""
    f = od.lib().orcd_sparse_prove
    f.restype = C.c_size_t
    indices, r, stream = _u64(indices), _u64(r), _u64(stream)
    cap = 1 << 24
    proof, comm = np.zeros(cap, dtype=np.uint8), np.zeros(cap, dtype=np.uint8)
    claim = np.zeros(4, dtype=np.uint64)
    n = f(int(kind), sz(C_), sz(log_m), sz(log_r), P(indices), sz(indices.shape[0]), P(r), P(stream),
          sz(stream.shape[0]), transcript.h, tape.h, P(proof), sz(cap), P(comm), sz(cap), P(claim))
    assert n > 0
    return proof[:n].tobytes(), _commitment_bytes(comm), claim


def sparse_verify(kind, C_, log_m, log_r, stream, commitment, proof, r, transcript):
    """SparsePolynomialEvaluationProof::verify of serialised bytes on an oracle transcript: 0 accepted, 1 rejected,
    2 the bytes do not parse"""
    stream, r = _u64(stream), _u64(r)
    return od.lib().orcd_sparse_verify(int(kind), sz(C_), sz(log_m), sz(log_r), P(stream), sz(stream.shape[0]),
                                       bytes(commitment), sz(len(commitment)), bytes(proof), sz(len(proof)), P(r),
                                       transcript.h)


def _custom(S, name):
    """the entry point for S's table form (the _fr one for (M, 4) tables) and its descriptor arguments"""
    if getattr(S, "fr_tables", False):
        args, keep = ocf._args(S)
        return getattr(oc.lib(), name + "_fr"), args, keep
    args, keep = oc._args(S)
    return getattr(oc.lib(), name), args, keep


def custom_prove(S, indices, r, gens, transcript, tape):
    """Densify -> commit -> prove with a lasso_b200.CustomStrategy on the oracle transcript and tape objects, advanced in
    place -> (proof bytes, commitment bytes, claimed evaluation)"""
    f, args, keep = _custom(S, "orc_custom_prove_transcript")
    f.restype = C.c_size_t
    indices, r, gens = _u64(indices), _u64(r), _u64(gens)
    cap = 1 << 24
    proof, comm = np.zeros(cap, dtype=np.uint8), np.zeros(cap, dtype=np.uint8)
    claim = np.zeros(4, dtype=np.uint64)
    n = f(*args, P(indices), sz(indices.shape[0]), P(r), P(gens), sz(gens.shape[0]), transcript.h, tape.h, P(proof),
          sz(cap), P(comm), sz(cap), P(claim))
    assert n > 0
    return proof[:n].tobytes(), _commitment_bytes(comm), claim


def custom_verify(S, gens, commitment, proof, r, transcript):
    """SparsePolynomialEvaluationProof::verify with a custom strategy of serialised bytes on an oracle transcript:
    0 accepted, 1 rejected, 2 the bytes do not parse"""
    f, args, keep = _custom(S, "orc_custom_verify_transcript")
    r, gens = _u64(r), _u64(gens)
    return f(*args, P(gens), sz(gens.shape[0]), bytes(commitment), sz(len(commitment)), bytes(proof), sz(len(proof)), P(r),
             transcript.h)
