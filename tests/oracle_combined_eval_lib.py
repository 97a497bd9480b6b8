"""ctypes wrappers of the oracle's DensePolynomial::merge and CombinedTableEvalProof::{prove, verify} (oracle_dense/, test
infrastructure only).  Transcripts and tapes are oracle_dense_lib objects; field elements are numpy uint64 arrays of shape
(..., 4)."""
import ctypes as C

import numpy as np

from oracle_dense_lib import _u64, lib
from oracle_lib import P, sz


def next_pow2(n):
    return 1 << max(int(n) - 1, 0).bit_length()


def proof_len(num_vars):
    """a serialised CombinedTableEvalProof is its PolyEvalProof: L_vec and R_vec of num_vars - num_vars // 2 points each,
    delta, beta, z1, z2"""
    lg = num_vars - num_vars // 2
    return 2 * (8 + 32 * lg) + 4 * 32


def merge(polys):
    """DensePolynomial::merge: the evaluations one after another, zero-padded to a power of two -> (2^v, 4)"""
    arrays = [_u64(p).reshape(-1, 4) for p in polys]
    lens = np.array([a.shape[0] for a in arrays], dtype=np.uint64)
    cap = next_pow2(int(lens.sum()))
    out = np.zeros((cap, 4), dtype=np.uint64)
    L = lib()
    L.orcd_merge.restype = C.c_size_t
    got = L.orcd_merge(P(_u64(np.concatenate(arrays))), P(lens), sz(len(arrays)), P(out), sz(cap))
    assert got == cap, (got, cap)
    return out


def prove(Z, evals, r, stream, transcript, tape):
    """CombinedTableEvalProof::prove on oracle transcript / tape objects -> proof bytes"""
    Z, evals, stream = _u64(Z), _u64(evals).reshape(-1, 4), _u64(stream)
    r = _u64(r).reshape(-1, 4)
    nv = Z.shape[0].bit_length() - 1
    cap = proof_len(nv)
    out = np.zeros(cap, dtype=np.uint8)
    L = lib()
    L.orcd_combined_eval_prove.restype = C.c_size_t
    n = L.orcd_combined_eval_prove(P(Z), sz(Z.shape[0]), P(evals), sz(evals.shape[0]), P(r), sz(r.shape[0]), P(stream),
                                   sz(stream.shape[0]), transcript.h, tape.h, P(out), sz(cap))
    assert n == cap, (n, cap)
    return out.tobytes()


def verify(stream, nv, comm, proof, evals, r, transcript):
    """CombinedTableEvalProof::verify: 0 accepted, 1 rejected, 2 does not parse"""
    stream, evals = _u64(stream), _u64(evals).reshape(-1, 4)
    r = _u64(r).reshape(-1, 4)
    return lib().orcd_combined_eval_verify(P(stream), sz(stream.shape[0]), sz(nv), bytes(comm), sz(len(comm)), bytes(proof),
                                           sz(len(proof)), P(evals), sz(evals.shape[0]), P(r), sz(r.shape[0]),
                                           transcript.h)
