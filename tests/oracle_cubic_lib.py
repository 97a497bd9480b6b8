"""ctypes wrapper of the oracle's SumcheckInstanceProof::prove_cubic_batched (oracle_dense/, test infrastructure only),
with the caller's claim, coefficients and num_rounds.  Transcripts are oracle_dense_lib.Transcript objects; field
elements are numpy uint64 arrays of shape (..., 4)."""
import ctypes

import numpy as np

from oracle_dense_lib import _u64, lib
from oracle_lib import P, sz


def cubic_prove(A, B, C, coeffs, claim, num_rounds, transcript):
    """prove_cubic_batched on copies of the n pairs (A[k], B[k]) and C, (len, 4) limbs each, on an oracle transcript
    -> dict(proof bytes, r, finals (2n + 1, 4): A_0.., B_0.., C)"""
    n, length = len(A), C.shape[0]
    A = _u64(np.stack([_u64(a) for a in A]))
    B = _u64(np.stack([_u64(b) for b in B]))
    cap = 8 + 104 * num_rounds
    out = np.zeros(cap, dtype=np.uint8)
    r = np.zeros((max(num_rounds, 1), 4), dtype=np.uint64)
    fin = np.zeros((2 * n + 1, 4), dtype=np.uint64)
    L = lib()
    L.orcd_cubic_prove.restype = ctypes.c_size_t
    got = L.orcd_cubic_prove(P(A), P(B), sz(n), P(_u64(C)), sz(length), P(_u64(coeffs).reshape(-1, 4)),
                             P(_u64(claim).reshape(4)), sz(num_rounds), transcript.h, P(out), sz(cap), P(r), P(fin))
    assert got == cap, (got, cap)
    return dict(proof=out.tobytes(), r=r[:num_rounds], finals=fin)
