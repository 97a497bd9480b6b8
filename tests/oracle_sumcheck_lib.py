"""ctypes wrappers of the oracle's SumcheckInstanceProof entry points (oracle_dense/, test infrastructure only):
prove_arbitrary with a combining function in the program format of lasso_comb_create, interpreted on the host, and
verify.  Transcripts are oracle_dense_lib.Transcript objects; field elements are numpy uint64 arrays of shape (..., 4)."""
import ctypes as C

import numpy as np

from oracle_dense_lib import _u64, lib
from oracle_lib import P, sz


def sumcheck_prove(polys, num_rounds, program, constants, degree, transcript, round_evals=False):
    """SumcheckInstanceProof::prove_arbitrary on copies of polys (k arrays of (len, 4) limbs) with the combining function
    interpreted on the host, on an oracle transcript -> dict(proof bytes, r, final_evals, claim[, round_evals])"""
    polys = _u64(np.stack([_u64(p) for p in polys]))
    k, n = polys.shape[0], polys.shape[1]
    program = np.ascontiguousarray(program, dtype=np.int32).reshape(-1, 3)
    constants = _u64(constants).reshape(-1, 4)
    cap = 8 + num_rounds * (8 + 32 * degree)
    out = np.zeros(cap, dtype=np.uint8)
    r = np.zeros((num_rounds, 4), dtype=np.uint64)
    fin = np.zeros((k, 4), dtype=np.uint64)
    claim = np.zeros(4, dtype=np.uint64)
    ev = np.zeros((num_rounds, degree + 1, 4), dtype=np.uint64) if round_evals else None
    L = lib()
    L.orcd_sumcheck_prove.restype = C.c_size_t
    got = L.orcd_sumcheck_prove(P(polys), sz(k), sz(n), sz(num_rounds), P(program), sz(program.shape[0]),
                                P(constants) if constants.size else None, sz(constants.shape[0]), sz(degree), transcript.h,
                                P(out), sz(cap), P(r), P(fin), P(claim), P(ev) if round_evals else None)
    assert got == cap, (got, cap)
    res = dict(proof=out.tobytes(), r=r, final_evals=fin, claim=claim)
    if round_evals:
        res["round_evals"] = ev
    return res


def sumcheck_verify(proof, claim, num_rounds, degree, transcript):
    """SumcheckInstanceProof::verify -> (0 accepted / 1 rejected / 2 does not parse, e, r)"""
    e = np.zeros(4, dtype=np.uint64)
    r = np.zeros((num_rounds, 4), dtype=np.uint64)
    rc = lib().orcd_sumcheck_verify(bytes(proof), sz(len(proof)), P(_u64(claim)), sz(num_rounds), sz(degree), transcript.h,
                                    P(e), P(r))
    return rc, e, r
