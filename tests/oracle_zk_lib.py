"""ctypes wrappers of the oracle's zero-knowledge sumcheck pieces (oracle_dense/, test infrastructure only): commitments
to short vectors, DotProductProof prove / verify and ZKSumcheckInstanceProof prove / verify, on the transcript and tape
objects of oracle_dense_lib.  A MultiCommitGens is a pair (G, h) of (n, 8) and (8,) uint64 affine points; field
elements are (..., 4) uint64 Montgomery limbs, points 32-byte compressed encodings."""
import ctypes as C

import numpy as np

import oracle_dense_lib as od
from oracle_lib import P, sz


def _lib():
    L = od.lib()
    for f in ("orcd_dot_prove", "orcd_zk_prove"):
        getattr(L, f).restype = C.c_size_t
    return L


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _gens(g):
    G, h = _u64(g[0]).reshape(-1, 8), _u64(g[1]).reshape(8)
    return G, h


def mc_gens(stream, n):
    """MultiCommitGens::new(n) of a stream: (stream[0..n), stream[n])"""
    return _u64(stream[:n]), _u64(stream[n])


def dot_gens(stream, n):
    """DotProductProofGens::new(n): (gens_1, gens_n) = (([s[n]], s[n+1]), (s[0..n), s[n+1]))"""
    return (_u64(stream[n:n + 1]), _u64(stream[n + 1])), (_u64(stream[:n]), _u64(stream[n + 1]))


def commit(gens, scalars, blind):
    """batch_commit(scalars, blind, gens) -> 32 bytes"""
    G, h = _gens(gens)
    s = _u64(scalars).reshape(-1, 4)
    assert s.shape[0] == G.shape[0]
    out = np.zeros(32, dtype=np.uint8)
    _lib().orcd_mc_commit(P(G), sz(G.shape[0]), P(h), P(s), P(_u64(blind)), P(out))
    return out.tobytes()


def dot_prove(gens_1, gens_n, transcript, tape, x, blind_x, a, y, blind_y):
    """DotProductProof::prove -> (proof bytes, Cx, Cy)"""
    G1, h1 = _gens(gens_1)
    Gn, hn = _gens(gens_n)
    x, a = _u64(x).reshape(-1, 4), _u64(a).reshape(-1, 4)
    n = x.shape[0]
    cap = 136 + 32 * n
    out = np.zeros(cap, dtype=np.uint8)
    cx, cy = np.zeros(32, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    got = _lib().orcd_dot_prove(P(G1), P(h1), P(Gn), sz(n), P(hn), transcript.h, tape.h, P(x), P(_u64(blind_x)), P(a),
                                P(_u64(y)), P(_u64(blind_y)), P(out), sz(cap), P(cx), P(cy))
    assert got == cap, (got, cap)
    return out.tobytes(), cx.tobytes(), cy.tobytes()


def dot_verify(gens_1, gens_n, proof, a, Cx, Cy, transcript):
    """DotProductProof::verify: 0 accepted, 1 rejected, 2 does not parse"""
    G1, h1 = _gens(gens_1)
    Gn, hn = _gens(gens_n)
    a = _u64(a).reshape(-1, 4)
    return _lib().orcd_dot_verify(P(G1), P(h1), P(Gn), sz(Gn.shape[0]), P(hn), bytes(proof), sz(len(proof)), P(a),
                                  bytes(Cx), bytes(Cy), transcript.h)


def zk_prove(polys, num_rounds, program, constants, degree, blind_claim, gens_1, gens_n, transcript, tape):
    """the ZK sumcheck prover on copies of polys (k arrays of (len, 4) limbs), the combining function in the program
    format of lasso_comb_create -> dict(proof, r, final_evals, claim, comm_claim, blind_eval)"""
    G1, h1 = _gens(gens_1)
    Gn, hn = _gens(gens_n)
    assert Gn.shape[0] == degree + 1
    polys = _u64(np.stack([_u64(p) for p in polys]))
    k, n = polys.shape[0], polys.shape[1]
    program = np.ascontiguousarray(program, dtype=np.int32).reshape(-1, 3)
    constants = _u64(constants).reshape(-1, 4)
    cap = 24 + num_rounds * (200 + 32 * (degree + 1))
    out = np.zeros(cap, dtype=np.uint8)
    r = np.zeros((num_rounds, 4), dtype=np.uint64)
    fin = np.zeros((k, 4), dtype=np.uint64)
    claim, blind_eval = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    cc = np.zeros(32, dtype=np.uint8)
    got = _lib().orcd_zk_prove(P(polys), sz(k), sz(n), sz(num_rounds), P(program), sz(program.shape[0]),
                               P(constants) if constants.size else None, sz(constants.shape[0]), sz(degree),
                               P(_u64(blind_claim)), P(G1), P(h1), P(Gn), P(hn), transcript.h, tape.h, P(out), sz(cap),
                               P(r), P(fin), P(claim), P(cc), P(blind_eval))
    assert got == cap, (got, cap)
    return dict(proof=out.tobytes(), r=r, final_evals=fin, claim=claim, comm_claim=cc.tobytes(), blind_eval=blind_eval)


def zk_verify(proof, comm_claim, num_rounds, degree, gens_1, gens_n, transcript):
    """ZKSumcheckInstanceProof::verify -> (0 accepted / 1 rejected / 2 does not parse, the last comm_eval, r)"""
    G1, h1 = _gens(gens_1)
    Gn, hn = _gens(gens_n)
    e = np.zeros(32, dtype=np.uint8)
    r = np.zeros((max(num_rounds, 1), 4), dtype=np.uint64)
    rc = _lib().orcd_zk_verify(bytes(proof), sz(len(proof)), bytes(comm_claim), sz(num_rounds), sz(degree), P(G1), P(h1),
                               P(Gn), P(hn), transcript.h, P(e), P(r))
    return rc, e.tobytes(), r[:num_rounds]
