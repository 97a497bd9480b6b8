"""ctypes wrappers of the oracle's Σ-protocols of committed scalars (oracle_dense/, test infrastructure only):
KnowledgeProof, EqualityProof and ProductProof prove / verify, restated from subprotocols/zk.rs, and a linear
combination of compressed points, on the transcript and tape objects of oracle_dense_lib.  gens is a MultiCommitGens
with n == 1, a pair (G, h) of (1, 8) and (8,) uint64 affine points as oracle_zk_lib makes them; field elements are (4,)
uint64 Montgomery limbs, points 32-byte compressed encodings."""
import ctypes as C

import numpy as np

import oracle_dense_lib as od
from oracle_lib import P, sz


def _sigma_lib():
    L = od.lib()
    for f in ("orcd_knowledge_prove", "orcd_equality_prove", "orcd_product_prove"):
        getattr(L, f).restype = C.c_size_t
    return L


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _g1(gens):
    G, h = _u64(gens[0]).reshape(-1, 8), _u64(gens[1]).reshape(8)
    assert G.shape[0] == 1
    return G, h


def _pts(k):
    return [np.zeros(32, dtype=np.uint8) for _ in range(k)]


def knowledge_prove(gens, transcript, tape, x, r):
    """KnowledgeProof::prove -> (proof bytes, C)"""
    G, h = _g1(gens)
    out, (c,) = np.zeros(96, dtype=np.uint8), _pts(1)
    got = _sigma_lib().orcd_knowledge_prove(P(G), P(h), transcript.h, tape.h, P(_u64(x)), P(_u64(r)), P(out), P(c))
    assert got == 96, got
    return out.tobytes(), c.tobytes()


def knowledge_verify(gens, proof, C, transcript):
    """KnowledgeProof::verify: 0 accepted, 1 rejected, 2 does not parse"""
    G, h = _g1(gens)
    return _sigma_lib().orcd_knowledge_verify(P(G), P(h), bytes(proof), sz(len(proof)), bytes(C), transcript.h)


def equality_prove(gens, transcript, tape, v1, s1, v2, s2):
    """EqualityProof::prove -> (proof bytes, C1, C2)"""
    G, h = _g1(gens)
    out, (c1, c2) = np.zeros(64, dtype=np.uint8), _pts(2)
    got = _sigma_lib().orcd_equality_prove(P(G), P(h), transcript.h, tape.h, *[P(_u64(v)) for v in (v1, s1, v2, s2)], P(out),
                                     P(c1), P(c2))
    assert got == 64, got
    return out.tobytes(), c1.tobytes(), c2.tobytes()


def equality_verify(gens, proof, C1, C2, transcript):
    """EqualityProof::verify: 0 accepted, 1 rejected, 2 does not parse"""
    G, h = _g1(gens)
    return _sigma_lib().orcd_equality_verify(P(G), P(h), bytes(proof), sz(len(proof)), bytes(C1), bytes(C2), transcript.h)


def product_prove(gens, transcript, tape, x, rX, y, rY, z, rZ):
    """ProductProof::prove -> (proof bytes, X, Y, Z)"""
    G, h = _g1(gens)
    out, (X, Y, Z) = np.zeros(256, dtype=np.uint8), _pts(3)
    got = _sigma_lib().orcd_product_prove(P(G), P(h), transcript.h, tape.h, *[P(_u64(v)) for v in (x, rX, y, rY, z, rZ)],
                                    P(out), P(X), P(Y), P(Z))
    assert got == 256, got
    return out.tobytes(), X.tobytes(), Y.tobytes(), Z.tobytes()


def product_verify(gens, proof, X, Y, Z, transcript):
    """ProductProof::verify: 0 accepted, 1 rejected, 2 does not parse"""
    G, h = _g1(gens)
    return _sigma_lib().orcd_product_verify(P(G), P(h), bytes(proof), sz(len(proof)), bytes(X), bytes(Y), bytes(Z),
                                      transcript.h)


def point_lincomb(points, scalars):
    """sum_i scalars[i] points[i] of 32-byte compressed points -> 32 bytes compressed"""
    pts = b"".join(bytes(p) for p in points)
    s = _u64(scalars).reshape(-1, 4)
    assert s.shape[0] * 32 == len(pts)
    out = np.zeros(32, dtype=np.uint8)
    rc = _sigma_lib().orcd_point_lincomb(pts, sz(s.shape[0]), P(s), P(out))
    assert rc == 0, rc
    return out.tobytes()
