"""ctypes wrappers of the oracle's hiding commitments and openings (oracle_dense/, test infrastructure only), on the
transcript and tape objects of oracle_dense_lib.  Field elements are (..., 4) uint64 Montgomery limbs, points 32-byte
compressed encodings."""
import ctypes as C

import numpy as np

import oracle_dense_lib as od
from oracle_lib import P, sz


def _lib():
    L = od.lib()
    for f in ("orcd_poly_commit_hiding", "orcd_poly_prove_hiding"):
        getattr(L, f).restype = C.c_size_t
    return L


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def commit_hiding(Z, stream, tape=None, blinds=None):
    """DensePolynomial::commit with blinds: drawn from `tape` as random_vector("poly_blinds", L), or the given (L, 4)
    blinds -> (commitment bytes, blinds)"""
    Z, stream = _u64(Z), _u64(stream)
    nv = Z.shape[0].bit_length() - 1
    L = 1 << (nv // 2)
    bl = np.zeros((L, 4), dtype=np.uint64) if blinds is None else _u64(blinds).copy()
    assert bl.shape == (L, 4)
    cap = 8 + 32 * L
    out = np.zeros(cap, dtype=np.uint8)
    n = _lib().orcd_poly_commit_hiding(P(Z), sz(Z.shape[0]), P(stream), sz(stream.shape[0]),
                                       None if tape is None else tape.h, P(bl), P(out), sz(cap))
    assert n > 0
    return out[:n].tobytes(), bl


def prove_hiding(Z, r, Zr, stream, transcript, tape, blinds=None, blind_Zr=None):
    """PolyEvalProof::prove with blinds / blind_Zr (None: None) -> (proof bytes, C_Zr bytes)"""
    Z, r, Zr, stream = _u64(Z), _u64(r), _u64(Zr), _u64(stream)
    bl = np.zeros((0, 4), dtype=np.uint64) if blinds is None else _u64(blinds)
    bz = None if blind_Zr is None else _u64(blind_Zr)
    cap = 1 << 16
    out = np.zeros(cap, dtype=np.uint8)
    czr = np.zeros(32, dtype=np.uint8)
    n = _lib().orcd_poly_prove_hiding(P(Z), sz(Z.shape[0]), P(bl), sz(bl.shape[0]), P(r), P(Zr),
                                      None if bz is None else P(bz), P(stream), sz(stream.shape[0]), transcript.h,
                                      tape.h, P(out), sz(cap), P(czr))
    assert n > 0
    return out[:n].tobytes(), czr.tobytes()


def verify(stream, nv, comm, proof, r, C_Zr, transcript):
    """PolyEvalProof::verify against a compressed C_Zr: 0 accepted, 1 rejected, 2 does not parse"""
    stream, r = _u64(stream), _u64(r)
    return _lib().orcd_poly_verify_czr(P(stream), sz(stream.shape[0]), sz(nv), bytes(comm), sz(len(comm)), bytes(proof),
                                       sz(len(proof)), P(r), bytes(C_Zr), transcript.h)
