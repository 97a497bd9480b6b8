"""ctypes loader for the oracle of dense polynomials on a caller's transcript (oracle_dense/, test infrastructure only).

Field elements are numpy uint64 arrays of shape (..., 4): Montgomery limbs; points are 32-byte compressed encodings."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import P, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle_dense", "_build", "liblasso_oracle_dense.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle_dense")])
        L = C.CDLL(SO)
        for f in ("orcd_transcript_new", "orcd_tape_new"):
            getattr(L, f).restype = C.c_void_p
        L.orcd_transcript_free.argtypes = [C.c_void_p]
        L.orcd_tape_free.argtypes = [C.c_void_p]
        L.orcd_transcript_append_u64.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]
        for f in ("orcd_poly_commit", "orcd_poly_prove"):
            getattr(L, f).restype = C.c_size_t
        _lib = L
    return _lib


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


class Transcript:
    """the oracle's ProofTranscript, one method per lasso_b200.Transcript method"""

    def __init__(self, label):
        self.h = C.c_void_p(lib().orcd_transcript_new(label))

    def __del__(self):
        lib().orcd_transcript_free(self.h)

    def append_message(self, label, msg):
        lib().orcd_transcript_append_message(self.h, label, bytes(msg), sz(len(msg)))

    def append_u64(self, label, x):
        lib().orcd_transcript_append_u64(self.h, label, int(x))

    def append_protocol_name(self, name):
        lib().orcd_transcript_append_protocol_name(self.h, name)

    def append_scalar(self, label, s):
        lib().orcd_transcript_append_scalar(self.h, label, P(_u64(s)))

    def append_scalars(self, label, s):
        s = _u64(s).reshape(-1, 4)
        lib().orcd_transcript_append_scalars(self.h, label, P(s), sz(s.shape[0]))

    def append_point(self, label, p):
        assert lib().orcd_transcript_append_point(self.h, label, bytes(p)) == 0

    def append_points(self, label, pts):
        b = b"".join(bytes(p) for p in pts) if not isinstance(pts, bytes) else pts
        assert lib().orcd_transcript_append_points(self.h, label, b, sz(len(b) // 32)) == 0

    def append_poly_commitment(self, label, comm):
        assert lib().orcd_transcript_append_poly_commitment(self.h, label, bytes(comm), sz(len(comm))) == 0

    def challenge_scalar(self, label):
        out = np.zeros(4, dtype=np.uint64)
        lib().orcd_transcript_challenge_scalar(self.h, label, P(out))
        return out

    def challenge_vector(self, label, n):
        out = np.zeros((n, 4), dtype=np.uint64)
        lib().orcd_transcript_challenge_vector(self.h, label, sz(n), P(out))
        return out


class RandomTape:
    def __init__(self, label, seed):
        self.h = C.c_void_p(lib().orcd_tape_new(label, P(_u64(seed))))

    def __del__(self):
        lib().orcd_tape_free(self.h)

    def random_vector(self, label, n):
        out = np.zeros((n, 4), dtype=np.uint64)
        lib().orcd_tape_random_vector(self.h, label, sz(n), P(out))
        return out

    def random_scalar(self, label):
        return self.random_vector(label, 1)[0]


def commit(Z, stream):
    Z, stream = _u64(Z), _u64(stream)
    cap = 8 + 32 * Z.shape[0]
    out = np.zeros(cap, dtype=np.uint8)
    n = lib().orcd_poly_commit(P(Z), sz(Z.shape[0]), P(stream), sz(stream.shape[0]), P(out), sz(cap))
    assert n > 0
    return out[:n].tobytes()


def evaluate(Z, r):
    Z, r = _u64(Z), _u64(r)
    out = np.zeros(4, dtype=np.uint64)
    lib().orcd_evaluate(P(Z), sz(Z.shape[0]), P(r), P(out))
    return out


def prove(Z, r, Zr, stream, transcript, tape):
    """PolyEvalProof::prove on the oracle transcript / tape objects -> (proof bytes, C_Zr bytes)"""
    Z, r, Zr, stream = _u64(Z), _u64(r), _u64(Zr), _u64(stream)
    cap = 1 << 16
    out = np.zeros(cap, dtype=np.uint8)
    czr = np.zeros(32, dtype=np.uint8)
    n = lib().orcd_poly_prove(P(Z), sz(Z.shape[0]), P(r), P(Zr), P(stream), sz(stream.shape[0]), transcript.h, tape.h,
                              P(out), sz(cap), P(czr))
    assert n > 0
    return out[:n].tobytes(), czr.tobytes()


def verify(stream, nv, comm, proof, r, Zr, transcript):
    """0 accepted, 1 rejected, 2 does not parse"""
    stream, r, Zr = _u64(stream), _u64(r), _u64(Zr)
    return lib().orcd_poly_verify(P(stream), sz(stream.shape[0]), sz(nv), bytes(comm), sz(len(comm)), bytes(proof),
                                  sz(len(proof)), P(r), P(Zr), transcript.h)
