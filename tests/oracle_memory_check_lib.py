"""ctypes wrappers for the oracle's MemoryCheckingProof::prove / verify on a caller-held transcript and tape (test
infrastructure only: oracle_dense/).  Transcripts and tapes are oracle_dense_lib objects; field elements are (..., 4)
uint64 Montgomery limbs."""
import ctypes as C

import numpy as np

import oracle_dense_lib as od
from oracle_lib import P, sz


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def prove(kind, C_, log_m, log_r, indices, gamma, tau, stream, transcript, tape, r=None):
    """Densify n x C indices, commit, and prove the memory check of a built-in strategy at (gamma, tau) on the oracle
    transcript and tape, advanced in place -> (proof bytes, sparse commitment bytes, combined-table commitment bytes).
    With r, the proof's prefix (surge.rs:129-186) runs first on the transcript and tape, and (gamma, tau) are drawn as
    surge.rs:188 draws them (the gamma and tau given are ignored)."""
    f = od.lib().orcd_memory_check_prove
    f.restype = C.c_size_t
    indices, stream = _u64(indices), _u64(stream)
    gamma, tau = _u64(gamma).reshape(4), _u64(tau).reshape(4)
    rr = None if r is None else _u64(r)
    cap = 1 << 24
    out, comm, derefs = (np.zeros(cap, dtype=np.uint8) for _ in range(3))
    nc, nd = C.c_size_t(0), C.c_size_t(0)
    n = f(int(kind), sz(C_), sz(log_m), sz(log_r), P(indices), sz(indices.shape[0]), P(gamma), P(tau),
          None if rr is None else P(rr), P(stream), sz(stream.shape[0]), transcript.h, tape.h, P(out), sz(cap), P(comm),
          sz(cap), C.byref(nc), P(derefs), sz(cap), C.byref(nd))
    assert n > 0
    return out[:n].tobytes(), comm[: nc.value].tobytes(), derefs[: nd.value].tobytes()


def verify(kind, C_, log_m, log_r, stream, commitment, derefs, proof, gamma, tau, transcript):
    """MemoryCheckingProof::verify of serialised bytes on an oracle transcript: 0 accepted, 1 rejected, 2 the bytes do
    not parse"""
    stream = _u64(stream)
    gamma, tau = _u64(gamma).reshape(4), _u64(tau).reshape(4)
    return od.lib().orcd_memory_check_verify(int(kind), sz(C_), sz(log_m), sz(log_r), P(stream), sz(stream.shape[0]),
                                             bytes(commitment), sz(len(commitment)), bytes(derefs), sz(len(derefs)),
                                             bytes(proof), sz(len(proof)), P(gamma), P(tau), transcript.h)
