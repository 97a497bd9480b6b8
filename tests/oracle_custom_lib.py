"""ctypes loader for the oracle of caller-defined strategies (oracle_custom/, test infrastructure only).

S is a lasso_b200.CustomStrategy: only its host description is read (tables, maps, program, constants, declared
degree), so none of these needs a GPU.  Field elements are numpy uint64 arrays of shape (..., 4): Montgomery limbs."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import P, sz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle_custom", "_build", "liblasso_oracle_custom.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle_custom")])
        _lib = C.CDLL(SO)
    return _lib


def _args(S):
    keep = [np.ascontiguousarray(np.stack(S.tables), dtype=np.uint32), S.memory_to_subtable, S.memory_to_dimension,
            np.ascontiguousarray(S.program, dtype=np.int32), np.ascontiguousarray(S.constants.reshape(-1, 4))]
    args = [sz(S.C), sz(S.log_m), sz(S.num_subtables), P(keep[0]), sz(S.num_memories), P(keep[1]), P(keep[2]),
            P(keep[3]), sz(S.program.shape[0]), P(keep[4]), sz(S.constants.shape[0]), sz(S.g_poly_degree)]
    return args, keep


def combine_lookups(S, vals):
    args, keep = _args(S)
    vals = np.ascontiguousarray(vals, dtype=np.uint64)
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_custom_combine_lookups(*args, P(vals), P(out))
    return out


def evaluate_subtable_mle(S, k, point):
    args, keep = _args(S)
    point = np.ascontiguousarray(point, dtype=np.uint64)
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_custom_evaluate_subtable_mle(*args, sz(k), P(point), sz(point.shape[0]), P(out))
    return out


def sumcheck_round(S, polys):
    """One round of prove_arbitrary's evaluation loop; polys = (num_memories + 1, len, 4), the last one eq."""
    args, keep = _args(S)
    polys = np.ascontiguousarray(polys, dtype=np.uint64)
    out = np.zeros((S.g_poly_degree + 2, 4), dtype=np.uint64)
    lib().orc_custom_sumcheck_round(*args, P(polys), sz(polys.shape[1]), P(out))
    return out


def prove(S, indices, r, gens, tape_seed, flags=1):
    """Densify -> commit -> prove (-> verify) with a custom strategy.  Returns dict(rc, proof, commitment, challenges)."""
    args, keep = _args(S)
    indices = np.ascontiguousarray(indices, dtype=np.uint64)
    cap = 1 << 24
    proof = np.zeros(cap, dtype=np.uint8)
    comm = np.zeros(cap, dtype=np.uint8)
    chal = np.zeros((1 << 16, 4), dtype=np.uint64)
    plen, clen, nch = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    r = np.ascontiguousarray(r, dtype=np.uint64)
    gens = np.ascontiguousarray(gens, dtype=np.uint64)
    tape_seed = np.ascontiguousarray(tape_seed, dtype=np.uint64)
    rc = lib().orc_custom_prove(*args, P(indices), sz(indices.shape[0]), P(r), P(gens), sz(gens.shape[0]),
                                P(tape_seed), int(flags), P(proof), sz(cap), C.byref(plen), P(comm), sz(cap),
                                C.byref(clen), P(chal), sz(chal.shape[0]), C.byref(nch))
    return dict(rc=rc, proof=bytes(proof[: plen.value]), commitment=bytes(comm[: clen.value]),
                challenges=chal[: nch.value].copy())
