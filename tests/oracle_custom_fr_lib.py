"""ctypes loader for the _fr entry points of the oracle for caller-defined strategies (oracle_custom/, test
infrastructure only): the same calls as oracle_custom_lib, for a lasso_b200.CustomStrategy whose tables are (M, 4)
Montgomery arrays (S.fr_tables).  A strategy with u32 tables is passed to oracle_custom_lib unchanged, so callers can
use this module for either kind."""
import ctypes as C

import numpy as np

import oracle_custom_lib as oc
from oracle_lib import P, sz

lib = oc.lib


def _fr_tables(S):
    return getattr(S, "fr_tables", False)


def _args(S):
    keep = [np.ascontiguousarray(np.stack(S.tables), dtype=np.uint64), S.memory_to_subtable, S.memory_to_dimension,
            np.ascontiguousarray(S.program, dtype=np.int32), np.ascontiguousarray(S.constants.reshape(-1, 4))]
    args = [sz(S.C), sz(S.log_m), sz(S.num_subtables), P(keep[0]), sz(S.num_memories), P(keep[1]), P(keep[2]),
            P(keep[3]), sz(S.program.shape[0]), P(keep[4]), sz(S.constants.shape[0]), sz(S.g_poly_degree)]
    return args, keep


def combine_lookups(S, vals):
    if not _fr_tables(S):
        return oc.combine_lookups(S, vals)
    args, keep = _args(S)
    vals = np.ascontiguousarray(vals, dtype=np.uint64)
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_custom_combine_lookups_fr(*args, P(vals), P(out))
    return out


def evaluate_subtable_mle(S, k, point):
    if not _fr_tables(S):
        return oc.evaluate_subtable_mle(S, k, point)
    args, keep = _args(S)
    point = np.ascontiguousarray(point, dtype=np.uint64)
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_custom_evaluate_subtable_mle_fr(*args, sz(k), P(point), sz(point.shape[0]), P(out))
    return out


def sumcheck_round(S, polys):
    """One round of prove_arbitrary's evaluation loop; polys = (num_memories + 1, len, 4), the last one eq."""
    if not _fr_tables(S):
        return oc.sumcheck_round(S, polys)
    args, keep = _args(S)
    polys = np.ascontiguousarray(polys, dtype=np.uint64)
    out = np.zeros((S.g_poly_degree + 2, 4), dtype=np.uint64)
    lib().orc_custom_sumcheck_round_fr(*args, P(polys), sz(polys.shape[1]), P(out))
    return out


def prove(S, indices, r, gens, tape_seed, flags=1):
    """Densify -> commit -> prove (-> verify) with a custom strategy.  Returns dict(rc, proof, commitment, challenges)."""
    if not _fr_tables(S):
        return oc.prove(S, indices, r, gens, tape_seed, flags)
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
    rc = lib().orc_custom_prove_fr(*args, P(indices), sz(indices.shape[0]), P(r), P(gens), sz(gens.shape[0]),
                                   P(tape_seed), int(flags), P(proof), sz(cap), C.byref(plen), P(comm), sz(cap),
                                   C.byref(clen), P(chal), sz(chal.shape[0]), C.byref(nch))
    return dict(rc=rc, proof=bytes(proof[: plen.value]), commitment=bytes(comm[: clen.value]),
                challenges=chal[: nch.value].copy())
