"""Shared pieces of the composed-protocol tests (test_compose_host.py, test_gpu_compose.py): the lookup outputs from the
oracle's own lookup polynomials and combine_lookups, and the claimed evaluation read out of proof bytes."""
import numpy as np

import oracle_custom_fr_lib as ocf
import oracle_lib as ol
from oracle_lib import P, sz


def dim_usize(indices, s):
    """DensifiedRepresentation::dim_usize (densified.rs:33-56): C x s, the padded lookups' indices 0"""
    idx = np.asarray(indices, dtype=np.uint64)
    out = np.zeros((idx.shape[1], s), dtype=np.uint64)
    out[:, : idx.shape[0]] = idx.T
    return np.ascontiguousarray(out)


def outputs(kind, C_, log_m, log_r, nz):
    """v[k] = combine_lookups(E_0[k], ..) from orc_lookup_polys + orc_combine_lookups -> (s, 4) Montgomery limbs"""
    L = ol.lib()
    s = nz.shape[1]
    alpha = int(L.orc_num_memories(kind, sz(C_), sz(log_m), sz(log_r)))
    E = np.zeros((alpha, s, 4), dtype=np.uint64)
    L.orc_lookup_polys(kind, sz(C_), sz(log_m), sz(log_r), P(np.ascontiguousarray(nz)), sz(s), P(E))
    v = np.zeros((s, 4), dtype=np.uint64)
    for k in range(s):
        col = np.ascontiguousarray(E[:, k])
        L.orc_combine_lookups(kind, sz(C_), sz(log_m), sz(log_r), P(col), P(v[k]))
    return v


def outputs_custom(S, nz):
    """the same for a lasso_b200.CustomStrategy (either table form), through the custom oracle's combine_lookups"""
    tabs = [t if t.ndim == 2 else ol.fr_array([int(x) for x in t]) for t in (np.asarray(t) for t in S.tables)]
    s = nz.shape[1]
    E = np.stack([tabs[S.memory_to_subtable[i]][nz[S.memory_to_dimension[i]].astype(np.int64)]
                  for i in range(S.num_memories)])
    return np.stack([ocf.combine_lookups(S, np.ascontiguousarray(E[:, k])) for k in range(s)])


def claim_in_proof(proof, log_s, sumcheck_degree):
    """PrimarySumcheck::claimed_evaluation at its offset in proof bytes (after comm_derefs and the primary sumcheck), as
    Montgomery limbs"""
    n_derefs = int.from_bytes(proof[:8], "little")
    at = 8 + 32 * n_derefs + 8 + log_s * (8 + 32 * sumcheck_degree)
    return ol.to_mont(int.from_bytes(proof[at:at + 32], "little"))
