"""ctypes wrappers of the oracle's grand-product entry points (oracle_dense/, test infrastructure only):
GrandProductCircuit + BatchedGrandProductArgument::prove, verify, and a polynomial formed pointwise by a combining
function in the program format of lasso_comb_create.  Transcripts are oracle_dense_lib.Transcript objects; field
elements are numpy uint64 arrays of shape (..., 4)."""
import ctypes as C

import numpy as np

from oracle_dense_lib import _u64, lib
from oracle_lib import P, sz


def proof_len(n, num_vars):
    """the size of a serialised BatchedGrandProductArgument: per layer i < num_vars, a sumcheck of i cubic rounds
    (8 + i (8 + 3 * 32) bytes) and two vectors of n claims"""
    return 8 + sum(8 + i * (8 + 96) + 2 * (8 + 32 * n) for i in range(num_vars))


def gp_prove(polys, transcript):
    """GrandProductCircuit::new over each polynomial (n arrays of (2^v, 4) limbs, v >= 1) and
    BatchedGrandProductArgument::prove on an oracle transcript (the products are not appended) -> dict(proof, products,
    r, claims)"""
    polys = _u64(np.stack([_u64(p) for p in polys]))
    n, length = polys.shape[0], polys.shape[1]
    v = length.bit_length() - 1
    cap = proof_len(n, v)
    out = np.zeros(cap, dtype=np.uint8)
    products = np.zeros((n, 4), dtype=np.uint64)
    r = np.zeros((v, 4), dtype=np.uint64)
    claims = np.zeros((n, 4), dtype=np.uint64)
    L = lib()
    L.orcd_gp_prove.restype = C.c_size_t
    got = L.orcd_gp_prove(P(polys), sz(n), sz(length), transcript.h, P(out), sz(cap), P(products), P(r), P(claims))
    assert got == cap, (got, cap)
    return dict(proof=out.tobytes(), products=products, r=r, claims=claims)


def gp_verify(proof, products, num_vars, transcript):
    """BatchedGrandProductArgument::verify -> (0 accepted / 1 rejected / 2 does not parse, claims (n, 4), rand)"""
    products = _u64(products).reshape(-1, 4)
    n = products.shape[0]
    claims = np.zeros((n, 4), dtype=np.uint64)
    r = np.zeros((max(num_vars, 1), 4), dtype=np.uint64)
    rc = lib().orcd_gp_verify(bytes(proof), sz(len(proof)), P(products), sz(n), sz(num_vars), transcript.h, P(claims), P(r))
    return rc, claims, r[:num_vars]


def comb_map(polys, program, constants):
    """out[i] = g(polys[0][i], ..), g interpreted on the host"""
    polys = _u64(np.stack([_u64(p) for p in polys]))
    k, length = polys.shape[0], polys.shape[1]
    program = np.ascontiguousarray(program, dtype=np.int32).reshape(-1, 3)
    constants = _u64(constants).reshape(-1, 4)
    out = np.zeros((length, 4), dtype=np.uint64)
    lib().orcd_comb_map(P(polys), sz(k), sz(length), P(program), sz(program.shape[0]),
                        P(constants) if constants.size else None, sz(constants.shape[0]), P(out))
    return out
