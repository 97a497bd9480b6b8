"""Caller-defined strategies over tables of arbitrary field elements on the GPU (lasso_strategy_create_fr): whole proofs
against the oracle for caller-defined strategies, the u32 route for tables whose entries all fit 32 bits, the
commitment paths without the 16-bit table and without any multiples table, sharded proofs, one proof at size against
a golden hash, and the three new launchers one launch at a time (tests/kernel_harness/harness_fr.cu, built by
Makefile.fr)."""
import ctypes as C
import hashlib
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import field_tables as ft
import kernel_harness_lib as kh
import oracle_custom_fr_lib as oc
import oracle_lib as ol
import test_gpu_prove as tgp
from oracle_lib import P, lib as orc, sz
from test_gpu_launchers import check, mont, ptr, rvals

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
L = ol.L_FR


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _gens(ctx, S, s):
    import lasso_b200 as lb

    need = lb.gens_points_needed(S.C, s, S.num_memories, S.log_m)
    stream = np.ascontiguousarray(ol.generators(max(need, 300))[:need])
    return stream, lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", S.C, s, S.num_memories, S.log_m,
                                                   stream=stream)


def _prove(ctx, S, idx, r, seed, s):
    import lasso_b200 as lb

    stream, gens = _gens(ctx, S, s)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, S.log_m)
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    return stream, com, proof


def _assert_oracle(S, idx, r, seed, stream, com, proof, what):
    ref = oc.prove(S, idx, r, stream, seed, flags=1)
    assert ref["rc"] == 0, what
    assert com == ref["commitment"], what + ": commitment differs"
    assert (proof.challenges.shape == ref["challenges"].shape and (proof.challenges == ref["challenges"]).all()), \
        what + ": challenges differ"
    assert proof.bytes == ref["proof"], what + ": proof differs"


# (C, log_m, degree, nsub, lookups): alpha = C * nsub from 1 to 16, degree 1..3, odd log_m, s = 2^10 .. 2^14
CONFIGS = [(1, 5, 1, 1, 1 << 10), (2, 7, 2, 2, 1 << 11), (4, 8, 3, 1, 3000), (8, 6, 1, 2, 1 << 10), (3, 9, 2, 1, 1 << 14)]
CASES = [(name, cfg) for name in sorted(ft.INTS) for cfg in CONFIGS if name == "random_full" or cfg == CONFIGS[1]]
CASES += [("edges", CONFIGS[4]), ("squares_40bit", CONFIGS[3]), ("differences", CONFIGS[2])]


@pytest.mark.parametrize("name,cfg", CASES, ids=["%s-C%d-m%d-d%d-a%d-n%d" % ((n,) + c[:3] + (c[0] * c[3], c[4]))
                                                 for n, c in CASES])
def test_prove_matches_oracle(ctx, name, cfg):
    C_, log_m, degree, nsub, n = cfg
    S = ft.strategy(ctx, name, C_, log_m, degree, nsub)
    idx, r, seed, s = tgp.make_inputs(C_, log_m, n, len(name) + C_, False)
    stream, com, proof = _prove(ctx, S, idx, r, seed, s)
    _assert_oracle(S, idx, r, seed, stream, com, proof, "%s %s" % (name, cfg))
    S.close()


def test_fr_entry_point_below_2_32_is_the_u32_route(ctx):
    """entries all below 2^32 through lasso_strategy_create_fr: the same bytes and the same launches as through
    lasso_strategy_create"""
    import lasso_b200 as lb

    rng = np.random.default_rng(8)
    t = rng.integers(0, 2**32, size=1 << 8, dtype=np.uint64)
    t[3], t[4] = 2**32 - 1, 0
    g = ft.g_of_degree(2)
    idx, r, seed, s = tgp.make_inputs(3, 8, 1 << 12, 5, False)
    out = {}
    for form in ("u32", "fr"):
        before = ctx.launches
        S = lb.CustomStrategy(ctx, 3, 8, [t if form == "u32" else lb.fr_from_ints(t.tolist())], g, 2)
        stream, com, proof = _prove(ctx, S, idx, r, seed, s)
        out[form] = (com, proof.bytes, ctx.launches - before)
        S.close()
    assert out["u32"] == out["fr"]


@pytest.mark.parametrize("env", [{"LASSO_B200_TABLE_GB": "0"}, {"LASSO_B200_NO_MULTIPLES": "1"}],
                         ids=["no_16bit_table", "no_multiples"])
@pytest.mark.parametrize("name", ["random_full", "squares_40bit", "edges"])
def test_prove_without_tables(monkeypatch, name, env):
    """the generators built without the 16-bit table (the Fr row kernel is unchanged) and without any multiples table
    (canonicalise + bucket MSM rows): the same bytes as the oracle"""
    import lasso_b200 as lb

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    c = lb.Context(0)
    try:
        S = ft.strategy(c, name, 2, 7, 2, 2)
        idx, r, seed, s = tgp.make_inputs(2, 7, 1 << 11, len(name), False)
        stream, com, proof = _prove(c, S, idx, r, seed, s)
        S.close()
    finally:
        for k in env:
            monkeypatch.delenv(k)
    _assert_oracle(S, idx, r, seed, stream, com, proof, "%s %s" % (name, env))
    c.close()


@pytest.mark.parametrize("nproc", [2, 4])
def test_sharded_one_gpu_bit_exact(nproc):
    """tools/sharded_check.py --fr: every field-element table, one proof sharded over nproc ranks on GPU 0"""
    sock = socket.socket()
    sock.bind(("127.0.0.1", 0))
    port = sock.getsockname()[1]
    sock.close()
    env = dict(os.environ, LASSO_SHARD_SAME_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sharded_check.py"), "--fr"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env)
    assert "SHARDED_CHECK PASS" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


def test_at_size_matches_golden(ctx):
    """C = 4, log_m = 16, 2^20 lookups, a full-width random table: hashes of tests/golden/field_tables_big.json"""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_fr as mg

    case = json.load(open(os.path.join(HERE, "golden", "field_tables_big.json")))["cases"][mg.NAME]
    S0, idx, r, seed, stream = mg.inputs()
    assert hashlib.sha256(idx.tobytes()).hexdigest() == case["indices_sha256"]
    assert hashlib.sha256(np.stack(S0.tables).tobytes()).hexdigest() == case["table_sha256"]
    import lasso_b200 as lb

    S = lb.CustomStrategy(ctx, mg.C, mg.LOG_M, S0.tables, ft.g_of_degree(1), 1)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", mg.C, 1 << mg.LOG_S, S.num_memories, mg.LOG_M,
                                           stream=stream)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, mg.LOG_M)
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    S.close()
    assert hashlib.sha256(com).hexdigest() == case["commitment_sha256"]
    assert len(proof.challenges) == case["n_challenges"]
    assert hashlib.sha256(np.ascontiguousarray(proof.challenges).tobytes()).hexdigest() == case["challenges_sha256"]
    assert hashlib.sha256(proof.bytes).hexdigest() == case["proof_sha256"]


# ---------------------------------------------------------------- one launch at a time
KH_FR = os.path.join(HERE, "kernel_harness", "_build", "libkernel_harness_fr.so")
_khfr = None


def _kh():
    """libkernel_harness_fr.so (tests/kernel_harness/Makefile.fr); the tables come from libkernel_harness.so"""
    global _khfr
    if _khfr is None:
        if not os.path.exists(KH_FR):
            raise RuntimeError("libkernel_harness_fr.so is missing: run `python -c 'import __graft_entry__ as g; "
                               "g.build()'` (nvcc, sm_90a).")
        L_ = C.CDLL(KH_FR)
        V, I, S_ = C.c_void_p, C.c_int, C.c_size_t
        L_.kh_msm_rows_direct_fr.argtypes = [V, V, I, I, I, I, I, V]
        L_.kh_bound_fr.argtypes = [V, V, S_, S_, V]
        L_.kh_multi_dot_fr.argtypes = [V, S_, I, V, S_, V]
        _khfr = L_
    return _khfr


def _call(name, *args):
    rc = getattr(_kh(), name)(*args)
    assert rc == 0, "%s returned %d (-1: the launcher threw, -2: CUDA error, -4: bad arguments)" % (name, rc)


@pytest.fixture(scope="module")
def gens():
    return np.ascontiguousarray(ol.generators(2 * 300 + 4))


@pytest.fixture(scope="module")
def tables(gens):
    t = kh.Tables(gens)
    yield t
    t.close()


FR_EDGES = [0, 1, L - 1, 2**252, 2**32 - 1, 2**32, L - 2**200]


def _fr_rows(rng, nrows, ncols, nw):
    """values of at most 8 nw - 2 bits (the widest nw windows cover): the window boundaries 2^(8k) - 1, 2^(8k),
    2^(8k) + 127, 128 * 2^(8k) below the top, the edges that fit, random values of the full width, an all-zero row and
    an all-equal row of the largest value"""
    bits = min(8 * nw - 2, 253)
    top = min(2**bits, L)
    edges = [v for v in FR_EDGES if v < top]
    for k in range(nw):
        for v in (2**(8 * k) - 1, 2**(8 * k), 2**(8 * k) + 127, 2**(8 * k) * 128, 2**(8 * k) * 129 - 1):
            if 0 <= v < top:
                edges.append(v)
    z = [int.from_bytes(rng.bytes(40), "little") % top for _ in range(nrows * ncols)]
    for i, v in enumerate(edges):
        z[(i * 7) % len(z)] = v
    if top > 1:
        z[(len(edges) * 7 + 3) % len(z)] = top - 1
    if nrows > 2:
        z[:ncols] = [0] * ncols
        z[ncols:2 * ncols] = [top - 1] * ncols
    return z


def _rows_check(tables, gens, nrows, ncols, nw, col_mul, col_add, seed):
    rng = np.random.default_rng(seed)
    z = _fr_rows(rng, nrows, ncols, nw)
    gsel = np.ascontiguousarray(np.concatenate([gens[[c * col_mul + col_add for c in range(ncols)]], gens[:1]]))
    out = np.zeros((nrows, 16), dtype=np.uint64)
    zm = mont(z)
    _call("kh_msm_rows_direct_fr", tables.h, ptr(zm), nrows, ncols, nw, col_mul, col_add, ptr(out))
    ref = np.zeros((nrows, 16), dtype=np.uint64)
    orc().orc_commit_rows(P(gsel), P(zm), sz(nrows), sz(ncols), P(ref))
    for i in range(nrows):
        aff = np.zeros(8, dtype=np.uint64)
        orc().orc_point_to_affine(P(np.ascontiguousarray(ref[i])), P(aff))
        assert (out[i][:8] == aff).all(), ("msm_rows_direct_fr nrows=%d ncols=%d nw=%d col_map=%d*c+%d: row %d differs"
                                           % (nrows, ncols, nw, col_mul, col_add, i))


@pytest.mark.parametrize("nw", list(range(1, 33)))
def test_msm_rows_direct_fr_every_window_count(tables, gens, nw):
    _rows_check(tables, gens, 4, 200, nw, 1, 0, nw)


@pytest.mark.parametrize("ncols", [1, 128, 300])
def test_msm_rows_direct_fr_shapes(tables, gens, ncols):
    """ncols not a multiple of the 128 threads, one column, many rows; full width"""
    _rows_check(tables, gens, 33, ncols, 32, 1, 0, ncols)


@pytest.mark.parametrize("nw", [6, 32])
def test_msm_rows_direct_fr_sharded_columns(tables, gens, nw):
    """one rank of a proof sharded over two GPUs: local column c <-> generator 2c + 1"""
    _rows_check(tables, gens, 9, 150, nw, 2, 1, 77 + nw)


@pytest.mark.parametrize("L_size,R_size", [(1, 8), (4, 300), (64, 64), (200, 33), (2048, 4)])
def test_bound_fr(L_size, R_size):
    """LZ[i] = sum_j L[j] Z[j R + i] mod l; (l-1)(l-1) everywhere in the longest per-thread run (2048 rows over 64
    chunks)"""
    rng = np.random.default_rng(L_size * 7 + R_size)
    Lv = rvals(rng, L_size)
    Z = rvals(rng, L_size * R_size)
    if L_size == 2048:
        Lv = [L - 1] * L_size
        Z = [L - 1] * (L_size * R_size)
    out = np.zeros((R_size, 4), dtype=np.uint64)
    _call("kh_bound_fr", ptr(mont(Z)), ptr(mont(Lv)), L_size, R_size, ptr(out))
    want = [sum(Lv[j] * Z[j * R_size + i] for j in range(L_size)) % L for i in range(R_size)]
    check("bound_fr L=%d R=%d" % (L_size, R_size), out, want)


@pytest.mark.parametrize("npolys,n,stride", [(1, 1, 1), (3, 1000, 1024), (16, 4096, 4096), (2, 1 << 17, 1 << 17)])
def test_multi_dot_fr(npolys, n, stride):
    """out[k] = <z_k, eq> mod l; the longest case puts l - 1 times l - 1 in every term of a thread's run"""
    rng = np.random.default_rng(npolys * 13 + n)
    if n == 1 << 17:
        base = [L - 1] * (npolys * stride)
        eq = [L - 1] * n
    else:
        base = rvals(rng, npolys * stride)
        eq = rvals(rng, n)
    out = np.zeros((npolys, 4), dtype=np.uint64)
    _call("kh_multi_dot_fr", ptr(mont(base)), stride, npolys, ptr(mont(eq)), n, ptr(out))
    want = [sum(base[k * stride + i] * eq[i] for i in range(n)) % L for k in range(npolys)]
    check("multi_dot_fr npolys=%d n=%d" % (npolys, n), out, want)
