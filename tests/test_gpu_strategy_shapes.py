"""The built-in strategies at the edges of the shapes the C ABI accepts (strategy_shapes.py restates
Strategy::valid()): round messages, subtables and gathers, and whole proofs, each bit-exact against the CPU oracle;
and every built-in entry point refusing the shape just past each boundary, LT proofs with C > 8 included, before any
launch."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import custom_builtins as cb
import oracle_lib as ol
import strategy_shapes as ss
import test_gpu_prove as tgp
from oracle_lib import P, lib as orc, sz

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGES = (0, 1, ol.L_FR - 1)
ERR_STRATEGY = 4  # LASSO_ERR_STRATEGY


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def sid(case):
    kind, C_, log_m, log_r = case[:4]
    return "%s_c%d_m%d_r%d" % (ss.NAMES.get(kind, "kind%d" % kind), C_, log_m, log_r)


def rand_polys(rng, npolys, n):
    """npolys random polynomials of n field elements, each with 0, 1 and l - 1 at random places"""
    if n >= 1 << 12:  # any residue below l is a field element in memory format: uniform below 2^252, made by numpy
        polys = rng.integers(0, 1 << 64, size=(npolys, n, 4), dtype=np.uint64)
        polys[:, :, 3] &= np.uint64((1 << 60) - 1)
    else:
        polys = ol.rand_fr(rng, npolys * n).reshape(npolys, n, 4)
    edges = ol.fr_array(EDGES)
    for k in range(npolys):
        for j, pos in enumerate(rng.choice(n, size=min(n, len(EDGES)), replace=False)):
            polys[k, pos] = edges[(j + k) % len(EDGES)]
    return polys


def oracle_round(S, polys):
    ref = np.zeros((S.sumcheck_poly_degree + 1, 4), dtype=np.uint64)
    orc().orc_sumcheck_round_arbitrary(S.kind, sz(S.C), sz(S.log_m), sz(S.log_r), P(np.ascontiguousarray(polys)),
                                       sz(polys.shape[1]), P(ref))
    return ref


def check_rounds(ctx, case, n):
    """one round over n elements, then (n >= 4) the bind to each r in {random, 0, l - 1} fused with the next round"""
    import lasso_b200 as lb

    S = lb.Strategy(*case)
    rng = np.random.default_rng(ss.seed_of(case, n))
    polys = rand_polys(rng, S.num_memories + 1, n)
    got = lb.sumcheck_round_arbitrary(ctx, S, list(polys))
    assert got.shape == (S.sumcheck_poly_degree + 1, 4)
    assert (got == oracle_round(S, polys)).all(), "round message"
    if n < 4:
        return
    for r in (ol.rand_fr(rng, 1)[0], ol.fr_array([0])[0], ol.fr_array([ol.L_FR - 1])[0]):
        bound = polys.copy()
        for k in range(bound.shape[0]):
            orc().orc_bind(1, P(bound[k]), sz(n), P(np.ascontiguousarray(r)))
        bound = np.ascontiguousarray(bound[:, : n // 2])
        got_polys, got = lb.sumcheck_bind_round_arbitrary(ctx, S, list(polys), r)
        assert (got == oracle_round(S, bound)).all(), ("bind round", ol.fr_ints(r))
        for k in range(bound.shape[0]):
            assert (got_polys[k] == bound[k]).all(), ("bound polynomial", k)


# ---------------------------------------------------------------- round messages
@pytest.mark.parametrize("n", ss.LT_ROUND_LENGTHS)
@pytest.mark.parametrize("case", ss.LT_ROUNDS, ids=sid)
def test_lt_round_every_c(ctx, case, n):
    """C = 1..16: the unrolled kernels (1-4), both C = 8 kernels, and the generic kernel (5-7, 9-16) that evaluates
    the C + 2 points six at a time"""
    check_rounds(ctx, case, n)


@pytest.mark.parametrize("case", ss.LT_GRID_STRIDE, ids=sid)
def test_lt_round_grid_stride(ctx, case):
    check_rounds(ctx, case, 1 << 16)


@pytest.mark.parametrize("case", ss.LT_TWO_LANE_BIND, ids=sid)
def test_lt_bind_round_two_lane_kernel(ctx, case):
    """n = 2^14: the round before the bind and the round after it both have at least 4096 pairs (sc_eval_lt2_kernel)"""
    check_rounds(ctx, case, 1 << 14)


@pytest.mark.parametrize("n", ss.LINEAR_ROUND_LENGTHS)
@pytest.mark.parametrize("case", ss.LINEAR_ROUNDS + ss.WEIGHT_BOUNDARY, ids=sid)
def test_linear_round(ctx, case, n):
    """AND, OR, XOR and RangeCheck: odd and even weight steps, C up to 16, the widest weights (shift 63)"""
    check_rounds(ctx, case, n)


# ---------------------------------------------------------------- subtables and gather
@pytest.mark.parametrize("case", ss.TABLES_SMALLEST + ss.TABLES_RANGE + ss.TABLES_LARGE + ss.GATHER_ALL_MEMORIES, ids=sid)
def test_materialize_and_gather(ctx, case):
    import lasso_b200 as lb

    kind, C_, log_m, log_r = case
    S = lb.Strategy(*case)
    M = 1 << log_m
    ref = np.zeros((S.num_subtables, M, 4), dtype=np.uint64)
    orc().orc_materialize_subtables(kind, sz(C_), sz(log_m), sz(log_r), P(ref))
    got = lb.materialize_subtables(ctx, S)
    for k in range(S.num_subtables):
        assert (got[k] == ref[k]).all(), ("subtable", k)
    if kind == ss.RANGE_CHECK:  # range_check.rs:15-34, restated: full, below 2^(log_r mod log_m), zero
        cut = 1 << (log_r % log_m)
        assert ol.fr_ints(got[1][: min(M, 64)]) == [i if i < cut else 0 for i in range(min(M, 64))]
        assert (got[2] == 0).all()
    rng = np.random.default_rng(ss.seed_of(case))
    s = 512
    nz = rng.integers(0, M, size=(C_, s), dtype=np.uint64)
    nz[:, 0], nz[:, 1] = 0, M - 1
    refE = np.zeros((S.num_memories, s, 4), dtype=np.uint64)
    orc().orc_lookup_polys(kind, sz(C_), sz(log_m), sz(log_r), P(nz), sz(s), P(refE))
    gotE = lb.gather_lookup_polys(ctx, S, [nz[d] for d in range(C_)])
    assert len(gotE) == S.num_memories
    for k in range(S.num_memories):
        assert (gotE[k] == refE[k]).all(), ("memory", k)


# ---------------------------------------------------------------- whole proofs
PROOFS = {c[0]: c for c in ss.PROOFS}
_oracle_proofs = {}


def proof_inputs(name):
    _, kind, C_, log_m, log_r, n, same = PROOFS[name]
    idx, r, seed, s = tgp.make_inputs(C_, log_m, n, ss.seed_of(name), same)
    need = gens_needed(kind, C_, log_m, s)
    return idx, r, seed, s, np.ascontiguousarray(ol.generators(9002)[:need])


def gens_needed(kind, C_, log_m, s):
    import lasso_b200 as lb

    return lb.gens_points_needed(C_, s, ss.num_memories(kind, C_) if kind in ss.KINDS else C_, log_m)


def oracle_proof(name):
    if name not in _oracle_proofs:
        _, kind, C_, log_m, log_r, n, same = PROOFS[name]
        idx, r, seed, s, stream = proof_inputs(name)
        ref = ol.prove(kind, C_, log_m, log_r, idx, r, stream, seed, flags=1)
        assert ref["rc"] == 0, "the oracle's verifier rejected"
        _oracle_proofs[name] = ref
    return _oracle_proofs[name]


def gpu_proof(ctx, name, strategy=None):
    """(commitment, proof) of the GPU path; strategy defaults to the built-in one"""
    import lasso_b200 as lb

    _, kind, C_, log_m, log_r, n, same = PROOFS[name]
    idx, r, seed, s, stream = proof_inputs(name)
    S = strategy if strategy is not None else lb.Strategy(kind, C_, log_m, log_r)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, s, S.num_memories, log_m, stream=stream)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    assert dense.s == s
    return dense.commit(gens), lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)


def assert_matches_oracle(name, commitment, proof):
    ref = oracle_proof(name)
    assert commitment == ref["commitment"]
    nch = min(len(proof.challenges), len(ref["challenges"]))
    first_bad = next((i for i in range(nch) if (proof.challenges[i] != ref["challenges"][i]).any()), None)
    assert first_bad is None, "Fiat-Shamir challenge %d diverges" % first_bad
    assert len(proof.challenges) == len(ref["challenges"])
    assert proof.bytes == ref["proof"]


@pytest.mark.parametrize("name", sorted(PROOFS))
def test_prove_matches_oracle(ctx, name):
    assert_matches_oracle(name, *gpu_proof(ctx, name))


@pytest.mark.parametrize("name", ss.PROOF_SUBSET)
def test_prove_as_custom_matches_oracle(ctx, name):
    """the same strategy as a caller-defined program (the interpreter kernels): the same bytes"""
    _, kind, C_, log_m, log_r, n, same = PROOFS[name]
    S = cb.as_custom(ctx, kind, C_, log_m, log_r)
    try:
        assert_matches_oracle(name, *gpu_proof(ctx, name, S))
    finally:
        S.close()


@pytest.mark.parametrize("name", ss.PROOF_SUBSET)
def test_prove_without_multiples_table(ctx, monkeypatch, name):
    """LASSO_B200_NO_MULTIPLES=1: the openings on the bucket MSM and per-step kernels, the same bytes"""
    monkeypatch.setenv("LASSO_B200_NO_MULTIPLES", "1")
    assert_matches_oracle(name, *gpu_proof(ctx, name))


def _run_sharded(nproc, args, timeout=1500):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, LASSO_SHARD_SAME_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sharded_check.py")] + [str(a) for a in args]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert "SHARDED_CHECK PASS" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.mark.parametrize("name", ss.PROOF_SUBSET)
def test_prove_sharded_two_ranks_one_gpu(name):
    """one proof over 2 ranks on GPU 0 (tools/sharded_check.py kind C log_m log_r lookups same) against the oracle"""
    _, kind, C_, log_m, log_r, n, same = PROOFS[name]
    _run_sharded(2, [kind, C_, log_m, log_r, n, int(same)])


# ---------------------------------------------------------------- rejections
ENTRIES = ["round", "bind_round", "materialize", "gather"]


def _entry_rc(ctx, entry, kind, C_, log_m, log_r):
    """the C ABI's return code for one built-in entry point, its buffers sized for the shape (so that an entry point
    that wrongly accepted it would compute, not read out of bounds)"""
    import lasso_b200 as lb

    L, C0 = lb.lib(), max(C_, 0)
    alpha = 2 * C0 if kind == ss.LT else C0
    n = 4
    if entry in ("round", "bind_round"):
        polys = [np.zeros((n, 4), dtype=np.uint64) for _ in range(alpha + 1)]
        out = np.zeros((C0 + 3, 4), dtype=np.uint64)
        if entry == "round":
            return L.lasso_sumcheck_round_arbitrary(ctx._h, kind, C_, log_m, log_r, lb.api._ptr_array(polys), C.c_size_t(n),
                                                    lb.api._p(out))
        r = ol.fr_array([5])[0]
        return L.lasso_sumcheck_bind_round_arbitrary(ctx._h, kind, C_, log_m, log_r, lb.api._ptr_array(polys),
                                                     C.c_size_t(n), lb.api._p(r), lb.api._p(out))
    if entry == "materialize":
        nsub = {ss.LT: 2, ss.RANGE_CHECK: 3}.get(kind, 1)
        tabs = [np.zeros((1 << log_m, 4), dtype=np.uint64) for _ in range(nsub)]
        return L.lasso_materialize_subtables(ctx._h, kind, C_, log_m, log_r, lb.api._ptr_array(tabs))
    nz = [np.zeros(n, dtype=np.uint64) for _ in range(max(C0, 1))]
    E = [np.zeros((n, 4), dtype=np.uint64) for _ in range(max(alpha, 1))]
    return L.lasso_gather_lookup_polys(ctx._h, kind, C_, log_m, log_r, lb.api._ptr_array(nz), C.c_size_t(n),
                                       lb.api._ptr_array(E))


def _prove_rc(ctx, kind, C_, log_m, log_r):
    """lasso_prove on a densified representation of the shape, with generators to match: (error code or 0, message,
    launches the call made)"""
    import lasso_b200 as lb

    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, np.zeros((4, C_), dtype=np.uint64), log_m)
    stream = np.ascontiguousarray(ol.generators(9002)[: gens_needed(kind, C_, log_m, 4)])
    alpha = ss.num_memories(kind, C_) if kind in ss.KINDS else C_
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, 4, alpha, log_m, stream=stream)
    before = ctx.launches
    try:
        lb.SparsePolynomialEvaluationProof.prove(ctx, lb.Strategy(kind, C_, log_m, log_r), dense, ol.fr_array([3, 4]),
                                                 gens, tape_seed=ol.fr_array([9])[0])
    except lb.LassoError as e:
        return e.code, str(e), ctx.launches - before
    return 0, "", ctx.launches - before


@pytest.mark.parametrize("case", ss.REJECTED, ids=[r[0] for r in ss.REJECTED])
def test_rejects_shape_past_boundary(ctx, monkeypatch, case):
    """LASSO_ERR_STRATEGY from round, bind-round, materialize, gather and prove, with no launch; the context still
    proves correctly afterwards"""
    import lasso_b200 as lb

    _, kind, C_, log_m, log_r = case
    for entry in ENTRIES:
        before = ctx.launches
        assert _entry_rc(ctx, entry, kind, C_, log_m, log_r) == ERR_STRATEGY, entry
        assert ctx.launches == before, entry
    if ss.C_MIN <= C_ <= ss.C_MAX:  # a shape lasso_densify takes: lasso_prove must refuse the strategy
        with monkeypatch.context() as m:
            m.setenv("LASSO_B200_NO_MULTIPLES", "1")  # no digit-multiples tables for generators that go unused
            code, _, launches = _prove_rc(ctx, kind, C_, log_m, log_r)
        assert code == ERR_STRATEGY and launches == 0
    else:  # C outside 1..16: lasso_densify refuses it already
        with pytest.raises(lb.LassoError) as e:
            lb.DensifiedRepresentation.from_lookup_indices(ctx, np.zeros((4, C_), dtype=np.uint64), log_m)
        assert e.value.code == ERR_STRATEGY
    assert_matches_oracle("lt_c2_m2_same", *gpu_proof(ctx, "lt_c2_m2_same"))


@pytest.mark.parametrize("case", ss.UNPROVABLE, ids=sid)
def test_rejects_lt_proof_above_circuit_batch(ctx, case):
    """LT with C > 8 (4C > 32 grand-product circuits): the round entry point takes it, lasso_prove refuses before any
    launch and names the limit, and the same context then proves a generic-kernel LT case bit-exactly"""
    assert _entry_rc(ctx, "round", *case) == 0
    code, msg, launches = _prove_rc(ctx, *case)
    assert (code, launches) == (ERR_STRATEGY, 0), msg
    assert "batch limit of 32" in msg
    assert_matches_oracle("lt_c5_m6", *gpu_proof(ctx, "lt_c5_m6"))
