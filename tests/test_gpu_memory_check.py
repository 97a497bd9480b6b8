"""Memory checking inside a caller's protocol on the GPU: Subtables (the lookup polynomials against a host gather, their
commitment against the proof's comm_derefs), the densified representation's polynomials, the lookup proof composed
step by step from public calls against lasso_prove_transcript (bytes and next challenge, at 2^10 and 2^14 lookups and
at the golden 2^20 / 2^24 configurations), the standalone MemoryCheckingProof against the oracle, GrandProducts.new
over a caller's memory against the oracle's fingerprints and host-uploaded circuits, the error table, launch counts,
and a sharded context's refusals.

Run as a script under torchrun it is the sharded worker (LASSO_SHARD_SAME_GPU=1: every rank on GPU 0)."""
import hashlib
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import custom_builtins as cb  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_lib as ol  # noqa: E402
import oracle_memory_check_lib as oml  # noqa: E402
import workloads as wl  # noqa: E402
from lasso_b200.api import (LASSO_ERR_GENS, LASSO_ERR_INDEX_RANGE, LASSO_ERR_LENGTH, LASSO_ERR_STRATEGY,  # noqa: E402
                            LASSO_ERR_VALUE)

pytestmark = pytest.mark.gpu

L_FR = ol.L_FR

# (name, kind, C, log_m, log_r)
BUILTINS = [("and", lb.AND, 4, 8, 0), ("or", lb.OR, 2, 16, 0), ("xor", lb.XOR, 4, 16, 0), ("lt", lb.LT, 4, 8, 0),
            ("range", lb.RANGE_CHECK, 4, 8, 28)]


@pytest.fixture(scope="module")
def ctx():
    c = lb.Context(0)
    yield c
    c.close()


def _custom_u32_g(v):
    return v[0] * v[1] + v[2] + v[3] * 5


def _custom_fr_g(v):
    return v[0] * v[1] + v[0] * 2


def custom_u32(ctx):
    """integer tables below 2^16, four memories over two dimensions"""
    rng = np.random.default_rng(11)
    tables = [rng.integers(0, 1 << 16, size=1 << 8, dtype=np.uint64) for _ in range(2)]
    return lb.CustomStrategy(ctx, 2, 8, tables, _custom_u32_g, 2), tables, _custom_u32_g


def custom_fr(ctx):
    """one table of uniform field elements (full width), two memories"""
    rng = np.random.default_rng(12)
    tables = [ol.rand_fr(rng, 1 << 6)]
    return lb.CustomStrategy(ctx, 2, 6, tables, _custom_fr_g, 2), tables, _custom_fr_g


CUSTOMS = {"custom_u32": custom_u32, "custom_fr": custom_fr}
ALL = [b[0] for b in BUILTINS] + list(CUSTOMS)


def strategy(ctx, name):
    """-> (S, C, log_m, tables as Montgomery limbs per subtable, memory -> subtable, memory -> dimension, g)"""
    if name in CUSTOMS:
        S, tables, g = CUSTOMS[name](ctx)
        tab = [t if t.ndim == 2 else ol.fr_array([int(x) for x in t]) for t in tables]
        return S, S.C, S.log_m, tab, list(S.memory_to_subtable), list(S.memory_to_dimension), g
    _, kind, C_, log_m, log_r = next(b for b in BUILTINS if b[0] == name)
    S = lb.Strategy(kind, C_, log_m, log_r)
    tab = [ol.fr_array([int(x) for x in t]) for t in cb.builtin_tables(kind, C_, log_m, log_r)]
    if kind == lb.LT:
        sub, dim = [i % 2 for i in range(2 * C_)], [i // 2 for i in range(2 * C_)]
    else:
        sub, dim = cb.builtin_maps(kind, C_, log_m, log_r)
        sub, dim = (sub or [0] * C_), (dim or list(range(C_)))
    g, _ = cb.builtin_g(kind, C_, log_m)
    return S, C_, log_m, tab, sub, dim, g


def setup(ctx, S, C_, log_m, n, seed):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    stream = ol.generators(lb.gens_points_needed(C_, dense.s, S.num_memories, log_m))
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, dense.s, S.num_memories, log_m, stream=stream)
    r = ol.rand_fr(rng, dense.s.bit_length() - 1)
    return idx, dense, stream, gens, r, ol.rand_fr(rng, 1)[0]


def _next(t):
    return t.challenge_scalar(b"next").tolist()


def _fr_bytes(a):
    return b"".join(int(x).to_bytes(32, "little") for x in ol.fr_ints(np.asarray(a).reshape(-1, 4)))


def _derefs_gens(ctx, alpha, s, stream):
    """the proof's gens_derefs (surge.rs:32-58): the view of num_vars log2(next_pow2(alpha s)) of the same stream"""
    return lb.PolyCommitmentGens.new(ctx, b"gens_derefs", (alpha * s - 1).bit_length(), stream=stream)


# ---------------------------------------------------------------- (a) Subtables
@pytest.mark.parametrize("name", ALL)
def test_lookup_polys_match_host_gather(ctx, name):
    S, C_, log_m, tab, sub, dim, _ = strategy(ctx, name)
    idx, dense, stream, gens, r, seed = setup(ctx, S, C_, log_m, 300, 1)
    nz = dense.dim_usize
    st = lb.Subtables(ctx, S, dense)
    assert len(st.lookup_polys) == S.num_memories
    for i, E in enumerate(st.lookup_polys):
        assert E.num_vars == dense.s.bit_length() - 1
        assert np.array_equal(E.to_numpy(), tab[sub[i]][nz[dim[i]].astype(np.int64)]), i
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=lb.Transcript(b"example"),
                                                     random_tape=lb.RandomTape(b"proof", seed)).bytes
    comm = st.commit(_derefs_gens(ctx, S.num_memories, dense.s, stream))
    assert proof[: len(comm)] == comm
    assert comm == st.combined_poly.commit(_derefs_gens(ctx, S.num_memories, dense.s, stream))


# ---------------------------------------------------------------- (b) the densified representation's polynomials
def test_dense_polys(ctx):
    C_, log_m = 3, 8
    dense = lb.DensifiedRepresentation.from_lookup_indices(
        ctx, np.random.default_rng(2).integers(0, 1 << log_m, size=(700, C_), dtype=np.uint64), log_m)
    dim, read, final = dense.dim, dense.read, dense.final
    one = np.ones(4, dtype=np.uint64)
    for j in range(C_):
        for p, want in ((dense.dim_poly(j), dim[j]), (dense.read_poly(j), read[j]), (dense.final_poly(j), final[j])):
            assert np.array_equal(p.to_numpy(), want)
            # integer-valued with the u32 mirror: accepted as the addresses of a memory of 2^12 cells
            lb.GrandProducts.new(ctx, _table(ctx, 1 << 12), p, p, _table(ctx, 1 << 12), (one, one))
    for bad in (0, 4):
        with pytest.raises(lb.LassoError) as e:
            dense._poly(bad, 0)
        assert e.value.code == LASSO_ERR_LENGTH
    with pytest.raises(lb.LassoError) as e:
        dense.dim_poly(C_)
    assert e.value.code == LASSO_ERR_LENGTH


def _table(ctx, M, seed=0):
    return lb.DensePolynomial(ctx, ol.rand_fr(np.random.default_rng(seed), M))


# ---------------------------------------------------------------- (c) the composed proof
def compose(ctx, S, g, dense, gens, stream, r, seed, label=b"example"):
    """surge.rs:129-199 step by step with public calls -> (proof bytes, next challenge)"""
    alpha = S.num_memories
    t, tape = lb.Transcript(label), lb.RandomTape(b"proof", seed)
    t.append_protocol_name(b"Lasso SparsePolynomialEvaluationProof")
    st = lb.Subtables(ctx, S, dense)
    pg = _derefs_gens(ctx, alpha, dense.s, stream)
    comm = st.commit(pg)
    t.append_combined_table_commitment(comm)
    claim = dense.outputs(S).evaluate(r)
    t.append_scalar(b"claim_eval_scalar_product", claim)
    comb = lb.Comb(lambda v: g(v[:alpha]) * v[alpha], alpha + 1, degree=S.sumcheck_poly_degree)
    sc = lb.SumcheckInstanceProof.prove_arbitrary(ctx, st.lookup_polys + [lb.DensePolynomial.eq(ctx, r)], comb, t)
    evals = lb.DensePolynomial.evaluate_batch(ctx, st.lookup_polys, sc.r)
    ce = lb.CombinedTableEvalProof.prove(ctx, st.combined_poly, evals, sc.r, pg, t, tape)
    gamma, tau = t.challenge_vector(b"challenge_r_hash", 2)
    mc = lb.MemoryCheckingProof.prove(ctx, S, dense, (gamma, tau), gens, t, tape)
    return comm + sc.bytes + _fr_bytes(claim) + _fr_bytes(evals) + ce.data + mc.bytes, _next(t)


@pytest.mark.parametrize("n", [1 << 10, 1 << 14])
@pytest.mark.parametrize("name", ["xor", "and", "range", "lt", "custom_u32", "custom_fr"])
def test_composed_proof_equals_lookup_proof(ctx, name, n):
    S, C_, log_m, _, _, _, g = strategy(ctx, name)
    if name in ("and", "range", "lt"):  # C = 4 built-ins
        assert C_ == 4
    idx, dense, stream, gens, r, seed = setup(ctx, S, C_, log_m, n, n + 3)
    t = lb.Transcript(b"example")
    want = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=t,
                                                    random_tape=lb.RandomTape(b"proof", seed)).bytes
    got, nxt = compose(ctx, S, g, dense, gens, stream, r, seed)
    assert got == want
    assert nxt == _next(t)


@pytest.mark.parametrize("name", ["xor_c4_s20", "rc40_c4_s24"])
def test_composed_proof_at_size(ctx, name):
    want = json.load(open(os.path.join(HERE, "golden", "big_proofs.json")))["cases"][name]["proof_sha256"]
    kind, C_, log_m, log_r, log_s, idx, r, seed = wl.config_inputs(name)
    S = lb.Strategy(kind, C_, log_m, log_r)
    stream = np.ascontiguousarray(ol.generators(wl.gens_needed(C_, log_s, S.num_memories, log_m)))
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, dense.s, S.num_memories, log_m, stream=stream)
    g, _ = cb.builtin_g(kind, C_, log_m)
    got, _ = compose(ctx, S, g, dense, gens, stream, r, seed)
    assert hashlib.sha256(got).hexdigest() == want


# ---------------------------------------------------------------- (d) the standalone memory check against the oracle
@pytest.mark.parametrize("kind,C_,log_m,n", [(lb.XOR, 2, 8, 200), (lb.LT, 2, 8, 130), (lb.AND, 3, 6, 64)])
def test_standalone_memory_check_matches_oracle(ctx, kind, C_, log_m, n):
    S = lb.Strategy(kind, C_, log_m)
    idx, dense, stream, gens, _, seed = setup(ctx, S, C_, log_m, n, 5)
    gamma, tau = ol.rand_fr(np.random.default_rng(n), 2)
    t = lb.Transcript(b"memory check")
    t.append_protocol_name(b"caller")
    mc = lb.MemoryCheckingProof.prove(ctx, S, dense, (gamma, tau), gens, t, lb.RandomTape(b"proof", seed))
    T = od.Transcript(b"memory check")
    T.append_protocol_name(b"caller")
    want, comm, derefs = oml.prove(kind, C_, log_m, 0, idx, gamma, tau, stream, T, od.RandomTape(b"proof", seed))
    assert mc.bytes == want
    assert _next(t) == T.challenge_scalar(b"next").tolist()
    assert comm == dense.commit(gens)
    V = od.Transcript(b"memory check")
    V.append_protocol_name(b"caller")
    assert oml.verify(kind, C_, log_m, 0, stream, comm, derefs, mc.bytes, gamma, tau, V) == 0


def test_memory_check_custom_equals_builtin(ctx):
    """a built-in strategy restated as a custom one proves the same memory check"""
    S = lb.Strategy(lb.LT, 2, 8)
    Sc = cb.as_custom(ctx, lb.LT, 2, 8)
    idx, dense, stream, gens, _, seed = setup(ctx, S, 2, 8, 500, 6)
    gamma, tau = ol.rand_fr(np.random.default_rng(6), 2)
    a = lb.MemoryCheckingProof.prove(ctx, S, dense, (gamma, tau), gens, lb.Transcript(b"x"), lb.RandomTape(b"p", seed))
    b = lb.MemoryCheckingProof.prove(ctx, Sc, dense, (gamma, tau), gens, lb.Transcript(b"x"), lb.RandomTape(b"p", seed))
    assert a.bytes == b.bytes


# ---------------------------------------------------------------- (e) GrandProducts.new over a caller's memory
def _host_fingerprints(T, dim, read, final, gamma, tau):
    """(init, read, write, final) in Python integers from Montgomery limbs"""
    g, t = ol.fr_ints(gamma.reshape(1, 4))[0], ol.fr_ints(tau.reshape(1, 4))[0]
    Tv, dv, rv, fv = (ol.fr_ints(x) for x in (T, dim, read, final))
    h = lambda a, v, ts: (ts * g * g + v * g + a - t) % L_FR  # noqa: E731
    init = [h(i, Tv[i], 0) for i in range(len(Tv))]
    fin = [h(i, Tv[i], fv[i]) for i in range(len(Tv))]
    rd = [h(a, Tv[a], ts) for a, ts in zip(dv, rv)]
    wr = [h(a, Tv[a], ts + 1) for a, ts in zip(dv, rv)]
    return [ol.fr_array(x) for x in (init, rd, wr, fin)]


def _oracle_fingerprints(T, dim_usize, read_ts, final_ts, gamma, tau):
    M, s = T.shape[0], dim_usize.shape[0]
    out = np.zeros((2 * M + 2 * s, 4), dtype=np.uint64)
    u = lambda a: np.ascontiguousarray(a, dtype=np.uint64)  # noqa: E731
    ol.lib().orc_gp_fingerprints(ol.P(u(T)), ol.sz(M), ol.P(u(dim_usize)), ol.P(u(read_ts)), ol.P(u(final_ts)),
                                 ol.sz(s), ol.P(u(gamma)), ol.P(u(tau)), ol.P(out))
    return out[:M], out[2 * M:2 * M + s], out[2 * M + s:], out[M:2 * M]


def _product(limbs):
    acc = 1
    for x in ol.fr_ints(limbs):
        acc = acc * x % L_FR
    return acc


@pytest.mark.parametrize("table", ["u16", "full", "eq"])
def test_fingerprints_of_a_densified_memory(ctx, table):
    """counters from a C = 1 densify: the oracle's fingerprints, and init * write = read * final"""
    log_m, n = 10, 3000
    rng = np.random.default_rng(7)
    M = 1 << log_m
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, rng.integers(0, M, size=(n, 1), dtype=np.uint64), log_m)
    if table == "u16":
        T = ol.fr_array([int(x) for x in rng.integers(0, 1 << 16, size=M)])
        Tp = lb.DensePolynomial(ctx, T)
    elif table == "full":
        T = ol.rand_fr(rng, M)
        Tp = lb.DensePolynomial(ctx, T)
    else:  # Spark: the memory is eq(r_x)
        Tp = lb.DensePolynomial.eq(ctx, ol.rand_fr(rng, log_m))
        T = Tp.to_numpy()
    gamma, tau = ol.rand_fr(rng, 2)
    gp = lb.GrandProducts.new(ctx, Tp, dense.dim_poly(0), dense.read_poly(0), dense.final_poly(0), (gamma, tau))
    want = _oracle_fingerprints(T, dense.dim_usize[0], ol.fr_ints(dense.read[0]), ol.fr_ints(dense.final[0]), gamma, tau)
    for got, w, name in zip(gp.polys, want, lb.GrandProducts.FIELDS):
        assert np.array_equal(got.to_numpy(), w), name
    hi, hr, hw, hf = (ol.fr_ints(getattr(gp, f).evaluate().reshape(1, 4))[0] for f in lb.GrandProducts.FIELDS)
    assert hi * hw % L_FR == hr * hf % L_FR
    assert hi == _product(want[0]) and hw == _product(want[2])


def test_fingerprints_of_arbitrary_field_counters(ctx):
    """read and final_ts may be any field elements (no mirror); dim any integers below M"""
    rng = np.random.default_rng(8)
    M, s = 1 << 6, 1 << 9
    T, rd, fn = ol.rand_fr(rng, M), ol.rand_fr(rng, s), ol.rand_fr(rng, M)
    dim = ol.fr_array([int(x) for x in rng.integers(0, M, size=s)])
    gamma, tau = ol.rand_fr(rng, 2)
    gp = lb.GrandProducts.new(ctx, lb.DensePolynomial(ctx, T), lb.DensePolynomial(ctx, dim), lb.DensePolynomial(ctx, rd),
                              lb.DensePolynomial(ctx, fn), (gamma, tau))
    for got, w in zip(gp.polys, _host_fingerprints(T, dim, rd, fn, gamma, tau)):
        assert np.array_equal(got.to_numpy(), w)


def _batched_bytes(ctx, gp_pairs):
    t = lb.Transcript(b"gp")
    out = [lb.BatchedGrandProductArgument.prove(ctx, pair, t).bytes for pair in gp_pairs]
    return out, _next(t)


@pytest.mark.parametrize("log_M,log_s", [(6, 10), (16, 20), (20, 20)])
def test_grand_products_equal_host_uploaded_circuits(ctx, log_M, log_s):
    rng = np.random.default_rng(log_M + log_s)
    M, s = 1 << log_M, 1 << log_s
    T = ol.rand_fr(rng, M)
    dim_u = rng.integers(0, M, size=s, dtype=np.uint64)
    read_u = rng.integers(0, 1 << 20, size=s, dtype=np.uint64)
    fin_u = rng.integers(0, 1 << 20, size=M, dtype=np.uint64)
    dim, read, fin = (lb.DensePolynomial(ctx, _u64_to_fr(x)) for x in (dim_u, read_u, fin_u))
    gamma, tau = ol.rand_fr(rng, 2)
    gp = lb.GrandProducts.new(ctx, lb.DensePolynomial(ctx, T), dim, read, fin, (gamma, tau))
    host = _oracle_fingerprints(T, dim_u, read_u, fin_u, gamma, tau)
    polys = [lb.DensePolynomial(ctx, h) for h in host]
    hc = [lb.GrandProductCircuit(ctx, p) for p in polys]
    got = _batched_bytes(ctx, [(gp.read, gp.write), (gp.init, gp.final)])
    want = _batched_bytes(ctx, [(hc[1], hc[2]), (hc[0], hc[3])])
    assert got == want


def _u64_to_fr(x):
    """integers as Montgomery limbs (the oracle's batch conversion)"""
    out = np.zeros((x.shape[0], 4), dtype=np.uint64)
    ol.lib().orc_fr_from_u64_batch(ol.P(np.ascontiguousarray(x, dtype=np.uint64)), ol.sz(x.shape[0]), ol.P(out))
    return out


# ---------------------------------------------------------------- (f) errors, (g) launch counts
def _raises(ctx, code, fn, *moved):
    """fn raises LassoError(code) with no launch, and leaves each (transcript, tape) pair as its twin"""
    l0 = ctx.launches
    with pytest.raises(lb.LassoError) as e:
        fn()
    assert e.value.code == code, (e.value.code, str(e.value))
    assert ctx.launches == l0
    for (t, twin) in moved:
        assert _next(t) == _next(twin)


def test_errors_before_anything_moves(ctx):
    S = lb.Strategy(lb.XOR, 4, 8)
    idx, dense, stream, gens, r, seed = setup(ctx, S, 4, 8, 256, 9)
    other = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", 4, dense.s * 2, 4, 8,
                                            stream=ol.generators(lb.gens_points_needed(4, dense.s * 2, 4, 8)))
    g = np.ones(4, dtype=np.uint64)
    bad = ol.int_to_limbs(L_FR)
    S_shape = custom_u32(ctx)[0]  # C = 2, log_m = 8: not the dense's C = 4
    L = lb.lib()

    def raw(t, tape, cap):
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        n = lb.api.C.c_size_t(0)
        rc = L.lasso_memory_check_prove(ctx._h, S.kind, S.log_r, dense._h, lb.api._p(g), lb.api._p(g), gens._h,
                                        t._h if t else None, tape._h if tape else None, lb.api._p(out),
                                        lb.api.C.c_size_t(cap), lb.api.C.byref(n))
        return rc, n.value

    def mc(S_=S, gamma=g, tau=g, gens_=gens, cap=None, t=None, tape=None):
        if cap is None:
            return lb.MemoryCheckingProof.prove(ctx, S_, dense, (gamma, tau), gens_, t, tape)
        rc, _ = raw(t, tape, cap)
        if rc:
            raise lb.LassoError(rc, "memory check")

    need = len(mc(t=lb.Transcript(b"x"), tape=lb.RandomTape(b"p", seed)).bytes)
    cases = [
        (LASSO_ERR_STRATEGY, dict(S_=lb.Strategy(9, 4, 8))),
        (LASSO_ERR_STRATEGY, dict(S_=S_shape)),
        (LASSO_ERR_GENS, dict(gens_=other)),
        (LASSO_ERR_VALUE, dict(gamma=bad)),
        (LASSO_ERR_VALUE, dict(tau=bad)),
        (LASSO_ERR_LENGTH, dict(cap=need - 1)),
    ]
    for code, kw in cases:
        t, twin = lb.Transcript(b"x"), lb.Transcript(b"x")
        tape, tape_twin = lb.RandomTape(b"p", seed), lb.RandomTape(b"p", seed)
        _raises(ctx, code, lambda: mc(t=t, tape=tape, **kw), (t, twin))
        assert tape.random_scalar(b"z").tolist() == tape_twin.random_scalar(b"z").tolist()
    # *proof_len reports the size needed with a short buffer; a null transcript or tape is refused
    assert raw(lb.Transcript(b"x"), lb.RandomTape(b"p", seed), need - 1) == (LASSO_ERR_LENGTH, need)
    assert raw(None, lb.RandomTape(b"p", seed), need)[0] == LASSO_ERR_LENGTH
    assert raw(lb.Transcript(b"x"), None, need)[0] == LASSO_ERR_LENGTH
    # Subtables: n_out != alpha
    hs = (lb.api.C.c_void_p * 8)()
    l0 = ctx.launches
    for n_out in (3, 5, 0):
        assert L.lasso_lookup_polys(ctx._h, S.kind, S.log_r, dense._h, hs, lb.api.C.c_size_t(n_out)) == LASSO_ERR_LENGTH
    assert ctx.launches == l0
    _raises(ctx, LASSO_ERR_STRATEGY, lambda: lb.Subtables(ctx, S_shape, dense))
    # fingerprints: lengths, dim out of range, non-canonical gamma / tau
    T, T2 = _table(ctx, 64), _table(ctx, 32)
    dim = lb.DensePolynomial(ctx, ol.fr_array([5] * 128))
    dim_hi = lb.DensePolynomial(ctx, ol.fr_array([63] * 127 + [64]))
    dim_wide = lb.DensePolynomial(ctx, ol.rand_fr(np.random.default_rng(1), 128))
    rd, rd2 = _table(ctx, 128, 1), _table(ctx, 64, 1)
    one = lb.DensePolynomial(ctx, ol.fr_array([1]))
    gt = (g, g)
    F = lb.GrandProducts.new
    _raises(ctx, LASSO_ERR_LENGTH, lambda: F(ctx, T, dim, rd, T2, gt))
    _raises(ctx, LASSO_ERR_LENGTH, lambda: F(ctx, T, dim, rd2, T, gt))
    _raises(ctx, LASSO_ERR_LENGTH, lambda: F(ctx, one, dim, rd, one, gt))
    _raises(ctx, LASSO_ERR_LENGTH, lambda: F(ctx, T, one, one, T, gt))
    _raises(ctx, LASSO_ERR_INDEX_RANGE, lambda: F(ctx, T, dim_hi, rd, T, gt))
    _raises(ctx, LASSO_ERR_INDEX_RANGE, lambda: F(ctx, T, dim_wide, rd, T, gt))
    _raises(ctx, LASSO_ERR_VALUE, lambda: F(ctx, T, dim, rd, T, (bad, g)))
    _raises(ctx, LASSO_ERR_VALUE, lambda: F(ctx, T, dim, rd, T, (g, bad)))
    ctx2 = lb.Context(0)
    T_other = _table(ctx2, 64)
    _raises(ctx, LASSO_ERR_STRATEGY, lambda: F(ctx, T_other, dim, rd, T, gt))
    del T_other
    ctx2.close()


def test_launch_counts(ctx):
    """Subtables: materialise + gather (a custom strategy's tables are uploaded: the gather only); dim_poly: the ingest
    pass, the read-back of its verdict and the u32 mirror; GrandProducts.new: two launches for the four fingerprints (plus the circuits' own)"""
    S = lb.Strategy(lb.XOR, 4, 8)
    idx, dense, stream, gens, r, seed = setup(ctx, S, 4, 8, 1 << 10, 10)
    l0 = ctx.launches
    lb.Subtables(ctx, S, dense)
    assert ctx.launches - l0 == 2
    Sc = custom_u32(ctx)[0]
    _, dc, _, _, _, _ = setup(ctx, Sc, 2, 8, 1 << 10, 10)
    l0 = ctx.launches
    lb.Subtables(ctx, Sc, dc)
    assert ctx.launches - l0 == 1
    l0 = ctx.launches
    d0 = dense.dim_poly(0)
    assert ctx.launches - l0 == 3
    rd, fn, T = dense.read_poly(0), dense.final_poly(0), _table(ctx, 1 << 8)
    g = np.ones(4, dtype=np.uint64)
    hs = (lb.api.C.c_void_p * 4)()
    l0 = ctx.launches
    assert lb.lib().lasso_memory_fingerprints(ctx._h, T._h, d0._h, rd._h, fn._h, lb.api._p(g), lb.api._p(g), hs) == 0
    assert ctx.launches - l0 == 2
    for h in hs:
        lb.DensePolynomial._wrap(ctx, lb.api.C.c_void_p(h))  # freed with the wrapper


# ---------------------------------------------------------------- sharded
def test_sharded_two_ranks_one_gpu(ctx):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, LASSO_SHARD_SAME_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env)
    assert "MEMORY_CHECK_SHARDED PASS" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


def _sharded_worker():
    """every new call returns LASSO_ERR_STRATEGY on a sharded context, on every rank"""
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(0)
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    C_, log_m, n = 2, 8, 1 << 10
    idx = np.random.default_rng(9).integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    S = lb.Strategy(lb.XOR, C_, log_m)
    c = lb.Context(0)
    c.init_comm()
    d = lb.DensifiedRepresentation.from_lookup_indices(c, idx, log_m)
    stream = ol.generators(lb.gens_points_needed(C_, n, 2, log_m))
    g = lb.SparsePolyCommitmentGens.new(c, b"gens_sparse_poly", C_, n, 2, log_m, stream=stream)
    P = lb.DensePolynomial(c, ol.fr_array(range(64)))
    one = np.ones(4, dtype=np.uint64)
    calls = [
        lambda: lb.Subtables(c, S, d),
        lambda: d.dim_poly(0),
        lambda: lb.MemoryCheckingProof.prove(c, S, d, (one, one), g, lb.Transcript(b"x"), lb.RandomTape(b"p", one)),
        lambda: lb.GrandProducts.new(c, P, P, P, P, (one, one)),
    ]
    codes = []
    for f in calls:
        try:
            f()
            codes.append(0)
        except lb.LassoError as e:
            codes.append(e.code)
    got = [None, None]
    dist.all_gather_object(got, codes)
    if rank == 0:
        ok = all(x == [LASSO_ERR_STRATEGY] * len(calls) for x in got)
        print("MEMORY_CHECK_SHARDED", "PASS" if ok else "FAIL %r" % (got,), flush=True)
    dist.barrier()
    del d, g, P
    c.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    _sharded_worker()
