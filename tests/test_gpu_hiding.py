"""Hiding commitments and openings of a caller's dense polynomials on the GPU: DensePolynomial.commit_hiding and
PolyEvalProof.prove with blinds / blind_Zr, bit for bit against the CPU oracle (oracle_dense/).  Covers the row
launchers every commitment form takes (u32 with the 16-bit tables, full width, <= 8 rows through the bucket MSM, the
all-zero polynomial), eq / merge / from_comb polynomials, generators without the multiples tables, the three blind
combinations of the opening, launch counts, a composed Lasso protocol on one transcript, every error of the two C
entry points, the blind-term kernel one launch at a time (tests/kernel_harness/harness_hiding.cu), and the sizes of
tests/golden/dense_poly_hiding.json."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import dense_poly_cases as dc
import kernel_harness_lib as kh
import oracle_combined_eval_lib as oce
import oracle_dense_lib as od
import oracle_hiding_lib as oh
import oracle_lib as ol
from test_gpu_dense_poly import _values
from test_gpu_launchers import mont, ptr
from test_gpu_msm_rows import Ref

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ERR_LENGTH, ERR_STRATEGY, ERR_GENS, ERR_VALUE = 1, 4, 5, 8
L_FR = ol.L_FR


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


_gens_cache = {}


def _gens(ctx, nv, no_multiples=False, monkeypatch=None):
    import lasso_b200 as lb

    key = (id(ctx), nv, no_multiples)
    if key not in _gens_cache:
        stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
        if no_multiples:
            monkeypatch.setenv("LASSO_B200_NO_MULTIPLES", "1")
        g = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream)
        if no_multiples:
            monkeypatch.delenv("LASSO_B200_NO_MULTIPLES")
        _gens_cache[key] = (g, stream)
    return _gens_cache[key]


def _seed(x):
    return ol.fr_array([x])[0]


def _commit_both(ctx, p, Z, gens, stream, seed):
    """commit_hiding on the GPU and the oracle on twin tapes; asserts bytes, blinds and the tapes' next draw"""
    import lasso_b200 as lb

    tape, otape = lb.RandomTape(b"commit", _seed(seed)), od.RandomTape(b"commit", _seed(seed))
    comm, blinds = p.commit_hiding(gens, tape)
    want, wblinds = oh.commit_hiding(Z, stream, tape=otape)
    assert blinds.shape == (1 << (p.num_vars // 2), 4)
    assert np.array_equal(blinds, wblinds)
    assert comm == want
    assert np.array_equal(tape.random_scalar(b"next"), otape.random_scalar(b"next"))
    return comm, blinds


@pytest.mark.parametrize("nv", [1, 2, 5, 7, 8, 9, 12, 16])
@pytest.mark.parametrize("kind", ["u32", "full", "zero"])
def test_commit_hiding_bytes(ctx, kind, nv):
    import lasso_b200 as lb

    Z = _values(kind, nv, 17 * nv + len(kind))
    gens, stream = _gens(ctx, nv)
    p = lb.DensePolynomial(ctx, Z)
    l0 = ctx.launches
    plain = p.commit(gens)
    l1 = ctx.launches
    comm, blinds = _commit_both(ctx, p, Z, gens, stream, nv)
    assert ctx.launches - l1 == (l1 - l0) + 1  # the blind term: one launch more than the plain commitment
    assert len(comm) == len(plain) and comm != plain
    if kind == "zero":  # rows are blind_i * h alone
        h = np.ascontiguousarray(stream[[dc.n_generators(nv) - 1]])
        hh = np.ascontiguousarray(np.concatenate([h, h, h]))  # one generator, Q and h: b G_0 = b h
        assert comm[8:] == b"".join(od.commit(np.ascontiguousarray(b[None]), hh)[8:] for b in blinds)


def test_commit_hiding_eq_merge_comb(ctx):
    import lasso_b200 as lb

    rng = np.random.default_rng(3)
    nv = 9
    gens, stream = _gens(ctx, nv)
    r = dc.random_full(rng, nv)
    eq = np.zeros((1 << nv, 4), dtype=np.uint64)
    ol.lib().orc_eq_evals(ol.P(np.ascontiguousarray(r)), ol.sz(nv), ol.P(eq))
    _commit_both(ctx, lb.DensePolynomial.eq(ctx, r), eq, gens, stream, 1)
    A, B = _values("u32", 8, 5), _values("full", 8, 6)
    merged = lb.DensePolynomial.merge(ctx, [lb.DensePolynomial(ctx, A), lb.DensePolynomial(ctx, B)])
    _commit_both(ctx, merged, oce.merge([A, B]), gens, stream, 2)
    X, Y = _values("full", nv, 7), _values("u8", nv, 8)
    comb = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda x: x[0] * x[1] + x[0], 2),
                                        [lb.DensePolynomial(ctx, X), lb.DensePolynomial(ctx, Y)])
    Q = ol.fr_array([(a * b + a) % L_FR for a, b in zip(ol.fr_ints(X), ol.fr_ints(Y))])
    _commit_both(ctx, comb, Q, gens, stream, 3)


def _prove_both(ctx, p, Z, nv, gens, stream, seed, blinds, blind_Zr):
    """the opening on the GPU and the oracle on twin transcripts and tapes -> (proof, C_Zr); asserts bytes and the
    next challenge"""
    import lasso_b200 as lb

    rng = np.random.default_rng(seed)
    r = dc.random_full(rng, nv)
    Zr = p.evaluate(r)
    t, tape = lb.Transcript(b"hiding"), lb.RandomTape(b"proof", _seed(seed))
    o, otape = od.Transcript(b"hiding"), od.RandomTape(b"proof", _seed(seed))
    proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, tape, blinds=blinds, blind_Zr=blind_Zr)
    want, czr = oh.prove_hiding(Z, r, Zr, stream, o, otape, blinds=blinds, blind_Zr=blind_Zr)
    assert proof.bytes == want and proof.C_Zr == czr
    assert np.array_equal(t.challenge_scalar(b"after"), o.challenge_scalar(b"after"))
    return proof, r


def _opening_cases(ctx, gens, stream, cases):
    import lasso_b200 as lb

    for nv, kind in cases:
        Z = _values(kind, nv, 3 * nv + 1)
        p = lb.DensePolynomial(ctx, Z)
        comm, blinds = p.commit_hiding(gens[nv], lb.RandomTape(b"commit", _seed(nv)))
        assert comm == oh.commit_hiding(Z, stream[nv], blinds=blinds)[0]
        bz = dc.random_full(np.random.default_rng(nv), 1)[0]
        for which, (bl, b_zr) in {"both": (blinds, bz), "blinds": (blinds, None), "blind_Zr": (None, bz)}.items():
            proof, r = _prove_both(ctx, p, Z, nv, gens[nv], stream[nv], 50 + nv, bl, b_zr)
            if bl is not None:  # the oracle's verifier against the hiding commitment and C_Zr
                v = od.Transcript(b"hiding")
                assert oh.verify(stream[nv], nv, comm, proof.bytes, r, proof.C_Zr, v) == 0, (nv, kind, which)


OPEN_CASES = [(1, "u32"), (2, "full"), (5, "u32"), (8, "full"), (11, "u32"), (16, "full")]


def test_eval_prove_hiding(ctx):
    gens = {nv: _gens(ctx, nv)[0] for nv, _ in OPEN_CASES}
    stream = {nv: _gens(ctx, nv)[1] for nv, _ in OPEN_CASES}
    _opening_cases(ctx, gens, stream, OPEN_CASES)


def test_no_multiples_tables(ctx, monkeypatch):
    """generators without the digit-multiples tables: the multiples of h are built for the call, the opening takes the
    bucket path; the bytes are the same"""
    import lasso_b200 as lb

    cases = [(2, "u32"), (7, "full"), (8, "u32"), (11, "full"), (12, "zero")]
    gens = {nv: _gens(ctx, nv, True, monkeypatch)[0] for nv, _ in cases}
    stream = {nv: _gens(ctx, nv, True, monkeypatch)[1] for nv, _ in cases}
    for nv, kind in cases:
        Z = _values(kind, nv, 11 * nv)
        with_tables, _ = _gens(ctx, nv)
        p = lb.DensePolynomial(ctx, Z)
        l0 = ctx.launches
        p.commit(gens[nv])
        l1 = ctx.launches
        a = p.commit_hiding(gens[nv], lb.RandomTape(b"commit", _seed(nv)))
        assert ctx.launches - l1 == (l1 - l0) + 2  # the multiples of h, then the blind term
        b = p.commit_hiding(with_tables, lb.RandomTape(b"commit", _seed(nv)))
        assert a[0] == b[0] and np.array_equal(a[1], b[1])
        _commit_both(ctx, p, Z, gens[nv], stream[nv], nv)
    _opening_cases(ctx, gens, stream, [(2, "u32"), (7, "full"), (11, "full")])


def test_no_blinds_is_the_plain_proof(ctx):
    """lasso_poly_eval_prove_hiding with neither blinds nor blind_Zr: lasso_poly_eval_prove's bytes and launches; plain
    calls launch the same before and after hiding calls on the same generators"""
    import lasso_b200 as lb

    L = lb.lib()
    for nv, kind in [(1, "full"), (6, "u32"), (13, "full")]:
        gens, _ = _gens(ctx, nv)
        Z = _values(kind, nv, nv)
        p = lb.DensePolynomial(ctx, Z)
        r = dc.random_full(np.random.default_rng(nv), nv)
        Zr = p.evaluate(r)

        def plain():
            l0 = ctx.launches
            c = p.commit(gens)
            l1 = ctx.launches
            pr = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, lb.Transcript(b"t"), lb.RandomTape(b"proof", _seed(1)))
            return c, pr.bytes, pr.C_Zr, l1 - l0, ctx.launches - l1

        before = plain()
        out = np.zeros(1 << 12, dtype=np.uint8)
        czr = np.zeros(32, dtype=np.uint8)
        n = ctypes.c_size_t(0)
        l0 = ctx.launches
        assert L.lasso_poly_eval_prove_hiding(ctx._h, p._h, gens._h, None, ctypes.c_size_t(0), lb.api._p(r),
                                              ctypes.c_size_t(nv), lb.api._p(Zr), None, lb.Transcript(b"t")._h,
                                              lb.RandomTape(b"proof", _seed(1))._h, lb.api._p(out),
                                              ctypes.c_size_t(out.shape[0]), ctypes.byref(n), lb.api._p(czr)) == 0
        assert (bytes(out[: n.value]), czr.tobytes(), ctx.launches - l0) == (before[1], before[2], before[4])
        zero = np.zeros(4, dtype=np.uint64)
        pz = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, lb.Transcript(b"t"), lb.RandomTape(b"proof", _seed(1)),
                                    blinds=np.zeros((1 << (nv // 2), 4), dtype=np.uint64), blind_Zr=zero)
        assert (pz.bytes, pz.C_Zr) == (before[1], before[2])  # zero blinds: the same bytes
        comm, blinds = p.commit_hiding(gens, lb.RandomTape(b"c", _seed(2)))
        lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, lb.Transcript(b"t"), lb.RandomTape(b"proof", _seed(1)),
                               blinds=blinds)
        assert plain() == before


def test_composed_protocol_hiding_outputs(ctx):
    """commit the lookup outputs v with hiding, absorb it and the sparse commitment, draw r, prove the Lasso proof and
    open v at r with its blinds on one transcript and tape: the oracle's replay gives the same bytes and accepts"""
    import lasso_b200 as lb
    import compose_cases as cc
    import oracle_compose_lib as ocl
    from test_gpu_compose import setup

    C_, log_m = 4, 16
    S = lb.Strategy(lb.XOR, C_, log_m)
    idx, dense, stream, gens, _, seed = setup(ctx, S, C_, log_m, 1 << 10, 2)
    log_s = dense.s.bit_length() - 1
    v_stream = ol.generators(lb.poly_gens_points_needed(log_s), b"gens_outputs")
    v_gens = lb.PolyCommitmentGens.new(ctx, b"gens_outputs", log_s, stream=v_stream)
    T, tape = lb.Transcript(b"compose"), lb.RandomTape(b"proof", seed)
    v = dense.outputs(S)
    comm_v, blinds = v.commit_hiding(v_gens, tape)
    T.append_poly_commitment(b"outputs", comm_v)
    comm_sparse = dense.commit(gens)
    T.append_sparse_commitment(comm_sparse)
    r = T.challenge_vector(b"r", log_s)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=T, random_tape=tape)
    blind_Zr = tape.random_scalar(b"blind_Zr")
    opening = lb.PolyEvalProof.prove(ctx, v, r, proof.claimed_evaluation, v_gens, T, tape, blinds=blinds,
                                     blind_Zr=blind_Zr)
    last = T.challenge_scalar(b"next")

    vals = cc.outputs(lb.XOR, C_, log_m, 0, cc.dim_usize(idx, dense.s))
    O, otape = od.Transcript(b"compose"), od.RandomTape(b"proof", seed)
    o_comm, o_blinds = oh.commit_hiding(vals, v_stream, tape=otape)
    assert o_comm == comm_v and np.array_equal(o_blinds, blinds)
    O.append_poly_commitment(b"outputs", o_comm)
    assert ocl.append_sparse_commitment(O, comm_sparse) == 0
    assert O.challenge_vector(b"r", log_s).tolist() == r.tolist()
    o_proof, _, claim = ocl.sparse_prove(lb.XOR, C_, log_m, 0, idx, r, stream, O, otape)
    assert o_proof == proof.bytes
    o_open, czr = oh.prove_hiding(vals, r, claim, v_stream, O, otape, blinds=blinds,
                                  blind_Zr=otape.random_scalar(b"blind_Zr"))
    assert o_open == opening.bytes and czr == opening.C_Zr
    assert O.challenge_scalar(b"next").tolist() == last.tolist()
    V = od.Transcript(b"compose")
    V.append_poly_commitment(b"outputs", comm_v)
    assert ocl.append_sparse_commitment(V, comm_sparse) == 0
    rv = V.challenge_vector(b"r", log_s)
    assert ocl.sparse_verify(lb.XOR, C_, log_m, 0, stream, comm_sparse, proof.bytes, rv, V) == 0
    assert oh.verify(v_stream, log_s, comm_v, opening.bytes, rv, opening.C_Zr, V) == 0


def test_errors(ctx):
    """every error of the two entry points, each before any launch and before the tape or the transcript moves"""
    import lasso_b200 as lb

    L = lb.lib()
    c_sz = ctypes.c_size_t
    nv = 6
    gens, _ = _gens(ctx, nv)
    other, _ = _gens(ctx, 8)  # R = 16 != 8
    Z = _values("u32", nv, 5)
    p = lb.DensePolynomial(ctx, Z)
    nrows = 1 << (nv // 2)
    r = dc.random_full(np.random.default_rng(1), nv)
    Zr = p.evaluate(r)
    bad_fr = ol.int_to_limbs(L_FR)
    blinds = dc.random_full(np.random.default_rng(2), nrows)
    bad_blinds = blinds.copy()
    bad_blinds[-1] = bad_fr
    bz = dc.random_full(np.random.default_rng(3), 1)[0]
    buf = np.zeros(1 << 16, dtype=np.uint8)
    bl_out = np.zeros((nrows, 4), dtype=np.uint64)
    czr = np.zeros(32, dtype=np.uint8)
    n = c_sz(0)
    t, tape = lb.Transcript(b"e"), lb.RandomTape(b"proof", _seed(1))

    def commit_rc(g=gens, tp=tape, cap=buf.shape[0], bcap=nrows, bo=bl_out):
        return L.lasso_poly_commit_hiding(ctx._h, p._h, g._h, None if tp is None else tp._h, lb.api._p(buf), c_sz(cap),
                                          ctypes.byref(n), None if bo is None else lb.api._p(bo), c_sz(bcap))

    def prove_rc(g=gens, bl=blinds, nb=nrows, rr=r, r_len=nv, zr=Zr, b_zr=bz, tr=t, tp=tape, cap=buf.shape[0]):
        return L.lasso_poly_eval_prove_hiding(
            ctx._h, p._h, g._h, None if bl is None else lb.api._p(bl), c_sz(nb), lb.api._p(rr), c_sz(r_len),
            lb.api._p(zr), None if b_zr is None else lb.api._p(b_zr), None if tr is None else tr._h,
            None if tp is None else tp._h, lb.api._p(buf), c_sz(cap), ctypes.byref(n), lb.api._p(czr))

    cases = [
        ("commit cap", ERR_LENGTH, lambda: commit_rc(cap=8 + 32 * nrows - 1)),
        ("commit blinds_cap", ERR_LENGTH, lambda: commit_rc(bcap=nrows - 1)),
        ("commit null blinds_out", ERR_LENGTH, lambda: commit_rc(bo=None)),
        ("commit null tape", ERR_LENGTH, lambda: commit_rc(tp=None)),
        ("commit other R", ERR_GENS, lambda: commit_rc(g=other)),
        ("prove cap", ERR_LENGTH, lambda: prove_rc(cap=8)),
        ("prove null transcript", ERR_LENGTH, lambda: prove_rc(tr=None)),
        ("prove null tape", ERR_LENGTH, lambda: prove_rc(tp=None)),
        ("prove n_blinds L-1", ERR_LENGTH, lambda: prove_rc(nb=nrows - 1)),
        ("prove n_blinds L+1", ERR_LENGTH, lambda: prove_rc(nb=nrows + 1)),
        ("prove r_len", ERR_LENGTH, lambda: prove_rc(r_len=nv - 1)),
        ("prove non-canonical blind", ERR_VALUE, lambda: prove_rc(bl=bad_blinds)),
        ("prove non-canonical blind_Zr", ERR_VALUE, lambda: prove_rc(b_zr=bad_fr)),
        ("prove non-canonical Zr", ERR_VALUE, lambda: prove_rc(zr=bad_fr)),
        ("prove non-canonical r", ERR_VALUE, lambda: prove_rc(rr=np.concatenate([r[:-1], bad_fr[None]]))),
        ("prove other R", ERR_GENS, lambda: prove_rc(g=other)),
    ]
    for name, code, f in cases:
        before = ctx.launches
        assert f() == code, (name, L.lasso_last_error())
        assert ctx.launches == before, name
    # the needed sizes were reported
    commit_rc(cap=8)
    assert n.value == 8 + 32 * nrows
    prove_rc(cap=8)
    assert n.value == 2 * (8 + 32 * (nv - nv // 2)) + 4 * 32
    # a polynomial of another context: LASSO_ERR_STRATEGY, as from every lasso_poly_* call
    other_ctx = lb.Context(0)
    p_other = lb.DensePolynomial(other_ctx, Z)
    before = ctx.launches
    assert L.lasso_poly_commit_hiding(ctx._h, p_other._h, gens._h, tape._h, lb.api._p(buf), c_sz(buf.shape[0]),
                                      ctypes.byref(n), lb.api._p(bl_out), c_sz(nrows)) == ERR_STRATEGY
    assert L.lasso_poly_eval_prove_hiding(ctx._h, p_other._h, gens._h, lb.api._p(blinds), c_sz(nrows), lb.api._p(r),
                                          c_sz(nv), lb.api._p(Zr), lb.api._p(bz), t._h, tape._h, lb.api._p(buf),
                                          c_sz(buf.shape[0]), ctypes.byref(n), lb.api._p(czr)) == ERR_STRATEGY
    assert ctx.launches == before
    del p_other
    other_ctx.close()
    # neither handle moved: the next challenge and draw equal fresh copies'
    assert np.array_equal(t.challenge_scalar(b"x"), lb.Transcript(b"e").challenge_scalar(b"x"))
    assert np.array_equal(tape.random_scalar(b"x"), lb.RandomTape(b"proof", _seed(1)).random_scalar(b"x"))
    # and the context stays usable
    assert commit_rc(tp=lb.RandomTape(b"c", _seed(1))) == 0 and prove_rc(tr=lb.Transcript(b"e")) == 0


# ---------------------------------------------------------------- the blind-term kernel one launch at a time
HCOL = 5  # h: generator 5 of a 6-point table; the rows R_i use generators 0..3
NCOLS = 4


@pytest.fixture(scope="module")
def tables():
    gens = np.ascontiguousarray(ol.generators(HCOL + 1))
    t = kh.Tables(gens)
    yield t, gens
    t.close()


def _raw_rows(t, rows, col_add=0):
    """un-normalised R_i of rows of integers (msm_rows_direct_fr with out_raw)"""
    ncols = len(rows[0])
    sc = np.ascontiguousarray(mont([v for row in rows for v in row]))
    out_raw = np.zeros((len(rows), 32), dtype=np.uint32)
    kh.call("kh_msm_rows_direct_raw", t.h, 1, ptr(sc), len(rows), ncols, 32, 1, col_add, 0, ptr(out_raw), None)
    return out_raw


def _reference(gens, rows, blinds):
    """the oracle's R_i + blind_i h: rows (row_i, blind_i) over (G_0 .. G_3, h)"""
    gsel = np.ascontiguousarray(np.concatenate([gens[:NCOLS], gens[HCOL:HCOL + 1], gens[:1]]))
    vals = mont([v for row, b in zip(rows, blinds) for v in list(row) + [b]])
    out = np.zeros((len(rows), 16), dtype=np.uint64)
    ol.lib().orc_commit_rows(ol.P(gsel), ol.P(np.ascontiguousarray(vals)), ol.sz(len(rows)), ol.sz(NCOLS + 1),
                             ol.P(out))
    return Ref(out).comp


KH_HIDING = os.path.join(HERE, "kernel_harness", "_build", "libkernel_harness_hiding.so")
_kh_hiding = None


def _kh():
    """libkernel_harness_hiding.so (tests/kernel_harness/Makefile.hiding); the tables come from libkernel_harness.so"""
    global _kh_hiding
    if _kh_hiding is None:
        if not os.path.exists(KH_HIDING):
            raise RuntimeError("libkernel_harness_hiding.so is missing: run `python -c 'import __graft_entry__ as g; "
                               "g.build()'` (nvcc, sm_90a).")
        L_ = ctypes.CDLL(KH_HIDING)
        L_.kh_row_blinds.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p,
                                     ctypes.c_int, ctypes.c_void_p]
        _kh_hiding = L_
    return _kh_hiding


def _row_blinds(t, source, raw_rows, blinds):
    nrows = raw_rows.shape[0]
    bl = np.ascontiguousarray(mont(blinds))
    out = np.zeros((nrows, 32), dtype=np.uint8)
    rc = _kh().kh_row_blinds(t.h, source, HCOL, ptr(np.ascontiguousarray(raw_rows)), ptr(bl), nrows, ptr(out))
    assert rc == 0, "kh_row_blinds returned %d (-1: the launcher threw, -2: CUDA error, -4: bad arguments)" % rc
    return out


EDGE_BLINDS = [0, 1, L_FR - 1, 2**252, int.from_bytes(b"\x7f" * 31, "little"), int.from_bytes(b"\x80" * 31, "little"),
               int.from_bytes(b"\x80" * 31 + b"\x0f", "little")]


@pytest.mark.parametrize("nrows", [1, 31, 32, 33, 1 << 14])
@pytest.mark.parametrize("source", [0, 1])
def test_row_blinds_kernel(tables, nrows, source):
    t, gens = tables
    rng = np.random.default_rng(nrows + 7 * source)
    import random

    prng = random.Random(nrows)
    blinds = [EDGE_BLINDS[i] if i < len(EDGE_BLINDS) and nrows > 1 else prng.randrange(L_FR) for i in range(nrows)]
    rows = [[int(x) for x in rng.integers(0, 2**62, size=NCOLS)] for _ in range(nrows)]
    rows[0] = [0] * NCOLS  # an identity row: the result is blind_0 h alone
    got = _row_blinds(t, source, _raw_rows(t, rows), blinds)
    want = _reference(gens, rows, blinds)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert not len(bad), "%d of %d rows differ, first row %d" % (len(bad), nrows, bad[0])


@pytest.mark.parametrize("source", [0, 1])
def test_row_blinds_cancel(tables, source):
    """R_i = -blind_i h: every row is the identity"""
    t, gens = tables
    blinds = EDGE_BLINDS[1:] + [random_b for random_b in (12345, L_FR // 3)]
    raw_rows = np.concatenate([_raw_rows(t, [[(L_FR - b) % L_FR]], col_add=HCOL) for b in blinds])
    got = _row_blinds(t, source, raw_rows, blinds)
    identity = _reference(gens, [[0] * NCOLS], [0])[0]
    assert all(bytes(row) == bytes(identity) for row in got)


# ---------------------------------------------------------------- at size
GOLD = json.load(open(os.path.join(HERE, "golden", "dense_poly_hiding.json")))["cases"]


@pytest.mark.parametrize("name", ["full_nv22", "u16_nv22", "full_nv24", "u16_nv24"])
def test_at_size_against_golden(ctx, name):
    import lasso_b200 as lb

    gold = GOLD[name]
    nv, Z, r, seed = dc.inputs(name)
    assert hashlib.sha256(Z.tobytes()).hexdigest() == gold["Z_sha256"]
    stream = np.ascontiguousarray(ol.generators(gold["n_generators"]))
    assert hashlib.sha256(stream.tobytes()).hexdigest() == gold["generators_sha256"]
    gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream)
    p = lb.DensePolynomial(ctx, Z)
    tape = lb.RandomTape(dc.TAPE_LABEL, seed)
    comm, blinds = p.commit_hiding(gens, tape)
    assert hashlib.sha256(comm).hexdigest() == gold["commitment_sha256"]
    assert hashlib.sha256(blinds.tobytes()).hexdigest() == gold["blinds_sha256"]
    t = lb.Transcript(dc.TRANSCRIPT_LABEL)
    t.append_poly_commitment(dc.COMMIT_LABEL, comm)
    Zr = p.evaluate(r)
    assert Zr.tobytes().hex() == gold["Zr_hex"]
    blind_Zr = tape.random_scalar(b"blind_Zr")
    assert blind_Zr.tobytes().hex() == gold["blind_Zr_hex"]
    proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, tape, blinds=blinds, blind_Zr=blind_Zr)
    assert hashlib.sha256(proof.bytes).hexdigest() == gold["proof_sha256"]
    assert proof.C_Zr.hex() == gold["C_Zr_hex"]
    assert t.challenge_scalar(b"after").tobytes().hex() == gold["after_challenge_hex"]
