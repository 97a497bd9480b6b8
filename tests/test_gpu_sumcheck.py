"""Sumchecks over a caller's polynomials on the GPU: SumcheckInstanceProof.prove_arbitrary with a traced combining
function on a caller-held Transcript, bit for bit against the CPU oracle (oracle_dense/).  Every case compares the proof
bytes, the challenges, the final evaluations, the claim and the transcript's next challenge.  Covers 1..16 inputs,
degrees 1..16, num_vars 1..20 with fewer rounds than variables, a polynomial passed twice, integer, full-width and l - 1
values, eq polynomials, CUDA-tensor polynomials, the caller's polynomials left unchanged, composition with commitments
and openings on one transcript, every argument error, the launch count, the fused and unfused rounds, and the sizes of
tests/golden/sumcheck.json."""
import hashlib
import json
import os

import numpy as np
import pytest

import dense_poly_cases as dc
import oracle_dense_lib as od
import oracle_lib as ol
import oracle_sumcheck_lib as osc
import sumcheck_cases as sc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ERR_LENGTH, ERR_STRATEGY = 1, 4
FUSED_MIN_Q = 1 << 15


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _values(kind, n, rng):
    if kind == "full":
        return dc.random_full(rng, n)
    if kind == "l-1":  # every other entry l - 1, the others small
        Z = dc.fr_from_u64(rng.integers(0, 256, size=n, dtype=np.uint64))
        Z[::2] = ol.fr_array([ol.L_FR - 1])[0]
        return Z
    return dc.fr_from_u64(rng.integers(0, 1 << {"u8": 8, "u32": 32}[kind], size=n, dtype=np.uint64))


def _both(ctx, fn, k, arrays, num_rounds=None, degree=None, polys=None, label=b"sumcheck"):
    """GPU and oracle on the same inputs; asserts every output equal and returns the GPU proof"""
    import lasso_b200 as lb

    comb = lb.Comb(fn, k, degree)
    if polys is None:
        polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    nv = polys[0].num_vars
    rounds = nv if num_rounds is None else num_rounds
    t = lb.Transcript(label)
    got = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, t, num_rounds)
    o = od.Transcript(label)
    want = osc.sumcheck_prove(arrays, rounds, comb.program, comb.constants, comb.degree, o)
    assert len(got.bytes) == 8 + rounds * (8 + 32 * comb.degree)
    assert got.bytes == want["proof"]
    assert np.array_equal(got.r, want["r"])
    assert np.array_equal(got.final_evals, want["final_evals"])
    assert np.array_equal(got.claim, want["claim"])
    assert np.array_equal(t.challenge_scalar(b"after"), o.challenge_scalar(b"after"))
    return got


def _kfun(k):
    """a degree-2 function of k inputs in which every input has its own weight"""
    return lambda v: sum((i + 1) * v[i] for i in range(k)) * v[k - 1] + v[0]


@pytest.mark.parametrize("k", list(range(1, 17)))
def test_inputs(ctx, k):
    rng = np.random.default_rng(k)
    _both(ctx, _kfun(k), k, [dc.random_full(rng, 1 << 7) for _ in range(k)])


@pytest.mark.parametrize("d", list(range(1, 17)))
def test_degrees(ctx, d):
    """x_0 x_1 x_0 x_1 ... (d factors), plus the same function declared one degree higher"""
    rng = np.random.default_rng(100 + d)
    arrays = [dc.random_full(rng, 1 << 6) for _ in range(2)]
    fn = (lambda v: sc.prod9([v[i % 2] for i in range(d)])) if d > 1 else (lambda v: v[0] + v[1])
    _both(ctx, fn, 2, arrays)
    if d < 16:
        _both(ctx, fn, 2, arrays, degree=d + 1)


@pytest.mark.parametrize("nv,rounds", [(1, 1), (2, 1), (2, 2), (3, 3), (5, 2), (8, 8), (12, 12), (12, 5), (16, 16),
                                       (17, 3), (18, 18), (20, 20), (20, 7)])
def test_num_vars_and_rounds(ctx, nv, rounds):
    rng = np.random.default_rng(1000 + nv)
    tau = dc.random_full(rng, nv)
    arrays = [sc.eq_evals(tau)] + [dc.random_full(rng, 1 << nv) for _ in range(3)]
    _both(ctx, sc.spartan, 4, arrays, num_rounds=rounds)


def test_same_poly_twice(ctx):
    import lasso_b200 as lb

    A = dc.random_full(np.random.default_rng(7), 1 << 10)
    p = lb.DensePolynomial(ctx, A)
    _both(ctx, lambda v: v[0] * v[1], 2, [A, A], polys=[p, p])
    _both(ctx, lambda v: v[0] * v[1] - v[2] * 3, 3, [A, A, A], polys=[p, p, p], num_rounds=4)


@pytest.mark.parametrize("kind", ["u8", "u32", "full", "l-1"])
def test_value_kinds(ctx, kind):
    rng = np.random.default_rng(len(kind))
    arrays = [_values(kind, 1 << 11, rng) for _ in range(3)]
    _both(ctx, sc.FUNCS["consts"][0], 3, arrays)


def test_eq_polynomial(ctx):
    """DensePolynomial.eq: its evaluations equal the oracle's, and it takes part in a sumcheck as any polynomial"""
    import lasso_b200 as lb

    rng = np.random.default_rng(3)
    for nv in (0, 1, 5, 12, 13, 23):
        tau = dc.random_full(rng, nv)
        e = lb.DensePolynomial.eq(ctx, tau)
        assert e.num_vars == nv
        x = dc.random_full(rng, nv)
        assert np.array_equal(e.evaluate(x), od.evaluate(sc.eq_evals(tau), x))
    tau = dc.random_full(rng, 9)
    arrays = [sc.eq_evals(tau)] + [dc.random_full(rng, 1 << 9) for _ in range(3)]
    polys = [lb.DensePolynomial.eq(ctx, tau)] + [lb.DensePolynomial(ctx, a) for a in arrays[1:]]
    _both(ctx, sc.spartan, 4, arrays, polys=polys)


def test_device_tensors(ctx):
    import torch

    import lasso_b200 as lb

    rng = np.random.default_rng(11)
    arrays = [dc.random_full(rng, 1 << 12) for _ in range(4)]
    wide = torch.zeros((1 << 12, 6), dtype=torch.int64, device="cuda")
    wide[:, 2:6] = torch.from_numpy(arrays[3].view(np.int64)).cuda()
    polys = [lb.DensePolynomial(ctx, torch.from_numpy(a.view(np.int64)).cuda()) for a in arrays[:2]]
    polys += [lb.DensePolynomial(ctx, arrays[2]), lb.DensePolynomial(ctx, wide[:, 2:6])]
    torch.cuda.synchronize()
    _both(ctx, sc.spartan, 4, arrays, polys=polys)


def test_final_evals_are_evaluations(ctx):
    import lasso_b200 as lb

    rng = np.random.default_rng(12)
    arrays = [_values(kind, 1 << 14, rng) for kind in ("full", "u32", "l-1", "full")]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    got = _both(ctx, sc.spartan, 4, arrays, polys=polys)
    for p, v in zip(polys, got.final_evals):
        assert np.array_equal(p.evaluate(got.r), v)


def _gens(ctx, nv):
    import lasso_b200 as lb

    stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
    return lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream), stream


def test_inputs_untouched(ctx):
    """every round and the final bind leave the caller's polynomials as they were: their commitments are unchanged,
    fused and unfused"""
    import lasso_b200 as lb

    nv = 18
    rng = np.random.default_rng(13)
    gens, _ = _gens(ctx, nv)
    arrays = [_values(kind, 1 << nv, rng) for kind in ("full", "u32", "full")]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    before = [p.commit(gens) for p in polys]
    comb = lb.Comb(lambda v: v[0] * v[1] + v[2], 3)
    for rounds in (nv, 1, 2, 5):
        lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, lb.Transcript(b"u"), rounds)
        assert [p.commit(gens) for p in polys] == before, rounds


def test_composition(ctx):
    """commit A, B, C -> draw tau -> sumcheck eq(tau) (A B - C) -> open A, B, C at r, one transcript and one tape: every
    byte equals the oracle's run of the same sequence, and the oracle's verifier accepts every part"""
    import lasso_b200 as lb

    nv = 10
    rng = np.random.default_rng(14)
    A, B = dc.random_full(rng, 1 << nv), _values("u32", 1 << nv, rng)
    C = ol.fr_array([a * b % ol.L_FR for a, b in zip(ol.fr_ints(A), ol.fr_ints(B))])  # a satisfied instance: claim 0
    gens, stream = _gens(ctx, nv)
    seed = ol.fr_array([99])[0]
    pa, pb, pc = (lb.DensePolynomial(ctx, X) for X in (A, B, C))
    comms = [p.commit(gens) for p in (pa, pb, pc)]
    t, tape = lb.Transcript(b"spartan"), lb.RandomTape(b"proof", seed)
    o, otape = od.Transcript(b"spartan"), od.RandomTape(b"proof", seed)
    for x in (t, o):
        for name, cm in zip((b"A", b"B", b"C"), comms):
            x.append_poly_commitment(name, cm)
    tau = t.challenge_vector(b"tau", nv)
    assert np.array_equal(tau, o.challenge_vector(b"tau", nv))
    comb = lb.Comb(sc.spartan, 4)
    sc_proof = lb.SumcheckInstanceProof.prove_arbitrary(ctx, [lb.DensePolynomial.eq(ctx, tau), pa, pb, pc], comb, t)
    want = osc.sumcheck_prove([sc.eq_evals(tau), A, B, C], nv, comb.program, comb.constants, 3, o)
    assert sc_proof.bytes == want["proof"] and ol.fr_ints(sc_proof.claim) == [0]
    r = sc_proof.r
    openings = [lb.PolyEvalProof.prove(ctx, p, r, sc_proof.final_evals[1 + i], gens, t, tape) for i, p in enumerate((pa, pb, pc))]
    wants = [od.prove(X, r, want["final_evals"][1 + i], stream, o, otape)[0] for i, X in enumerate((A, B, C))]
    assert [p.bytes for p in openings] == wants
    assert np.array_equal(t.challenge_scalar(b"end"), o.challenge_scalar(b"end"))
    # the verifier's replay
    v = od.Transcript(b"spartan")
    for name, cm in zip((b"A", b"B", b"C"), comms):
        v.append_poly_commitment(name, cm)
    vtau = v.challenge_vector(b"tau", nv)
    rc, e, vr = osc.sumcheck_verify(sc_proof.bytes, sc_proof.claim, nv, 3, v)
    assert rc == 0 and np.array_equal(vr, r)
    eq_r = np.zeros(4, dtype=np.uint64)
    ol.lib().orc_eq_evaluate(ol.P(np.ascontiguousarray(vtau)), ol.P(np.ascontiguousarray(vr)), ol.sz(nv), ol.P(eq_r))
    ea, eb, ec = ol.fr_ints(sc_proof.final_evals[1:])
    assert ol.fr_ints(e)[0] == ol.fr_ints(eq_r)[0] * (ea * eb - ec) % ol.L_FR
    for i, cm in enumerate(comms):
        assert od.verify(stream, nv, cm, openings[i].bytes, vr, sc_proof.final_evals[1 + i], v) == 0


def _expected_launches(nv, rounds):
    """DESIGN.md §3.9: the first round's evaluation, then per round one fused kernel from q = 2^15 pairs up (q = 2^(nv - j
    - 1) in round j), else a bind and an evaluation, and one final kernel"""
    fused = sum(1 for j in range(1, rounds) if (1 << (nv - j - 1)) >= FUSED_MIN_Q)
    return 1 + fused + 2 * (rounds - 1 - fused) + 1


@pytest.mark.parametrize("nv,rounds", [(1, 1), (4, 4), (18, 18), (18, 2), (20, 20)])
def test_launch_count(ctx, nv, rounds):
    import lasso_b200 as lb

    rng = np.random.default_rng(nv)
    polys = [lb.DensePolynomial(ctx, dc.random_full(rng, 1 << nv)) for _ in range(2)]
    comb = lb.Comb(lambda v: v[0] * v[1], 2)
    before = ctx.launches
    lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, lb.Transcript(b"n"), rounds)
    assert ctx.launches - before == _expected_launches(nv, rounds)


@pytest.mark.parametrize("nv,name", [(18, "spartan"), (17, "wide16"), (16, "prod9")])
def test_fused_equals_unfused(ctx, monkeypatch, nv, name):
    import lasso_b200 as lb

    fn, k = sc.FUNCS[name]
    rng = np.random.default_rng(nv + k)
    polys = [lb.DensePolynomial(ctx, dc.random_full(rng, 1 << nv)) for _ in range(k)]
    comb = lb.Comb(fn, k)
    fused = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, lb.Transcript(b"f"))
    monkeypatch.setenv("LASSO_B200_UNFUSED_SUMCHECK", "1")
    before = ctx.launches
    unfused = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, lb.Transcript(b"f"))
    assert ctx.launches - before == 2 * nv
    assert fused.bytes == unfused.bytes and np.array_equal(fused.final_evals, unfused.final_evals)


def test_errors(ctx):
    """each error before any launch with the transcript untouched, then a correct proof on the same context"""
    import ctypes

    import lasso_b200 as lb

    rng = np.random.default_rng(15)
    A, B = dc.random_full(rng, 1 << 6), dc.random_full(rng, 1 << 6)
    pa, pb, small = lb.DensePolynomial(ctx, A), lb.DensePolynomial(ctx, B), lb.DensePolynomial(ctx, A[:32])
    other = lb.Context(0)
    foreign = lb.DensePolynomial(other, B)
    comb = lb.Comb(lambda v: v[0] * v[1], 2)
    cases = [
        ([pa], None, ERR_STRATEGY),  # n_polys != n_inputs
        ([pa, pb, pb], None, ERR_STRATEGY),
        ([pa, foreign], None, ERR_STRATEGY),  # a polynomial of another context
        ([pa, small], None, ERR_LENGTH),  # different num_vars
        ([pa, pb], 0, ERR_LENGTH),  # num_rounds outside 1..num_vars
        ([pa, pb], 7, ERR_LENGTH),
    ]
    for polys, rounds, code in cases:
        t, twin = lb.Transcript(b"err"), lb.Transcript(b"err")
        before = ctx.launches
        with pytest.raises(lb.LassoError) as e:
            lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, t, rounds)
        assert e.value.code == code, (len(polys), rounds, str(e.value))
        assert ctx.launches == before
        assert np.array_equal(t.challenge_scalar(b"x"), twin.challenge_scalar(b"x"))
        _both(ctx, lambda v: v[0] * v[1], 2, [A, B], polys=[pa, pb])
    # proof_cap too small, through the C ABI
    t, twin = lb.Transcript(b"err"), lb.Transcript(b"err")
    arr = (ctypes.c_void_p * 2)(pa._h.value, pb._h.value)
    need = 8 + 6 * (8 + 64)
    out = np.zeros(need, dtype=np.uint8)
    r, fin, n = np.zeros((6, 4), dtype=np.uint64), np.zeros((2, 4), dtype=np.uint64), ctypes.c_size_t(0)
    before = ctx.launches
    rc = lb.lib().lasso_sumcheck_prove(ctx._h, comb._h, arr, ctypes.c_size_t(2), ctypes.c_size_t(6), t._h, out.ctypes.data,
                                       ctypes.c_size_t(need - 1), ctypes.byref(n), r.ctypes.data, fin.ctypes.data, None)
    assert rc == ERR_LENGTH and n.value == need and ctx.launches == before
    assert np.array_equal(t.challenge_scalar(b"x"), twin.challenge_scalar(b"x"))
    _both(ctx, lambda v: v[0] * v[1], 2, [A, B], polys=[pa, pb])
    del foreign
    other.close()


GOLDEN = json.load(open(os.path.join(HERE, "golden", "sumcheck.json")))


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_at_size_against_golden(ctx, name):
    """the seeded cases of tests/golden/sumcheck.json: SHA-256 of proof bytes || r || final_evals, the claim and the
    next challenge equal the oracle's, with eq(tau) made on the GPU"""
    import lasso_b200 as lb

    fname, nv, tau, arrays = sc.golden_inputs(name)
    g = GOLDEN["cases"][name]
    fn, k = sc.FUNCS[fname]
    polys = [lb.DensePolynomial.eq(ctx, tau)] + [lb.DensePolynomial(ctx, a) for a in arrays[1:]]
    del arrays
    t = lb.Transcript(sc.TRANSCRIPT_LABEL)
    got = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, lb.Comb(fn, k), t)
    digest = hashlib.sha256(got.bytes + got.r.tobytes() + got.final_evals.tobytes()).hexdigest()
    assert digest == g["sha256"]
    assert got.claim.tobytes().hex() == g["claim_hex"]
    assert t.challenge_scalar(b"after").tobytes().hex() == g["after_challenge_hex"]
