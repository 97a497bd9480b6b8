"""Many polynomials per call on the GPU: DensePolynomial.merge, DensePolynomial.evaluate_batch and
CombinedTableEvalProof.prove, bit for bit against the CPU oracle (oracle_dense/).  Covers merges of equal, unequal,
repeated and single inputs with and without padding over zero, u32, full-width, l - 1 and mixed values (commitments,
evaluations at random and boolean points, the u32 mirror, no launch, inputs unchanged); batched evaluation of 1..64
polynomials of num_vars 0..22 in both forms with its launch count; combined proofs (bytes, the next challenge, the
oracle's verifier, a wrong claim); offline memory checking on one transcript; the derefs of a Lasso proof; merged
polynomials of 2^24 evaluations; the sizes of tests/golden/combined_eval.json; and every argument error."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import combined_eval_cases as cc
import dense_poly_cases as dc
import oracle_combined_eval_lib as oce
import oracle_dense_lib as od
import oracle_grand_product_lib as ogp
import oracle_lib as ol
import workloads

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ERR_LENGTH, ERR_STRATEGY, ERR_GENS, ERR_VALUE = 1, 4, 5, 8
L = ol.L_FR
BAD = np.full(4, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)  # limbs of no canonical residue
TAPE_SEED = ol.fr_array([11])[0]


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _values(kind, n, rng):
    if kind == "full":
        return dc.random_full(rng, n)
    if kind == "zero":
        return np.zeros((n, 4), dtype=np.uint64)
    if kind == "l-1":
        Z = dc.fr_from_u64(rng.integers(0, 256, size=n, dtype=np.uint64))
        Z[::2] = ol.fr_array([L - 1])[0]
        return Z
    return dc.fr_from_u64(rng.integers(0, 1 << 32, size=n, dtype=np.uint64))  # "u32"


_GENS = {}


def _gens(ctx, nv):
    """generators for num_vars, one object per num_vars up to 16 for the module"""
    import lasso_b200 as lb

    if nv > 16:  # the device tables of a large R are not kept for the module
        stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
        return lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream), stream
    if nv not in _GENS:
        stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
        _GENS[nv] = (lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream), stream)
    return _GENS[nv]


def _eq_launches(ell):
    return 1 if ell <= 11 else (3 if ell <= 22 else 5)


def _has_mirror(ctx, p):
    """a polynomial with a u32 mirror is evaluated in the u32 form: next to a full-width one, a batch takes two dot
    launches and their reductions (DESIGN.md §3.11: the eq table, 2 per form, 1 read-back)"""
    import lasso_b200 as lb

    full = lb.DensePolynomial.eq(ctx, dc.random_full(np.random.default_rng(0), p.num_vars))
    before = ctx.launches
    lb.DensePolynomial.evaluate_batch(ctx, [p, full], dc.random_full(np.random.default_rng(1), p.num_vars))
    forms, odd = divmod(ctx.launches - before - _eq_launches(p.num_vars) - 1, 2)
    assert forms in (1, 2) and not odd
    return forms == 2


# ------------------------------------------------------------------ merge
MERGES = {  # name -> component sizes (log2), value kinds
    "equal": ([5, 5, 5, 5], ["u32"] * 4), "unequal": ([6, 3, 4], ["full", "full", "full"]),
    "one": ([7], ["full"]), "pad": ([4, 4, 4], ["u32"] * 3), "pad_unequal": ([5, 0, 2, 1], ["u32", "full", "u32", "u32"]),
    "zero": ([4, 4], ["zero", "zero"]), "l-1": ([3, 5], ["l-1", "l-1"]), "mixed": ([4, 4, 4], ["zero", "u32", "full"]),
    "u32_zero": ([4, 3, 4], ["u32", "zero", "u32"]), "big": ([12, 10, 9], ["full", "u32", "u32"]),
}


@pytest.mark.parametrize("name", sorted(MERGES))
def test_merge(ctx, name):
    """commitment and evaluations (random and boolean points) of the merged polynomial equal the oracle's merge; no
    launch; a mirror exactly when every input is integer; the inputs unchanged"""
    import lasso_b200 as lb

    logs, kinds = MERGES[name]
    rng = np.random.default_rng(len(name) * 7 + sum(logs))
    arrays = [_values(k, 1 << n, rng) for n, k in zip(logs, kinds)]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    gens_in = [_gens(ctx, p.num_vars)[0] if p.num_vars else None for p in polys]
    before_comm = [p.commit(g) if g else None for p, g in zip(polys, gens_in)]
    before = ctx.launches
    m = lb.DensePolynomial.merge(ctx, polys)
    assert ctx.launches == before
    want = oce.merge(arrays)
    mv = want.shape[0].bit_length() - 1
    assert m.num_vars == mv
    gens, _ = _gens(ctx, mv)
    assert m.commit(gens) == od.commit(want, _gens(ctx, mv)[1])
    x = dc.random_full(rng, mv)
    assert np.array_equal(m.evaluate(x), od.evaluate(want, x))
    for idx in (0, len(arrays[0]) - 1, want.shape[0] - 1, int(rng.integers(0, want.shape[0]))):  # boolean points
        b = ol.fr_array([(idx >> (mv - 1 - i)) & 1 for i in range(mv)])
        assert np.array_equal(m.evaluate(b), want[idx]), idx
    integer = all(k in ("u32", "zero") for k in kinds)
    assert _has_mirror(ctx, m) == integer
    assert [p.commit(g) if g else None for p, g in zip(polys, gens_in)] == before_comm


def test_merge_repeated_and_owned(ctx):
    """the same polynomial three times; the merged polynomial keeps its own copy after the inputs are dropped"""
    import lasso_b200 as lb

    rng = np.random.default_rng(5)
    A, B = _values("full", 1 << 6, rng), _values("u32", 1 << 5, rng)
    pa, pb = lb.DensePolynomial(ctx, A), lb.DensePolynomial(ctx, B)
    m = lb.DensePolynomial.merge(ctx, [pa, pb, pa, pa])
    want = oce.merge([A, B, A, A])
    del pa, pb
    x = dc.random_full(rng, m.num_vars)
    assert np.array_equal(m.evaluate(x), od.evaluate(want, x))
    assert m.commit(_gens(ctx, m.num_vars)[0]) == od.commit(want, _gens(ctx, m.num_vars)[1])


# ------------------------------------------------------------------ evaluate_batch
@pytest.mark.parametrize("k", [1, 7, 8, 9, 64])
def test_evaluate_batch_sizes(ctx, k):
    import lasso_b200 as lb

    rng = np.random.default_rng(200 + k)
    nv = 9
    kinds = ["u32", "full", "l-1", "zero"]
    arrays = [_values(kinds[j % 4], 1 << nv, rng) for j in range(k)]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    r = dc.random_full(rng, nv)
    before = ctx.launches
    got = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
    forms = len({kinds[j % 4] in ("u32", "zero") for j in range(k)})
    assert ctx.launches - before == _eq_launches(nv) + 2 * forms + 1
    assert got.shape == (k, 4)
    assert np.array_equal(got, np.stack([od.evaluate(a, r) for a in arrays]))
    assert np.array_equal(got, np.stack([p.evaluate(r) for p in polys]))


@pytest.mark.parametrize("nv", [0, 1, 2, 5, 11, 12, 16, 20, 22])
@pytest.mark.parametrize("forms", ["u32", "full", "mixed"])
def test_evaluate_batch_num_vars(ctx, nv, forms):
    import lasso_b200 as lb

    rng = np.random.default_rng(300 + nv)
    kinds = {"u32": ["u32"] * 10, "full": ["full"] * 10, "mixed": ["full", "u32", "l-1", "u32", "full", "zero",
                                                                    "u32", "full", "u32", "u32"]}[forms]
    if nv >= 20:
        kinds = kinds[:3]
    arrays = [_values(k, 1 << nv, rng) for k in kinds]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    polys.append(polys[0])  # a repeated input
    r = dc.random_full(rng, nv)
    before = ctx.launches
    got = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
    n_forms = len({k in ("u32", "zero") for k in kinds})
    assert ctx.launches - before == _eq_launches(nv) + 2 * n_forms + 1
    each = np.stack([p.evaluate(r) for p in polys])
    assert np.array_equal(got, each)
    if nv <= 16:
        assert np.array_equal(got[:-1], np.stack([od.evaluate(a, r) for a in arrays]))


# ------------------------------------------------------------------ the combined proof
def _combined_both(ctx, arrays, r, label=b"ce", wrong=None):
    """merge, evaluate_batch and the combined proof on the GPU and the oracle; asserts the bytes and the next challenge
    equal and the oracle's verifier accepts; returns (merged poly, evals, proof bytes, commitment, stream)"""
    import lasso_b200 as lb

    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    m = lb.DensePolynomial.merge(ctx, polys)
    gens, stream = _gens(ctx, m.num_vars)
    evals = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
    claims = evals if wrong is None else wrong
    t, tape = lb.Transcript(label), lb.RandomTape(b"proof", TAPE_SEED)
    proof = lb.CombinedTableEvalProof.prove(ctx, m, claims, r, gens, t, tape)
    Z = oce.merge(arrays)
    o = od.Transcript(label)
    want = oce.prove(Z, claims, r, stream, o, od.RandomTape(b"proof", TAPE_SEED))
    assert proof.data == want and len(want) == lb.CombinedTableEvalProof.proof_len(m.num_vars)
    assert np.array_equal(t.challenge_scalar(b"after"), o.challenge_scalar(b"after"))
    comm = m.commit(gens)
    return m, evals, proof.data, comm, stream


@pytest.mark.parametrize("k,nv", [(1, 3), (2, 1), (3, 4), (4, 5), (5, 2), (8, 6), (17, 3), (32, 2), (64, 1), (3, 0)])
def test_combined_proof(ctx, k, nv):
    rng = np.random.default_rng(400 + 10 * k + nv)
    kinds = ["u32", "full", "l-1", "zero"]
    arrays = [_values(kinds[j % 4], 1 << nv, rng) for j in range(k)]
    r = dc.random_full(rng, nv)
    m, evals, proof, comm, stream = _combined_both(ctx, arrays, r)
    assert np.array_equal(evals, np.stack([od.evaluate(a, r) for a in arrays]))
    assert oce.verify(stream, m.num_vars, comm, proof, evals, r, od.Transcript(b"ce")) == 0


def test_combined_proof_wrong_claim(ctx):
    """a proof made from a wrong claim matches the oracle's bytes, and the oracle's verifier rejects it"""
    rng = np.random.default_rng(450)
    arrays = [_values("full", 1 << 5, rng) for _ in range(3)]
    r = dc.random_full(rng, 5)
    true = np.stack([od.evaluate(a, r) for a in arrays])
    wrong = true.copy()
    wrong[2] = ol.fr_array([(ol.fr_ints(true[2])[0] + 1) % L])[0]
    m, evals, proof, comm, stream = _combined_both(ctx, arrays, r, wrong=wrong)
    assert np.array_equal(evals, true)
    assert oce.verify(stream, m.num_vars, comm, proof, true, r, od.Transcript(b"ce")) == 1
    assert oce.verify(stream, m.num_vars, comm, proof, wrong, r, od.Transcript(b"ce")) == 1


GOLDEN = json.load(open(os.path.join(HERE, "golden", "combined_eval.json")))


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_against_golden(ctx, name):
    """the seeded cases of tests/golden/combined_eval.json: SHA-256 of evals || proof, the merged commitment and the next
    challenge equal the oracle's"""
    import lasso_b200 as lb

    nv, comps, r, seed = cc.golden_inputs(name)
    g = GOLDEN["cases"][name]
    polys = [lb.DensePolynomial(ctx, a) for a in comps]
    m = lb.DensePolynomial.merge(ctx, polys)
    gens, _ = _gens(ctx, m.num_vars)
    evals = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
    t = lb.Transcript(cc.TRANSCRIPT_LABEL)
    proof = lb.CombinedTableEvalProof.prove(ctx, m, evals, r, gens, t, lb.RandomTape(cc.TAPE_LABEL, seed))
    assert len(proof.data) == g["proof_len"] and m.num_vars == g["merged_num_vars"]
    assert hashlib.sha256(cc.digest_input(evals, proof.data)).hexdigest() == g["sha256"]
    assert hashlib.sha256(m.commit(gens)).hexdigest() == g["commitment_sha256"]
    assert t.challenge_scalar(b"after").tobytes().hex() == g["after_challenge_hex"]


@pytest.mark.parametrize("k,nv,kind", [(16, 20, "u32"), (4, 22, "full")])
def test_at_size(ctx, k, nv, kind):
    """merged polynomials of 2^24 evaluations: the evals equal the per-polynomial evaluations and the oracle's verifier
    accepts the proof against the GPU's commitment"""
    import lasso_b200 as lb

    rng = np.random.default_rng(500 + nv)
    polys = [lb.DensePolynomial(ctx, _values(kind, 1 << nv, rng)) for _ in range(k)]
    m = lb.DensePolynomial.merge(ctx, polys)
    assert m.num_vars == 24
    r = dc.random_full(rng, nv)
    evals = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
    assert np.array_equal(evals, np.stack([p.evaluate(r) for p in polys]))
    gens, stream = _gens(ctx, 24)
    t = lb.Transcript(b"at_size")
    proof = lb.CombinedTableEvalProof.prove(ctx, m, evals, r, gens, t, lb.RandomTape(b"proof", TAPE_SEED))
    comm = m.commit(gens)
    v = od.Transcript(b"at_size")
    assert oce.verify(stream, 24, comm, proof.data, evals, r, v) == 0
    assert np.array_equal(v.challenge_scalar(b"after"), t.challenge_scalar(b"after"))


# ------------------------------------------------------------------ composed protocols
def _h(a, v, t, gamma, tau):
    return (t * gamma * gamma + v * gamma + a - tau) % L


def test_offline_memory_checking_one_transcript(ctx):
    """merge (a, v, t) of 2^12 reads, commit once, draw gamma and tau, form the read fingerprints with from_comb, append
    the product, prove the grand product, evaluate a, v, t at its rand in one batch and open all three with one combined
    proof.  The oracle replays all of it: the commitment, the grand product, the claim h(a, v, t) at rand and the
    combined opening."""
    import lasso_b200 as lb

    nv = 12
    rng = np.random.default_rng(77)
    cols = [rng.integers(0, 1 << 10, size=1 << nv, dtype=np.uint64), rng.integers(0, 1 << 32, size=1 << nv, dtype=np.uint64),
            rng.integers(0, 1 << 8, size=1 << nv, dtype=np.uint64)]
    Z = [dc.fr_from_u64(c) for c in cols]
    P = [lb.DensePolynomial(ctx, z) for z in Z]
    merged = lb.DensePolynomial.merge(ctx, P)
    gens, stream = _gens(ctx, merged.num_vars)
    comm = merged.commit(gens)
    t, tape = lb.Transcript(b"memory"), lb.RandomTape(b"proof", TAPE_SEED)
    t.append_poly_commitment(b"comm_avt", comm)
    gamma, tau = ol.fr_ints(t.challenge_vector(b"challenge_r_hash", 2))
    g2 = gamma * gamma % L
    read = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda x: x[2] * g2 + x[1] * gamma + x[0] - tau, 3), P)
    circuit = lb.GrandProductCircuit(ctx, read)
    product = circuit.evaluate()
    t.append_scalar(b"claim_hash_read", product)
    gp = lb.BatchedGrandProductArgument.prove(ctx, [circuit], t)
    evals = lb.DensePolynomial.evaluate_batch(ctx, P, gp.r)
    proof = lb.CombinedTableEvalProof.prove(ctx, merged, evals, gp.r, gens, t, tape)
    end = t.challenge_scalar(b"end")

    v = od.Transcript(b"memory")
    v.append_poly_commitment(b"comm_avt", od.commit(oce.merge(Z), stream))
    assert ol.fr_ints(v.challenge_vector(b"challenge_r_hash", 2)) == [gamma, tau]
    v.append_scalar(b"claim_hash_read", product)
    rc, claims, rand = ogp.gp_verify(gp.bytes, product.reshape(1, 4), nv, v)
    assert rc == 0 and np.array_equal(rand, gp.r)
    a, vv, tt = ol.fr_ints(evals)
    assert ol.fr_ints(claims) == [_h(a, vv, tt, gamma, tau)]
    assert oce.verify(stream, merged.num_vars, comm, proof.data, evals, rand, v) == 0
    assert np.array_equal(v.challenge_scalar(b"end"), end)


@pytest.mark.parametrize("name", ["s10", "xor_c4_s20"])
def test_lasso_derefs(ctx, name):
    """the E polynomials of an XOR C=4 proof as lasso_polys: their merge commits to comm_derefs and evaluate_batch at
    r_z (the primary sumcheck's challenges) gives eval_derefs, both read from the proof bytes"""
    import lasso_b200 as lb

    if name == "s10":
        C_, log_m, log_s = 4, 16, 10
        rng = np.random.default_rng(1)
        col = rng.integers(0, 1 << log_m, size=(1 << log_s, 1), dtype=np.uint64)
        idx = np.ascontiguousarray(np.repeat(col, C_, axis=1))
        r, seed = ol.rand_fr(rng, log_s), ol.rand_fr(rng, 1)[0]
    else:
        _, C_, log_m, _, log_s, idx, r, seed = workloads.config_inputs(name)
    S = lb.Strategy(lb.XOR, C_, log_m)
    alpha = S.num_memories
    stream = lb.sample_generators(b"gens_sparse_poly", lb.gens_points_needed(C_, 1 << log_s, alpha, log_m))
    sgens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, 1 << log_s, alpha, log_m, stream=stream)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, sgens, tape_seed=seed)
    b = proof.bytes
    n_pts = int.from_bytes(b[:8], "little")
    comm_derefs = b[: 8 + 32 * n_pts]
    at = 8 + 32 * n_pts
    rounds = int.from_bytes(b[at: at + 8], "little")
    at += 8
    for _ in range(rounds):
        at += 8 + 32 * int.from_bytes(b[at: at + 8], "little")
    at += 32  # claimed_eval
    eval_derefs = [int.from_bytes(b[at + 32 * i: at + 32 * (i + 1)], "little") for i in range(alpha)]
    r_z = proof.challenges[:log_s]
    E = lb.gather_lookup_polys(ctx, S, [np.ascontiguousarray(idx[:, d]) for d in range(C_)])
    polys = [lb.DensePolynomial(ctx, e) for e in E]
    m = lb.DensePolynomial.merge(ctx, polys)
    nv_d = m.num_vars
    pgens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv_d, stream=stream)
    assert m.commit(pgens) == comm_derefs
    assert ol.fr_ints(lb.DensePolynomial.evaluate_batch(ctx, polys, r_z)) == eval_derefs
    if name == "s10":
        assert _has_mirror(ctx, m)


def test_smoke_launch_count_unchanged():
    """lasso_launch_count() after smoke(), the 2^10 XOR proof of a fresh process, is 421"""
    import subprocess
    import sys

    root = os.path.dirname(HERE)
    out = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], cwd=root, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert " 421 kernel launches" in out.stdout, out.stdout


# ------------------------------------------------------------------ errors
def _raises(ctx, code, fn, transcript=None, tape=None):
    """fn fails with `code`, launches nothing, and leaves the transcript and the tape as they were"""
    import lasso_b200 as lb

    twin_t, twin_tape = lb.Transcript(b"err"), lb.RandomTape(b"tape", TAPE_SEED)
    before = ctx.launches
    with pytest.raises(lb.LassoError) as e:
        fn()
    assert e.value.code == code, str(e.value)
    assert ctx.launches == before
    if transcript is not None:
        assert np.array_equal(transcript.challenge_scalar(b"x"), twin_t.challenge_scalar(b"x"))
    if tape is not None:
        assert np.array_equal(tape.random_scalar(b"x"), twin_tape.random_scalar(b"x"))


def test_errors(ctx):
    """every error before any launch with the transcript and tape untouched, then correct results on the same context"""
    import lasso_b200 as lb

    rng = np.random.default_rng(15)
    A, B = dc.random_full(rng, 1 << 6), dc.random_full(rng, 1 << 6)
    pa, pb, small = lb.DensePolynomial(ctx, A), lb.DensePolynomial(ctx, B), lb.DensePolynomial(ctx, A[:32])
    other = lb.Context(0)
    foreign = lb.DensePolynomial(other, B)
    r6 = dc.random_full(rng, 6)
    # merge
    _raises(ctx, ERR_LENGTH, lambda: lb.DensePolynomial.merge(ctx, []))
    _raises(ctx, ERR_STRATEGY, lambda: lb.DensePolynomial.merge(ctx, [pa, foreign]))
    big = lb.DensePolynomial.eq(ctx, dc.random_full(rng, 27))  # 2^27 evaluations made on the device
    _raises(ctx, ERR_LENGTH, lambda: lb.DensePolynomial.merge(ctx, [big, big, pa]))
    del big
    out = ctypes.c_void_p()
    arr = (ctypes.c_void_p * 1)(pa._h.value)
    for args in ((None, 1, ctypes.byref(out)), (arr, 1, None)):
        before = ctx.launches
        assert lb.lib().lasso_poly_create_merge(ctx._h, args[0], ctypes.c_size_t(args[1]), args[2]) == ERR_LENGTH
        assert ctx.launches == before
    # evaluate_batch
    _raises(ctx, ERR_LENGTH, lambda: lb.DensePolynomial.evaluate_batch(ctx, [], r6))
    _raises(ctx, ERR_LENGTH, lambda: lb.DensePolynomial.evaluate_batch(ctx, [pa] * 65, r6))
    _raises(ctx, ERR_LENGTH, lambda: lb.DensePolynomial.evaluate_batch(ctx, [pa, small], r6))
    _raises(ctx, ERR_LENGTH, lambda: lb.DensePolynomial.evaluate_batch(ctx, [pa, pb], r6[:5]))
    _raises(ctx, ERR_VALUE, lambda: lb.DensePolynomial.evaluate_batch(ctx, [pa, pb], np.vstack([r6[:5], BAD])))
    _raises(ctx, ERR_STRATEGY, lambda: lb.DensePolynomial.evaluate_batch(ctx, [pa, foreign], r6))
    arr2 = (ctypes.c_void_p * 2)(pa._h.value, pb._h.value)
    before = ctx.launches
    assert lb.lib().lasso_poly_evaluate_batch(ctx._h, arr2, ctypes.c_size_t(2), r6.ctypes.data, ctypes.c_size_t(6), None) == ERR_LENGTH
    assert ctx.launches == before
    # the combined proof: merged polynomial of 3 x 2^6 -> 2^8 (r of 6 coordinates, 3 claims)
    m = lb.DensePolynomial.merge(ctx, [pa, pb, pa])
    gens8, _ = _gens(ctx, 8)
    gens5, _ = _gens(ctx, 5)
    evals = lb.DensePolynomial.evaluate_batch(ctx, [pa, pb, pa], r6)
    m_foreign = lb.DensePolynomial.merge(other, [foreign] * 4)
    cases = [
        (ERR_LENGTH, dict(r=r6[:5])), (ERR_LENGTH, dict(evals=evals[:1])), (ERR_LENGTH, dict(evals=np.vstack([evals] * 2))),
        (ERR_GENS, dict(gens=gens5)), (ERR_VALUE, dict(evals=np.vstack([evals[:2], BAD]))),
        (ERR_VALUE, dict(r=np.vstack([r6[:5], BAD]))), (ERR_STRATEGY, dict(combined=m_foreign)),
    ]
    for code, over in cases:
        t, tape = lb.Transcript(b"err"), lb.RandomTape(b"tape", TAPE_SEED)
        a = dict(combined=m, evals=evals, r=r6, gens=gens8)
        a.update(over)
        _raises(ctx, code, lambda: lb.CombinedTableEvalProof.prove(ctx, a["combined"], a["evals"], a["r"], a["gens"], t, tape),
                transcript=t, tape=tape)
    # n_evals == 0, proof_cap too small, a null transcript or tape, through the C ABI
    need = lb.CombinedTableEvalProof.proof_len(8)
    buf, n = np.zeros(need, dtype=np.uint8), ctypes.c_size_t(0)
    for n_evals, cap, use_t, use_tape in ((0, need, True, True), (3, need - 1, True, True), (3, need, False, True),
                                          (3, need, True, False)):
        t, tape = lb.Transcript(b"err"), lb.RandomTape(b"tape", TAPE_SEED)
        n.value = 0
        before = ctx.launches
        rc = lb.lib().lasso_combined_eval_prove(ctx._h, m._h, gens8._h, evals.ctypes.data, ctypes.c_size_t(n_evals),
                                                r6.ctypes.data, ctypes.c_size_t(6), t._h if use_t else None,
                                                tape._h if use_tape else None, buf.ctypes.data, ctypes.c_size_t(cap),
                                                ctypes.byref(n))
        assert rc == ERR_LENGTH and ctx.launches == before, (n_evals, cap, use_t, use_tape)
        if n_evals and cap < need:
            assert n.value == need
        twin_t, twin_tape = lb.Transcript(b"err"), lb.RandomTape(b"tape", TAPE_SEED)
        assert np.array_equal(t.challenge_scalar(b"x"), twin_t.challenge_scalar(b"x"))
        assert np.array_equal(tape.random_scalar(b"x"), twin_tape.random_scalar(b"x"))
    # the context still proves correctly
    _combined_both(ctx, [A, B, A], r6)
    del foreign, m_foreign
    other.close()
