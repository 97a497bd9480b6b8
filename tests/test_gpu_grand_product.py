"""Grand products over a caller's polynomials on the GPU: GrandProductCircuit and BatchedGrandProductArgument.prove on a
caller-held Transcript, bit for bit against the CPU oracle (oracle_dense/).  Every proof case compares the proof bytes,
the products, rand, the final claims and the transcript's next challenge.  Covers 1..32 circuits, num_vars 1..20 around
the tree build's 4096-element tail and the round kernels' q = 2048 switch, integer, full-width, l - 1 and zero values,
CUDA-tensor and eq polynomials, the caller's polynomials left unchanged, every argument error, the launch counts,
DensePolynomial.from_comb, the sizes of tests/golden/grand_product.json, and offline memory checking end to end on one
transcript."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import dense_poly_cases as dc
import grand_product_cases as gc
import oracle_dense_lib as od
import oracle_grand_product_lib as ogp
import oracle_lib as ol
import sumcheck_cases as sc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ERR_LENGTH, ERR_STRATEGY = 1, 4
L = ol.L_FR


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _values(kind, n, rng):
    if kind == "full":
        return dc.random_full(rng, n)
    if kind == "zero":  # a few zeros among full-width values: the product is 0
        Z = dc.random_full(rng, n)
        Z[rng.integers(0, n, size=max(1, n // 64))] = 0
        return Z
    if kind == "l-1":
        Z = dc.fr_from_u64(rng.integers(1, 256, size=n, dtype=np.uint64))
        Z[::2] = ol.fr_array([L - 1])[0]
        return Z
    return dc.fr_from_u64(rng.integers(1, 1 << 32, size=n, dtype=np.uint64))  # "u32"


def _both(ctx, arrays, polys=None, label=b"gp"):
    """GPU and oracle on the same inputs; asserts every output equal and returns (GPU proof, circuits)"""
    import lasso_b200 as lb

    if polys is None:
        polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    circuits = [lb.GrandProductCircuit(ctx, p) for p in polys]
    t = lb.Transcript(label)
    got = lb.BatchedGrandProductArgument.prove(ctx, circuits, t)
    o = od.Transcript(label)
    want = ogp.gp_prove(arrays, o)
    nv = polys[0].num_vars
    assert len(got.bytes) == ogp.proof_len(len(arrays), nv) == lb.BatchedGrandProductArgument.proof_len(len(arrays), nv)
    assert np.array_equal(np.stack([c.evaluate() for c in circuits]), want["products"])
    assert got.bytes == want["proof"]
    assert np.array_equal(got.r, want["r"])
    assert np.array_equal(got.claims, want["claims"])
    assert np.array_equal(t.challenge_scalar(b"after"), o.challenge_scalar(b"after"))
    return got, circuits


@pytest.mark.parametrize("n", list(range(1, 33)))
def test_batch_sizes(ctx, n):
    rng = np.random.default_rng(n)
    _both(ctx, [dc.random_full(rng, 1 << 5) for _ in range(n)])


@pytest.mark.parametrize("nv,n", [(1, 1), (1, 32), (2, 1), (2, 7), (3, 2), (3, 32), (12, 3), (12, 32), (13, 2), (13, 17),
                                  (14, 4), (20, 2)])
def test_num_vars(ctx, nv, n):
    rng = np.random.default_rng(100 * nv + n)
    _both(ctx, [dc.random_full(rng, 1 << nv) for _ in range(n)])


@pytest.mark.parametrize("kind", ["u32", "full", "l-1", "zero"])
def test_value_kinds(ctx, kind):
    rng = np.random.default_rng(len(kind))
    got, circuits = _both(ctx, [_values(kind, 1 << 12, rng) for _ in range(3)])
    if kind == "zero":
        assert all(ol.fr_ints(c.evaluate()) == [0] for c in circuits)


def test_device_tensors(ctx):
    import torch

    import lasso_b200 as lb

    rng = np.random.default_rng(11)
    arrays = [dc.random_full(rng, 1 << 13) for _ in range(3)]
    wide = torch.zeros((1 << 13, 6), dtype=torch.int64, device="cuda")
    wide[:, 1:5] = torch.from_numpy(arrays[2].view(np.int64)).cuda()
    polys = [lb.DensePolynomial(ctx, torch.from_numpy(arrays[0].view(np.int64)).cuda()), lb.DensePolynomial(ctx, arrays[1]),
             lb.DensePolynomial(ctx, wide[:, 1:5])]
    torch.cuda.synchronize()
    _both(ctx, arrays, polys=polys)


def test_eq_leaves(ctx):
    import lasso_b200 as lb

    rng = np.random.default_rng(12)
    taus = [dc.random_full(rng, 9) for _ in range(2)]
    _both(ctx, [sc.eq_evals(tau) for tau in taus], polys=[lb.DensePolynomial.eq(ctx, tau) for tau in taus])


def _gens(ctx, nv):
    import lasso_b200 as lb

    stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
    return lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream), stream


@pytest.mark.parametrize("nv", [1, 2, 3, 13])
def test_polynomials_untouched(ctx, nv):
    """creating and proving leave the caller's polynomials as they were (evaluation at a random point, commitment), and
    the final claims are the polynomials evaluated at rand"""
    import lasso_b200 as lb

    rng = np.random.default_rng(13 + nv)
    gens, _ = _gens(ctx, nv)
    arrays = [_values(kind, 1 << nv, rng) for kind in ("full", "u32", "l-1")]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    x = dc.random_full(rng, nv)
    before = [(p.evaluate(x).tobytes(), p.commit(gens)) for p in polys]
    got, _ = _both(ctx, arrays, polys=polys)
    assert [(p.evaluate(x).tobytes(), p.commit(gens)) for p in polys] == before
    for p, claim in zip(polys, got.claims):
        assert np.array_equal(p.evaluate(got.r), claim)


def _eq_launches(ell):
    return 1 if ell <= 11 else (3 if ell <= 22 else 5)


def _create_launches(nv):
    """DESIGN.md §3.10: layer 1 from the caller's buffer, then the tree from N/2 (one launch per layer above 4096
    elements, one tail kernel); N = 2: one read-back"""
    if nv == 1:
        return 1
    return 2 + sum(1 for k in range(nv - 1, 0, -1) if (1 << k) > 4096)


def _prove_launches(nv):
    """DESIGN.md §3.10: per layer with ell rounds the eq table, then the top layer's pack and read-back of its heads
    (ell = 0) or the first evaluation and one kernel per round; layer 0 adds the evaluation after its out-of-place first
    bind (nv >= 3), or the pack and read-back of its heads (nv = 2)"""
    extra = 1 if nv >= 3 else (2 if nv == 2 else 0)
    return sum(_eq_launches(ell) + (2 if ell == 0 else 1 + ell) for ell in range(nv)) + extra


@pytest.mark.parametrize("nv,n", [(1, 1), (2, 3), (3, 1), (12, 2), (14, 5), (20, 2), (24, 1)])
def test_launch_count(ctx, nv, n):
    import lasso_b200 as lb

    rng = np.random.default_rng(nv)
    polys = [lb.DensePolynomial(ctx, dc.random_full(rng, 1 << nv)) for _ in range(n)]
    before = ctx.launches
    circuits = [lb.GrandProductCircuit(ctx, p) for p in polys]
    assert ctx.launches - before == n * _create_launches(nv)
    before = ctx.launches
    lb.BatchedGrandProductArgument.prove(ctx, circuits, lb.Transcript(b"n"))
    assert ctx.launches - before == _prove_launches(nv)


def test_errors(ctx):
    """each error before any launch with the transcript untouched, then a correct proof on the same context"""
    import lasso_b200 as lb

    rng = np.random.default_rng(15)
    A, B = dc.random_full(rng, 1 << 6), dc.random_full(rng, 1 << 6)
    pa, pb, small = lb.DensePolynomial(ctx, A), lb.DensePolynomial(ctx, B), lb.DensePolynomial(ctx, A[:32])
    other = lb.Context(0)
    foreign = lb.GrandProductCircuit(other, lb.DensePolynomial(other, B))
    ca, cs = lb.GrandProductCircuit(ctx, pa), lb.GrandProductCircuit(ctx, small)
    proven = lb.GrandProductCircuit(ctx, pb)
    lb.BatchedGrandProductArgument.prove(ctx, [proven], lb.Transcript(b"once"))
    many = [lb.GrandProductCircuit(ctx, pa) for _ in range(33)]
    cases = [
        ([], ERR_STRATEGY), (many, ERR_STRATEGY), ([ca, foreign], ERR_STRATEGY), ([ca, proven], ERR_STRATEGY),
        ([ca, ca], ERR_STRATEGY), ([ca, cs], ERR_LENGTH),
    ]
    for circuits, code in cases:
        t, twin = lb.Transcript(b"err"), lb.Transcript(b"err")
        before = ctx.launches
        with pytest.raises(lb.LassoError) as e:
            lb.BatchedGrandProductArgument.prove(ctx, circuits, t)
        assert e.value.code == code, (len(circuits), str(e.value))
        assert ctx.launches == before
        assert np.array_equal(t.challenge_scalar(b"x"), twin.challenge_scalar(b"x"))
    # proof_cap too small and a null transcript, through the C ABI
    arr = (ctypes.c_void_p * 1)(ca._h.value)
    need = ogp.proof_len(1, 6)
    out, r, claims, n = np.zeros(need, dtype=np.uint8), np.zeros((6, 4), dtype=np.uint64), np.zeros((1, 4), dtype=np.uint64), ctypes.c_size_t(0)
    for cap, tr in ((need - 1, lb.Transcript(b"err")), (need, None)):
        twin = lb.Transcript(b"err")
        before = ctx.launches
        rc = lb.lib().lasso_gp_prove(ctx._h, arr, ctypes.c_size_t(1), tr._h if tr else None, out.ctypes.data,
                                     ctypes.c_size_t(cap), ctypes.byref(n), r.ctypes.data, claims.ctypes.data)
        assert rc == ERR_LENGTH and n.value == need and ctx.launches == before
        if tr:
            assert np.array_equal(tr.challenge_scalar(b"x"), twin.challenge_scalar(b"x"))
    # creation: num_vars 0, a polynomial of another context
    for p, code in ((lb.DensePolynomial(ctx, A[:1]), ERR_LENGTH), (lb.DensePolynomial(other, A), ERR_STRATEGY)):
        before = ctx.launches
        with pytest.raises(lb.LassoError) as e:
            lb.GrandProductCircuit(ctx, p)
        assert e.value.code == code and ctx.launches == before
    # from_comb: inputs that do not match the combining function, different num_vars, another context
    comb = lb.Comb(lambda v: v[0] * v[1], 2)
    for polys, code in (([pa], ERR_STRATEGY), ([pa, small], ERR_LENGTH), ([pa, lb.DensePolynomial(other, B)], ERR_STRATEGY)):
        before = ctx.launches
        with pytest.raises(lb.LassoError) as e:
            lb.DensePolynomial.from_comb(ctx, comb, polys)
        assert e.value.code == code and ctx.launches == before
    # the context still proves correctly
    _both(ctx, [A, B])
    del foreign, many
    other.close()


GOLDEN = json.load(open(os.path.join(HERE, "golden", "grand_product.json")))


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_at_size_against_golden(ctx, name):
    """the seeded cases of tests/golden/grand_product.json: SHA-256 of proof || products || rand || claims and the next
    challenge equal the oracle's"""
    import lasso_b200 as lb

    nv, arrays = gc.golden_inputs(name)
    g = GOLDEN["cases"][name]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    del arrays
    circuits = [lb.GrandProductCircuit(ctx, p) for p in polys]
    t = lb.Transcript(gc.TRANSCRIPT_LABEL)
    got = lb.BatchedGrandProductArgument.prove(ctx, circuits, t)
    res = dict(proof=got.bytes, products=np.stack([c.evaluate() for c in circuits]), r=got.r, claims=got.claims)
    assert len(got.bytes) == g["proof_len"]
    assert hashlib.sha256(gc.digest_input(res)).hexdigest() == g["sha256"]
    assert t.challenge_scalar(b"after").tobytes().hex() == g["after_challenge_hex"]


@pytest.mark.parametrize("nv", [0, 1, 5, 13])
def test_from_comb(ctx, nv):
    """DensePolynomial.from_comb equals the oracle's pointwise map (evaluated at a random point), and committing it gives
    the bytes of the same values made with DensePolynomial(ctx, values)"""
    import lasso_b200 as lb

    rng = np.random.default_rng(40 + nv)
    arrays = [_values(kind, 1 << nv, rng) for kind in ("full", "u32", "l-1")]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    comb = lb.Comb(sc.FUNCS["consts"][0], 3)
    before = ctx.launches
    q = lb.DensePolynomial.from_comb(ctx, comb, polys)
    assert ctx.launches - before == 1 and q.num_vars == nv
    want = ogp.comb_map(arrays, comb.program, comb.constants)
    x = dc.random_full(rng, nv)
    assert np.array_equal(q.evaluate(x), od.evaluate(want, x))
    if nv:
        gens, _ = _gens(ctx, nv)
        assert q.commit(gens) == lb.DensePolynomial(ctx, want).commit(gens)


def _h(a, v, t, gamma, tau):
    return (t * gamma * gamma + v * gamma + a - tau) % L


def test_offline_memory_checking(ctx):
    """A caller's memory of 2^10 cells read 2^14 times, proven on one transcript: commit the addresses a, values v and
    timestamps t of the reads (and the memory's values and final timestamps), draw gamma and tau, form the fingerprints
    with from_comb, append the four products, prove [read, write] and [init, final] as two batched grand products, open
    every committed polynomial at its rand.  The oracle's replay accepts every part; changing one read value breaks the
    multiset equation init * write = read * final."""
    import lasso_b200 as lb

    log_m, log_s = 10, 14
    M, S = 1 << log_m, 1 << log_s
    rng = np.random.default_rng(77)
    mem = rng.integers(0, 1 << 32, size=M, dtype=np.uint64)
    addr = rng.integers(0, M, size=S, dtype=np.uint64)
    counter = np.zeros(M, dtype=np.uint64)
    ts = np.zeros(S, dtype=np.uint64)
    for j, a in enumerate(addr):  # read timestamp = the cell's counter; the write stores it + 1
        ts[j] = counter[a]
        counter[a] += 1
    cols = {"a": addr, "v": mem[addr], "t": ts, "idx": np.arange(M, dtype=np.uint64), "mem": mem, "fin": counter}
    Z = {k: dc.fr_from_u64(x) for k, x in cols.items()}
    P = {k: lb.DensePolynomial(ctx, z) for k, z in Z.items()}
    (gens_s, stream_s), (gens_m, stream_m) = _gens(ctx, log_s), _gens(ctx, log_m)
    committed = {"a": gens_s, "v": gens_s, "t": gens_s, "mem": gens_m, "fin": gens_m}
    comms = {k: P[k].commit(g) for k, g in committed.items()}
    seed = ol.fr_array([5])[0]
    t, tape = lb.Transcript(b"memory"), lb.RandomTape(b"proof", seed)
    for k in committed:
        t.append_poly_commitment(k.encode(), comms[k])
    r_hash = t.challenge_vector(b"challenge_r_hash", 2)
    gamma, tau = ol.fr_ints(r_hash)

    def fingerprints(P):
        g2 = gamma * gamma % L
        read = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda x: x[2] * g2 + x[1] * gamma + x[0] - tau, 3), [P["a"], P["v"], P["t"]])
        write = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda x: x[2] * g2 + x[1] * gamma + x[0] + (g2 - tau), 3),
                                             [P["a"], P["v"], P["t"]])
        init = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda x: x[1] * gamma + x[0] - tau, 2), [P["idx"], P["mem"]])
        final = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda x: x[2] * g2 + x[1] * gamma + x[0] - tau, 3),
                                             [P["idx"], P["mem"], P["fin"]])
        return {"init": init, "read": read, "write": write, "final": final}

    fp = fingerprints(P)
    C = {k: lb.GrandProductCircuit(ctx, p) for k, p in fp.items()}
    products = {k: c.evaluate() for k, c in C.items()}
    for k in ("init", "read", "write", "final"):
        t.append_scalar(("claim_hash_" + k).encode(), products[k])
    proof_rw = lb.BatchedGrandProductArgument.prove(ctx, [C["read"], C["write"]], t)
    proof_if = lb.BatchedGrandProductArgument.prove(ctx, [C["init"], C["final"]], t)
    openings = {}
    for k in committed:
        r = proof_rw.r if committed[k] is gens_s else proof_if.r
        y = P[k].evaluate(r)
        openings[k] = (y, lb.PolyEvalProof.prove(ctx, P[k], r, y, committed[k], t, tape).bytes)
    end = t.challenge_scalar(b"end")

    # the verifier's replay
    v = od.Transcript(b"memory")
    for k in committed:
        v.append_poly_commitment(k.encode(), comms[k])
    assert np.array_equal(v.challenge_vector(b"challenge_r_hash", 2), r_hash)
    for k in ("init", "read", "write", "final"):
        v.append_scalar(("claim_hash_" + k).encode(), products[k])
    hi, hr, hw, hf = (ol.fr_ints(products[k])[0] for k in ("init", "read", "write", "final"))
    assert hi * hw % L == hr * hf % L
    rc, claims_rw, r_rw = ogp.gp_verify(proof_rw.bytes, np.stack([products["read"], products["write"]]), log_s, v)
    assert rc == 0 and np.array_equal(r_rw, proof_rw.r) and np.array_equal(claims_rw, proof_rw.claims)
    rc, claims_if, r_if = ogp.gp_verify(proof_if.bytes, np.stack([products["init"], products["final"]]), log_m, v)
    assert rc == 0 and np.array_equal(r_if, proof_if.r) and np.array_equal(claims_if, proof_if.claims)
    ev = {k: ol.fr_ints(y)[0] for k, (y, _) in openings.items()}
    idx_r = ol.fr_ints(od.evaluate(Z["idx"], r_if))[0]  # the cell index is public: the verifier evaluates it
    assert ol.fr_ints(claims_rw) == [_h(ev["a"], ev["v"], ev["t"], gamma, tau), _h(ev["a"], ev["v"], ev["t"] + 1, gamma, tau)]
    assert ol.fr_ints(claims_if) == [_h(idx_r, ev["mem"], 0, gamma, tau), _h(idx_r, ev["mem"], ev["fin"], gamma, tau)]
    for k in committed:
        nv, stream, r = (log_s, stream_s, r_rw) if committed[k] is gens_s else (log_m, stream_m, r_if)
        assert od.verify(stream, nv, comms[k], openings[k][1], r, openings[k][0], v) == 0, k
    assert np.array_equal(v.challenge_scalar(b"end"), end)

    # one read value changed: the multiset equation fails
    bad = cols["v"].copy()
    bad[S // 3] ^= np.uint64(1)
    Pb = dict(P, v=lb.DensePolynomial(ctx, dc.fr_from_u64(bad)))
    pb = {k: ol.fr_ints(lb.GrandProductCircuit(ctx, p).evaluate())[0] for k, p in fingerprints(Pb).items()}
    assert pb["init"] * pb["write"] % L != pb["read"] * pb["final"] % L
