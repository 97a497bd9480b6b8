"""Zero-knowledge sumchecks on the GPU: MultiCommitGens commitments, DotProductProof.prove and
ZKSumcheckInstanceProof.prove bit for bit against the CPU oracle (oracle_dense/), the oracle's verifiers accepting the
GPU's bytes, a composed Spartan-style check over hiding commitments and openings on one transcript and tape, every
argument error with nothing moved, the launch counts of DESIGN §3.16, and the calls on a sharded context."""
import ctypes
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import dense_poly_cases as dc  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_hiding_lib as oh  # noqa: E402
import oracle_lib as ol  # noqa: E402
import oracle_zk_lib as oz  # noqa: E402
import sumcheck_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu
ERR_LENGTH, ERR_STRATEGY, ERR_GENS, ERR_VALUE = 1, 4, 5, 8
FUSED_MIN_Q = 1 << 15
SEED = ol.fr_array([777])[0]
MARK = "ZK_SHARDED"


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _dot_gens(ctx, n, label=b"zk_gens"):
    """-> (gens_1, gens_n) on the GPU and their (G, h) pairs for the oracle, DotProductProofGens::new(n, label)"""
    import lasso_b200 as lb

    g = lb.DotProductProofGens.new(ctx, n, label)
    stream = ol.generators(n + 2, label)
    assert np.array_equal(g.gens_n.G, stream[:n]) and np.array_equal(g.gens_1.h, stream[n + 1])
    return g.gens_1, g.gens_n, oz.dot_gens(stream, n)


@pytest.mark.parametrize("n", [1, 2, 17, 1024])
def test_commit(ctx, n):
    import lasso_b200 as lb

    rng = np.random.default_rng(n)
    stream = ol.generators(n + 1, b"mc")
    g = lb.MultiCommitGens(ctx, stream[:n], stream[n])
    assert lb.lib().lasso_mc_gens_n(g._h) == n
    for s, b in ((ol.rand_fr(rng, n), ol.rand_fr(rng, 1)[0]), (np.zeros((n, 4), np.uint64), np.zeros(4, np.uint64)),
                 (ol.rand_fr(rng, n), np.zeros(4, np.uint64)), (np.zeros((n, 4), np.uint64), ol.rand_fr(rng, 1)[0])):
        assert g.commit(s, b) == oz.commit(oz.mc_gens(stream, n), s, b)
    assert lb.MultiCommitGens.new(ctx, n, b"mc").commit(s, b) == g.commit(s, b)


@pytest.mark.parametrize("n", [1, 3, 17, 200])
def test_dot_product_proof(ctx, n):
    import lasso_b200 as lb

    rng = np.random.default_rng(20 + n)
    g1, gn, (og1, ogn) = _dot_gens(ctx, n)
    x, a = ol.rand_fr(rng, n), ol.rand_fr(rng, n)
    bx, by = ol.rand_fr(rng, 2)
    y = ol.fr_array([sum(p * q for p, q in zip(ol.fr_ints(x), ol.fr_ints(a))) % ol.L_FR])[0]
    t, tape = lb.Transcript(b"dp"), lb.RandomTape(b"tape", SEED)
    o, otape = od.Transcript(b"dp"), od.RandomTape(b"tape", SEED)
    before = ctx.launches
    proof, Cx, Cy = lb.DotProductProof.prove(ctx, g1, gn, t, tape, x, bx, a, y, by)
    assert ctx.launches - before == 4
    want = oz.dot_prove(og1, ogn, o, otape, x, bx, a, y, by)
    assert (proof, Cx, Cy) == want
    assert np.array_equal(t.challenge_scalar(b"after"), o.challenge_scalar(b"after"))
    assert np.array_equal(tape.random_scalar(b"after"), otape.random_scalar(b"after"))
    assert oz.dot_verify(og1, ogn, proof, a, Cx, Cy, od.Transcript(b"dp")) == 0


def _zk_both(ctx, fn, k, arrays, num_rounds=None, degree=None, polys=None, label=b"zk"):
    """GPU and oracle ZK sumchecks on the same inputs: every output equal, and the oracle's verifier accepts"""
    import lasso_b200 as lb

    comb = lb.Comb(fn, k, degree)
    if polys is None:
        polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    rounds = polys[0].num_vars if num_rounds is None else num_rounds
    g1, gn, (og1, ogn) = _dot_gens(ctx, comb.degree + 1)
    bc = ol.rand_fr(np.random.default_rng(rounds), 1)[0]
    t, tape = lb.Transcript(label), lb.RandomTape(b"tape", SEED)
    got = lb.ZKSumcheckInstanceProof.prove(ctx, comb, polys, num_rounds, bc, g1, gn, t, tape)
    o, otape = od.Transcript(label), od.RandomTape(b"tape", SEED)
    want = oz.zk_prove(arrays, rounds, comb.program, comb.constants, comb.degree, bc, og1, ogn, o, otape)
    assert len(got.data) == lb.ZKSumcheckInstanceProof.proof_len(rounds, comb.degree)
    assert got.data == want["proof"]
    for f in ("r", "final_evals", "claim", "blind_eval"):
        assert np.array_equal(getattr(got, f), want[f]), f
    assert got.comm_claim == want["comm_claim"]
    assert np.array_equal(t.challenge_scalar(b"after"), o.challenge_scalar(b"after"))
    assert np.array_equal(tape.random_scalar(b"after"), otape.random_scalar(b"after"))
    rc, _, vr = oz.zk_verify(got.data, got.comm_claim, rounds, comb.degree, og1, ogn, od.Transcript(label))
    assert rc == 0 and np.array_equal(vr, got.r)
    return got


def _kfun(k):
    return lambda v: sum((i + 1) * v[i] for i in range(k)) * v[k - 1] + v[0]


@pytest.mark.parametrize("k", [1, 2, 5, 9, 16])
def test_inputs(ctx, k):
    rng = np.random.default_rng(k)
    _zk_both(ctx, _kfun(k), k, [dc.random_full(rng, 1 << 6) for _ in range(k)])


@pytest.mark.parametrize("d", list(range(1, 17)))
def test_degrees(ctx, d):
    rng = np.random.default_rng(100 + d)
    arrays = [dc.random_full(rng, 1 << 5) for _ in range(2)]
    fn = (lambda v: sc.prod9([v[i % 2] for i in range(d)])) if d > 1 else (lambda v: v[0] + v[1])
    _zk_both(ctx, fn, 2, arrays)


@pytest.mark.parametrize("nv,rounds", [(1, 1), (2, 1), (3, 3), (8, 5), (12, 12), (16, 16), (17, 4), (20, 20)])
def test_num_vars_and_rounds(ctx, nv, rounds):
    """eq(tau) (A B - C) with eq made on the GPU, full-width and u32-mirrored inputs"""
    import lasso_b200 as lb

    rng = np.random.default_rng(1000 + nv)
    tau = dc.random_full(rng, nv)
    arrays = [sc.eq_evals(tau), dc.random_full(rng, 1 << nv),
              dc.fr_from_u64(rng.integers(0, 1 << 32, size=1 << nv, dtype=np.uint64)), dc.random_full(rng, 1 << nv)]
    polys = [lb.DensePolynomial.eq(ctx, tau)] + [lb.DensePolynomial(ctx, a) for a in arrays[1:]]
    got = _zk_both(ctx, sc.spartan, 4, arrays, num_rounds=rounds, polys=polys)
    if rounds == nv:  # the final evaluations are the polynomials at r, which are unchanged
        for p, v in zip(polys, got.final_evals):
            assert np.array_equal(p.evaluate(got.r), v)


def test_same_poly_and_tensors(ctx):
    import torch

    import lasso_b200 as lb

    rng = np.random.default_rng(7)
    A, B = dc.random_full(rng, 1 << 10), dc.random_full(rng, 1 << 10)
    p = lb.DensePolynomial(ctx, A)
    _zk_both(ctx, lambda v: v[0] * v[1] - v[2] * 3, 3, [A, A, A], polys=[p, p, p], num_rounds=4)
    q = lb.DensePolynomial(ctx, torch.from_numpy(B.view(np.int64)).cuda())
    torch.cuda.synchronize()
    _zk_both(ctx, lambda v: v[0] * v[1], 2, [A, B], polys=[p, q])


def test_spartan_composition(ctx):
    """hiding commitments of A, B, C -> tau -> ZK sumcheck of eq(tau) (A B - C) with claim 0 -> hiding openings of A, B,
    C at r, on one transcript and tape: equal to the oracle's run, and its verifiers accept every part"""
    import lasso_b200 as lb

    nv = 10
    rng = np.random.default_rng(14)
    A, B = dc.random_full(rng, 1 << nv), dc.fr_from_u64(rng.integers(0, 1 << 32, size=1 << nv, dtype=np.uint64))
    C = ol.fr_array([a * b % ol.L_FR for a, b in zip(ol.fr_ints(A), ol.fr_ints(B))])
    stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
    pgens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream)
    g1, gn, (og1, ogn) = _dot_gens(ctx, 4)
    t, tape = lb.Transcript(b"spartan"), lb.RandomTape(b"proof", SEED)
    o, otape = od.Transcript(b"spartan"), od.RandomTape(b"proof", SEED)
    polys = [lb.DensePolynomial(ctx, X) for X in (A, B, C)]
    comms, blinds = [], []
    for X, p in zip((A, B, C), polys):
        cm, bl = p.commit_hiding(pgens, tape)
        ocm, obl = oh.commit_hiding(X, stream, otape)
        assert cm == ocm and np.array_equal(bl, obl)
        comms.append(cm)
        blinds.append(bl)
    for x in (t, o):
        for name, cm in zip((b"A", b"B", b"C"), comms):
            x.append_poly_commitment(name, cm)
    tau = t.challenge_vector(b"tau", nv)
    assert np.array_equal(tau, o.challenge_vector(b"tau", nv))
    comb = lb.Comb(sc.spartan, 4)
    bc = np.zeros(4, dtype=np.uint64)
    zk = lb.ZKSumcheckInstanceProof.prove(ctx, comb, [lb.DensePolynomial.eq(ctx, tau)] + polys, nv, bc, g1, gn, t, tape)
    want = oz.zk_prove([sc.eq_evals(tau), A, B, C], nv, comb.program, comb.constants, 3, bc, og1, ogn, o, otape)
    assert zk.data == want["proof"] and ol.fr_ints(zk.claim) == [0]
    r = zk.r
    ev_blinds = ol.rand_fr(rng, 3)
    opens = [lb.PolyEvalProof.prove(ctx, p, r, zk.final_evals[1 + i], pgens, t, tape, blinds=blinds[i], blind_Zr=ev_blinds[i])
             for i, p in enumerate(polys)]
    wants = [oh.prove_hiding(X, r, want["final_evals"][1 + i], stream, o, otape, blinds[i], ev_blinds[i])
             for i, X in enumerate((A, B, C))]
    assert [(p.bytes, p.C_Zr) for p in opens] == wants
    assert np.array_equal(t.challenge_scalar(b"end"), o.challenge_scalar(b"end"))
    # the verifier's replay on one transcript
    v = od.Transcript(b"spartan")
    for name, cm in zip((b"A", b"B", b"C"), comms):
        v.append_poly_commitment(name, cm)
    v.challenge_vector(b"tau", nv)
    rc, _, vr = oz.zk_verify(zk.data, zk.comm_claim, nv, 3, og1, ogn, v)
    assert rc == 0 and np.array_equal(vr, r)
    for i, cm in enumerate(comms):
        assert oh.verify(stream, nv, cm, opens[i].bytes, vr, opens[i].C_Zr, v) == 0


def _plain_launches(nv, rounds):
    fused = sum(1 for j in range(1, rounds) if (1 << (nv - j - 1)) >= FUSED_MIN_Q)
    return 1 + fused + 2 * (rounds - 1 - fused) + 1


def _zk_launches(nv, rounds):
    """DESIGN §3.16: the plain call's, two per delta MSM (two rounds each) and six per round"""
    return _plain_launches(nv, rounds) + 2 * ((rounds + 1) // 2) + 6 * rounds


@pytest.mark.parametrize("nv,rounds", [(1, 1), (4, 3), (18, 18), (20, 20)])
def test_launch_count(ctx, nv, rounds):
    import lasso_b200 as lb

    rng = np.random.default_rng(nv)
    polys = [lb.DensePolynomial(ctx, dc.random_full(rng, 1 << nv)) for _ in range(2)]
    comb = lb.Comb(lambda v: v[0] * v[1], 2)
    g1, gn, _ = _dot_gens(ctx, 3)
    before = ctx.launches
    lb.ZKSumcheckInstanceProof.prove(ctx, comb, polys, rounds, np.zeros(4, np.uint64), g1, gn, lb.Transcript(b"n"),
                                     lb.RandomTape(b"t", SEED))
    assert ctx.launches - before == _zk_launches(nv, rounds)
    before = ctx.launches
    g1.commit(ol.rand_fr(rng, 1), ol.rand_fr(rng, 1)[0])
    assert ctx.launches - before == 2


def test_errors(ctx):
    """each error before any launch with the transcript and the tape untouched"""
    import lasso_b200 as lb

    L = lb.lib()
    rng = np.random.default_rng(15)
    A, B = dc.random_full(rng, 1 << 6), dc.random_full(rng, 1 << 6)
    pa, pb = lb.DensePolynomial(ctx, A), lb.DensePolynomial(ctx, B)
    comb = lb.Comb(lambda v: v[0] * v[1], 2)
    g1, g3, _ = _dot_gens(ctx, 3)
    _, g4, _ = _dot_gens(ctx, 4)
    other = lb.Context(0)
    foreign = lb.MultiCommitGens.new(other, 3, b"zk_gens")
    bad = ol.fr_array([0])[0].copy()
    bad[:] = np.uint64(0xFFFFFFFFFFFFFFFF)
    good = np.zeros(4, dtype=np.uint64)
    P = lambda a: a.ctypes.data  # noqa: E731
    arr = (ctypes.c_void_p * 2)(pa._h.value, pb._h.value)
    need = lb.ZKSumcheckInstanceProof.proof_len(6, 2)
    out = np.zeros(need, dtype=np.uint8)
    r, fin = np.zeros((6, 4), np.uint64), np.zeros((2, 4), np.uint64)

    def zk(gens_1, gens_n, bc, cap, tape_ok=True, n=None):
        t, tape = lb.Transcript(b"e"), lb.RandomTape(b"t", SEED)
        ln = ctypes.c_size_t(0)
        rc = L.lasso_zk_sumcheck_prove(ctx._h, comb._h, arr, ctypes.c_size_t(2), ctypes.c_size_t(6), P(bc),
                                       gens_1._h if gens_1 else None, gens_n._h if gens_n else None, t._h,
                                       tape._h if tape_ok else None, P(out), ctypes.c_size_t(cap), ctypes.byref(ln), P(r),
                                       P(fin), None, None, None)
        return rc, ln.value, t, tape

    cases = [((None, g3, good, need), ERR_GENS), ((g1, None, good, need), ERR_GENS), ((g3, g3, good, need), ERR_GENS),
             ((g1, g4, good, need), ERR_GENS), ((g1, foreign, good, need), ERR_GENS), ((g1, g3, bad, need), ERR_VALUE),
             ((g1, g3, good, need - 1), ERR_LENGTH)]
    for args, code in cases:
        before = ctx.launches
        rc, ln, t, tape = zk(*args)
        assert rc == code, (args, rc)
        assert ctx.launches == before
        assert np.array_equal(t.challenge_scalar(b"x"), lb.Transcript(b"e").challenge_scalar(b"x"))
        assert np.array_equal(tape.random_scalar(b"x"), lb.RandomTape(b"t", SEED).random_scalar(b"x"))
        if code == ERR_LENGTH:
            assert ln == need
    before = ctx.launches
    assert zk(g1, g3, good, need, tape_ok=False)[0] == ERR_LENGTH and ctx.launches == before
    # dot product proof: gens_n.n != n, a non-canonical y, a short buffer
    x = ol.rand_fr(rng, 3)
    for gn, y, cap, code in ((g4, good, 232, ERR_GENS), (g3, bad, 232, ERR_VALUE), (g3, good, 231, ERR_LENGTH)):
        t, tape = lb.Transcript(b"e"), lb.RandomTape(b"t", SEED)
        o, ln = np.zeros(232, np.uint8), ctypes.c_size_t(0)
        cx, cy = np.zeros(32, np.uint8), np.zeros(32, np.uint8)
        before = ctx.launches
        rc = L.lasso_dot_product_prove(ctx._h, g1._h, gn._h, t._h, tape._h, P(x), P(good), P(x), ctypes.c_size_t(3), P(y),
                                       P(good), P(o), ctypes.c_size_t(cap), ctypes.byref(ln), P(cx), P(cy))
        assert rc == code and ctx.launches == before
        assert np.array_equal(t.challenge_scalar(b"x"), lb.Transcript(b"e").challenge_scalar(b"x"))
        assert np.array_equal(tape.random_scalar(b"x"), lb.RandomTape(b"t", SEED).random_scalar(b"x"))
    # gens and commitments
    for n in (0, 1025):
        with pytest.raises(lb.LassoError) as e:
            lb.MultiCommitGens(ctx, np.zeros((n, 8), np.uint64), np.zeros(8, np.uint64))
        assert e.value.code == ERR_LENGTH
    with pytest.raises(lb.LassoError) as e:
        g3.commit(x, bad)
    assert e.value.code == ERR_VALUE
    rc = L.lasso_mc_commit(ctx._h, g3._h, P(x), ctypes.c_size_t(2), P(good), P(np.zeros(32, np.uint8)))
    assert rc == ERR_GENS
    _zk_both(ctx, lambda v: v[0] * v[1], 2, [A, B], polys=[pa, pb])
    del foreign
    other.close()


def _zk_calls(ctx):
    """gens, commit and dot-product bytes, and the ZK sumcheck's return code"""
    import lasso_b200 as lb

    rng = np.random.default_rng(33)
    g = lb.DotProductProofGens.new(ctx, 5, b"zk_gens")
    x, a = ol.rand_fr(rng, 5), ol.rand_fr(rng, 5)
    bx, y, by = ol.rand_fr(rng, 3)
    comm = g.gens_n.commit(x, bx)
    dp = lb.DotProductProof.prove(ctx, g.gens_1, g.gens_n, lb.Transcript(b"s"), lb.RandomTape(b"t", SEED), x, bx, a, y, by)
    g3 = lb.DotProductProofGens.new(ctx, 3, b"zk_gens").gens_n
    polys = [lb.DensePolynomial(ctx, dc.random_full(rng, 1 << 8)) for _ in range(2)]
    try:
        lb.ZKSumcheckInstanceProof.prove(ctx, lb.Comb(lambda v: v[0] * v[1], 2), polys, 8, np.zeros(4, np.uint64),
                                         g.gens_1, g3, lb.Transcript(b"s"), lb.RandomTape(b"t", SEED))
        code = 0
    except lb.LassoError as e:
        code = e.code
    return comm, dp, code


def test_sharded_two_ranks_one_gpu():
    """on 2 ranks of one GPU the gens, commit and dot-product bytes equal a single-GPU context's; the ZK sumcheck
    returns LASSO_ERR_STRATEGY"""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert MARK + " PASS" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]


def _worker():
    import torch
    import torch.distributed as dist

    import lasso_b200 as lb

    rank, G = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo")
    single = [None]
    if rank == 0:
        c1 = lb.Context(0)
        single = [_zk_calls(c1)]
        c1.close()
    dist.broadcast_object_list(single, src=0)
    c = lb.Context(0)
    c.init_comm()
    got = [None] * G
    dist.all_gather_object(got, _zk_calls(c))
    if rank == 0:
        want = single[0]
        fails = [g for g, x in enumerate(got) if x[:2] != want[:2] or x[2] != ERR_STRATEGY or want[2] != 0]
        print(MARK, "PASS" if not fails else "FAIL %r" % fails, flush=True)
    dist.barrier()
    c.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker()
