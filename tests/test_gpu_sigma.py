"""Σ-protocols of committed scalars on the GPU: KnowledgeProof, EqualityProof and ProductProof bit for bit against the
CPU oracle (oracle_dense/), with random values and the edges; the oracle's verifiers accepting the GPU's bytes; one
short MSM (2 launches) per proof; every argument error with nothing moved; 2 ranks on one GPU; and the end of a Spartan
phase one composed on one transcript and tape: ZK sumcheck, knowledge, product and equality proofs, replayed by the
verifier (DESIGN §3.17)."""
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
import oracle_lib as ol  # noqa: E402
import oracle_sigma_lib as osg  # noqa: E402
import oracle_zk_lib as oz  # noqa: E402
import sumcheck_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu
ERR_LENGTH, ERR_GENS, ERR_VALUE = 1, 5, 8
L = ol.L_FR
SEED = ol.fr_array([919])[0]
MARK = "SIGMA_SHARDED"


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _fr(v):
    return ol.fr_array([v % L])[0]


def _gens(ctx, label=b"sigma_gens"):
    """gens_1 of DotProductProofGens::new(3, label), the gens a ZK sumcheck's comm_evals are on -> (GPU, oracle)"""
    import lasso_b200 as lb

    g = lb.DotProductProofGens.new(ctx, 3, label).gens_1
    og = oz.dot_gens(ol.generators(5, label), 3)[0]
    assert np.array_equal(g.G, og[0]) and np.array_equal(g.h, og[1])
    return g, og


def _provers():
    import lasso_b200 as lb

    return {"knowledge": (lb.KnowledgeProof.prove, osg.knowledge_prove, osg.knowledge_verify, [(0, 1)]),
            "equality": (lb.EqualityProof.prove, osg.equality_prove, osg.equality_verify, [(0, 1), (2, 3)]),
            "product": (lb.ProductProof.prove, osg.product_prove, osg.product_verify, [(0, 1), (2, 3), (4, 5)])}


def _both(ctx, kind, vals, label=b"sigma"):
    """GPU and oracle proofs of `kind` over vals: everything equal, every commitment the right one, the oracle's
    verifier accepting -> the GPU's (proof, commitments..)"""
    import lasso_b200 as lb

    gpu, cpu, verify, pairs = _provers()[kind]
    g, og = _gens(ctx)
    t, tape = lb.Transcript(label), lb.RandomTape(b"tape", SEED)
    o, otape = od.Transcript(label), od.RandomTape(b"tape", SEED)
    before = ctx.launches
    got = gpu(ctx, g, t, tape, *vals)
    assert ctx.launches - before == 2
    want = cpu(og, o, otape, *vals)
    assert got == want
    assert len(got[0]) == {"knowledge": 96, "equality": 64, "product": 256}[kind]
    for C, (i, j) in zip(got[1:], pairs):
        assert C == oz.commit(og, vals[i], vals[j])
    assert np.array_equal(t.challenge_scalar(b"after"), o.challenge_scalar(b"after"))
    assert np.array_equal(tape.random_scalar(b"after"), otape.random_scalar(b"after"))
    assert verify(og, *got, od.Transcript(label)) == 0
    return got


EDGES = [0, 1, L - 1]


@pytest.mark.parametrize("x", [None] + EDGES)
def test_knowledge(ctx, x):
    rng = np.random.default_rng(11)
    if x is None:
        _both(ctx, "knowledge", list(ol.rand_fr(rng, 2)))
    else:
        _both(ctx, "knowledge", [_fr(x), _fr(0)])
        _both(ctx, "knowledge", [_fr(x), ol.rand_fr(rng, 1)[0]])


@pytest.mark.parametrize("v", [None] + EDGES)
def test_equality(ctx, v):
    import lasso_b200 as lb

    rng = np.random.default_rng(12)
    val = ol.rand_fr(rng, 1)[0] if v is None else _fr(v)
    s1, s2 = ol.rand_fr(rng, 2)
    _both(ctx, "equality", [val, s1, val, s2])
    _both(ctx, "equality", [val, _fr(0), val, _fr(0)])
    _both(ctx, "equality", [val, s1, val, s1])
    # a false statement: the bytes still match, and the verifier rejects them
    g, og = _gens(ctx)
    other = _fr(ol.fr_ints(val)[0] + 1)
    got = lb.EqualityProof.prove(ctx, g, lb.Transcript(b"f"), lb.RandomTape(b"tape", SEED), val, s1, other, s2)
    assert got == osg.equality_prove(og, od.Transcript(b"f"), od.RandomTape(b"tape", SEED), val, s1, other, s2)
    assert osg.equality_verify(og, *got, od.Transcript(b"f")) == 1


@pytest.mark.parametrize("xy", [(None, None), (0, 0), (1, 1), (L - 1, L - 1), (0, L - 1), (1, L - 1), (L - 1, 7)])
def test_product(ctx, xy):
    import lasso_b200 as lb

    rng = np.random.default_rng(13)
    x, y = [ol.rand_fr(rng, 1)[0] if v is None else _fr(v) for v in xy]
    z = _fr(ol.fr_ints(x)[0] * ol.fr_ints(y)[0])
    rX, rY, rZ = ol.rand_fr(rng, 3)
    _both(ctx, "product", [x, rX, y, rY, z, rZ])
    zero = _fr(0)
    _both(ctx, "product", [x, zero, y, zero, z, zero])
    # z != x y: the bytes still match, and the verifier rejects them
    g, og = _gens(ctx)
    bad = _fr(ol.fr_ints(z)[0] + 1)
    vals = [x, rX, y, rY, bad, rZ]
    got = lb.ProductProof.prove(ctx, g, lb.Transcript(b"f"), lb.RandomTape(b"tape", SEED), *vals)
    assert got == osg.product_prove(og, od.Transcript(b"f"), od.RandomTape(b"tape", SEED), *vals)
    assert osg.product_verify(og, *got, od.Transcript(b"f")) == 1


def test_mc_gens_of_its_own(ctx):
    """a MultiCommitGens made from explicit points, not a DotProductProofGens half"""
    import lasso_b200 as lb

    rng = np.random.default_rng(14)
    stream = ol.generators(2, b"own")
    g, og = lb.MultiCommitGens(ctx, stream[:1], stream[1]), oz.mc_gens(stream, 1)
    vals = list(ol.rand_fr(rng, 6))
    vals[4] = _fr(ol.fr_ints(vals[0])[0] * ol.fr_ints(vals[2])[0])
    got = lb.ProductProof.prove(ctx, g, lb.Transcript(b"o"), lb.RandomTape(b"tape", SEED), *vals)
    assert got == osg.product_prove(og, od.Transcript(b"o"), od.RandomTape(b"tape", SEED), *vals)
    assert osg.product_verify(og, *got, od.Transcript(b"o")) == 0


def test_errors(ctx):
    """every error code before any launch, with the transcript and the tape untouched"""
    import lasso_b200 as lb

    Lb = lb.lib()
    rng = np.random.default_rng(15)
    g, _ = _gens(ctx)
    g3 = lb.DotProductProofGens.new(ctx, 3, b"sigma_gens").gens_n
    other = lb.Context(0)
    foreign = lb.MultiCommitGens.new(other, 1, b"sigma_gens")
    bad = np.full(4, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    calls = {"knowledge": (Lb.lasso_knowledge_prove, 2, 96, 1), "equality": (Lb.lasso_equality_prove, 4, 64, 2),
             "product": (Lb.lasso_product_prove, 6, 256, 3)}
    for kind, (fn, nv, plen, npts) in calls.items():
        vals = [ol.rand_fr(rng, 1)[0] for _ in range(nv)]
        out, pts = np.zeros(plen, np.uint8), [np.zeros(32, np.uint8) for _ in range(npts)]

        def call(gens, t_ok=True, tape_ok=True, vals=vals, outs=None):
            t, tape = lb.Transcript(b"e"), lb.RandomTape(b"t", SEED)
            outs = [out] + pts if outs is None else outs
            rc = fn(ctx._h, gens._h if gens else None, t._h if t_ok else None, tape._h if tape_ok else None,
                    *[P(v) if v is not None else None for v in vals], *[P(o) if o is not None else None for o in outs])
            return rc, t, tape

        cases = [(dict(gens=None), ERR_GENS), (dict(gens=g3), ERR_GENS), (dict(gens=foreign), ERR_GENS),
                 (dict(gens=g, t_ok=False), ERR_LENGTH), (dict(gens=g, tape_ok=False), ERR_LENGTH)]
        for i in range(nv):
            cases.append((dict(gens=g, vals=vals[:i] + [None] + vals[i + 1:]), ERR_LENGTH))
            cases.append((dict(gens=g, vals=vals[:i] + [bad] + vals[i + 1:]), ERR_VALUE))
        for i in range(1 + npts):
            outs = [out] + pts
            cases.append((dict(gens=g, outs=outs[:i] + [None] + outs[i + 1:]), ERR_LENGTH))
        for args, code in cases:
            before = ctx.launches
            rc, t, tape = call(**args)
            assert rc == code, (kind, args.keys(), rc)
            assert ctx.launches == before
            assert np.array_equal(t.challenge_scalar(b"x"), lb.Transcript(b"e").challenge_scalar(b"x"))
            assert np.array_equal(tape.random_scalar(b"x"), lb.RandomTape(b"t", SEED).random_scalar(b"x"))
        before = ctx.launches
        assert call(g)[0] == 0 and ctx.launches - before == 2
    with pytest.raises(lb.LassoError) as e:
        lb.KnowledgeProof.prove(ctx, g, lb.Transcript(b"e"), lb.RandomTape(b"t", SEED), bad, vals[0])
    assert e.value.code == ERR_VALUE
    del foreign
    other.close()


def test_spartan_phase_one_tail(ctx):
    """the end of a Spartan phase one on one transcript and tape: the ZK sumcheck of eq(tau) (A B - C) with claim 0,
    blinds for Az, Bz, Cz and Az Bz, KnowledgeProof(Cz), ProductProof(Az, Bz, Az Bz) and EqualityProof tying
    eq (C_prod - C_Cz) to the last comm_eval; equal to the oracle's run, and replayed by the verifier"""
    import lasso_b200 as lb

    nv = 10
    rng = np.random.default_rng(16)
    A, B = dc.random_full(rng, 1 << nv), dc.random_full(rng, 1 << nv)
    C = ol.fr_array([a * b % L for a, b in zip(ol.fr_ints(A), ol.fr_ints(B))])
    gens = lb.DotProductProofGens.new(ctx, 4, b"gens_sc")
    og1, ogn = oz.dot_gens(ol.generators(6, b"gens_sc"), 4)
    comb = lb.Comb(sc.spartan, 4)
    bc = np.zeros(4, dtype=np.uint64)

    def run(gpu):
        """the prover's steps -> every proof, commitment and the last transcript and tape draws"""
        if gpu:
            t, tape = lb.Transcript(b"spartan"), lb.RandomTape(b"proof", SEED)
        else:
            t, tape = od.Transcript(b"spartan"), od.RandomTape(b"proof", SEED)
        tau = t.challenge_vector(b"challenge_tau", nv)
        if gpu:
            polys = [lb.DensePolynomial.eq(ctx, tau)] + [lb.DensePolynomial(ctx, X) for X in (A, B, C)]
            zk = lb.ZKSumcheckInstanceProof.prove(ctx, comb, polys, nv, bc, gens.gens_1, gens.gens_n, t, tape)
            zk = dict(proof=zk.data, final_evals=zk.final_evals, blind_eval=zk.blind_eval, comm_claim=zk.comm_claim)
            g1 = gens.gens_1
            know = lambda *a: lb.KnowledgeProof.prove(ctx, g1, t, tape, *a)  # noqa: E731
            prod = lambda *a: lb.ProductProof.prove(ctx, g1, t, tape, *a)  # noqa: E731
            eq = lambda *a: lb.EqualityProof.prove(ctx, g1, t, tape, *a)  # noqa: E731
        else:
            zk = oz.zk_prove([sc.eq_evals(tau), A, B, C], nv, comb.program, comb.constants, 3, bc, og1, ogn, t, tape)
            know = lambda *a: osg.knowledge_prove(og1, t, tape, *a)  # noqa: E731
            prod = lambda *a: osg.product_prove(og1, t, tape, *a)  # noqa: E731
            eq = lambda *a: osg.equality_prove(og1, t, tape, *a)  # noqa: E731
        tau_r, Az, Bz, Cz = (ol.fr_ints(f)[0] for f in zk["final_evals"])
        b_Az, b_Bz, b_Cz, b_prod = (tape.random_scalar(lb_) for lb_ in (b"Az_blind", b"Bz_blind", b"Cz_blind",
                                                                        b"prod_Az_Bz_blind"))
        pok, C_Cz = know(_fr(Cz), b_Cz)
        pprod, C_Az, C_Bz, C_prod = prod(_fr(Az), b_Az, _fr(Bz), b_Bz, _fr(Az * Bz), b_prod)
        for name, cm in ((b"comm_Az_claim", C_Az), (b"comm_Bz_claim", C_Bz), (b"comm_Cz_claim", C_Cz),
                         (b"comm_prod_Az_Bz_claims", C_prod)):
            t.append_point(name, cm)
        v = _fr(tau_r * (Az * Bz - Cz))
        s1 = _fr(tau_r * (ol.fr_ints(b_prod)[0] - ol.fr_ints(b_Cz)[0]))
        peq, C1, C2 = eq(v, s1, v, zk["blind_eval"])
        return dict(zk=zk["proof"], comm_claim=zk["comm_claim"], tau_r=tau_r, pok=pok, C_Cz=C_Cz, pprod=pprod,
                    C_Az=C_Az, C_Bz=C_Bz, C_prod=C_prod, peq=peq, C1=C1, C2=C2, claim=v,
                    end=(t.challenge_scalar(b"end"), tape.random_scalar(b"end")))

    got, want = run(True), run(False)
    for k in want:
        if k == "end":
            assert all(np.array_equal(a, b) for a, b in zip(got[k], want[k]))
        else:
            assert np.array_equal(got[k], want[k]) if isinstance(got[k], np.ndarray) else got[k] == want[k], k
    # the verifier's replay: zk_verify gives the last comm_eval, the product and the knowledge proof their commitments,
    # and eq (C_prod - C_Cz) the other side of the equality
    vt = od.Transcript(b"spartan")
    tau = ol.fr_ints(vt.challenge_vector(b"challenge_tau", nv))
    rc, comm_eval, vr = oz.zk_verify(got["zk"], got["comm_claim"], nv, 3, og1, ogn, vt)
    assert rc == 0
    eq_r = 1
    for ti, ri in zip(tau, ol.fr_ints(vr)):
        eq_r = eq_r * (ti * ri + (1 - ti) * (1 - ri)) % L
    assert eq_r == got["tau_r"]
    assert osg.knowledge_verify(og1, got["pok"], got["C_Cz"], vt) == 0
    assert osg.product_verify(og1, got["pprod"], got["C_Az"], got["C_Bz"], got["C_prod"], vt) == 0
    for name, k in ((b"comm_Az_claim", "C_Az"), (b"comm_Bz_claim", "C_Bz"), (b"comm_Cz_claim", "C_Cz"),
                    (b"comm_prod_Az_Bz_claims", "C_prod")):
        vt.append_point(name, got[k])
    expected = osg.point_lincomb([got["C_prod"], got["C_Cz"]], [_fr(eq_r), _fr(-eq_r)])
    assert got["C1"] == expected and got["C2"] == comm_eval
    assert osg.equality_verify(og1, got["peq"], expected, comm_eval, vt) == 0


def _sigma_calls(ctx):
    """the three proofs' bytes and commitments"""
    import lasso_b200 as lb

    rng = np.random.default_rng(17)
    g = lb.DotProductProofGens.new(ctx, 2, b"sigma_gens").gens_1
    x, r, y, ry, rz = ol.rand_fr(rng, 5)
    z = _fr(ol.fr_ints(x)[0] * ol.fr_ints(y)[0])
    t, tape = lb.Transcript(b"s"), lb.RandomTape(b"t", SEED)
    return (lb.KnowledgeProof.prove(ctx, g, t, tape, x, r), lb.EqualityProof.prove(ctx, g, t, tape, x, r, x, ry),
            lb.ProductProof.prove(ctx, g, t, tape, x, r, y, ry, z, rz), bytes(t.challenge_scalar(b"end")))


def test_sharded_two_ranks_one_gpu():
    """on 2 ranks of one GPU every rank's bytes equal a single-GPU context's"""
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
        single = [_sigma_calls(c1)]
        c1.close()
    dist.broadcast_object_list(single, src=0)
    c = lb.Context(0)
    c.init_comm()
    got = [None] * G
    dist.all_gather_object(got, _sigma_calls(c))
    if rank == 0:
        fails = [g for g, x in enumerate(got) if x != single[0]]
        print(MARK, "PASS" if not fails else "FAIL %r" % fails, flush=True)
    dist.barrier()
    c.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker()
