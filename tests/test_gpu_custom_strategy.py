"""Caller-defined strategies on the GPU (lasso_strategy_create, lasso_sumcheck_round_custom, lasso_prove_custom):
round messages against the oracle, proofs of the built-ins re-expressed as programs against the built-in path, proofs
of new tables against the oracle for caller-defined strategies (oracle_custom/), the descriptor checks, and a sharded proof."""
import ctypes as C
import hashlib
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import custom_builtins as cb
import oracle_custom_lib as oc
import oracle_lib as ol
import test_gpu_prove as tgp
import workloads as wl

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def random_program(rng, alpha, degree, width=0):
    """combine_lookups of exactly `degree`: a product of `degree` memory values, scaled, plus random lower-degree terms;
    width > 0 first forms `width` products that all stay live until they are summed"""
    picks = [int(x) for x in rng.integers(0, alpha, size=degree)]
    k = [int(x) for x in rng.integers(-2**40, 2**40, size=6)]
    ops = [int(x) for x in rng.integers(0, 3, size=alpha)]

    def g(v):
        p = v[picks[0]] * k[0]
        for j in picks[1:]:
            p = p * v[j]
        acc = p + k[1]
        for i in range(alpha):
            acc = acc + v[i] * k[2] if ops[i] == 0 else (acc - v[i] if ops[i] == 1 else k[3] - acc)
        if width:
            prods = [v[i % alpha] * v[(i + 1) % alpha] for i in range(width)]
            s = prods[0]
            for q in prods[1:]:
                s = s + q
            acc = acc + s * k[4]
        return acc
    return g


def _tables(rng, nsub, log_m):
    return [rng.integers(0, 2**32, size=1 << log_m, dtype=np.uint64) for _ in range(nsub)]


def _rand_polys(rng, n, length):
    return np.stack([ol.rand_fr(rng, length) for _ in range(n)])


def test_round_against_oracle_alpha_and_degree(ctx):
    """alpha = 1..16 memories, degree = 1..16"""
    import lasso_b200 as lb

    rng = np.random.default_rng(11)
    pairs = [(a, d) for a in range(1, 17) for d in range(1, 17) if a == d or a in (1, 16) or d in (1, 16)]
    for alpha, deg in pairs:
        S = lb.CustomStrategy(ctx, 1, 2, _tables(rng, 1, 2), random_program(rng, alpha, deg), deg,
                              memory_to_subtable=[0] * alpha, memory_to_dimension=[0] * alpha)
        polys = _rand_polys(rng, alpha + 1, 16)
        got = lb.sumcheck_round_custom(ctx, S, list(polys))
        assert got.shape == (deg + 2, 4)
        assert (got == oc.sumcheck_round(S, polys)).all(), (alpha, deg)
        S.close()


@pytest.mark.parametrize("length", [2, 1 << 12, 1 << 15])
def test_round_many_ctas_and_live_slots(ctx, length):
    """long rounds (many CTAs, the last one publishes), a declared degree above the program's, and 16 live slots (15
    products and the running sum)"""
    import lasso_b200 as lb

    rng = np.random.default_rng(length)
    alpha = 16
    S = lb.CustomStrategy(ctx, 1, 2, _tables(rng, 1, 2), random_program(rng, alpha, 3, width=15), 5,
                          memory_to_subtable=[0] * alpha, memory_to_dimension=[0] * alpha)
    polys = _rand_polys(rng, alpha + 1, length)
    assert (lb.sumcheck_round_custom(ctx, S, list(polys)) == oc.sumcheck_round(S, polys)).all()


@pytest.mark.parametrize("kind,C,log_m,log_r", [(0, 4, 8, 0), (1, 2, 8, 0), (2, 3, 16, 0), (3, 1, 4, 0), (3, 4, 8, 0),
                                                (3, 8, 16, 0), (4, 3, 8, 20)])
def test_round_matches_builtin_round(ctx, kind, C, log_m, log_r):
    import lasso_b200 as lb

    rng = np.random.default_rng(kind * 10 + C)
    S = cb.as_custom(ctx, kind, C, log_m, log_r)
    B = lb.Strategy(kind, C, log_m, log_r)
    for length in (4, 1 << 13):
        polys = list(_rand_polys(rng, S.num_memories + 1, length))
        assert (lb.sumcheck_round_custom(ctx, S, polys) == lb.sumcheck_round_arbitrary(ctx, B, polys)).all()


def _gens(ctx, S, s, need_min=300):
    import lasso_b200 as lb

    need = lb.gens_points_needed(S.C, s, S.num_memories, S.log_m)
    stream = np.ascontiguousarray(ol.generators(max(need, need_min))[:need])
    return stream, lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", S.C, s, S.num_memories, S.log_m,
                                                   stream=stream)


@pytest.mark.parametrize("name,kind,C,log_m,log_r,n,same", tgp.CASES, ids=[c[0] for c in tgp.CASES])
def test_prove_builtin_as_custom_matches_builtin(ctx, name, kind, C, log_m, log_r, n, same):
    import lasso_b200 as lb

    idx, r, seed, s = tgp.make_inputs(C, log_m, n, len(name), same)
    S = cb.as_custom(ctx, kind, C, log_m, log_r)
    _, gens = _gens(ctx, S, s)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    want = lb.SparsePolynomialEvaluationProof.prove(ctx, lb.Strategy(kind, C, log_m, log_r), dense, r, gens,
                                                    tape_seed=seed)
    got = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    assert got.bytes == want.bytes
    assert got.challenges.shape == want.challenges.shape and (got.challenges == want.challenges).all()


@pytest.mark.parametrize("name", ["xor_c4_s20", "lt_c8_s22"])
def test_prove_at_size_matches_golden(ctx, name):
    import lasso_b200 as lb

    g = json.load(open(os.path.join(HERE, "golden", "big_proofs.json")))["cases"][name]
    kind, C, log_m, log_r, log_s, idx, r, tape_seed = wl.config_inputs(name)
    S = cb.as_custom(ctx, kind, C, log_m, log_r)
    stream, gens = _gens(ctx, S, 1 << log_s, 0)
    assert hashlib.sha256(stream.tobytes()).hexdigest() == g["generators_sha256"]
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    assert hashlib.sha256(dense.commit(gens)).hexdigest() == g["commitment_sha256"]
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=tape_seed)
    assert len(proof.challenges) == g["n_challenges"]
    assert hashlib.sha256(proof.bytes).hexdigest() == g["proof_sha256"]


@pytest.mark.parametrize("name", sorted(cb.NEW_TABLES))
@pytest.mark.parametrize("n", [40, 1 << 12])
def test_prove_new_tables_matches_oracle(ctx, name, n):
    import lasso_b200 as lb

    S = cb.NEW_TABLES[name](ctx)
    idx, r, seed, s = tgp.make_inputs(S.C, S.log_m, n, len(name) + n, False)
    stream, gens = _gens(ctx, S, s)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, S.log_m)
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    ref = oc.prove(S, idx, r, stream, seed, flags=1)
    assert ref["rc"] == 0, "the oracle's verifier rejected"
    assert com == ref["commitment"]
    assert (proof.challenges == ref["challenges"]).all()
    assert proof.bytes == ref["proof"]


# ---------------------------------------------------------------- errors
def _create(ctx, C_=2, log_m=4, nsub=1, alpha=2, sub=None, dim=None, prog=None, consts=None, deg=1):
    import lasso_b200 as lb

    tables = [np.ascontiguousarray(np.arange(1 << log_m), dtype=np.uint32) for _ in range(max(nsub, 1))]
    sub = np.ascontiguousarray(sub if sub is not None else [0] * alpha, dtype=np.int32)
    dim = np.ascontiguousarray(dim if dim is not None else [i % C_ for i in range(alpha)], dtype=np.int32)
    prog = np.ascontiguousarray(prog if prog is not None else [[0, 0, 1]], dtype=np.int32)
    consts = np.ascontiguousarray(consts if consts is not None else np.zeros((0, 4)), dtype=np.uint64)
    h = C.c_void_p()
    rc = lb.lib().lasso_strategy_create(ctx._h, C_, log_m, nsub, lb.api._ptr_array(tables), alpha, lb.api._p(sub),
                                        lb.api._p(dim), lb.api._p(prog), int(prog.shape[0]), lb.api._p(consts),
                                        int(consts.shape[0]), deg, C.byref(h))
    if rc == 0:
        lb.lib().lasso_strategy_destroy(h)
    return rc


def test_create_rejects_malformed_descriptors(ctx):
    assert _create(ctx) == 0
    assert _create(ctx, prog=[[3, 0, 0]], consts=ol.fr_array([5])) == 0
    bad = {
        "operand names the slot being written": dict(prog=[[0, 0, 2]]),
        "operand names a later slot": dict(prog=[[0, 0, 1], [0, 4, 0]]),
        "negative operand": dict(prog=[[0, -1, 0]]),
        "constant index out of range": dict(prog=[[3, 0, 1]], consts=ol.fr_array([5])),
        "unknown opcode": dict(prog=[[7, 0, 1]]),
        "non-canonical constant": dict(prog=[[3, 0, 0]], consts=np.full((1, 4), 2**64 - 1, dtype=np.uint64)),
        "subtable map out of range": dict(sub=[0, 1]),
        "dimension map out of range": dict(dim=[0, 2]),
        "more than 16 memories": dict(alpha=17, prog=[[0, 0, 16]]),
        "declared degree too low": dict(prog=[[2, 0, 1]], deg=1),
        "declared degree above 16": dict(deg=17),
        "too many instructions": dict(prog=[[0, 0, 1]] + [[0, 2 + j, 0] for j in range(128)]),
        "no instructions": dict(prog=np.zeros((0, 3))),
        "more subtables than memories": dict(nsub=3),
        "C above 16": dict(C_=17),
        "log_m below 2": dict(log_m=1),
        "more than 16 live values": dict(alpha=2, prog=[[2, 0, 1]] * 17 + [[0, 2 + j, 3 + j] for j in range(16)], deg=2),
    }
    for why, kw in bad.items():
        assert _create(ctx, **kw) == 4, why


def test_prove_custom_errors(ctx):
    import lasso_b200 as lb

    idx, r, seed, s = tgp.make_inputs(2, 4, 16, 1, True)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, 4)
    S = cb.as_custom(ctx, cb.XOR, 2, 4)
    _, gens = _gens(ctx, S, s)
    with pytest.raises(lb.LassoError) as e:  # assert_eq!(r.len(), log2(s)) surge.rs:131
        lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r[:-1], gens, tape_seed=seed)
    assert e.value.code == 1
    for other in (cb.as_custom(ctx, cb.XOR, 3, 4), cb.as_custom(ctx, cb.XOR, 2, 6)):
        with pytest.raises(lb.LassoError) as e:
            lb.SparsePolynomialEvaluationProof.prove(ctx, other, dense, r, gens, tape_seed=seed)
        assert e.value.code == 4
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)  # still usable
    assert proof.bytes == lb.SparsePolynomialEvaluationProof.prove(ctx, lb.Strategy(lb.XOR, 2, 4), dense, r, gens,
                                                                   tape_seed=seed).bytes


# ---------------------------------------------------------------- sharded
def test_sharded_custom_two_ranks_one_gpu_bit_exact():
    """tools/sharded_check.py --custom: the built-in cases as programs and the new tables, 2 ranks on GPU 0"""
    sock = socket.socket()
    sock.bind(("127.0.0.1", 0))
    port = sock.getsockname()[1]
    sock.close()
    env = dict(os.environ, LASSO_SHARD_SAME_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sharded_check.py"), "--custom"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env)
    assert "SHARDED_CHECK PASS" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
