"""Lookups inside a caller's protocol on the GPU: SparsePolynomialEvaluationProof.prove on a caller's transcript and tape
against the label path (bytes, launches, claimed evaluation), the composed protocol against the oracle (outputs v
committed and opened at r, the sparse commitment absorbed, the proof on the same transcript), DensifiedRepresentation
.outputs against the oracle's combine of the lookup polynomials, the error table, a sharded run and the 2^20 golden.

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

import compose_cases as cc  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import oracle_compose_lib as ocl  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_lib as ol  # noqa: E402
import workloads as wl  # noqa: E402
from lasso_b200.api import LASSO_ERR_GENS, LASSO_ERR_LENGTH, LASSO_ERR_STRATEGY, LASSO_ERR_VALUE  # noqa: E402

pytestmark = pytest.mark.gpu

# (name, kind, C, log_m, log_r)
BUILTINS = [("and", lb.AND, 4, 8, 0), ("or", lb.OR, 2, 16, 0), ("xor", lb.XOR, 4, 16, 0), ("lt", lb.LT, 8, 8, 0),
            ("lt2", lb.LT, 2, 16, 0), ("range", lb.RANGE_CHECK, 4, 8, 28)]


@pytest.fixture(scope="module")
def ctx():
    c = lb.Context(0)
    yield c
    c.close()


def custom_u32(ctx):
    """integer tables below 2^16, four memories over two dimensions, g = v0 v1 + v2 + 5 v3"""
    rng = np.random.default_rng(11)
    tables = [rng.integers(0, 1 << 16, size=1 << 8, dtype=np.uint64) for _ in range(2)]
    return lb.CustomStrategy(ctx, 2, 8, tables, lambda v: v[0] * v[1] + v[2] + v[3] * 5, 2)


def custom_fr(ctx):
    """one table of uniform field elements (full width), two memories, g = v0 v1 + 2 v0"""
    rng = np.random.default_rng(12)
    return lb.CustomStrategy(ctx, 2, 6, [ol.rand_fr(rng, 1 << 6)], lambda v: v[0] * v[1] + v[0] * 2, 2)


CUSTOMS = {"custom_u32": custom_u32, "custom_fr": custom_fr}
ALL = [b[0] for b in BUILTINS] + list(CUSTOMS)


def strategy(ctx, name):
    """-> (S, C, log_m, sumcheck degree, oracle outputs of a dim_usize matrix)"""
    if name in CUSTOMS:
        S = CUSTOMS[name](ctx)
        return S, S.C, S.log_m, S.sumcheck_poly_degree, lambda nz: cc.outputs_custom(S, nz)
    _, kind, C_, log_m, log_r = next(b for b in BUILTINS if b[0] == name)
    S = lb.Strategy(kind, C_, log_m, log_r)
    return S, C_, log_m, S.sumcheck_poly_degree, lambda nz: cc.outputs(kind, C_, log_m, log_r, nz)


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


# ---------------------------------------------------------------- 1. the transcript path is the label path
@pytest.mark.parametrize("name", ALL)
def test_transcript_path_equals_label_path(ctx, name):
    S, C_, log_m, deg, _ = strategy(ctx, name)
    idx, dense, stream, gens, r, seed = setup(ctx, S, C_, log_m, 300, 1)
    l0 = ctx.launches
    a = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    l1 = ctx.launches
    t, tape = lb.Transcript(b"example"), lb.RandomTape(b"proof", seed)
    b = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=t, random_tape=tape)
    l2 = ctx.launches
    assert b.bytes == a.bytes and b.challenges is None
    assert l2 - l1 == l1 - l0
    assert b.claimed_evaluation.tolist() == cc.claim_in_proof(b.bytes, len(r), deg).tolist()
    # the handles moved exactly as the label path's: its last challenge is the next one a twin would not draw
    assert t.challenge_scalar(b"after").tolist() != lb.Transcript(b"example").challenge_scalar(b"after").tolist()


# ---------------------------------------------------------------- 2. the composed protocol against the oracle
def compose_gpu(ctx, S, dense, gens, seed, log_s):
    T, tape = lb.Transcript(b"compose"), lb.RandomTape(b"proof", seed)
    T.append_protocol_name(b"Lasso composed")
    v = dense.outputs(S)
    v_gens = lb.PolyCommitmentGens.new(ctx, b"gens_outputs", log_s,
                                       stream=ol.generators(lb.poly_gens_points_needed(log_s), b"gens_outputs"))
    comm_v = v.commit(v_gens)
    T.append_poly_commitment(b"outputs", comm_v)
    comm_sparse = dense.commit(gens)
    T.append_sparse_commitment(comm_sparse)
    r = T.challenge_vector(b"r", log_s)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=T, random_tape=tape)
    opening = lb.PolyEvalProof.prove(ctx, v, r, proof.claimed_evaluation, v_gens, T, tape)
    return dict(v=v, comm_v=comm_v, comm_sparse=comm_sparse, r=r, proof=proof, opening=opening, last=_next(T))


def compose_oracle(S, kind_args, idx, stream, seed, log_s, v):
    """the same steps in the oracle; kind_args = (kind, C, log_m, log_r) or None for a custom strategy"""
    v_stream = ol.generators(lb.poly_gens_points_needed(log_s), b"gens_outputs")
    T, tape = od.Transcript(b"compose"), od.RandomTape(b"proof", seed)
    T.append_protocol_name(b"Lasso composed")
    comm_v = od.commit(v, v_stream)
    T.append_poly_commitment(b"outputs", comm_v)
    scratch = (od.Transcript(b"scratch"), od.RandomTape(b"scratch", seed), np.zeros((log_s, 4), dtype=np.uint64))
    if kind_args:
        _, comm_sparse, _ = ocl.sparse_prove(*kind_args, idx, scratch[2], stream, scratch[0], scratch[1])
    else:
        _, comm_sparse, _ = ocl.custom_prove(S, idx, scratch[2], stream, scratch[0], scratch[1])
    assert ocl.append_sparse_commitment(T, comm_sparse) == 0
    r = T.challenge_vector(b"r", log_s)
    if kind_args:
        proof, _, claim = ocl.sparse_prove(*kind_args, idx, r, stream, T, tape)
    else:
        proof, _, claim = ocl.custom_prove(S, idx, r, stream, T, tape)
    opening, _ = od.prove(v, r, claim, v_stream, T, tape)
    return dict(comm_v=comm_v, comm_sparse=comm_sparse, r=r, proof=proof, opening=opening, last=_next(T))


def verify_composed(S, kind_args, stream, got, log_s):
    """the oracle's verifiers on the GPU's bytes, replaying the caller's steps -> (sparse verdict, opening verdict)"""
    v_stream = ol.generators(lb.poly_gens_points_needed(log_s), b"gens_outputs")
    V = od.Transcript(b"compose")
    V.append_protocol_name(b"Lasso composed")
    V.append_poly_commitment(b"outputs", got["comm_v"])
    assert ocl.append_sparse_commitment(V, got["comm_sparse"]) == 0
    r = V.challenge_vector(b"r", log_s)
    proof = got["proof"].bytes
    if kind_args:
        ok = ocl.sparse_verify(*kind_args, stream, got["comm_sparse"], proof, r, V)
    else:
        ok = ocl.custom_verify(S, stream, got["comm_sparse"], proof, r, V)
    deg = S.sumcheck_poly_degree
    return ok, od.verify(v_stream, log_s, got["comm_v"], got["opening"].bytes, r, cc.claim_in_proof(proof, log_s, deg), V)


@pytest.mark.parametrize("name,n", [("xor", 1 << 10), ("xor", 1000), ("custom_fr", 300), ("custom_u32", 200),
                                    ("lt2", 77)])
def test_composed_protocol_matches_oracle(ctx, name, n):
    S, C_, log_m, deg, _ = strategy(ctx, name)
    idx, dense, stream, gens, _, seed = setup(ctx, S, C_, log_m, n, 2)
    log_s = dense.s.bit_length() - 1
    got = compose_gpu(ctx, S, dense, gens, seed, log_s)
    v = got["v"]
    kind_args = None if name in CUSTOMS else next((b[1], b[2], b[3], b[4]) for b in BUILTINS if b[0] == name)
    want = compose_oracle(S, kind_args, idx, stream, seed, log_s, strategy(ctx, name)[4](cc.dim_usize(idx, dense.s)))
    assert got["comm_v"] == want["comm_v"] and got["comm_sparse"] == want["comm_sparse"]
    assert got["r"].tolist() == want["r"].tolist()
    assert got["proof"].bytes == want["proof"] and got["opening"].bytes == want["opening"]
    assert got["last"] == want["last"]
    assert v.evaluate(got["r"]).tolist() == got["proof"].claimed_evaluation.tolist()
    assert verify_composed(S, kind_args, stream, got, log_s) == (0, 0)


# ---------------------------------------------------------------- 3. the outputs
@pytest.mark.parametrize("name", ALL)
@pytest.mark.parametrize("n", [2, 3, 100, 1 << 12, (1 << 16) - 5])
def test_outputs_match_oracle(ctx, name, n):
    S, C_, log_m, deg, oracle = strategy(ctx, name)
    rng = np.random.default_rng(n)
    idx = rng.integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    l0 = ctx.launches
    v = dense.outputs(S)
    launches = ctx.launches - l0
    want = oracle(cc.dim_usize(idx, dense.s))
    nv = dense.s.bit_length() - 1
    assert v.num_vars == nv
    # the values themselves: v is multilinear, so its evaluations at the boolean points are its entries
    for k in list(range(min(dense.s, 8))) + [dense.s - 1, int(rng.integers(0, dense.s))]:
        point = ol.fr_array([(k >> (nv - 1 - j)) & 1 for j in range(nv)])
        assert v.evaluate(point).tolist() == want[k].tolist(), k
    r = ol.rand_fr(rng, nv)
    assert v.evaluate(r).tolist() == od.evaluate(want, r).tolist()
    widest = max(ol.fr_ints(want)).bit_length()
    # the outputs kernel, the width read-back and, for integer values, the u32 mirror
    assert launches == 2 + (widest <= 32)
    if n <= 1 << 12:
        g = lb.PolyCommitmentGens.new(ctx, b"gens_outputs", nv, stream=ol.generators(lb.poly_gens_points_needed(nv),
                                                                                      b"gens_outputs"))
        assert v.commit(g) == od.commit(want, g.stream)


@pytest.mark.parametrize("name", ALL)
def test_outputs_evaluate_to_the_claimed_evaluation(ctx, name):
    S, C_, log_m, _, _ = strategy(ctx, name)
    idx, dense, stream, gens, r, seed = setup(ctx, S, C_, log_m, 513, 3)
    p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=lb.Transcript(b"t"),
                                                 random_tape=lb.RandomTape(b"p", seed))
    assert dense.outputs(S).evaluate(r).tolist() == p.claimed_evaluation.tolist()


def test_integer_outputs_take_the_16_bit_path(ctx):
    """XOR at C log_m / 2 = 16 bits: every output below 2^32, so v has the u32 mirror, and its commitment equals the
    oracle's; a full-width custom output commits through the Fr windows to the oracle's bytes too"""
    for name in ("xor", "custom_fr"):
        S, C_, log_m, _, oracle = strategy(ctx, name)
        idx = np.random.default_rng(5).integers(0, 1 << log_m, size=(1 << 10, C_), dtype=np.uint64)
        dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
        want = oracle(cc.dim_usize(idx, dense.s))
        assert (max(ol.fr_ints(want)).bit_length() <= 32) == (name == "xor")
        v = dense.outputs(S)
        g = lb.PolyCommitmentGens.new(ctx, b"gens_outputs", 10, stream=ol.generators(lb.poly_gens_points_needed(10),
                                                                                      b"gens_outputs"))
        assert v.commit(g) == od.commit(want, g.stream)


# ---------------------------------------------------------------- 4. errors leave the handles untouched
def _raw_prove(ctx, S, dense, r, gens, t, tape, cap=1 << 22, proof_len=True, r_len=None):
    import ctypes as C

    from lasso_b200.api import _p, lib

    out = np.zeros(max(cap, 1), dtype=np.uint8)
    n = C.c_size_t(0)
    r = np.ascontiguousarray(r, dtype=np.uint64).reshape(-1, 4)
    tail = (dense._h, _p(r), C.c_size_t(r.shape[0] if r_len is None else r_len), gens._h if gens else None,
            t._h if t else None, tape._h if tape else None, _p(out), C.c_size_t(cap), C.byref(n) if proof_len else None,
            None)
    if isinstance(S, lb.CustomStrategy):
        rc = lib().lasso_prove_custom_transcript(ctx._h, S._h, *tail)
    else:
        rc = lib().lasso_prove_transcript(ctx._h, S.kind, S.log_r, *tail)
    return rc, n.value


def _raw_prove_labels(ctx, S, dense, r, gens, seed, cap=1 << 22, label=b"example"):
    """lasso_prove / lasso_prove_custom -> (error code, *proof_len)"""
    import ctypes as C

    from lasso_b200.api import _p, lib

    out = np.zeros(max(cap, 1), dtype=np.uint8)
    n = C.c_size_t(0)
    r = np.ascontiguousarray(r, dtype=np.uint64).reshape(-1, 4)
    seed = np.ascontiguousarray(seed, dtype=np.uint64)
    tail = (dense._h, _p(r), C.c_size_t(r.shape[0]), gens._h, label, b"proof", _p(seed), _p(out), C.c_size_t(cap),
            C.byref(n), None, C.c_size_t(0), None)
    if isinstance(S, lb.CustomStrategy):
        rc = lib().lasso_prove_custom(ctx._h, S._h, *tail)
    else:
        rc = lib().lasso_prove(ctx._h, S.kind, S.log_r, *tail)
    return rc, n.value


def test_errors_before_anything_moves(ctx):
    S, C_, log_m, _, _ = strategy(ctx, "xor")
    idx, dense, stream, gens, r, seed = setup(ctx, S, C_, log_m, 256, 4)
    need = len(lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed).bytes)
    other = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, dense.s * 2, S.num_memories, log_m,
                                            stream=ol.generators(lb.gens_points_needed(C_, dense.s * 2, 4, log_m)))
    ctx2 = lb.Context(0)
    S_other = custom_u32(ctx2)
    S_shape = custom_u32(ctx)  # C = 2, log_m = 8: not the dense's (4, 16)
    bad_r = r.copy()
    bad_r[0] = ol.int_to_limbs(ol.L_FR)
    cases = [
        (dict(S=lb.Strategy(9, C_, log_m)), LASSO_ERR_STRATEGY),
        (dict(S=S_other), LASSO_ERR_STRATEGY),
        (dict(S=S_shape), LASSO_ERR_STRATEGY),
        (dict(r_len=len(r) - 1), LASSO_ERR_LENGTH),
        (dict(t=None), LASSO_ERR_LENGTH),
        (dict(tape=None), LASSO_ERR_LENGTH),
        (dict(proof_len=False), LASSO_ERR_LENGTH),
        (dict(cap=need - 1), LASSO_ERR_LENGTH),
        (dict(gens=other), LASSO_ERR_GENS),
        (dict(gens=None), LASSO_ERR_GENS),
        (dict(r=bad_r), LASSO_ERR_VALUE),
    ]
    for over, code in cases:
        t, tape = lb.Transcript(b"example"), lb.RandomTape(b"proof", seed)
        kw = dict(S=S, r=r, gens=gens, t=t, tape=tape)
        kw.update(over)
        l0 = ctx.launches
        rc, plen = _raw_prove(ctx, kw.pop("S"), dense, kw.pop("r"), kw.pop("gens"), kw.pop("t"), kw.pop("tape"), **kw)
        assert rc == code, (over, rc)
        assert ctx.launches == l0
        if over.get("cap"):
            assert plen == need
        assert _next(t) == _next(lb.Transcript(b"example"))
        assert tape.random_scalar(b"x").tolist() == lb.RandomTape(b"proof", seed).random_scalar(b"x").tolist()
    # the label path takes the same checks, built-in and custom: each error before any launch
    for name in ("xor", "custom_u32"):
        S_l, C_l, log_m_l, _, _ = strategy(ctx, name)
        _, d_l, _, g_l, r_l, seed_l = setup(ctx, S_l, C_l, log_m_l, 256, 5)
        need_l = len(lb.SparsePolynomialEvaluationProof.prove(ctx, S_l, d_l, r_l, g_l, tape_seed=seed_l).bytes)
        n_other = lb.gens_points_needed(C_l, d_l.s * 2, S_l.num_memories, log_m_l)
        other_l = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_l, d_l.s * 2, S_l.num_memories, log_m_l,
                                                  stream=ol.generators(n_other))
        bad_r_l = r_l.copy()
        bad_r_l[0] = ol.int_to_limbs(ol.L_FR)
        for over, code in [(dict(gens=other_l), LASSO_ERR_GENS), (dict(r=bad_r_l), LASSO_ERR_VALUE),
                           (dict(seed=ol.int_to_limbs(ol.L_FR)), LASSO_ERR_VALUE), (dict(label=None), LASSO_ERR_LENGTH),
                           (dict(cap=need_l - 1), LASSO_ERR_LENGTH)]:
            kw = dict(r=r_l, gens=g_l, seed=seed_l)
            kw.update(over)
            l0 = ctx.launches
            rc, plen = _raw_prove_labels(ctx, S_l, d_l, **kw)
            assert rc == code, (name, over, rc)
            assert ctx.launches == l0
            if over.get("cap"):
                assert plen == need_l
    # LT with C = 8 is provable, with C = 9 not (its memories make 36 circuits)
    idx9 = np.zeros((16, 9), dtype=np.uint64)
    d9 = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx9, 4)
    g9 = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", 9, 16, 18, 4,
                                         stream=ol.generators(lb.gens_points_needed(9, 16, 18, 4)))
    t = lb.Transcript(b"example")
    rc, _ = _raw_prove(ctx, lb.Strategy(lb.LT, 9, 4), d9, ol.rand_fr(np.random.default_rng(0), 4), g9, t,
                       lb.RandomTape(b"proof", seed))
    assert rc == LASSO_ERR_STRATEGY and _next(t) == _next(lb.Transcript(b"example"))
    with pytest.raises(lb.LassoError) as e:
        d9.outputs(lb.Strategy(lb.LT, 9, 4))
    assert e.value.code == LASSO_ERR_STRATEGY
    with pytest.raises(lb.LassoError) as e:
        dense.outputs(S_other)
    assert e.value.code == LASSO_ERR_STRATEGY
    del S_other
    ctx2.close()


def test_label_path_shares_generators_across_contexts(ctx):
    """lasso_prove on a second context of the same GPU with the first context's generators, whose tables are only read
    (the batched-throughput mode of bench.py): the first context's bytes"""
    S, C_, log_m, _, _ = strategy(ctx, "xor")
    idx, dense, stream, gens, r, seed = setup(ctx, S, C_, log_m, 256, 6)
    want = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed).bytes
    ctx2 = lb.Context(0)
    d2 = lb.DensifiedRepresentation.from_lookup_indices(ctx2, idx, log_m)
    assert lb.SparsePolynomialEvaluationProof.prove(ctx2, S, d2, r, gens, tape_seed=seed).bytes == want
    del d2
    ctx2.close()


# ---------------------------------------------------------------- 5. sharded
def test_sharded_two_ranks_one_gpu(ctx):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, LASSO_SHARD_SAME_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env)
    assert "COMPOSE_SHARDED PASS" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


def _sharded_worker():
    """every rank proves on its own transcript and tape in the same state; every rank must get the single-GPU bytes,
    the same next challenge, and LASSO_ERR_STRATEGY from outputs"""
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(0)
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    C_, log_m, n = 4, 16, 1 << 11
    rng = np.random.default_rng(9)
    idx = rng.integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    r, seed = ol.rand_fr(rng, 11), ol.rand_fr(rng, 1)[0]
    S = lb.Strategy(lb.XOR, C_, log_m)
    stream = ol.generators(lb.gens_points_needed(C_, n, 4, log_m))
    single = None
    if rank == 0:  # the single-GPU bytes, before the collective context exists
        c1 = lb.Context(0)
        d1 = lb.DensifiedRepresentation.from_lookup_indices(c1, idx, log_m)
        g1 = lb.SparsePolyCommitmentGens.new(c1, b"gens_sparse_poly", C_, n, 4, log_m, stream=stream)
        t1 = lb.Transcript(b"example")
        t1.append_protocol_name(b"prefix")
        single = (lb.SparsePolynomialEvaluationProof.prove(c1, S, d1, r, g1, transcript=t1,
                                                           random_tape=lb.RandomTape(b"proof", seed)).bytes, _next(t1))
        del d1, g1
        c1.close()
    dist.barrier()
    c = lb.Context(0)
    c.init_comm()
    d = lb.DensifiedRepresentation.from_lookup_indices(c, idx, log_m)
    g = lb.SparsePolyCommitmentGens.new(c, b"gens_sparse_poly", C_, n, 4, log_m, stream=stream)
    t = lb.Transcript(b"example")
    t.append_protocol_name(b"prefix")
    p = lb.SparsePolynomialEvaluationProof.prove(c, S, d, r, g, transcript=t, random_tape=lb.RandomTape(b"proof", seed))
    got = [None, None]
    dist.all_gather_object(got, (hashlib.sha256(p.bytes).hexdigest(), _next(t)))
    try:
        d.outputs(S)
        out_code = 0
    except lb.LassoError as e:
        out_code = e.code
    codes = [None, None]
    dist.all_gather_object(codes, out_code)
    if rank == 0:
        want = (hashlib.sha256(single[0]).hexdigest(), single[1])
        ok = all(tuple(x) == want for x in got) and all(x == LASSO_ERR_STRATEGY for x in codes)
        print("COMPOSE_SHARDED", "PASS" if ok else "FAIL %r %r %r" % (got, want, codes), flush=True)
    dist.barrier()
    del d, g
    c.close()
    dist.destroy_process_group()


# ---------------------------------------------------------------- 6. at size
def test_at_size_xor_2_20(ctx):
    name = "xor_c4_s20"
    g = json.load(open(os.path.join(HERE, "golden", "big_proofs.json")))["cases"][name]
    kind, C_, log_m, log_r, log_s, idx, r, seed = wl.config_inputs(name)
    S = lb.Strategy(kind, C_, log_m, log_r)
    stream = np.ascontiguousarray(ol.generators(wl.gens_needed(C_, log_s, 4, log_m)))
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, dense.s, 4, log_m, stream=stream)
    p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=lb.Transcript(b"example"),
                                                 random_tape=lb.RandomTape(b"proof", seed))
    assert hashlib.sha256(p.bytes).hexdigest() == g["proof_sha256"]
    got = compose_gpu(ctx, S, dense, gens, seed, log_s)
    assert got["v"].evaluate(got["r"]).tolist() == got["proof"].claimed_evaluation.tolist()
    assert verify_composed(S, (kind, C_, log_m, log_r), stream, got, log_s) == (0, 0)


if __name__ == "__main__":
    _sharded_worker()
