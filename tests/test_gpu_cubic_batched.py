"""Batched cubic sumchecks over a caller's polynomials on the GPU: SumcheckInstanceProof.prove_cubic_batched with a
caller's claim and coefficients on a caller-held Transcript, bit for bit against the CPU oracle (oracle_dense/
orcd_cubic_prove).  Every case compares the proof bytes, the challenges, the finals A_0.., B_0.., C and the
transcript's next challenge.  Covers n = 1, 2, 7, 32 pairs at num_vars 1, 2, 3, 10 and 13 with full and partial rounds,
C = eq(tau) and C random, repeated polynomials, zero coefficients, integer and full-width values, numpy and CUDA inputs,
the caller's polynomials left unchanged, the oracle verifier, prove_arbitrary on the same polynomial, the sizes of
tests/golden/cubic_batched.json, every argument error and the launch count.

Sharded contexts: run as a script under torch.distributed.run the file is the worker (2 and 4 ranks time-slicing GPU 0,
or one rank per GPU).  Rank 0 first runs every case on a plain context; every rank must return the same bytes, r and
finals on the sharded one."""
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

import cubic_batched_cases as cb  # noqa: E402
import oracle_cubic_lib as ocb  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_lib as ol  # noqa: E402
import oracle_sumcheck_lib as osc  # noqa: E402

pytestmark = pytest.mark.gpu
ERR_LENGTH, ERR_STRATEGY, ERR_VALUE = 1, 4, 8
MARK = "CUBIC_BATCHED"
LABEL = b"cubic"


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _gpu(ctx, A, B, C, coeffs, claim, rounds, polys=None, label=LABEL):
    """-> (proof, next challenge) on the GPU; polys = (A polys, B polys, C poly) when given"""
    import lasso_b200 as lb

    if polys is None:
        cache = {}

        def mk(Z):  # one polynomial per distinct array object: repeated arrays are passed as the same polynomial
            if id(Z) not in cache:
                cache[id(Z)] = lb.DensePolynomial(ctx, Z)
            return cache[id(Z)]

        polys = ([mk(a) for a in A], [mk(b) for b in B], mk(C))
    t = lb.Transcript(label)
    got = lb.SumcheckInstanceProof.prove_cubic_batched(ctx, polys[0], polys[1], polys[2], coeffs, claim, t, rounds)
    return got, t.challenge_scalar(b"after")


def _oracle(A, B, C, coeffs, claim, rounds, label=LABEL):
    o = od.Transcript(label)
    want = ocb.cubic_prove(A, B, C, coeffs, claim, rounds, o)
    return want, o.challenge_scalar(b"after")


def _both(ctx, A, B, C, coeffs, claim, rounds, polys=None, label=LABEL):
    got, after = _gpu(ctx, A, B, C, coeffs, claim, rounds, polys, label)
    want, o_after = _oracle(A, B, C, coeffs, claim, rounds, label)
    assert len(got.bytes) == 8 + 104 * rounds
    assert got.bytes == want["proof"]
    assert np.array_equal(got.r, want["r"])
    assert np.array_equal(got.final_evals, want["finals"])
    assert np.array_equal(after, o_after)
    return got


def _claim(rng):
    """the claim is not checked: any canonical value gives the oracle's bytes"""
    return ol.rand_fr(rng, 1)[0]


SHAPES = [(n, nv, rounds) for n in (1, 2, 7, 32) for nv in (1, 2, 3, 10, 13)
          for rounds in sorted({nv, max(1, nv - 2)}) if not (n == 32 and nv == 13 and rounds != nv)]


@pytest.mark.parametrize("n,nv,rounds", SHAPES)
def test_shapes(ctx, n, nv, rounds):
    ckind = "eq" if (n + nv) % 2 else "random"
    kinds = ("full", "u32") if nv % 2 else ("u32", "full")
    A, B, C, coeffs = cb.random_case(n, nv, 1000 * n + 10 * nv + rounds, ckind, kinds)
    _both(ctx, A, B, C, coeffs, _claim(np.random.default_rng(nv)), rounds)


@pytest.mark.parametrize("nv,rounds", [(1, 1), (3, 2), (10, 10), (10, 7)])
def test_repeated(ctx, nv, rounds):
    """A_0 = B_0, A_1 = B_2 = C, B_1 = A_0: the caller's buffers are read several times and bound once per slot"""
    A, B, C, coeffs = cb.random_case(3, nv, 77 + nv)
    A[1] = B[2] = C
    B[0] = B[1] = A[0]
    _both(ctx, A, B, C, coeffs, _claim(np.random.default_rng(1)), rounds)


@pytest.mark.parametrize("n,nv,rounds,zeros", [(2, 3, 3, [1]), (7, 10, 8, [0]), (32, 10, 10, [5]), (2, 10, 10, "all"),
                                               (1, 1, 1, "all"), (32, 3, 2, "all"), (32, 13, 13, "all")])
def test_zero_coefficients(ctx, n, nv, rounds, zeros):
    A, B, C, coeffs = cb.random_case(n, nv, 500 + n + nv)
    coeffs[list(range(n)) if zeros == "all" else zeros] = 0
    _both(ctx, A, B, C, coeffs, _claim(np.random.default_rng(2)), rounds)


def test_cuda_inputs(ctx):
    import torch

    import lasso_b200 as lb

    A, B, C, coeffs = cb.random_case(3, 10, 31, "eq", ("u32", "full"))
    polys = ([lb.DensePolynomial(ctx, torch.from_numpy(a.view(np.int64)).cuda()) for a in A],
             [lb.DensePolynomial(ctx, torch.from_numpy(b.view(np.int64)).cuda()) for b in B],
             lb.DensePolynomial(ctx, torch.from_numpy(C.view(np.int64)).cuda()))
    torch.cuda.synchronize()
    _both(ctx, A, B, C, coeffs, _claim(np.random.default_rng(3)), 9, polys)


def test_inputs_unchanged_and_verified(ctx):
    """the caller's polynomials keep their commitments, and the oracle verifier accepts the proof of the true claim with
    the final claim C(r) sum_k coeff_k A_k(r) B_k(r)"""
    import lasso_b200 as lb

    nv, n = 10, 4
    A, B, C, coeffs = cb.random_case(n, nv, 41, "eq")
    claim = cb.true_claim(A, B, C, coeffs)
    polys = ([lb.DensePolynomial(ctx, a) for a in A], [lb.DensePolynomial(ctx, b) for b in B], lb.DensePolynomial(ctx, C))
    gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=ol.generators(lb.poly_gens_points_needed(nv)))
    every = polys[0] + polys[1] + [polys[2]]
    before = [p.commit(gens) for p in every]
    got = _both(ctx, A, B, C, coeffs, claim, nv, polys)
    assert [p.commit(gens) for p in every] == before
    rc, e, r = osc.sumcheck_verify(got.bytes, claim, nv, 3, od.Transcript(LABEL))
    assert rc == 0 and np.array_equal(r, got.r)
    f = ol.fr_ints(got.final_evals)
    want = sum(k * f[i] * f[n + i] for i, k in enumerate(ol.fr_ints(coeffs))) * f[2 * n] % ol.L_FR
    assert ol.fr_ints(e)[0] == want


@pytest.mark.parametrize("n,nv,rounds", [(1, 1, 1), (2, 5, 5), (2, 10, 6), (7, 8, 8)])
def test_equals_prove_arbitrary(ctx, n, nv, rounds):
    """with the true claim, prove_arbitrary over [A_0.., B_0.., C] with g = C sum_k coeff_k A_k B_k gives the same bytes,
    r and finals: both prove the same round polynomials"""
    import lasso_b200 as lb

    A, B, C, coeffs = cb.random_case(n, nv, 900 + n + nv, "eq" if n % 2 else "random")
    claim = cb.true_claim(A, B, C, coeffs)
    ks = ol.fr_ints(coeffs)

    def g(v):
        acc = v[0] * v[n] * ks[0]
        for k in range(1, n):
            acc = acc + v[k] * v[n + k] * ks[k]
        return acc * v[2 * n]

    got = _both(ctx, A, B, C, coeffs, claim, rounds)
    t = lb.Transcript(LABEL)
    polys = [lb.DensePolynomial(ctx, Z) for Z in list(A) + list(B) + [C]]
    arb = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, lb.Comb(g, 2 * n + 1, 3), t, rounds)
    assert arb.bytes == got.bytes
    assert np.array_equal(arb.r, got.r)
    assert np.array_equal(arb.final_evals, got.final_evals)
    assert np.array_equal(arb.claim, claim)


def test_golden(ctx):
    doc = json.load(open(os.path.join(HERE, "golden", "cubic_batched.json")))["cases"]
    for name in sorted(cb.GOLDEN):
        g = doc[name]
        A, B, C, coeffs, rounds = cb.golden_inputs(name)
        claim = np.frombuffer(bytes.fromhex(g["claim_hex"]), dtype=np.uint64)
        got, after = _gpu(ctx, A, B, C, coeffs, claim, rounds, label=cb.TRANSCRIPT_LABEL)
        assert len(got.bytes) == g["proof_len"], name
        assert hashlib.sha256(cb.digest_input(got.bytes, got.r, got.final_evals)).hexdigest() == g["sha256"], name
        assert after.tobytes().hex() == g["after_challenge_hex"], name


def test_launch_count(ctx):
    """single GPU, every coefficient non-zero: one evaluation for round 1; before round 2 an out-of-place bind of the
    caller's arrays and an evaluation; one fused bind + evaluation for every later round; one finals kernel.
    launches = R + 2 for R >= 2 rounds, 2 for R = 1."""
    import lasso_b200 as lb

    for n, nv, rounds in [(1, 1, 1), (2, 3, 1), (2, 3, 2), (7, 10, 10), (32, 13, 13), (3, 13, 5)]:
        A, B, C, coeffs = cb.random_case(n, nv, 60 + nv)
        polys = ([lb.DensePolynomial(ctx, a) for a in A], [lb.DensePolynomial(ctx, b) for b in B], lb.DensePolynomial(ctx, C))
        before = ctx.launches
        _gpu(ctx, A, B, C, coeffs, _claim(np.random.default_rng(4)), rounds, polys)
        assert ctx.launches - before == (rounds + 2 if rounds >= 2 else 2), (n, nv, rounds)


def test_errors(ctx):
    """every error comes before any launch and leaves the transcript as it was"""
    import lasso_b200 as lb
    from lasso_b200.api import LassoError

    A, B, C, coeffs = cb.random_case(2, 4, 5)
    pa, pb, pc = [lb.DensePolynomial(ctx, a) for a in A], [lb.DensePolynomial(ctx, b) for b in B], lb.DensePolynomial(ctx, C)
    other = lb.DensePolynomial(ctx, C[:8])
    claim = _claim(np.random.default_rng(5))
    bad = coeffs.copy()
    bad[1] = ol.int_to_limbs(ol.L_FR)  # l itself: not canonical
    ctx2 = lb.Context(0)
    foreign = lb.DensePolynomial(ctx2, C)
    many = cb.random_case(33, 2, 6)
    pm = [lb.DensePolynomial(ctx, a) for a in many[0]]
    cases = [
        (ERR_STRATEGY, ([], [], pc, coeffs[:0], claim, 4)),
        (ERR_STRATEGY, (pm, pm, lb.DensePolynomial(ctx, many[2]), many[3], claim, 2)),
        (ERR_STRATEGY, ([pa[0], foreign], pb, pc, coeffs, claim, 4)),
        (ERR_STRATEGY, (pa, pb, foreign, coeffs, claim, 4)),
        (ERR_LENGTH, ([pa[0], other], pb, pc, coeffs, claim, 4)),
        (ERR_LENGTH, (pa, pb, other, coeffs, claim, 3)),
        (ERR_LENGTH, (pa, pb, pc, coeffs, claim, 0)),
        (ERR_LENGTH, (pa, pb, pc, coeffs, claim, 5)),
        (ERR_VALUE, (pa, pb, pc, bad, claim, 4)),
        (ERR_VALUE, (pa, pb, pc, coeffs, ol.int_to_limbs(ol.L_FR + 5), 4)),
    ]
    fresh = lb.Transcript(LABEL).challenge_scalar(b"after")
    for code, (a, b, c, k, e, rounds) in cases:
        t = lb.Transcript(LABEL)
        before = ctx.launches
        with pytest.raises(LassoError) as ei:
            lb.SumcheckInstanceProof.prove_cubic_batched(ctx, a, b, c, k, e, t, rounds)
        assert ei.value.code == code, (code, ei.value)
        assert ctx.launches == before
        assert np.array_equal(t.challenge_scalar(b"after"), fresh)
    # the C ABI's own checks: a short output buffer (with *proof_len still set) and a null transcript
    import ctypes as C_

    from lasso_b200.api import _p, _poly_handles, lib

    out, r, fin = np.zeros(100, dtype=np.uint8), np.zeros((4, 4), dtype=np.uint64), np.zeros((5, 4), dtype=np.uint64)
    need = C_.c_size_t(0)
    t = lb.Transcript(LABEL)
    before = ctx.launches
    for tr, cap in ((t._h, 100), (None, 8 + 104 * 4)):
        rc = lib().lasso_sumcheck_prove_cubic_batched(
            ctx._h, _poly_handles(pa), _poly_handles(pb), C_.c_size_t(2), pc._h, _p(np.ascontiguousarray(coeffs)),
            _p(np.ascontiguousarray(claim)), C_.c_size_t(4), tr, _p(out), C_.c_size_t(cap), C_.byref(need), _p(r),
            _p(fin[:2]), _p(fin[2:4]), _p(fin[4:]))
        assert rc == ERR_LENGTH and need.value == 8 + 104 * 4
    assert ctx.launches == before
    assert np.array_equal(t.challenge_scalar(b"after"), fresh)
    del foreign
    ctx2.close()


# ------------------------------------------------------------------------------------------------ sharded contexts
def _run(nproc, same_gpu, timeout=1500):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ)
    if same_gpu:
        env["LASSO_SHARD_SAME_GPU"] = "1"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert MARK + " PASS" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]


def test_sharded_two_ranks_one_gpu():
    _run(2, True)


def test_sharded_four_ranks_one_gpu():
    _run(4, True)


def test_sharded_two_ranks_two_gpus():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (the one-GPU runs cover the same code)")
    _run(2, False)


def _sharded_cases(G):
    """(name, n, nv, rounds, C kind, zero coefficients, repeated, CUDA input): the smallest num_vars G allows with full
    and partial rounds, rounds that end while sharded and rounds that end in the replicated tail"""
    nv0 = max(1, 2 * (G.bit_length() - 1) - 1)
    out = [("min_full", 2, nv0, nv0, "eq", [], False, False), ("min_one", 3, nv0, 1, "random", [], False, False),
           ("n1_nv10", 1, 10, 10, "eq", [], False, True), ("n7_nv10_tail", 7, 10, 9, "random", [], True, False),
           ("n32_nv13", 32, 13, 13, "eq", [], False, False), ("n4_nv13_sharded_end", 4, 13, 3, "random", [], False, True),
           ("zero_one", 3, 10, 10, "eq", [1], False, False), ("zero_all", 2, 10, 6, "random", "all", False, False),
           ("zero_all_32", 32, nv0 + 2, nv0 + 1, "random", "all", False, False)]
    return out


def _sharded_suite(ctx, G, dev):
    import torch

    import lasso_b200 as lb

    res = {}
    for name, n, nv, rounds, ckind, zeros, repeated, cuda in _sharded_cases(G):
        A, B, C, coeffs = cb.random_case(n, nv, 7000 + n + nv + rounds, ckind, ("u32", "full"))
        if zeros:
            coeffs[list(range(n)) if zeros == "all" else zeros] = 0
        if repeated:
            A[1] = B[2] = C
            B[0] = A[0]
        claim = cb.true_claim(A, B, C, coeffs) if n <= 7 else _claim(np.random.default_rng(nv))
        mk = (lambda Z: lb.DensePolynomial(ctx, torch.from_numpy(Z.view(np.int64)).to(dev))) if cuda else \
            (lambda Z: lb.DensePolynomial(ctx, Z))
        cache = {}
        for Z in list(A) + list(B) + [C]:
            if id(Z) not in cache:
                cache[id(Z)] = mk(Z)
        if cuda:
            torch.cuda.synchronize()
        polys = ([cache[id(a)] for a in A], [cache[id(b)] for b in B], cache[id(C)])
        got, after = _gpu(ctx, A, B, C, coeffs, claim, rounds, polys)
        res[name] = (got.bytes.hex(), got.r.tobytes().hex(), got.final_evals.tobytes().hex(), after.tobytes().hex())
        if n <= 7:
            want, o_after = _oracle(A, B, C, coeffs, claim, rounds)
            res[name + " oracle"] = (want["proof"].hex(), want["r"].tobytes().hex(), want["finals"].tobytes().hex(),
                                     o_after.tobytes().hex())
    return res


def _worker():
    import torch
    import torch.distributed as dist

    import lasso_b200 as lb

    rank, local = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    G = int(os.environ.get("WORLD_SIZE", 1))
    if os.environ.get("LASSO_SHARD_SAME_GPU") == "1":
        local = 0
        torch.cuda.set_device(0)
        dist.init_process_group("gloo")
    else:
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    single = [None]
    if rank == 0:  # the single-GPU results, before the collective context exists
        c1 = lb.Context(local)
        single = [_sharded_suite(c1, G, dev)]
        c1.close()
    dist.broadcast_object_list(single, src=0)
    res1 = single[0]
    c = lb.Context(local)
    c.init_comm()
    res = _sharded_suite(c, G, dev)
    got = [None] * G
    dist.all_gather_object(got, res)
    if rank == 0:
        fails = []
        for g, rg in enumerate(got):
            fails += ["rank %d %s" % (g, k) for k in sorted(set(res1) | set(rg)) if res1.get(k) != rg.get(k)]
        fails += ["oracle %s" % k for k in res1 if k + " oracle" in res1 and res1[k] != res1[k + " oracle"]]
        print(MARK, "PASS" if not fails else "FAIL %r" % fails[:40], "(%d items)" % len(res1), flush=True)
    dist.barrier()
    c.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker()
