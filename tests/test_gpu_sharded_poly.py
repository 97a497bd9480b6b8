"""A caller's dense polynomials on a sharded context: create (host arrays, CUDA tensors, strided views), commit, hiding
commit, evaluate, open, merge, batched evaluation, the combined opening, the eq and comb constructors and the composed
protocol of DESIGN §3.12 are collective over G ranks, and every rank must return the bytes of a single-GPU context.

Rank 0 first runs the same steps on a plain context; every rank then runs them on the sharded one and the results are
compared, item by item.  Run as a script under torch.distributed.run it is the worker: 2 and 4 ranks time-slicing
GPU 0 (LASSO_SHARD_SAME_GPU=1, gloo for the plumbing), or one rank per GPU.  The ranks other than 0 build one set of
generators without the digit-multiples tables, so that ranks holding different tables are covered too."""
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

import combined_eval_cases as cec  # noqa: E402
import compose_cases as cc  # noqa: E402
import dense_poly_cases as dc  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_hiding_lib as oh  # noqa: E402
import oracle_lib as ol  # noqa: E402
from lasso_b200.api import LASSO_ERR_LENGTH, LASSO_ERR_STRATEGY, LASSO_ERR_VALUE  # noqa: E402

pytestmark = pytest.mark.gpu
MARK = "SHARDED_POLY"


def _run(nproc, same_gpu, mode="main", timeout=1500):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ)
    env.pop("LASSO_B200_NO_MULTIPLES", None)
    if same_gpu:
        env["LASSO_SHARD_SAME_GPU"] = "1"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__), mode]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert MARK + " PASS" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]


def test_two_ranks_one_gpu():
    _run(2, True)


def test_four_ranks_one_gpu():
    _run(4, True)


def test_two_ranks_two_gpus():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (the one-GPU runs cover the same code)")
    _run(2, False)


def test_at_size_two_ranks_one_gpu():
    """2^22 evaluations, full width and 16-bit, against tests/golden/dense_poly.json and dense_poly_hiding.json"""
    _run(2, True, "at_size")


# ------------------------------------------------------------------------------------------------ the worker
def _h(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def _a(x):
    return np.ascontiguousarray(x).tobytes().hex()


def _values(kind, n, rng):
    if kind == "full":
        return dc.random_full(rng, n)
    bits = {"u16": 16, "u32": 32}[kind]
    return dc.fr_from_u64(rng.integers(0, 1 << bits, size=n, dtype=np.uint64))


def _nv_min(G):
    return max(0, 2 * (G.bit_length() - 1) - 1)


def _cases(G):
    return [(_nv_min(G), k) for k in ("u16", "full")] + [(nv, k) for nv in (13, 16) for k in ("u16", "u32", "full")]


_STREAMS = {}


def _stream(nv, label=b"gens_sparse_poly"):
    key = (nv, label)
    if key not in _STREAMS:
        _STREAMS[key] = np.ascontiguousarray(ol.generators(lb.poly_gens_points_needed(nv), label))
    return _STREAMS[key]


def _open(ctx, p, gens, r, seed, label):
    """commit, evaluate, open on a transcript that absorbed the commitment -> dict of results"""
    comm = p.commit(gens)
    Zr = p.evaluate(r)
    t = lb.Transcript(label)
    t.append_poly_commitment(b"poly", comm)
    proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, lb.RandomTape(b"proof", seed))
    return dict(comm=comm.hex(), eval=_a(Zr), proof=proof.bytes.hex(), czr=proof.C_Zr.hex(),
                next=_a(t.challenge_scalar(b"next")))


def _open_hiding(ctx, p, gens, r, seed, label):
    tape = lb.RandomTape(b"proof", seed)
    comm, blinds = p.commit_hiding(gens, tape)
    Zr = p.evaluate(r)
    t = lb.Transcript(label)
    t.append_poly_commitment(b"poly", comm)
    blind_Zr = tape.random_scalar(b"blind_Zr")
    proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, tape, blinds=blinds, blind_Zr=blind_Zr)
    return dict(hcomm=comm.hex(), blinds=_a(blinds), hproof=proof.bytes.hex(), hczr=proof.C_Zr.hex(),
                hnext=_a(t.challenge_scalar(b"next")))


def _suite(ctx, G, dev, mixed_tables):
    """every collective call of the feature on ctx -> {item: hex}; the same on a single-GPU context and a sharded one"""
    import torch

    out = {}
    for i, (nv, kind) in enumerate(_cases(G)):
        rng = np.random.default_rng(1000 + 37 * nv + i)
        Z, r, seed = _values(kind, 1 << nv, rng), dc.random_full(rng, nv), dc.random_full(rng, 1)[0]
        gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=_stream(nv))
        p = lb.DensePolynomial(ctx, Z)
        key = "%d/%s/" % (nv, kind)
        for k, v in _open(ctx, p, gens, r, seed, b"sharded_poly").items():
            out[key + k] = v
        for k, v in _open_hiding(ctx, p, gens, r, seed, b"sharded_poly_hiding").items():
            out[key + k] = v
        # the same polynomial from a contiguous int64 CUDA tensor and from a strided view of one
        t = torch.from_numpy(Z.view(np.int64)).to(dev)
        wide = torch.zeros((Z.shape[0], 7), dtype=torch.int64, device=dev)
        wide[:, 2:6] = t
        for name, src in (("dev", t), ("strided", wide[:, 2:6])):
            q = lb.DensePolynomial(ctx, src)
            out[key + name] = q.commit(gens).hex() + _a(q.evaluate(r))
            del q
        del p, gens
    # merge of unequal sizes, batched evaluation, and the combined opening of the golden cases
    rng = np.random.default_rng(77)
    sizes = [max(_nv_min(G), v) for v in (6, 4, 5)]
    parts = [lb.DensePolynomial(ctx, _values(k, 1 << v, rng)) for v, k in zip(sizes, ("full", "u16", "u32"))]
    m = lb.DensePolynomial.merge(ctx, parts)
    mr = dc.random_full(rng, m.num_vars)
    mg = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", m.num_vars, stream=_stream(m.num_vars))
    for k, v in _open(ctx, m, mg, mr, dc.random_full(rng, 1)[0], b"merged").items():
        out["merge/" + k] = v
    same = [lb.DensePolynomial(ctx, _values(k, 1 << 7, rng)) for k in ("u32", "full", "u16", "u32")]
    out["batch"] = _a(lb.DensePolynomial.evaluate_batch(ctx, same, dc.random_full(rng, 7)))
    for name in cec.SMALL:
        nv, comps, r, seed = cec.golden_inputs(name)
        polys = [lb.DensePolynomial(ctx, a) for a in comps]
        cm = lb.DensePolynomial.merge(ctx, polys)
        cg = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", cm.num_vars, stream=_stream(cm.num_vars))
        evals = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
        t = lb.Transcript(cec.TRANSCRIPT_LABEL)
        proof = lb.CombinedTableEvalProof.prove(ctx, cm, evals, r, cg, t, lb.RandomTape(cec.TAPE_LABEL, seed))
        out["combined/" + name] = json.dumps(dict(digest=_h(cec.digest_input(evals, proof.data)), comm=_h(cm.commit(cg)),
                                                  after=_a(t.challenge_scalar(b"after"))))
    # the constructors
    nv = max(_nv_min(G), 9)
    rng = np.random.default_rng(99)
    eg = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=_stream(nv))
    eq = lb.DensePolynomial.eq(ctx, dc.random_full(rng, nv))
    out["eq"] = eq.commit(eg).hex()
    a, b = (lb.DensePolynomial(ctx, _values(k, 1 << nv, rng)) for k in ("u16", "full"))
    q = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda v: v[0] * v[1] + v[2] * 3, 3), [a, b, eq])
    out["comb"] = q.commit(eg).hex() + _a(q.evaluate(dc.random_full(rng, nv)))
    # generators built on every rank but 0 without the multiples tables (the opening's bucket path, the commitments'
    # bucket row-MSM): the exchanges must still line up and give the same bytes
    nv = 14
    if mixed_tables:
        os.environ["LASSO_B200_NO_MULTIPLES"] = "1"
    try:
        xg = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=_stream(nv))
    finally:
        os.environ.pop("LASSO_B200_NO_MULTIPLES", None)
    for kind in ("u16", "full"):
        rng = np.random.default_rng(140 + len(kind))
        p = lb.DensePolynomial(ctx, _values(kind, 1 << nv, rng))
        r, seed = dc.random_full(rng, nv), dc.random_full(rng, 1)[0]
        for k, v in list(_open(ctx, p, xg, r, seed, b"mixed").items()) + list(_open_hiding(ctx, p, xg, r, seed, b"mixed").items()):
            out["mixed/%s/%s" % (kind, k)] = v
    out.update(_composed(ctx, G))
    return out


def _composed(ctx, G):
    """DESIGN §3.12 with v from the host: commit v, absorb it and the sparse commitment, draw r, prove the lookups on the
    same transcript, open v at the claimed evaluation"""
    C_, log_m, n = 4, 16, 1 << 11
    log_s = 11
    rng = np.random.default_rng(311)
    idx = rng.integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    seed = dc.random_full(rng, 1)[0]
    S = lb.Strategy(lb.XOR, C_, log_m)
    v = cc.outputs(lb.XOR, C_, log_m, 0, cc.dim_usize(idx, n))
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, n, 4, log_m,
                                           stream=ol.generators(lb.gens_points_needed(C_, n, 4, log_m)))
    T, tape = lb.Transcript(b"compose"), lb.RandomTape(b"proof", seed)
    T.append_protocol_name(b"Lasso composed")
    vp = lb.DensePolynomial(ctx, v)
    v_gens = lb.PolyCommitmentGens.new(ctx, b"gens_outputs", log_s, stream=_stream(log_s, b"gens_outputs"))
    comm_v = vp.commit(v_gens)
    T.append_poly_commitment(b"outputs", comm_v)
    comm_sparse = dense.commit(gens)
    T.append_sparse_commitment(comm_sparse)
    r = T.challenge_vector(b"r", log_s)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=T, random_tape=tape)
    opening = lb.PolyEvalProof.prove(ctx, vp, r, proof.claimed_evaluation, v_gens, T, tape)
    ev = vp.evaluate(r)
    return {"compose": json.dumps(dict(comm_v=_h(comm_v), sparse=_h(comm_sparse), proof=_h(proof.bytes),
                                       claim=_a(proof.claimed_evaluation), ev=_a(ev), opening=_h(opening.bytes),
                                       czr=opening.C_Zr.hex(), last=_a(T.challenge_scalar(b"next"))))}


def _code(fn):
    try:
        fn()
        return 0
    except lb.LassoError as e:
        return e.code


def _errors(ctx, G, rank, dev):
    """-> {check: code or verdict}; the same on every rank"""
    import torch

    out = {}
    nv = max(_nv_min(G), 6)
    rng = np.random.default_rng(5)
    Z = _values("u16", 1 << nv, rng)
    gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=_stream(nv))
    good = lb.DensePolynomial(ctx, Z)
    bad = Z.copy()
    bad[G - 1 + G * 3] = ol.fr_array([0])[0]
    bad[G - 1 + G * 3, 3] = np.uint64(2**64 - 1)  # not a canonical residue, in the last rank's rows
    out["bad_host"] = _code(lambda: lb.DensePolynomial(ctx, bad))
    out["bad_device"] = _code(lambda: lb.DensePolynomial(ctx, torch.from_numpy(bad.view(np.int64)).to(dev)))
    out["commit_after"] = _h(good.commit(gens))
    t = lb.Transcript(b"errors")
    small = _nv_min(G) - 1
    if small >= 0:
        before = lb.Transcript(b"errors").challenge_scalar(b"c").tolist()
        out["small_poly"] = _code(lambda: lb.DensePolynomial(ctx, _values("u16", 1 << small, rng)))
        out["small_dev"] = _code(lambda: lb.DensePolynomial(ctx, torch.from_numpy(_values("full", 1 << small, rng).view(np.int64)).to(dev)))
        out["small_eq"] = _code(lambda: lb.DensePolynomial.eq(ctx, dc.random_full(rng, small)))
        out["small_gens"] = _code(lambda: lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", small, stream=_stream(small)))
        out["transcript_untouched"] = t.challenge_scalar(b"c").tolist() == before
    out["sumcheck"] = _code(lambda: lb.SumcheckInstanceProof.prove_arbitrary(ctx, [good, good], lb.Comb(lambda v: v[0] * v[1], 2), t))
    out["gp_circuit"] = _code(lambda: lb.GrandProductCircuit(ctx, good))
    idx = np.random.default_rng(6).integers(0, 1 << 8, size=(64, 2), dtype=np.uint64)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, 8)
    out["outputs"] = _code(lambda: dense.outputs(lb.Strategy(lb.AND, 2, 8)))
    out["commit_end"] = _h(good.commit(gens))
    return out


def _expected_errors(G, single_commit):
    want = dict(bad_host=LASSO_ERR_VALUE, bad_device=LASSO_ERR_VALUE, commit_after=single_commit,
                sumcheck=LASSO_ERR_STRATEGY, gp_circuit=LASSO_ERR_STRATEGY, outputs=LASSO_ERR_STRATEGY, commit_end=single_commit)
    if _nv_min(G) >= 1:
        want.update(small_poly=LASSO_ERR_LENGTH, small_dev=LASSO_ERR_LENGTH, small_eq=LASSO_ERR_LENGTH,
                    small_gens=LASSO_ERR_LENGTH, transcript_untouched=True)
    return want


def _oracle_checks(res, G):
    """the oracle's verifiers accept the small proofs (rank 0, on the sharded context's bytes)"""
    bad = []
    for i, (nv, kind) in enumerate(_cases(G)):
        if nv > 13:
            continue
        rng = np.random.default_rng(1000 + 37 * nv + i)
        _values(kind, 1 << nv, rng)
        r = dc.random_full(rng, nv)
        key = "%d/%s/" % (nv, kind)
        comm, proof = bytes.fromhex(res[key + "comm"]), bytes.fromhex(res[key + "proof"])
        v = od.Transcript(b"sharded_poly")
        v.append_poly_commitment(b"poly", comm)
        Zr = np.frombuffer(bytes.fromhex(res[key + "eval"]), dtype=np.uint64)
        if od.verify(_stream(nv), nv, comm, proof, r, Zr, v) != 0:
            bad.append(key + "proof")
        hcomm, hproof = bytes.fromhex(res[key + "hcomm"]), bytes.fromhex(res[key + "hproof"])
        v = od.Transcript(b"sharded_poly_hiding")
        v.append_poly_commitment(b"poly", hcomm)
        if oh.verify(_stream(nv), nv, hcomm, hproof, r, bytes.fromhex(res[key + "hczr"]), v) != 0:
            bad.append(key + "hproof")
    for name in cec.SMALL:
        g = json.load(open(os.path.join(HERE, "golden", "combined_eval.json")))["cases"].get(name)
        got = json.loads(res["combined/" + name])
        if g and (got["digest"] != g["sha256"] or got["comm"] != g["commitment_sha256"]):
            bad.append("combined golden " + name)
    return bad


def _at_size(ctx, dev):
    """-> list of mismatches against the golden hashes"""
    import torch

    bad = []
    plain = json.load(open(os.path.join(HERE, "golden", "dense_poly.json")))["cases"]
    hiding = json.load(open(os.path.join(HERE, "golden", "dense_poly_hiding.json")))["cases"]
    for name in ("full_nv22", "u16_nv22"):
        nv, Z, r, seed = dc.inputs(name)
        gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=np.ascontiguousarray(ol.generators(dc.n_generators(nv))))
        for src_name, src in (("host", Z), ("device", torch.from_numpy(Z.view(np.int64)).to(dev))):
            p = lb.DensePolynomial(ctx, src)
            g = plain[name]
            comm = p.commit(gens)
            Zr = p.evaluate(r)
            t = lb.Transcript(dc.TRANSCRIPT_LABEL)
            t.append_poly_commitment(dc.COMMIT_LABEL, comm)
            proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, lb.RandomTape(dc.TAPE_LABEL, seed))
            got = (_h(comm), Zr.tobytes().hex(), _h(proof.bytes), proof.C_Zr.hex(), t.challenge_scalar(b"after").tobytes().hex())
            want = (g["commitment_sha256"], g["Zr_hex"], g["proof_sha256"], g["C_Zr_hex"], g["after_challenge_hex"])
            if got != want:
                bad.append("%s %s plain" % (name, src_name))
            del p
        p = lb.DensePolynomial(ctx, Z)
        g = hiding[name]
        tape = lb.RandomTape(dc.TAPE_LABEL, seed)
        comm, blinds = p.commit_hiding(gens, tape)
        t = lb.Transcript(dc.TRANSCRIPT_LABEL)
        t.append_poly_commitment(dc.COMMIT_LABEL, comm)
        Zr = p.evaluate(r)
        blind_Zr = tape.random_scalar(b"blind_Zr")
        proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, tape, blinds=blinds, blind_Zr=blind_Zr)
        got = (_h(comm), _h(blinds.tobytes()), _h(proof.bytes), proof.C_Zr.hex(), t.challenge_scalar(b"after").tobytes().hex())
        want = (g["commitment_sha256"], g["blinds_sha256"], g["proof_sha256"], g["C_Zr_hex"], g["after_challenge_hex"])
        if got != want:
            bad.append("%s hiding" % name)
        del p, gens
    return bad


def _worker(mode):
    import torch
    import torch.distributed as dist

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
    if mode == "at_size":
        c = lb.Context(local)
        c.init_comm()
        bad = _at_size(c, dev)
        got = [None] * G
        dist.all_gather_object(got, bad)
        if rank == 0:
            fails = [(g, b) for g, b in enumerate(got) if b]
            print(MARK, "PASS" if not fails else "FAIL %r" % fails, flush=True)
        dist.barrier()
        c.close()
        dist.destroy_process_group()
        return
    single = [None]
    if rank == 0:  # the single-GPU results, before the collective context exists
        c1 = lb.Context(local)
        res1 = _suite(c1, G, dev, False)
        nv = max(_nv_min(G), 6)
        Z = _values("u16", 1 << nv, np.random.default_rng(5))
        g1 = lb.PolyCommitmentGens.new(c1, b"gens_sparse_poly", nv, stream=_stream(nv))
        single = [(res1, _h(lb.DensePolynomial(c1, Z).commit(g1)))]
        del g1
        c1.close()
    dist.broadcast_object_list(single, src=0)
    res1, commit1 = single[0]
    c = lb.Context(local)
    c.init_comm()
    res = _suite(c, G, dev, rank != 0)
    errs = _errors(c, G, rank, dev)
    got = [None] * G
    dist.all_gather_object(got, (res, errs))
    if rank == 0:
        fails = []
        want_err = _expected_errors(G, commit1)
        for g, (rg, eg) in enumerate(got):
            fails += ["rank %d %s" % (g, k) for k in sorted(set(res1) | set(rg)) if res1.get(k) != rg.get(k)]
            fails += ["rank %d error %s: %r != %r" % (g, k, eg.get(k), want_err[k]) for k in want_err if eg.get(k) != want_err[k]]
        fails += _oracle_checks(res, G)
        print(MARK, "PASS" if not fails else "FAIL %r" % fails[:40], "(%d items)" % len(res1), flush=True)
    dist.barrier()
    c.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker(sys.argv[1] if len(sys.argv) > 1 else "main")
