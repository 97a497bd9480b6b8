"""Commit, evaluate and open a caller's polynomial on a context sharded over G ranks (one rank per GPU), against the same
calls on one GPU: G = 1 is the run with one process, which uses a plain context.
Cases of tests/dense_poly_cases.py: 2^22 and 2^24 evaluations, full width and 16-bit integers (the integer path: the
u32 mirror and, where the tables fit, the 16-bit multiples).  Each call is timed with the host clock around the library
call on every rank after a barrier; every call ends in a device synchronise.  A rank's time is the slowest rank's, W
warm-ups, then the median and range of N runs.  Every commitment, evaluation and proof is checked against
tests/golden/dense_poly.json on every rank.  Prints one JSON object with the card's name and power limit.
usage: torchrun --nproc-per-node G tools/sharded_poly_bench.py [--warmup W] [--reps N] [--cases a,b]
       (LASSO_SHARD_SAME_GPU=1: every rank on GPU 0 -- a check of the exchanges, not a measurement of scaling)"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import dense_poly_cases as dc  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import oracle_lib as ol  # noqa: E402

CASES = ("full_nv22", "u16_nv22", "full_nv24", "u16_nv24")


def card(device):
    try:
        return subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def slowest(ms, world):
    """the slowest rank's time of one call"""
    if world == 1:
        return ms
    t = torch.tensor([ms], dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def timed(fn, world):
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    out = fn()
    return out, slowest((time.perf_counter() - t0) * 1e3, world)


def run_case(ctx, name, warmup, reps, world, gold):
    nv, Z, r, seed = dc.inputs(name)
    gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=np.ascontiguousarray(ol.generators(dc.n_generators(nv))))
    p = lb.DensePolynomial(ctx, Z)
    times = {"commit": [], "evaluate": [], "prove": []}
    ok = True
    for it in range(warmup + reps):
        comm, t_c = timed(lambda: p.commit(gens), world)
        Zr, t_e = timed(lambda: p.evaluate(r), world)
        t = lb.Transcript(dc.TRANSCRIPT_LABEL)
        t.append_poly_commitment(dc.COMMIT_LABEL, comm)
        proof, t_p = timed(lambda: lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, lb.RandomTape(dc.TAPE_LABEL, seed)), world)
        ok = ok and (hashlib.sha256(comm).hexdigest(), Zr.tobytes().hex(), hashlib.sha256(proof.bytes).hexdigest()) == (
            gold["commitment_sha256"], gold["Zr_hex"], gold["proof_sha256"])
        if it >= warmup:
            times["commit"].append(t_c)
            times["evaluate"].append(t_e)
            times["prove"].append(t_p)
    del p, gens
    return {k: stats(v) for k, v in times.items()}, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", 1))
    rank, local = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    same_gpu = os.environ.get("LASSO_SHARD_SAME_GPU") == "1"
    if same_gpu:
        local = 0
    torch.cuda.set_device(local)
    if world > 1:  # gloo carries the job id and the timings; the library exchanges through its own peer buffers
        dist.init_process_group("gloo")
    ctx = lb.Context(local)
    if world > 1:
        ctx.init_comm()
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "dense_poly.json")))["cases"]
    res, all_ok = {}, True
    for name in a.cases.split(","):
        res[name], ok = run_case(ctx, name, a.warmup, a.reps, world, gold[name])
        all_ok = all_ok and ok
    if world > 1:
        flags = [None] * world
        dist.all_gather_object(flags, all_ok)
        all_ok = all(flags)
    if rank == 0:
        print(json.dumps({"G": world, "same_gpu": same_gpu and world > 1, "card": card(local), "golden_ok": all_ok,
                          "ms": res}), flush=True)
    if world > 1:
        dist.barrier()
    ctx.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
