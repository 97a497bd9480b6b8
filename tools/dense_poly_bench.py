"""DensePolynomial::new / commit / evaluate and PolyEvalProof::prove on the GPU, each timed separately, for num_vars
20, 22 and 24 with full-width and 16-bit values (tests/dense_poly_cases.py inputs), the evaluations given from the host
(a numpy array) and from the device (a torch CUDA tensor), alternating in one process.
Each call is timed with the host clock around the library call; every call ends in a device synchronise (the verdict
of the ingest, the commitment's points, Z(r), the proof's last message).  W warm-ups, then the median and range of N
runs.  Every commitment and proof is checked against tests/golden/dense_poly.json.  Also prints the card's name and
power limit, and (--cpu) the CPU oracle's commit and prove at 2^20 with 8 threads for comparison.
--hiding adds a leg per case: the plain commit + prove and the hiding ones (DensePolynomial.commit_hiding, the proof
with blinds and blind_Zr) alternating on one polynomial, hiding results checked against
tests/golden/dense_poly_hiding.json where it has the case, with the launches of each call.
usage: python tools/dense_poly_bench.py [--warmup W] [--reps N] [--cases a,b] [--cpu] [--hiding] [--out FILE.json]"""
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

import dense_poly_cases as dc  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_lib as ol  # noqa: E402

CASES = ("full_nv20", "u16_nv20", "full_nv22", "u16_nv22", "full_nv24", "u16_nv24")


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def ms_since(t0):
    return (time.perf_counter() - t0) * 1e3


def one(ctx, src, gens, r, seed):
    t = {}
    t0 = time.perf_counter()
    p = lb.DensePolynomial(ctx, src)
    t["create"] = ms_since(t0)
    t0 = time.perf_counter()
    comm = p.commit(gens)
    t["commit"] = ms_since(t0)
    t0 = time.perf_counter()
    Zr = p.evaluate(r)
    t["evaluate"] = ms_since(t0)
    tr = lb.Transcript(dc.TRANSCRIPT_LABEL)
    tr.append_poly_commitment(dc.COMMIT_LABEL, comm)
    tape = lb.RandomTape(dc.TAPE_LABEL, seed)
    t0 = time.perf_counter()
    proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, tr, tape)
    t["prove"] = ms_since(t0)
    return t, hashlib.sha256(comm).hexdigest(), hashlib.sha256(proof.bytes).hexdigest()


def run_case(ctx, name, warmup, reps, gold):
    nv, Z, r, seed = dc.inputs(name)
    stream = np.ascontiguousarray(ol.generators(gold["n_generators"]))
    t0 = time.perf_counter()
    gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream)
    gens_ms = ms_since(t0)
    inputs = {"host_numpy": Z, "cuda_int64": torch.from_numpy(Z.view(np.int64)).cuda()}
    torch.cuda.synchronize()
    times = {k: {s: [] for s in ("create", "commit", "evaluate", "prove")} for k in inputs}
    match = True
    for i in range(warmup + reps):
        for k, src in inputs.items():  # alternating
            t, hc, hp = one(ctx, src, gens, r, seed)
            match &= hc == gold["commitment_sha256"] and hp == gold["proof_sha256"]
            if i >= warmup:
                for s, v in t.items():
                    times[k][s].append(v)
    out = {"num_vars": nv, "values": dc.CASES[name][1], "golden_match": bool(match), "gens_create_ms": round(gens_ms, 1)}
    for k in inputs:
        out[k] = {s: stats(v) for s, v in times[k].items()}
    return out


def run_hiding(ctx, name, warmup, reps, gold):
    """plain and hiding commit + prove alternating on one polynomial (host input)"""
    nv, Z, r, seed = dc.inputs(name)
    stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
    gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream)
    p = lb.DensePolynomial(ctx, Z)
    Zr = p.evaluate(r)
    times = {k: {"commit": [], "prove": []} for k in ("plain", "hiding")}
    launches = {k: {} for k in times}
    match = True
    for i in range(warmup + reps):
        for k in ("plain", "hiding"):
            tape = lb.RandomTape(dc.TAPE_LABEL, seed)
            l0, t0 = ctx.launches, time.perf_counter()
            if k == "plain":
                comm = p.commit(gens)
            else:
                comm, blinds = p.commit_hiding(gens, tape)
            tc, l1 = ms_since(t0), ctx.launches
            tr = lb.Transcript(dc.TRANSCRIPT_LABEL)
            tr.append_poly_commitment(dc.COMMIT_LABEL, comm)
            kw = {} if k == "plain" else {"blinds": blinds, "blind_Zr": tape.random_scalar(b"blind_Zr")}
            t0 = time.perf_counter()
            proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, tr, tape, **kw)
            tp = ms_since(t0)
            launches[k] = {"commit": l1 - l0, "prove": ctx.launches - l1}
            if k == "hiding" and gold:
                match &= (hashlib.sha256(comm).hexdigest() == gold["commitment_sha256"]
                          and hashlib.sha256(proof.bytes).hexdigest() == gold["proof_sha256"])
            if i >= warmup:
                times[k]["commit"].append(tc)
                times[k]["prove"].append(tp)
    out = {"num_vars": nv, "values": dc.CASES[name][1], "hiding_golden_match": bool(match) if gold else None}
    for k in times:
        out[k] = {s: stats(v) for s, v in times[k].items()}
        out[k]["launches"] = launches[k]
    return out


def cpu_oracle(reps):
    """the CPU oracle (the restatement of the reference, OpenMP) at 2^20 with 8 threads: commit and prove"""
    ol.lib().orc_set_num_threads(8)
    res = {}
    for name in ("full_nv20", "u16_nv20"):
        nv, Z, r, seed = dc.inputs(name)
        stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
        Zr = od.evaluate(Z, r)
        tc, tp = [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            od.commit(Z, stream)
            tc.append(ms_since(t0))
            t0 = time.perf_counter()
            od.prove(Z, r, Zr, stream, od.Transcript(dc.TRANSCRIPT_LABEL), od.RandomTape(dc.TAPE_LABEL, seed))
            tp.append(ms_since(t0))
        res[name] = {"commit": stats(tc), "prove": stats(tp), "threads": 8}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--cpu-reps", type=int, default=3)
    ap.add_argument("--hiding", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "dense_poly.json")))["cases"]
    doc = {"card": card(), "warmup": a.warmup, "reps": a.reps, "cases": {}}
    print("card:", doc["card"], flush=True)
    ctx = lb.Context(0)
    for name in a.cases.split(","):
        doc["cases"][name] = run_case(ctx, name, a.warmup, a.reps, gold[name])
        print(name, json.dumps(doc["cases"][name]), flush=True)
    if a.hiding:
        gold_h = json.load(open(os.path.join(ROOT, "tests", "golden", "dense_poly_hiding.json")))["cases"]
        doc["hiding"] = {}
        for name in a.cases.split(","):
            doc["hiding"][name] = run_hiding(ctx, name, a.warmup, a.reps, gold_h.get(name))
            print("hiding", name, json.dumps(doc["hiding"][name]), flush=True)
    if a.cpu:
        doc["cpu_oracle"] = cpu_oracle(a.cpu_reps)
        print("cpu_oracle", json.dumps(doc["cpu_oracle"]), flush=True)
    doc["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
