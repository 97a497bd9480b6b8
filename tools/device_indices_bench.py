"""Densify + commit + prove with the lookup indices on the host (a numpy u64 matrix, lasso_densify) against the same
matrix already on the GPU (a torch CUDA int64 tensor, lasso_densify_device), alternating in one process, for
XOR C=4 2^20, LT C=8 2^22 and RangeCheck<40> C=4 2^24 (tests/workloads.py inputs).
Per workload and input it prints the median and range of
  e2e      host clock around densify + commit + prove (prove ends in a device synchronise);
  densify  the library's wall time of the densify call (Context.last_timings_ms);
  Densify  the span of the same name under LASSO_B200_SPANS=1 (a separate pass: spans synchronise around every step);
checks every proof against tests/golden/big_proofs.json, and prints the card's name and power limit.
usage: python tools/device_indices_bench.py [--warmup W] [--reps N] [--configs a,b] [--out FILE.json]"""
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

import lasso_b200 as lb  # noqa: E402
import oracle_lib as ol  # noqa: E402
import workloads as wl  # noqa: E402

CONFIGS = ("xor_c4_s20", "lt_c8_s22", "rc40_c4_s24")


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def one(ctx, S, src, log_m, gens, r, seed):
    t0 = time.perf_counter()
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, src, log_m)
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    e2e = (time.perf_counter() - t0) * 1e3
    return e2e, ctx.last_timings_ms()["densify"], hashlib.sha256(com).hexdigest(), hashlib.sha256(proof.bytes).hexdigest()


def run_config(name, warmup, reps, gold):
    kind, C, log_m, log_r, log_s, idx, r, seed = wl.config_inputs(name)
    S = lb.Strategy(kind, C, log_m, log_r)
    stream = np.ascontiguousarray(ol.generators(gold["n_generators"]))
    inputs = {"host_numpy": idx, "cuda_int64": torch.from_numpy(idx.astype(np.int64)).cuda()}
    torch.cuda.synchronize()
    row = {}
    ctx = lb.Context(0)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C, 1 << log_s, S.num_memories, log_m, stream=stream)
    e2e, dz, ok = {k: [] for k in inputs}, {k: [] for k in inputs}, {k: True for k in inputs}
    for rep in range(warmup + reps):
        for k, src in inputs.items():
            t, d, hc, hp = one(ctx, S, src, log_m, gens, r, seed)
            ok[k] = ok[k] and hc == gold["commitment_sha256"] and hp == gold["proof_sha256"]
            if rep >= warmup:
                e2e[k].append(t)
                dz[k].append(d)
    del gens
    ctx.close()
    os.environ["LASSO_B200_SPANS"] = "1"
    ctx = lb.Context(0)  # the span switch is read when a context is created
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C, 1 << log_s, S.num_memories, log_m, stream=stream)
    span = {k: [] for k in inputs}
    for rep in range(max(3, reps // 2) + 1):
        for k, src in inputs.items():
            ctx.spans()
            one(ctx, S, src, log_m, gens, r, seed)
            if rep:
                span[k].append(ctx.spans()["Densify"])
    del gens
    ctx.close()
    del os.environ["LASSO_B200_SPANS"]
    for k in inputs:
        row[k] = {"e2e_ms": stats(e2e[k]), "densify_ms": stats(dz[k]), "Densify_span_ms": stats(span[k]),
                  "matches_golden": ok[k]}
        print("%-12s %-10s e2e %8.2f ms (%.2f-%.2f)  densify %7.2f ms (%.2f-%.2f)  Densify span %7.2f ms (%.2f-%.2f)  "
              "golden %s" % (name, k, row[k]["e2e_ms"]["median"], row[k]["e2e_ms"]["min"], row[k]["e2e_ms"]["max"],
                             row[k]["densify_ms"]["median"], row[k]["densify_ms"]["min"], row[k]["densify_ms"]["max"],
                             row[k]["Densify_span_ms"]["median"], row[k]["Densify_span_ms"]["min"],
                             row[k]["Densify_span_ms"]["max"], ok[k]), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None, help="also write the results as JSON")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("device_indices_bench needs a CUDA device")
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "big_proofs.json")))["cases"]
    results = {"card": card(), "warmup": args.warmup, "reps": args.reps, "configs": {}}
    print("card: %s" % results["card"], flush=True)
    for name in args.configs.split(","):
        results["configs"][name] = run_config(name, args.warmup, args.reps, gold[name])
    print("card: %s" % card(), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    ok = all(v["matches_golden"] for row in results["configs"].values() for v in row.values())
    print("DEVICE_INDICES_BENCH", "PASS" if ok else "FAIL")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
