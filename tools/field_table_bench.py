"""Cost of caller-defined tables of arbitrary field elements (lasso_strategy_create_fr), in one process, alternating four
strategies over the same workload: C = 4, log_m = 16, 2^20 lookups (tests/golden/make_golden_fr.py inputs), g = the sum
of the four lookups, one table of
  u32      2^16 random integers below 2^32 through lasso_strategy_create;
  u32_fr   the same integers through lasso_strategy_create_fr (must give the same bytes and time as u32);
  full     2^16 uniform field elements (253-bit commitments and Montgomery openings; its proof must match the golden hash);
  bits40   squares of 20-bit values (40 bits: 6 signed 8-bit windows).
For each it prints the per-proof time (host clock around a prove call, which ends in a device synchronise; median and
range), the spans Subtables.commit, CombinedEval.prove and HashLayer.prove (LASSO_B200_SPANS=1, a separate pass: spans
synchronise around every step), and the card's name and power limit.
usage: python tools/field_table_bench.py [--reps N] [--out FILE.json]"""
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402

import field_tables as ft  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import make_golden_fr as mg  # noqa: E402

SPANS = ("Subtables.commit", "CombinedEval.prove", "HashLayer.prove")


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def tables():
    rng = np.random.default_rng(2024)
    small = rng.integers(0, 2**32, size=1 << mg.LOG_M, dtype=np.uint64)
    full = mg.inputs()[0].tables[0]
    return {"u32": small.astype(np.uint32), "u32_fr": lb.fr_from_ints(small.tolist()), "full": full,
            "bits40": lb.fr_from_ints(ft.ints_squares_40(mg.LOG_M))}


def make(ctx, t):
    return lb.CustomStrategy(ctx, mg.C, mg.LOG_M, [t], ft.g_of_degree(1), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed proofs per table (after one warm-up each)")
    ap.add_argument("--out", default=None, help="also write the results as JSON")
    args = ap.parse_args()
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "field_tables_big.json")))["cases"][mg.NAME]
    _, idx, r, seed, stream = mg.inputs()
    tabs = tables()
    results = {"card": card(), "workload": "C=4 log_m=16 2^20 lookups, g = sum", "tables": {}}
    print("card: %s" % results["card"], flush=True)
    ctx = lb.Context(0)
    forms = {k: make(ctx, t) for k, t in tabs.items()}
    s = 1 << mg.LOG_S
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", mg.C, s, mg.C, mg.LOG_M, stream=stream)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, mg.LOG_M)
    proofs, times, launches = {}, {k: [] for k in forms}, {}
    for k, S in forms.items():  # warm-up
        before = ctx.launches
        proofs[k] = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed).bytes
        launches[k] = ctx.launches - before
    for _ in range(args.reps):
        for k, S in forms.items():
            t0 = time.perf_counter()
            p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
            times[k].append((time.perf_counter() - t0) * 1e3)
            assert p.bytes == proofs[k], "%s: proof changed between runs" % k
    for S in forms.values():
        S.close()
    del gens, dense, p
    os.environ["LASSO_B200_SPANS"] = "1"
    ctx2 = lb.Context(0)  # the span switch is read when a context is created
    forms2 = {k: make(ctx2, t) for k, t in tabs.items()}
    gens2 = lb.SparsePolyCommitmentGens.new(ctx2, b"gens_sparse_poly", mg.C, s, mg.C, mg.LOG_M, stream=stream)
    dense2 = lb.DensifiedRepresentation.from_lookup_indices(ctx2, idx, mg.LOG_M)
    spans = {k: {n: [] for n in SPANS} for k in forms}
    for _ in range(max(2, args.reps // 2)):
        for k, S in forms2.items():
            ctx2.spans()
            lb.SparsePolynomialEvaluationProof.prove(ctx2, S, dense2, r, gens2, tape_seed=seed)
            got = ctx2.spans()
            for n in SPANS:
                spans[k][n].append(got.get(n))
    for S in forms2.values():
        S.close()
    del gens2, dense2
    ctx2.close()
    del os.environ["LASSO_B200_SPANS"]
    for k in forms:
        row = {"prove_ms_median": statistics.median(times[k]), "prove_ms": [round(t, 2) for t in times[k]],
               "launches": launches[k], "proof_sha256": hashlib.sha256(proofs[k]).hexdigest()}
        for n in SPANS:
            v = spans[k][n]
            row[n + "_ms_median"] = statistics.median(v) if None not in v else None
        results["tables"][k] = row
        print("%-7s prove %8.2f ms (median of %d; range %.2f-%.2f)  %d launches  %s" % (
            k, row["prove_ms_median"], len(times[k]), min(times[k]), max(times[k]), launches[k],
            "  ".join("%s %s ms" % (n, "%.2f" % row[n + "_ms_median"] if row[n + "_ms_median"] is not None else "n/a")
                      for n in SPANS)), flush=True)
    results["u32_fr_identical"] = proofs["u32"] == proofs["u32_fr"] and launches["u32"] == launches["u32_fr"]
    results["full_matches_golden"] = results["tables"]["full"]["proof_sha256"] == gold["proof_sha256"]
    print("u32 and u32_fr proofs and launches identical: %s; full-width proof matches the golden hash: %s"
          % (results["u32_fr_identical"], results["full_matches_golden"]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    ctx.close()
    ok = results["u32_fr_identical"] and results["full_matches_golden"]
    print("FIELD_TABLE_BENCH", "PASS" if ok else "FAIL")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
