"""Built-in strategy against the same strategy written as a caller-defined program (lasso_b200.CustomStrategy), in one
process, alternating the two: XOR C=4 with 2^20 lookups and LT C=8 with 2^22 lookups (tests/workloads.py inputs).
For each form it prints the per-proof time (host clock around a prove call, which ends in a device synchronise), the
Sumcheck.prove span (LASSO_B200_SPANS=1, a separate pass: spans synchronise around every step), whether the two
forms' proofs are identical and match the golden hash (tests/golden/big_proofs.json), and the card's name and power
limit.  usage: python tools/custom_strategy_bench.py [--reps N] [--configs xor_c4_s20,lt_c8_s22] [--out FILE.json]"""
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

import custom_builtins as cb  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import workloads as wl  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed proofs per form (after one warm-up each)")
    ap.add_argument("--configs", default="xor_c4_s20,lt_c8_s22")
    ap.add_argument("--out", default=None, help="also write the results as JSON")
    args = ap.parse_args()
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "big_proofs.json")))["cases"]
    ctx = lb.Context(0)
    results = {"card": card(), "configs": {}}
    print("card: %s" % results["card"], flush=True)
    for name in args.configs.split(","):
        kind, C, log_m, log_r, log_s, idx, r, seed = wl.config_inputs(name)
        forms = {"builtin": lb.Strategy(kind, C, log_m, log_r), "custom": cb.as_custom(ctx, kind, C, log_m, log_r)}
        s = 1 << log_s
        alpha = forms["builtin"].num_memories
        import oracle_lib as ol  # generator stream (cached sampling)

        stream = np.ascontiguousarray(ol.generators(lb.gens_points_needed(C, s, alpha, log_m)))
        gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C, s, alpha, log_m, stream=stream)
        dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
        proofs, times, spans = {}, {k: [] for k in forms}, {k: [] for k in forms}
        for k, S in forms.items():  # warm-up
            proofs[k] = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed).bytes
        for _ in range(args.reps):
            for k, S in forms.items():
                t0 = time.perf_counter()
                p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
                times[k].append((time.perf_counter() - t0) * 1e3)
                assert p.bytes == proofs[k], "%s %s: proof changed between runs" % (name, k)
        forms["custom"].close()
        del gens, dense, p  # free the generator tables before the second context builds its own
        os.environ["LASSO_B200_SPANS"] = "1"
        ctx2 = lb.Context(0)  # the span switch is read when a context is created
        forms2 = {"builtin": forms["builtin"], "custom": cb.as_custom(ctx2, kind, C, log_m, log_r)}
        gens2 = lb.SparsePolyCommitmentGens.new(ctx2, b"gens_sparse_poly", C, s, alpha, log_m, stream=stream)
        dense2 = lb.DensifiedRepresentation.from_lookup_indices(ctx2, idx, log_m)
        for _ in range(max(2, args.reps // 2)):
            for k, S in forms2.items():
                ctx2.spans()
                lb.SparsePolynomialEvaluationProof.prove(ctx2, S, dense2, r, gens2, tape_seed=seed)
                spans[k].append(ctx2.spans().get("Sumcheck.prove"))
        del forms2, gens2, dense2
        ctx2.close()
        del os.environ["LASSO_B200_SPANS"]
        golden = gold.get(name, {}).get("proof_sha256")
        row = {"identical": proofs["builtin"] == proofs["custom"]}
        for k in forms:
            h = hashlib.sha256(proofs[k]).hexdigest()
            row[k] = {"prove_ms_median": statistics.median(times[k]), "prove_ms": [round(t, 2) for t in times[k]],
                      "sumcheck_ms_median": statistics.median(spans[k]) if None not in spans[k] else None,
                      "matches_golden": golden == h}
            print("%-11s %-7s prove %8.2f ms (median of %d; range %.2f-%.2f)  Sumcheck.prove %s ms  golden hash %s"
                  % (name, k, row[k]["prove_ms_median"], len(times[k]), min(times[k]), max(times[k]),
                     "%.2f" % row[k]["sumcheck_ms_median"] if row[k]["sumcheck_ms_median"] is not None else "n/a",
                     "match" if row[k]["matches_golden"] else "MISMATCH"), flush=True)
        print("%-11s builtin and custom proofs identical: %s" % (name, row["identical"]), flush=True)
        results["configs"][name] = row
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    ctx.close()
    ok = all(r["identical"] and r["builtin"]["matches_golden"] and r["custom"]["matches_golden"]
             for r in results["configs"].values())
    print("CUSTOM_STRATEGY_BENCH", "PASS" if ok else "FAIL")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
