"""ZKSumcheckInstanceProof.prove against SumcheckInstanceProof.prove_arbitrary on the same polynomials, alternating in
one process: eq * (A * B - C) (4 inputs, degree 3, eq(tau) made on the GPU) and A * B (2 inputs, degree 2), at 2^20,
2^22 and 2^24 evaluations, every variable bound.  Each call is timed with the host clock around the library call, which
ends in a device synchronise (the final evaluations are read back).  W warm-ups per path, then the median and range of
N runs per path.  A second context made with LASSO_B200_SPANS=1 runs each ZK call once more and reports its total and
the McMsm.wait span: a span synchronises the device before it starts, so that span is the host side of the commitment
waits (decode and compression) only, and the commitment MSMs' device time stays in the rest.  That pass is not used
for the timing table.  Prints the card's name and power limit.
usage: python tools/zk_sumcheck_bench.py [--warmup W] [--reps N] [--sizes 20,22,24] [--out FILE.json]"""
import argparse
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

import lasso_b200 as lb  # noqa: E402
import sumcheck_cases as sc  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def polys_for(ctx, stmt, nv, rng):
    """device polynomials of a statement, generated on the GPU from seeded eq tables (no 2^24 host upload per input)"""
    rnd = lambda: rng.integers(1, 1 << 62, size=(nv, 4), dtype=np.uint64) % np.uint64(1 << 60)  # noqa: E731
    if stmt == "spartan":
        return [lb.DensePolynomial.eq(ctx, rnd()) for _ in range(4)], lb.Comb(sc.spartan, 4)
    return [lb.DensePolynomial.eq(ctx, rnd()) for _ in range(2)], lb.Comb(lambda v: v[0] * v[1], 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = lb.Context(0)
    res = {"card": card(), "warmup": a.warmup, "reps": a.reps, "cases": {}}
    seed = np.zeros(4, dtype=np.uint64)
    seed[0] = 5
    bc = np.zeros(4, dtype=np.uint64)
    for nv in [int(x) for x in a.sizes.split(",")]:
        for stmt in ("spartan", "ab"):
            rng = np.random.default_rng(nv)
            polys, comb = polys_for(ctx, stmt, nv, rng)
            g = lb.DotProductProofGens.new(ctx, comb.degree + 1, b"zk_bench")
            times = {"plain": [], "zk": []}

            def plain():
                lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, lb.Transcript(b"b"))

            def zk(c=ctx, ps=polys, gens=g):
                return lb.ZKSumcheckInstanceProof.prove(c, comb, ps, None, bc, gens.gens_1, gens.gens_n, lb.Transcript(b"b"),
                                                        lb.RandomTape(b"t", seed))

            for i in range(a.warmup + a.reps):
                for name, fn in (("plain", plain), ("zk", zk)):
                    t0 = time.perf_counter()
                    fn()
                    dt = (time.perf_counter() - t0) * 1e3
                    if i >= a.warmup:
                        times[name].append(dt)
            case = {k: stats(v) for k, v in times.items()}
            case["zk_minus_plain_ms"] = round(case["zk"]["median"] - case["plain"]["median"], 3)
            case["zk_minus_plain_per_round_us"] = round(1e3 * case["zk_minus_plain_ms"] / nv, 1)
            res["cases"]["%s_nv%d" % (stmt, nv)] = case
            print(json.dumps({"%s_nv%d" % (stmt, nv): case}), flush=True)
            del polys
    # the per-round split, from spans, on a context of its own
    os.environ["LASSO_B200_SPANS"] = "1"
    sctx = lb.Context(0)
    for nv in [int(x) for x in a.sizes.split(",")]:
        for stmt in ("spartan", "ab"):
            polys, comb = polys_for(sctx, stmt, nv, np.random.default_rng(nv))
            g = lb.DotProductProofGens.new(sctx, comb.degree + 1, b"zk_bench")
            for _ in range(2):  # the second call's spans
                sctx.spans()
                lb.ZKSumcheckInstanceProof.prove(sctx, comb, polys, None, bc, g.gens_1, g.gens_n, lb.Transcript(b"b"),
                                                 lb.RandomTape(b"t", seed))
                sp = sctx.spans()
            total, waits = sp.get("ZKSumcheck.prove", 0.0), sp.get("McMsm.wait", 0.0)
            res["cases"]["%s_nv%d" % (stmt, nv)]["spans_ms"] = {
                "total": round(total, 3), "commit_decode": round(waits, 3), "commit_decode_per_round": round(waits / nv, 4),
                "rest": round(total - waits, 3)}
            del polys
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
