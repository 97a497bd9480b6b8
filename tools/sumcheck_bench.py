"""SumcheckInstanceProof.prove_arbitrary over a caller's polynomials on the GPU, fused and unfused rounds alternating in
one process, for the seeded cases of tests/golden/sumcheck.json: eq * (A * B - C) at 2^20, 2^22 and 2^24 (4 inputs,
degree 3) and eq * prod_{i < 8} P_i at 2^20 (9 inputs, degree 9).  eq(tau) is made on the GPU.
Each call is timed with the host clock around the library call, which ends in a device synchronise (the final
evaluations are read back).  W warm-ups per path, then the median and range of N runs per path.  Bytes per call are the
algorithmic traffic computed from the shapes (32 B per element read or written once: round 1 reads every input, a fused
round reads 4q and writes 2q per input, an unfused one reads 4q, writes 2q and reads 2q again), and GB/s is that over the
median.  Every proof is checked against the golden hash.  Also prints the card's name and power limit, and (--cpu) the CPU
oracle's time at 2^20.
usage: python tools/sumcheck_bench.py [--warmup W] [--reps N] [--cases a,b] [--cpu] [--out FILE.json]"""
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

import lasso_b200 as lb  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_sumcheck_lib as osc  # noqa: E402
import sumcheck_cases as sc  # noqa: E402

CASES = ("spartan_nv20", "spartan_nv22", "spartan_nv24", "prod9_nv20")
FUSED_MIN_Q = 1 << 15


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def bytes_per_call(k, nv, fused):
    total = (1 << nv) * k  # round 1: every input read once
    for j in range(1, nv):
        q = 1 << (nv - j - 1)
        total += k * (4 * q + 2 * q + (0 if fused and q >= FUSED_MIN_Q else 2 * q))
    return 32 * total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "sumcheck.json")))["cases"]
    ctx = lb.Context(0)
    res = {"card": card(), "warmup": a.warmup, "reps": a.reps, "cases": {}}
    for name in a.cases.split(","):
        fname, nv, tau, arrays = sc.golden_inputs(name)
        fn, k = sc.FUNCS[fname]
        polys = [lb.DensePolynomial.eq(ctx, tau)] + [lb.DensePolynomial(ctx, x) for x in arrays[1:]]
        comb = lb.Comb(fn, k)
        want = golden[name]["sha256"]
        times = {"fused": [], "unfused": []}
        match = True
        for i in range(a.warmup + a.reps):
            for mode in ("fused", "unfused"):
                if mode == "unfused":
                    os.environ["LASSO_B200_UNFUSED_SUMCHECK"] = "1"
                else:
                    os.environ.pop("LASSO_B200_UNFUSED_SUMCHECK", None)
                t = lb.Transcript(sc.TRANSCRIPT_LABEL)
                t0 = time.perf_counter()
                p = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, t)
                dt = (time.perf_counter() - t0) * 1e3
                match &= hashlib.sha256(p.bytes + p.r.tobytes() + p.final_evals.tobytes()).hexdigest() == want
                if i >= a.warmup:
                    times[mode].append(dt)
        os.environ.pop("LASSO_B200_UNFUSED_SUMCHECK", None)
        row = {"num_vars": nv, "n_inputs": k, "degree": comb.degree, "golden_match": bool(match)}
        for mode in ("fused", "unfused"):
            b = bytes_per_call(k, nv, mode == "fused")
            s = stats(times[mode])
            row[mode] = dict(ms=s, bytes=b, GBps=round(b / s["median"] / 1e6, 1))
        if a.cpu and nv == 20:
            t = od.Transcript(sc.TRANSCRIPT_LABEL)
            t0 = time.perf_counter()
            osc.sumcheck_prove(arrays, nv, comb.program, comb.constants, comb.degree, t)
            row["cpu_oracle_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        res["cases"][name] = row
        print(json.dumps({name: row}), flush=True)
        del polys, arrays
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
