"""Grand products over a caller's polynomials on the GPU: GrandProductCircuit creation and
BatchedGrandProductArgument.prove for n in {2, 8} circuits at 2^20, 2^22 and 2^24 elements each (seeded uniform
canonical residues).  A circuit can be proven once, so every run creates the n circuits again and then proves them.
Each call is timed with the host clock around the library call, which ends in a device synchronise (creation reads the
top layer back, a proof reads every layer's claims back).  W warm-ups, then the median and range of N runs; launches
per call are the library's launch counter.  Every proof of a shape must give the same bytes.  Also prints the card's
name and power limit, read in the same run, and (--cpu) the CPU oracle's time at 2^20.
A proof over num_vars v is a chain of v (v - 1) / 2 dependent rounds (276 at v = 24), each a device round trip.
usage: python tools/grand_product_bench.py [--warmup W] [--reps N] [--shapes 2x20,8x24] [--cpu] [--out FILE.json]"""
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

import dense_poly_cases as dc  # noqa: E402
import lasso_b200 as lb  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_grand_product_lib as ogp  # noqa: E402

SHAPES = ("2x20", "8x20", "2x22", "8x22", "2x24", "8x24")


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = lb.Context(0)
    res = {"card": card(), "warmup": a.warmup, "reps": a.reps, "shapes": {}}
    for shape in a.shapes.split(","):
        n, nv = (int(x) for x in shape.split("x"))
        rng = np.random.default_rng(1000 * n + nv)
        arrays = [dc.random_full(rng, 1 << nv) for _ in range(n)]
        polys = [lb.DensePolynomial(ctx, x) for x in arrays]
        t_create, t_prove, digests = [], [], set()
        launches = {}
        for i in range(a.warmup + a.reps):
            l0 = ctx.launches
            t0 = time.perf_counter()
            circuits = [lb.GrandProductCircuit(ctx, p) for p in polys]
            t1 = time.perf_counter()
            l1 = ctx.launches
            p = lb.BatchedGrandProductArgument.prove(ctx, circuits, lb.Transcript(b"grand_product_bench"))
            t2 = time.perf_counter()
            launches = {"create": l1 - l0, "prove": ctx.launches - l1}
            digests.add(hashlib.sha256(p.bytes).hexdigest())
            del circuits
            if i >= a.warmup:
                t_create.append((t1 - t0) * 1e3)
                t_prove.append((t2 - t1) * 1e3)
        row = {"n_circuits": n, "num_vars": nv, "create_ms": stats(t_create), "prove_ms": stats(t_prove),
               "launches": launches, "rounds": nv * (nv - 1) // 2, "deterministic": len(digests) == 1}
        if a.cpu and nv == 20:
            t0 = time.perf_counter()
            want = ogp.gp_prove(arrays, od.Transcript(b"grand_product_bench"))
            row["cpu_oracle_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            row["oracle_match"] = hashlib.sha256(want["proof"]).hexdigest() in digests
        res["shapes"][shape] = row
        print(json.dumps({shape: row}), flush=True)
        del polys, arrays
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
