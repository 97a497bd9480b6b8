"""KnowledgeProof.prove, EqualityProof.prove and ProductProof.prove on one GPU, and the three in a row on one transcript
and tape as at the end of a Spartan phase one (knowledge, product, equality: 11 points from three short MSMs).  For
comparison, 11 separate gens.commit calls, each its own device round trip: what a caller rebuilding these proofs from
commitments pays for the same points.  Every call ends in a host wait for its points, so the host clock around it is the
call's time.  W warm-ups, then the median and range of N runs per case, cases alternating.  Prints the card's name and
power limit.
usage: python tools/sigma_bench.py [--warmup W] [--reps N] [--out FILE.json]"""
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
import oracle_lib as ol  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median_us": round(statistics.median(v), 1), "min_us": round(min(v), 1), "max_us": round(max(v), 1),
            "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = lb.Context(0)
    g = lb.DotProductProofGens.new(ctx, 4, b"sigma_bench").gens_1
    rng = np.random.default_rng(1)
    x, rX, y, rY, rZ, s2 = ol.rand_fr(rng, 6)
    L = ol.L_FR
    z = ol.fr_array([ol.fr_ints(x)[0] * ol.fr_ints(y)[0] % L])[0]
    seed = ol.fr_array([5])[0]

    def io():
        return lb.Transcript(b"b"), lb.RandomTape(b"t", seed)

    def knowledge():
        lb.KnowledgeProof.prove(ctx, g, *io(), x, rX)

    def equality():
        lb.EqualityProof.prove(ctx, g, *io(), z, rZ, z, s2)

    def product():
        lb.ProductProof.prove(ctx, g, *io(), x, rX, y, rY, z, rZ)

    def tail():
        t, tape = io()
        lb.KnowledgeProof.prove(ctx, g, t, tape, x, rX)
        lb.ProductProof.prove(ctx, g, t, tape, x, rX, y, rY, z, rZ)
        lb.EqualityProof.prove(ctx, g, t, tape, z, rZ, z, s2)

    def commits():
        for _ in range(11):
            g.commit(x, rX)

    cases = {"knowledge": knowledge, "equality": equality, "product": product, "tail": tail, "commit_x11": commits}
    launches = {}
    for name, fn in cases.items():
        before = ctx.launches
        fn()
        launches[name] = ctx.launches - before
    times = {k: [] for k in cases}
    for i in range(a.warmup + a.reps):
        for name, fn in cases.items():
            t0 = time.perf_counter()
            fn()
            dt = (time.perf_counter() - t0) * 1e6
            if i >= a.warmup:
                times[name].append(dt)
    res = {"card": card(), "warmup": a.warmup, "reps": a.reps,
           "cases": {k: dict(stats(v), launches=launches[k]) for k, v in times.items()}}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
