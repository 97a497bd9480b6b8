"""Opening k of a caller's polynomials at one point on the GPU, two ways, at component sizes 2^20 and 2^22 for k in
{4, 16}, integer (values below 2^32) and full-width (uniform canonical residues) components:
  separate: k x (DensePolynomial.evaluate + PolyEvalProof.prove), one opening per component;
  combined: DensePolynomial.merge + DensePolynomial.evaluate_batch + one CombinedTableEvalProof.prove;
and, alone, k evaluate calls against one evaluate_batch.  Each leg is timed with the host clock around calls that end
in a device synchronise (an evaluation reads its values back, a proof its points; the merge is timed together with the
batch evaluation that follows it).  Commitments and generator creation are not timed.  W warm-ups, then the median and
range of N runs, alternating the legs.  Also prints the proof bytes of both ways, the launches per leg and the card's
name and power limit, read before and after the run.
usage: python tools/combined_eval_bench.py [--warmup W] [--reps N] [--shapes 4x20u,16x22f] [--out FILE.json]"""
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

import dense_poly_cases as dc  # noqa: E402
import lasso_b200 as lb  # noqa: E402

SHAPES = ("4x20u", "4x20f", "16x20u", "16x20f", "4x22u", "4x22f", "16x22u", "16x22f")


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def gens(ctx, nv):
    return lb.PolyCommitmentGens.new(ctx, b"combined_eval_bench", nv,
                                     stream=lb.sample_generators(b"combined_eval_bench", lb.poly_gens_points_needed(nv)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = lb.Context(0)
    res = {"card": card(), "warmup": a.warmup, "reps": a.reps, "shapes": {}}
    seed = dc.random_full(np.random.default_rng(9), 1)[0]
    for shape in a.shapes.split(","):
        k, nv, kind = int(shape.split("x")[0]), int(shape.split("x")[1][:-1]), shape[-1]
        rng = np.random.default_rng(100 * k + nv)
        polys = []
        for _ in range(k):
            Z = (dc.random_full(rng, 1 << nv) if kind == "f"
                 else dc.fr_from_u64(rng.integers(0, 1 << 32, size=1 << nv, dtype=np.uint64)))
            polys.append(lb.DensePolynomial(ctx, Z))
        del Z
        r = dc.random_full(rng, nv)
        g_one = gens(ctx, nv)
        mv = nv + (k - 1).bit_length()
        g_all = gens(ctx, mv)
        t = {"separate": [], "combined": [], "evaluate_k": [], "evaluate_batch": []}
        launches, nbytes = {}, {}
        for i in range(a.warmup + a.reps):
            l0 = ctx.launches
            t0 = time.perf_counter()
            proofs = []
            for p in polys:
                y = p.evaluate(r)
                proofs.append(lb.PolyEvalProof.prove(ctx, p, r, y, g_one, lb.Transcript(b"ce"), lb.RandomTape(b"proof", seed)))
            t1 = time.perf_counter()
            l1 = ctx.launches
            m = lb.DensePolynomial.merge(ctx, polys)
            evals = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
            cp = lb.CombinedTableEvalProof.prove(ctx, m, evals, r, g_all, lb.Transcript(b"ce"), lb.RandomTape(b"proof", seed))
            t2 = time.perf_counter()
            l2 = ctx.launches
            ys = [p.evaluate(r) for p in polys]
            t3 = time.perf_counter()
            l3 = ctx.launches
            yb = lb.DensePolynomial.evaluate_batch(ctx, polys, r)
            t4 = time.perf_counter()
            assert np.array_equal(np.stack(ys), yb) and np.array_equal(evals, yb)
            launches = {"separate": l1 - l0, "combined": l2 - l1, "evaluate_k": l3 - l2, "evaluate_batch": ctx.launches - l3}
            nbytes = {"separate": sum(len(q.bytes) for q in proofs), "combined": len(cp.data)}
            del m
            if i >= a.warmup:
                for name, dt in (("separate", t1 - t0), ("combined", t2 - t1), ("evaluate_k", t3 - t2),
                                 ("evaluate_batch", t4 - t3)):
                    t[name].append(dt * 1e3)
        row = {"k": k, "num_vars": nv, "values": "u32" if kind == "u" else "full", "merged_num_vars": mv,
               "ms": {n: stats(v) for n, v in t.items()}, "launches": launches, "proof_bytes": nbytes}
        res["shapes"][shape] = row
        print(json.dumps({shape: row}), flush=True)
        del polys, g_one, g_all
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
