"""Lookups inside a caller's protocol on the GPU, three measurements:
  outputs:  DensifiedRepresentation.outputs: the outputs kernel's CUDA time (torch.profiler, a run of its own) and the
            whole call (host clock around `--iters` calls and a device synchronise: the kernel, the width read-back
            and, for integer outputs, the u32 mirror), at 2^20, 2^22 and
            2^24 lookups for XOR C=4 M=2^16, LT C=8 M=2^16, RangeCheck<40> C=4 M=2^16 and a full-width custom table
            (C=4, M=2^16, one table of uniform field elements, g = sum of the four), with bytes/s of the call over traffic() below;
  paths:    SparsePolynomialEvaluationProof.prove through the label path and through the transcript path, alternating
            in one process, at 2^20 lookups (XOR C=4): median, range and spread of each;
  compose:  outputs + commit of v + sparse commit + prove + opening of v at 2^20 and 2^22 (XOR C=4), each step timed
            with the host clock around calls that end in a device synchronise, and its share of the total.
The card's name and power limit are read in the same run.
usage: python tools/compose_bench.py [--iters N] [--reps N] [--sizes 20,22,24] [--out FILE.json]"""
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
import workloads as wl  # noqa: E402


def traffic(C_, s, integer):
    """bytes the outputs pass needs per call: 4 C bytes of indices read and 32 bytes written per lookup, plus 4 bytes of
    u32 mirror (and the 32 bytes it reads back) for integer outputs; tables of a custom strategy are not counted"""
    return s * (4 * C_ + 32 + (4 + 32 if integer else 0))


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3),
            "spread_pct": round(100 * (max(v) - min(v)) / statistics.median(v), 1), "n": len(v)}


def strategies(ctx):
    rng = np.random.default_rng(3)
    M = 1 << 16
    table = lb.api.fr_from_ints([int.from_bytes(rng.bytes(31), "little") >> 4 for _ in range(M)])
    custom = lb.CustomStrategy(ctx, 4, 16, [table], lambda v: v[0] + v[1] + v[2] + v[3], 1)
    return {"xor_c4": (lb.Strategy(lb.XOR, 4, 16), 4), "lt_c8": (lb.Strategy(lb.LT, 8, 16), 8),
            "rc40_c4": (lb.Strategy(lb.RANGE_CHECK, 4, 16, 40), 4), "custom_fr_c4": (custom, 4)}


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = lb.Context(0)
    res = {"card_before": card(), "outputs": {}, "paths": {}, "compose": {}}
    sizes = [int(x) for x in a.sizes.split(",")]
    for name, (S, C_) in strategies(ctx).items():
        for log_s in sizes:
            rng = np.random.default_rng(log_s)
            idx = rng.integers(0, 1 << 16, size=(1 << log_s, C_), dtype=np.uint64)
            dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, 16)
            del idx
            v = dense.outputs(S)  # warm-up
            del v
            integer = name in ("xor_c4", "lt_c8")  # RangeCheck<40> and the custom table are wider than 32 bits
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.iters):
                v = dense.outputs(S)
                del v
            torch.cuda.synchronize()
            call_ms = 1e3 * (time.perf_counter() - t0) / a.iters
            # kernel time: CUDA activity of the outputs kernel alone, in a profiled run of its own
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    v = dense.outputs(S)
                    del v
                torch.cuda.synchronize()
            us = [getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                  for e in prof.key_averages() if "lookup_outputs" in e.key]
            ms = sum(us) / 1e3 / a.iters
            nbytes = traffic(C_, 1 << log_s, integer)
            res["outputs"]["%s_s%d" % (name, log_s)] = {"kernel_ms": round(ms, 4), "call_ms": round(call_ms, 4),
                                                        "traffic_bytes": nbytes,
                                                        "GB_per_s_call": round(nbytes / call_ms / 1e6, 1)}
            print(name, log_s, res["outputs"]["%s_s%d" % (name, log_s)], flush=True)
            del dense
    # label vs transcript path, alternating
    kind, C_, log_m, log_r, log_s, idx, r, seed = wl.config_inputs("xor_c4_s20")
    S = lb.Strategy(kind, C_, log_m, log_r)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, dense.s, 4, log_m,
                                           stream=lb.sample_generators(b"gens_sparse_poly",
                                                                       lb.gens_points_needed(C_, dense.s, 4, log_m)))
    t = {"label": [], "transcript": []}
    for i in range(a.reps + 1):
        for leg in ("label", "transcript"):
            t0 = time.perf_counter()
            if leg == "label":
                p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
            else:
                p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, transcript=lb.Transcript(b"example"),
                                                             random_tape=lb.RandomTape(b"proof", seed))
            if i:
                t[leg].append(1e3 * (time.perf_counter() - t0))
    res["paths"] = {k: stats(v) for k, v in t.items()}
    print("paths", res["paths"], flush=True)
    del dense, gens
    # the composed protocol
    for log_s in [x for x in (20, 22) if x in sizes]:
        rng = np.random.default_rng(100 + log_s)
        idx = rng.integers(0, 1 << 16, size=(1 << log_s, 4), dtype=np.uint64)
        dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, 16)
        gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", 4, dense.s, 4, 16,
                                               stream=lb.sample_generators(b"gens_sparse_poly",
                                                                           lb.gens_points_needed(4, dense.s, 4, 16)))
        v_gens = lb.PolyCommitmentGens.new(ctx, b"gens_outputs", log_s)
        steps = {k: [] for k in ("outputs", "commit_v", "commit_sparse", "prove", "open_v")}
        for i in range(a.reps + 1):
            T, tape = lb.Transcript(b"compose"), lb.RandomTape(b"proof", np.zeros(4, dtype=np.uint64))
            tm = {}
            t0 = time.perf_counter()
            v = dense.outputs(S)
            tm["outputs"] = time.perf_counter()
            T.append_poly_commitment(b"outputs", v.commit(v_gens))
            tm["commit_v"] = time.perf_counter()
            T.append_sparse_commitment(dense.commit(gens))
            tm["commit_sparse"] = time.perf_counter()
            rr = T.challenge_vector(b"r", log_s)
            p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, rr, gens, transcript=T, random_tape=tape)
            tm["prove"] = time.perf_counter()
            lb.PolyEvalProof.prove(ctx, v, rr, p.claimed_evaluation, v_gens, T, tape)
            tm["open_v"] = time.perf_counter()
            if i:
                prev = t0
                for k in steps:
                    steps[k].append(1e3 * (tm[k] - prev))
                    prev = tm[k]
            del v
        total = sum(statistics.median(v) for v in steps.values())
        res["compose"]["xor_c4_s%d" % log_s] = {k: dict(stats(v), share_pct=round(100 * statistics.median(v) / total, 1))
                                                for k, v in steps.items()}
        res["compose"]["xor_c4_s%d" % log_s]["total_ms_median_sum"] = round(total, 3)
        print("compose", log_s, res["compose"]["xor_c4_s%d" % log_s], flush=True)
        del dense, gens, v_gens
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
