"""Memory checking inside a caller's protocol on the GPU, three measurements:
  1. MemoryCheckingProof.prove on its own at XOR C=4, log_m=16, 2^20 lookups, next to the ProductLayer.prove +
     HashLayer.prove spans of one lasso_prove on the same inputs (a second context with LASSO_B200_SPANS=1, whose span
     timers synchronise the device around each span);
  2. GrandProducts.new (the four fingerprint polynomials only: lasso_memory_fingerprints, no circuits) at
     M in {2^16, 2^20} and s in {2^20, 2^24}, with GB/s from shape-derived bytes, against the host path it replaces:
     fingerprints on the host (the oracle's single-threaded C++), upload of the four polynomials and four
     GrandProductCircuits; the GPU path gets the same circuits after its fingerprints;
  3. the lookup proof composed step by step from public calls (tests/test_gpu_memory_check.py compose) against
     lasso_prove_transcript, XOR C=4, 2^20 lookups.
Each call is timed with the host clock around the library call and a device synchronise: W warm-ups, then the median
and range of N runs (the host path of 2 runs once).  The fingerprint bytes per op are read: the 4-byte address, the
gathered 32-byte table entry, the 4-byte timestamp (the counters' u32 mirror), written: two 32-byte fingerprints; per
cell 64 read (table, final) and 64 written.  The table entry is counted although it is served from L2 when the table
fits.  Prints the card's name and power limit, read in the same run, and one JSON line per measurement.
usage: python tools/memory_check_bench.py [--warmup W] [--reps N] [--out FILE.json]"""
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


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def timed(fn, warmup, reps):
    import torch

    out = []
    for i in range(warmup + reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        if i >= warmup:
            out.append((time.perf_counter() - t0) * 1e3)
        del r
    return stats(out)


def xor_inputs(ctx, n):
    import oracle_lib as ol

    C_, log_m = 4, 16
    rng = np.random.default_rng(1)
    idx = rng.integers(0, 1 << log_m, size=(n, C_), dtype=np.uint64)
    S = lb.Strategy(lb.XOR, C_, log_m)
    stream = ol.generators(lb.gens_points_needed(C_, n, 4, log_m))
    r = ol.rand_fr(rng, n.bit_length() - 1)
    return S, idx, stream, r, ol.rand_fr(rng, 1)[0]


def standalone(ctx, warmup, reps):
    import oracle_lib as ol

    n = 1 << 20
    S, idx, stream, r, seed = xor_inputs(ctx, n)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, 16)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", 4, n, 4, 16, stream=stream)
    gamma, tau = ol.rand_fr(np.random.default_rng(2), 2)
    mc = timed(lambda: lb.MemoryCheckingProof.prove(ctx, S, dense, (gamma, tau), gens, lb.Transcript(b"x"),
                                                    lb.RandomTape(b"p", seed)), warmup, reps)
    os.environ["LASSO_B200_SPANS"] = "1"
    c2 = lb.Context(0)
    os.environ.pop("LASSO_B200_SPANS")
    d2 = lb.DensifiedRepresentation.from_lookup_indices(c2, idx, 16)
    g2 = lb.SparsePolyCommitmentGens.new(c2, b"gens_sparse_poly", 4, n, 4, 16, stream=stream)
    lb.SparsePolynomialEvaluationProof.prove(c2, S, d2, r, g2, tape_seed=seed)
    sp = c2.spans()
    del d2, g2
    c2.close()
    return {"case": "standalone_xor_c4_s20", "memory_check_ms": mc,
            "in_lasso_prove_ms": round(sp.get("ProductLayer.prove", 0) + sp.get("HashLayer.prove", 0), 3),
            "spans": {k: round(sp[k], 3) for k in ("ProductLayer.prove", "HashLayer.prove") if k in sp}}


def grand_products(ctx, log_M, log_s, warmup, reps):
    import ctypes as C

    import torch

    import oracle_lib as ol

    M, s = 1 << log_M, 1 << log_s
    rng = np.random.default_rng(log_M + log_s)
    T_h = ol.rand_fr(rng, M)
    dim_u = rng.integers(0, M, size=s, dtype=np.uint64)
    read_u = rng.integers(0, 1 << 20, size=s, dtype=np.uint64)
    fin_u = rng.integers(0, 1 << 20, size=M, dtype=np.uint64)

    def fr(x):
        out = np.zeros((x.shape[0], 4), dtype=np.uint64)
        ol.lib().orc_fr_from_u64_batch(ol.P(np.ascontiguousarray(x)), ol.sz(x.shape[0]), ol.P(out))
        return out

    T, dim, read, fin = (lb.DensePolynomial(ctx, a) for a in (T_h, fr(dim_u), fr(read_u), fr(fin_u)))
    gamma, tau = ol.rand_fr(rng, 2)
    L = lb.lib()

    def fingerprints():
        hs = (C.c_void_p * 4)()
        assert L.lasso_memory_fingerprints(ctx._h, T._h, dim._h, read._h, fin._h, lb.api._p(gamma), lb.api._p(tau),
                                           hs) == 0
        return [lb.DensePolynomial._wrap(ctx, C.c_void_p(h)) for h in hs]

    k = timed(fingerprints, warmup, reps)
    gb = (s * (4 + 32 + 4 + 64) + M * (64 + 64)) / 1e9
    full = timed(lambda: [lb.GrandProductCircuit(ctx, p) for p in fingerprints()], warmup, reps)

    def host():
        out = np.zeros((2 * M + 2 * s, 4), dtype=np.uint64)
        ol.lib().orc_gp_fingerprints(ol.P(T_h), ol.sz(M), ol.P(dim_u), ol.P(read_u), ol.P(fin_u), ol.sz(s),
                                     ol.P(gamma), ol.P(tau), ol.P(out))
        parts = (out[:M], out[2 * M:2 * M + s], out[2 * M + s:], out[M:2 * M])
        return [lb.GrandProductCircuit(ctx, lb.DensePolynomial(ctx, np.ascontiguousarray(p))) for p in parts]

    h = timed(host, 0, 1)
    torch.cuda.synchronize()
    return {"case": "grand_products_M%d_s%d" % (log_M, log_s), "fingerprints_ms": k,
            "fingerprints_GBps": round(gb / (k["median"] / 1e3), 1), "shape_GB": round(gb, 4),
            "gpu_with_circuits_ms": full, "host_fingerprints_upload_circuits_ms": h}


def composed(ctx, warmup, reps):
    import test_gpu_memory_check as t

    n = 1 << 20
    S, idx, stream, r, seed = xor_inputs(ctx, n)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, 16)
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", 4, n, 4, 16, stream=stream)
    import custom_builtins as cb

    g, _ = cb.builtin_g(lb.XOR, 4, 16)
    whole = timed(lambda: lb.SparsePolynomialEvaluationProof.prove(
        ctx, S, dense, r, gens, transcript=lb.Transcript(b"example"), random_tape=lb.RandomTape(b"proof", seed)),
        warmup, reps)
    comp = timed(lambda: t.compose(ctx, S, g, dense, gens, stream, r, seed), warmup, reps)
    return {"case": "composed_xor_c4_s20", "lasso_prove_transcript_ms": whole, "composed_ms": comp}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    ctx = lb.Context(0)
    rows = [standalone(ctx, a.warmup, a.reps)]
    print(json.dumps(rows[-1]), flush=True)
    for log_M in (16, 20):
        for log_s in (20, 24):
            rows.append(grand_products(ctx, log_M, log_s, a.warmup, a.reps))
            print(json.dumps(rows[-1]), flush=True)
    rows.append(composed(ctx, a.warmup, a.reps))
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
