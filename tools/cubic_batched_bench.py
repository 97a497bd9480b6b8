"""SumcheckInstanceProof.prove_cubic_batched over a caller's polynomials on the GPU: n = 2, 8 and 32 pairs and a random C
at 2^20, 2^22 and 2^24, every round (num_rounds = num_vars).  For n <= 7 the same inputs also go through prove_arbitrary
with g = C sum_k coeff_k A_k B_k (2n + 1 inputs, degree 3) and its true claim, alternating with the cubic call in one
process, and each row reports whether the two proofs and finals are equal.  The inputs are uniform residues made on the GPU with torch (no host copy of 2^24-element arrays).
Each call is timed with the host clock around the library call, which ends in a device synchronise (the finals are read
back): W warm-ups per path, then the median and range of N runs.  Prints the card's name and power limit, read in the
same run, and one JSON line per case.  Sharded contexts are not timed here.
usage: python tools/cubic_batched_bench.py [--warmup W] [--reps N] [--cases n2_nv20,...] [--out FILE.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402

import lasso_b200 as lb  # noqa: E402

CASES = tuple("n%d_nv%d" % (n, nv) for nv in (20, 22, 24) for n in (2, 8, 32))
L_FR = 2**252 + 27742317777372353535851937790883648493


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "n": len(v)}


def residues(gen, n):
    """n uniform canonical Montgomery residues on the GPU: four random limbs, the top one below 2^60"""
    import torch

    z = torch.randint(-2**63, 2**63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=gen)
    z[:, 3] &= 2**60 - 1
    return z


def to_limbs(x):
    return np.array([(x >> (64 * i)) & (2**64 - 1) for i in range(4)], dtype=np.uint64)


def run_case(ctx, name, warmup, reps):
    import torch

    n, nv = (int(s[1:]) for s in name.replace("nv", "v").split("_"))
    gen = torch.Generator(device="cuda")
    gen.manual_seed(n * 100 + nv)
    A = [lb.DensePolynomial(ctx, residues(gen, 1 << nv)) for _ in range(n)]
    B = [lb.DensePolynomial(ctx, residues(gen, 1 << nv)) for _ in range(n)]
    C = lb.DensePolynomial(ctx, residues(gen, 1 << nv))
    torch.cuda.synchronize()
    rng = np.random.default_rng(n + nv)
    ks = [int.from_bytes(rng.bytes(40), "little") % L_FR for _ in range(n)]
    coeffs = np.stack([to_limbs(k * 2**256 % L_FR) for k in ks])
    claim = to_limbs(12345)  # not checked: any claim times the same work
    paths = {}
    if n <= 7:
        def g(v):
            acc = v[0] * v[n] * ks[0]
            for k in range(1, n):
                acc = acc + v[k] * v[n + k] * ks[k]
            return acc * v[2 * n]

        comb = lb.Comb(g, 2 * n + 1, 3)
        polys = A + B + [C]
        paths["prove_arbitrary"] = lambda t: lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, t)
        claim = paths["prove_arbitrary"](lb.Transcript(b"bench")).claim  # the true claim: both paths prove the same
    paths["cubic"] = lambda t: lb.SumcheckInstanceProof.prove_cubic_batched(ctx, A, B, C, coeffs, claim, t)
    times = {p: [] for p in paths}
    proofs = {}
    for i in range(warmup + reps):
        for p, fn in paths.items():
            t = lb.Transcript(b"bench")
            t0 = time.perf_counter()
            out = fn(t)
            dt = (time.perf_counter() - t0) * 1e3
            if i >= warmup:
                times[p].append(dt)
            proofs[p] = (out.bytes, out.final_evals.tobytes())
    res = {"case": name, "n": n, "num_vars": nv, "ms": {p: stats(v) for p, v in times.items()}}
    if "prove_arbitrary" in proofs:
        res["same_proof_and_finals"] = proofs["cubic"] == proofs["prove_arbitrary"]
    # algorithmic traffic of the cubic path: round 1 reads 2n + 1 arrays, the out-of-place bind reads them and writes half,
    # then a fused round reads 4q and writes 2q per array
    elems = (2 * n + 1) << nv
    elems += ((2 * n + 1) << nv) + ((2 * n + 1) << (nv - 1))
    for j in range(2, nv):
        elems += (2 * n + 1) * 6 * (1 << (nv - j - 1))
    res["cubic_GBps"] = round(32 * elems / (res["ms"]["cubic"]["median"] * 1e-3) / 1e9, 1)
    del A, B, C, paths
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = lb.Context(0)
    head = {"card": card(), "sharded_one_rank_per_gpu": "not measured"}
    print(json.dumps(head), flush=True)
    rows = []
    for name in a.cases.split(","):
        r = run_case(ctx, name, a.warmup, a.reps)
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"head": head, "rows": rows}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
