"""Deriving polynomials and reading them back on one GPU: DensePolynomial.bound_top / bound_bot of k variables in one
call (passes of up to 8 variables) against chains of k single-variable calls, at k = 2, 4, 8, 12 and 2^20..2^24
full-width evaluations (and the top bind of a 16-bit polynomial, whose first pass reads the u32 mirror); to_numpy and
to_tensor; new_padded from host and device memory.  Each call is timed with the host clock around the call and a
device synchronise, W warm-ups, then the median and range of N runs.  Rates are algorithmic: the bytes the operation
must move at least (inputs read once, outputs written once) over the time, against the data sheet's 3.35 TB/s of HBM3
(PCIe for the host forms).  Prints the card's name and power limit, read in the same run, and one JSON line per row.
Sharded contexts are not timed here.
usage: python tools/poly_transform_bench.py [--warmup W] [--reps N] [--nv 20,22,24] [--out FILE.json]"""
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

HBM = 3.35e12
U16 = lb.fr_from_ints(range(1 << 16))  # the Montgomery form of every 16-bit integer


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        return None


def stats(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4), "n": len(v)}


def timed(fn, warmup, reps):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
        del res
    return out


def residues(gen, n):
    import torch

    z = torch.randint(-2**63, 2**63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=gen)
    z[:, 3] &= 2**60 - 1
    return z


def row(name, ms, nbytes, peak=HBM):
    med = statistics.median(ms)
    r = {"case": name, "ms": stats(ms), "bytes": nbytes, "TBps": round(nbytes / med / 1e9, 3)}
    if peak:
        r["of_peak"] = round(nbytes / med / 1e9 / (peak / 1e12), 3)
    print(json.dumps(r), flush=True)
    return r


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--nv", default="20,22,24")
    ap.add_argument("--out")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    ctx = lb.Context(0)
    gen = torch.Generator(device="cuda")
    rows = []
    for nv in (int(x) for x in a.nv.split(",")):
        gen.manual_seed(nv)
        n = 1 << nv
        Z = residues(gen, n)
        p = lb.DensePolynomial(ctx, Z)
        small = lb.DensePolynomial(ctx, U16[np.random.default_rng(nv).integers(0, 1 << 16, size=n)])
        r = np.ascontiguousarray(residues(gen, 12).cpu().numpy().view(np.uint64))
        for k in (2, 4, 8, 12):
            out_b = (n >> k) * 32
            for d in ("top", "bot"):
                one = getattr(p, "bound_" + d)
                rows.append(row("%s_nv%d_k%d_onepass" % (d, nv, k), timed(lambda: one(r[:k]), a.warmup, a.reps), n * 32 + out_b))

                def chain():
                    q = p
                    for j in range(k):
                        q = getattr(q, "bound_" + d)(r[j])
                    return q

                chain_b = sum((n >> j) * 32 + (n >> (j + 1)) * 32 for j in range(k))
                rows.append(row("%s_nv%d_k%d_chain" % (d, nv, k), timed(chain, a.warmup, a.reps), chain_b))
            rows.append(row("top_u16_nv%d_k%d_onepass" % (nv, k), timed(lambda: small.bound_top(r[:k]), a.warmup, a.reps),
                            n * 4 + out_b))
        rows.append(row("read_host_nv%d" % nv, timed(p.to_numpy, a.warmup, a.reps), n * 32, None))
        dst = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        rows.append(row("read_device_nv%d" % nv, timed(lambda: p.copy_to(dst), a.warmup, a.reps), 2 * n * 32))
        host = Z.cpu().numpy()[: n - 1].copy()
        rows.append(row("padded_host_nv%d" % nv, timed(lambda: lb.DensePolynomial.new_padded(ctx, host), a.warmup, a.reps),
                        n * 32, None))
        dev = Z[: n - 1]
        rows.append(row("padded_device_nv%d" % nv, timed(lambda: lb.DensePolynomial.new_padded(ctx, dev), a.warmup, a.reps),
                        2 * n * 32))
        del p, small, Z, dst
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump({"card": card(), "rows": rows}, open(a.out, "w"), indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
