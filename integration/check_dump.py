#!/usr/bin/env python
"""Check the vectors dumped by the reference itself (integration/rust/reference_patch/, run on any machine with
cargo) against this repository: the CPU oracle must reproduce the Rust commitment and proof bytes from the same
explicit inputs, and — with --gpu on an H100 — so must liblasso_b200.so.  A PASS pins everything the repository calls
"bit-exact" to the real Rust binary (SURVEY.md §8c, DESIGN.md §5).

    python integration/check_dump.py /tmp/lasso_vectors [--gpu]
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def load_case(d):
    man = json.load(open(os.path.join(d, "manifest.json")))
    C = man["C"]
    idx = np.fromfile(os.path.join(d, "indices.u64"), dtype=np.uint64).reshape(-1, C)
    r = np.fromfile(os.path.join(d, "r.fr"), dtype=np.uint64).reshape(-1, 4)
    gens = np.fromfile(os.path.join(d, "gens.aff"), dtype=np.uint64).reshape(-1, 8)
    seed = np.fromfile(os.path.join(d, "tape_seed.fr"), dtype=np.uint64).reshape(4)
    com = open(os.path.join(d, "commitment.bin"), "rb").read()
    proof = open(os.path.join(d, "proof.bin"), "rb").read()
    assert idx.shape[0] == man["lookups"] and gens.shape[0] == man["n_generators"]
    return man, np.ascontiguousarray(idx), np.ascontiguousarray(r), np.ascontiguousarray(gens), seed, com, proof


def first_diff(a, b):
    n = min(len(a), len(b))
    for i in range(n):
        if a[i] != b[i]:
            return i
    return None if len(a) == len(b) else n


def main():
    root = sys.argv[1]
    use_gpu = "--gpu" in sys.argv[2:]
    import oracle_lib as ol

    ok = True
    for case in sorted(os.listdir(root)):
        d = os.path.join(root, case)
        if not os.path.exists(os.path.join(d, "manifest.json")):
            continue
        man, idx, r, gens, seed, com, proof = load_case(d)
        if not man.get("deterministic_test_rng", False):
            print("%s: WARNING dumped without DETERMINISTIC_TEST_RNG=1: tape_seed.fr may not be the seed RandomTape::new drew" % case)
        # 1. the generator stream: the oracle's restatement of MultiCommitGens::new must sample the same points
        mine = np.zeros_like(gens)
        ol.lib().orc_sample_generators(ol.sz(gens.shape[0]), man["generator_label"].encode(), ol.P(mine))
        gens_ok = bool((mine == gens).all())
        # 2. oracle prover on the explicit inputs
        res = ol.prove(man["kind"], man["C"], man["log_m"], man["log_r"], idx, r, gens, seed, flags=1)
        o_ok = res["rc"] == 0 and res["commitment"] == com and res["proof"] == proof
        line = "%-18s generators %s | oracle commitment %s proof %s" % (
            case, "same" if gens_ok else "DIFFER", "same" if res["commitment"] == com else "DIFFER@%s" % first_diff(res["commitment"], com),
            "same" if res["proof"] == proof else "DIFFER@%s" % first_diff(res["proof"], proof))
        ok = ok and gens_ok and o_ok
        if use_gpu:
            import lasso_b200 as lb

            ctx = lb.Context(0)
            S = lb.Strategy(man["kind"], man["C"], man["log_m"], man["log_r"])
            s = 1 << max(0, (idx.shape[0] - 1).bit_length())
            g = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", man["C"], s, S.num_memories, man["log_m"], stream=gens)
            dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, man["log_m"])
            gcom = dense.commit(g)
            gproof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, g, tape_seed=seed)
            g_ok = gcom == com and gproof.bytes == proof
            line += " | gpu commitment %s proof %s" % ("same" if gcom == com else "DIFFER", "same" if gproof.bytes == proof else "DIFFER")
            ok = ok and g_ok
            ctx.close()
        print(line, flush=True)
    print("CHECK_DUMP", "PASS" if ok else "FAIL")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
