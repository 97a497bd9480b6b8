"""Golden hashes of sumchecks over a caller's polynomials AT SIZE (tests/golden/sumcheck.json).

    python tests/golden/make_golden_sumcheck.py [spartan_nv20 spartan_nv22 spartan_nv24 prod9_nv20 ...]

Runs the CPU oracle's SumcheckInstanceProof::prove_arbitrary (oracle_dense/ over the restatement in oracle/) on the
seeded inputs of tests/sumcheck_cases.py, with polys[0] = eq(tau):
- spartan_nv20/22/24: eq * (A * B - C), 4 inputs, degree 3;
- prod9_nv20: eq * prod_{i < 8} P_i, 9 inputs, degree 9.
The oracle's verifier must accept every proof, and its final claim must equal g(final_evals).  Only SHA-256 hashes of
proof bytes || r || final_evals are committed (with the claim and a challenge drawn after the proof);
tests/test_gpu_sumcheck.py and tools/sumcheck_bench.py compare the GPU's outputs with them.

Oracle CPU time (proof and verification, the inputs' generation excluded), on an 8-core x86-64 host: spartan_nv20
0.4 s, spartan_nv22 1.9 s, spartan_nv24 7.2 s, prod9_nv20 2.5 s."""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import oracle_dense_lib as od  # noqa: E402
import oracle_lib as ol  # noqa: E402
import oracle_sumcheck_lib as osc  # noqa: E402
import sumcheck_cases as sc  # noqa: E402

OUT = os.path.join(HERE, "sumcheck.json")


def main():
    import lasso_b200 as lb  # the tracer only (host code): no GPU is used

    names = sys.argv[1:] or sorted(sc.GOLDEN)
    doc = json.load(open(OUT)) if os.path.exists(OUT) else {"cases": {}}
    for name in names:
        fname, nv, tau, polys = sc.golden_inputs(name)
        fn, k = sc.FUNCS[fname]
        prog, consts, degree = lb.trace_combine_lookups(fn, k)
        t0 = time.time()
        t = od.Transcript(sc.TRANSCRIPT_LABEL)
        got = osc.sumcheck_prove(polys, nv, prog, consts, degree, t)
        after = t.challenge_scalar(b"after")
        rc, e, r = osc.sumcheck_verify(got["proof"], got["claim"], nv, degree, od.Transcript(sc.TRANSCRIPT_LABEL))
        assert rc == 0 and np.array_equal(r, got["r"]), name
        assert ol.fr_ints(e)[0] == sc.g_int(fname, ol.fr_ints(got["final_evals"])), name
        dt = time.time() - t0
        doc["cases"][name] = {
            "function": fname, "num_vars": nv, "seed": sc.GOLDEN[name][2], "degree": degree, "n_inputs": k,
            "sha256": hashlib.sha256(got["proof"] + got["r"].tobytes() + got["final_evals"].tobytes()).hexdigest(),
            "proof_len": len(got["proof"]), "claim_hex": got["claim"].tobytes().hex(),
            "after_challenge_hex": after.tobytes().hex(), "oracle_seconds": round(dt, 1), "oracle_verifier": "accepted",
        }
        print(name, "done in %.1f s" % dt, flush=True)
        with open(OUT, "w") as f:
            json.dump(doc, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
