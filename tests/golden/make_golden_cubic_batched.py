"""Golden hashes of batched cubic sumchecks over a caller's polynomials (tests/golden/cubic_batched.json).

    python tests/golden/make_golden_cubic_batched.py [n2_nv20_eq n8_nv20_partial n2_nv22_eq ...]

Runs the CPU oracle's SumcheckInstanceProof::prove_cubic_batched (oracle_dense/ over the restatement in oracle/) on the
seeded inputs of tests/cubic_batched_cases.py, with their true claim, on a transcript labelled TRANSCRIPT_LABEL to which
nothing is appended first.  The oracle's sumcheck verifier must accept every proof at degree 3 on a fresh transcript,
with the same r.  Committed: the claim, and SHA-256 of proof || r || finals (with the proof length and a challenge drawn
after the proof); tests/test_gpu_cubic_batched.py compares the GPU's outputs with them."""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import cubic_batched_cases as cb  # noqa: E402
import oracle_cubic_lib as ocb  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_sumcheck_lib as osc  # noqa: E402

OUT = os.path.join(HERE, "cubic_batched.json")


def main():
    names = sys.argv[1:] or sorted(cb.GOLDEN)
    doc = json.load(open(OUT)) if os.path.exists(OUT) else {"cases": {}}
    for name in names:
        A, B, C, coeffs, rounds = cb.golden_inputs(name)
        claim = cb.true_claim(A, B, C, coeffs)
        t0 = time.time()
        t = od.Transcript(cb.TRANSCRIPT_LABEL)
        got = ocb.cubic_prove(A, B, C, coeffs, claim, rounds, t)
        after = t.challenge_scalar(b"after")
        rc, _, r = osc.sumcheck_verify(got["proof"], claim, rounds, 3, od.Transcript(cb.TRANSCRIPT_LABEL))
        assert rc == 0 and np.array_equal(r, got["r"]), name
        dt = time.time() - t0
        n, nv, seed, ckind, _ = cb.GOLDEN[name]
        doc["cases"][name] = {
            "n": n, "num_vars": nv, "seed": seed, "C": ckind, "num_rounds": rounds, "claim_hex": claim.tobytes().hex(),
            "sha256": hashlib.sha256(cb.digest_input(got["proof"], got["r"], got["finals"])).hexdigest(),
            "proof_len": len(got["proof"]), "after_challenge_hex": after.tobytes().hex(), "oracle_seconds": round(dt, 1),
            "oracle_verifier": "accepted",
        }
        print(name, "done in %.1f s" % dt, flush=True)
        with open(OUT, "w") as f:
            json.dump(doc, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
