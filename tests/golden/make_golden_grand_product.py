"""Golden hashes of batched grand products over a caller's polynomials (tests/golden/grand_product.json).

    python tests/golden/make_golden_grand_product.py [n3_nv6 n2_nv10 n2_nv20 n2_nv22 ...]

Runs the CPU oracle's GrandProductCircuit::new and BatchedGrandProductArgument::prove (oracle_dense/ over the
restatement in oracle/) on the seeded inputs of tests/grand_product_cases.py, on a transcript labelled
TRANSCRIPT_LABEL to which nothing is appended first.  The oracle's verifier must accept every proof on a fresh
transcript, with the same rand and final claims.  Only SHA-256 hashes of proof || products || rand || claims are
committed (with the proof length and a challenge drawn after the proof); tests/test_grand_product_host.py reproduces the
small cases with the oracle, tests/test_gpu_grand_product.py compares the GPU's outputs with all of them."""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import grand_product_cases as gc  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_grand_product_lib as ogp  # noqa: E402

OUT = os.path.join(HERE, "grand_product.json")


def main():
    names = sys.argv[1:] or sorted(gc.GOLDEN)
    doc = json.load(open(OUT)) if os.path.exists(OUT) else {"cases": {}}
    for name in names:
        nv, polys = gc.golden_inputs(name)
        t0 = time.time()
        t = od.Transcript(gc.TRANSCRIPT_LABEL)
        got = ogp.gp_prove(polys, t)
        after = t.challenge_scalar(b"after")
        rc, claims, r = ogp.gp_verify(got["proof"], got["products"], nv, od.Transcript(gc.TRANSCRIPT_LABEL))
        assert rc == 0 and np.array_equal(r, got["r"]) and np.array_equal(claims, got["claims"]), name
        dt = time.time() - t0
        doc["cases"][name] = {
            "n_circuits": len(polys), "num_vars": nv, "seed": gc.GOLDEN[name][2],
            "sha256": hashlib.sha256(gc.digest_input(got)).hexdigest(), "proof_len": len(got["proof"]),
            "after_challenge_hex": after.tobytes().hex(), "oracle_seconds": round(dt, 1), "oracle_verifier": "accepted",
        }
        print(name, "done in %.1f s" % dt, flush=True)
        with open(OUT, "w") as f:
            json.dump(doc, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
