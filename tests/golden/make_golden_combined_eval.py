"""Golden hashes of combined openings of merged polynomials (tests/golden/combined_eval.json).

    python tests/golden/make_golden_combined_eval.py [k3_nv4_full k5_nv6_u32 ...]

Runs the CPU oracle (oracle_dense/ over the restatement in oracle/) on the seeded inputs of tests/combined_eval_cases.py:
DensePolynomial::merge of the k components, their evaluations at r as the claims, and CombinedTableEvalProof::prove on a
transcript labelled TRANSCRIPT_LABEL to which nothing is appended first, with a tape seeded from the case.  The oracle's
verifier must accept every proof against the merged polynomial's commitment on a fresh transcript.  Only SHA-256 hashes
of evals || proof are committed (with the proof length, the merged commitment's hash and a challenge drawn after the
proof); tests/test_combined_eval_host.py reproduces the small cases with the oracle, tests/test_gpu_combined_eval.py
compares the GPU's outputs with all of them."""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import combined_eval_cases as cc  # noqa: E402
import dense_poly_cases as dc  # noqa: E402
import oracle_combined_eval_lib as oce  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_lib as ol  # noqa: E402

OUT = os.path.join(HERE, "combined_eval.json")


def main():
    names = sys.argv[1:] or sorted(cc.GOLDEN)
    doc = json.load(open(OUT)) if os.path.exists(OUT) else {"cases": {}}
    for name in names:
        nv, comps, r, seed = cc.golden_inputs(name)
        t0 = time.time()
        Z = oce.merge(comps)
        mv = Z.shape[0].bit_length() - 1
        stream = np.ascontiguousarray(ol.generators(dc.n_generators(mv)))
        evals = np.stack([od.evaluate(c, r) for c in comps])
        t = od.Transcript(cc.TRANSCRIPT_LABEL)
        proof = oce.prove(Z, evals, r, stream, t, od.RandomTape(cc.TAPE_LABEL, seed))
        after = t.challenge_scalar(b"after")
        comm = od.commit(Z, stream)
        assert oce.verify(stream, mv, comm, proof, evals, r, od.Transcript(cc.TRANSCRIPT_LABEL)) == 0, name
        dt = time.time() - t0
        k, _, kind, s = cc.GOLDEN[name]
        doc["cases"][name] = {
            "k": k, "num_vars": nv, "merged_num_vars": mv, "values": kind, "seed": s,
            "sha256": hashlib.sha256(cc.digest_input(evals, proof)).hexdigest(), "proof_len": len(proof),
            "commitment_sha256": hashlib.sha256(comm).hexdigest(), "after_challenge_hex": after.tobytes().hex(),
            "oracle_seconds": round(dt, 1), "oracle_verifier": "accepted",
        }
        print(name, "done in %.1f s" % dt, flush=True)
        with open(OUT, "w") as f:
            json.dump(doc, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
