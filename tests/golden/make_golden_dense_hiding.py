"""Golden hashes of HIDING dense-polynomial commitments and openings at size (tests/golden/dense_poly_hiding.json).

    python tests/golden/make_golden_dense_hiding.py [full_nv22 u16_nv22 full_nv24 u16_nv24 ...]

Runs the CPU oracle (oracle_dense/) on the seeded inputs of tests/dense_poly_cases.py, with one tape throughout:
commit_hiding (blinds drawn as random_vector("poly_blinds", L)), the commitment absorbed, Zr = evaluate(r),
blind_Zr = random_scalar("blind_Zr"), PolyEvalProof::prove with the blinds and blind_Zr, then a challenge drawn after
the proof.  The oracle's verifier must accept every proof against its C_Zr.  Only SHA-256 hashes of the bytes are
committed; tests/test_gpu_hiding.py compares the GPU's bytes with them."""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import dense_poly_cases as dc  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_hiding_lib as oh  # noqa: E402
import oracle_lib as ol  # noqa: E402

OUT = os.path.join(HERE, "dense_poly_hiding.json")


def main():
    names = sys.argv[1:] or ["full_nv22", "u16_nv22", "full_nv24", "u16_nv24"]
    doc = json.load(open(OUT)) if os.path.exists(OUT) else {"generator_label": "gens_sparse_poly", "cases": {}}
    for name in names:
        nv, Z, r, seed = dc.inputs(name)
        need = dc.n_generators(nv)
        stream = np.ascontiguousarray(ol.generators(need))
        t0 = time.time()
        tape = od.RandomTape(dc.TAPE_LABEL, seed)
        comm, blinds = oh.commit_hiding(Z, stream, tape=tape)
        t = od.Transcript(dc.TRANSCRIPT_LABEL)
        t.append_poly_commitment(dc.COMMIT_LABEL, comm)
        Zr = od.evaluate(Z, r)
        blind_Zr = tape.random_scalar(b"blind_Zr")
        proof, czr = oh.prove_hiding(Z, r, Zr, stream, t, tape, blinds=blinds, blind_Zr=blind_Zr)
        after = t.challenge_scalar(b"after")
        v = od.Transcript(dc.TRANSCRIPT_LABEL)
        v.append_poly_commitment(dc.COMMIT_LABEL, comm)
        assert oh.verify(stream, nv, comm, proof, r, czr, v) == 0, name
        dt = time.time() - t0
        doc["cases"][name] = {
            "num_vars": nv, "values": dc.CASES[name][1], "seed": dc.CASES[name][2], "n_generators": need,
            "generators_sha256": hashlib.sha256(stream.tobytes()).hexdigest(),
            "Z_sha256": hashlib.sha256(Z.tobytes()).hexdigest(),
            "commitment_sha256": hashlib.sha256(comm).hexdigest(), "commitment_len": len(comm),
            "blinds_sha256": hashlib.sha256(blinds.tobytes()).hexdigest(),
            "proof_sha256": hashlib.sha256(proof).hexdigest(), "proof_len": len(proof),
            "Zr_hex": Zr.tobytes().hex(), "blind_Zr_hex": blind_Zr.tobytes().hex(), "C_Zr_hex": czr.hex(),
            "after_challenge_hex": after.tobytes().hex(), "oracle_seconds": round(dt, 1), "oracle_verifier": "accepted",
        }
        print(name, "done in %.1f s" % dt, flush=True)
        with open(OUT, "w") as f:
            json.dump(doc, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
