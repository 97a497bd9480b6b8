"""Golden hashes of the BASELINE configurations AT SIZE (tests/golden/big_proofs.json).

    python tests/golden/make_golden_big.py xor_c4_s20 lt_c8_s22 rc40_c4_s24 xor_c4_s14 lt_c8_s14 rc40_c4_s14

Runs the CPU oracle (oracle/: the restatement of the reference prover AND verifier, pinned against the reference's
own known-answer tests by tests/test_oracle_kats.py) on the seeded workloads of tests/workloads.py — minutes to
tens of minutes of CPU and tens of GB of RAM for the large ones, which is why only the SHA-256 of the commitment
and proof bytes is committed.  The oracle's verifier must accept every proof it hashes.  The GPU tests
(tests/test_gpu_big_configs.py) and bench.py compare the bytes produced on the GPU with these hashes."""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as ol  # noqa: E402
import workloads as wl  # noqa: E402

OUT = os.path.join(HERE, "big_proofs.json")


def main():
    names = sys.argv[1:] or ["xor_c4_s14", "lt_c8_s14", "rc40_c4_s14"]
    doc = json.load(open(OUT)) if os.path.exists(OUT) else {"generator_label": "gens_sparse_poly", "cases": {}}
    for name in names:
        kind, C, log_m, log_r, log_s, idx, r, tape_seed = wl.config_inputs(name)
        need = wl.gens_needed(C, log_s, wl.num_memories(kind, C), log_m)
        gens = np.ascontiguousarray(ol.generators(need))
        t0 = time.time()
        res = ol.prove(kind, C, log_m, log_r, idx, r, gens, tape_seed, flags=1)  # flags=1: run the verifier too
        dt = time.time() - t0
        assert res["rc"] == 0, (name, res["rc"])
        doc["cases"][name] = {
            "kind": kind, "C": C, "log_m": log_m, "log_r": log_r, "log_s": log_s, "seed": wl.CONFIGS[name][5],
            "n_generators": need, "generators_sha256": hashlib.sha256(gens.tobytes()).hexdigest(),
            "indices_sha256": hashlib.sha256(idx.tobytes()).hexdigest(),
            "commitment_sha256": hashlib.sha256(res["commitment"]).hexdigest(), "commitment_len": len(res["commitment"]),
            "proof_sha256": hashlib.sha256(res["proof"]).hexdigest(), "proof_len": len(res["proof"]),
            "n_challenges": int(len(res["challenges"])),
            "last_challenge_hex": res["challenges"][-1].tobytes().hex(),
            "oracle_seconds": round(dt, 1), "oracle_verifier": "accepted",
        }
        import resource
        print(name, "done in %.1f s, peak RSS %.1f GB" % (dt, resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6), flush=True)
        with open(OUT, "w") as f:
            json.dump(doc, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
