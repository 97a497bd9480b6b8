"""Golden hashes of a caller-defined strategy over a full-width field-element table AT SIZE
(tests/golden/field_tables_big.json):

    python tests/golden/make_golden_fr.py

C = 4, log_m = 16, 2^20 lookups of tests/workloads.py's seeded inputs, one table of 2^16 uniform field elements
(tests/field_tables.py "random_full"), g = the sum of the four lookups.  Runs the CPU oracle for caller-defined
strategies (oracle_custom/), whose verifier must accept the proof it hashes; a minute or more of CPU.  The GPU test
(tests/test_gpu_field_tables.py) compares the bytes it produces with these hashes: 2^11-row commitments of 253-bit
values and openings whose bound runs over many row chunks."""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import field_tables as ft  # noqa: E402
import oracle_custom_fr_lib as oc  # noqa: E402
import oracle_lib as ol  # noqa: E402
import workloads as wl  # noqa: E402

OUT = os.path.join(HERE, "field_tables_big.json")
NAME, C, LOG_M, LOG_S, SEED = "random_full_c4_s20", 4, 16, 20, wl.BENCH_SEED + 20


def inputs():
    idx, r, tape_seed = wl.make_inputs(LOG_S, C, LOG_M, SEED)
    S = ft.strategy(None, "random_full", C, LOG_M, 1)
    need = wl.gens_needed(C, LOG_S, S.num_memories, LOG_M)
    return S, idx, r, tape_seed, np.ascontiguousarray(ol.generators(need))


def main():
    S, idx, r, tape_seed, gens = inputs()
    t0 = time.time()
    res = oc.prove(S, idx, r, gens, tape_seed, flags=1)  # flags=1: run the verifier too
    dt = time.time() - t0
    assert res["rc"] == 0, res["rc"]
    doc = {"cases": {NAME: {
        "C": C, "log_m": LOG_M, "log_s": LOG_S, "seed": SEED, "table": "random_full", "n_generators": int(gens.shape[0]),
        "table_sha256": hashlib.sha256(np.stack(S.tables).tobytes()).hexdigest(),
        "indices_sha256": hashlib.sha256(idx.tobytes()).hexdigest(),
        "commitment_sha256": hashlib.sha256(res["commitment"]).hexdigest(), "commitment_len": len(res["commitment"]),
        "proof_sha256": hashlib.sha256(res["proof"]).hexdigest(), "proof_len": len(res["proof"]),
        "challenges_sha256": hashlib.sha256(res["challenges"].tobytes()).hexdigest(),
        "n_challenges": int(len(res["challenges"])),
        "oracle_seconds": round(dt, 1), "oracle_verifier": "accepted",
    }}}
    print(NAME, "done in %.1f s" % dt, flush=True)
    with open(OUT, "w") as f:
        json.dump(doc, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
