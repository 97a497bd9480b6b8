"""BASELINE.json configs 2-4 AT SIZE on one H100: the commitment and proof bytes must hash to the golden values the
CPU oracle produced offline (tests/golden/big_proofs.json, tests/golden/make_golden_big.py; the oracle's verifier
accepted every one of them).  Mirrors the reference's end-to-end tests (src/e2e_test.rs:64-99,
src/subtables/range_check.rs:101-128) at the benchmark sizes."""
import hashlib
import json
import os

import numpy as np
import pytest

import workloads as wl

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DOC = json.load(open(os.path.join(HERE, "golden", "big_proofs.json")))


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("name", ["and_c1_s10", "xor_c4_s14", "lt_c8_s14", "rc40_c4_s14", "xor_c4_s20", "lt_c8_s22", "rc40_c4_s24"])
def test_config_bytes_match_golden(ctx, name):
    import lasso_b200 as lb
    import oracle_lib as ol

    g = DOC["cases"].get(name)
    if g is None:
        pytest.skip("no golden entry for %s (run tests/golden/make_golden_big.py %s)" % (name, name))
    kind, C, log_m, log_r, log_s, idx, r, tape_seed = wl.config_inputs(name)
    assert hashlib.sha256(idx.tobytes()).hexdigest() == g["indices_sha256"]
    S = lb.Strategy(kind, C, log_m, log_r)
    s = 1 << log_s
    need = lb.gens_points_needed(C, s, S.num_memories, log_m)
    assert need == g["n_generators"]
    stream = np.ascontiguousarray(ol.generators(need))
    assert hashlib.sha256(stream.tobytes()).hexdigest() == g["generators_sha256"]
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C, s, S.num_memories, log_m, stream=stream)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=tape_seed)
    assert len(com) == g["commitment_len"] and len(proof.bytes) == g["proof_len"]
    assert hashlib.sha256(com).hexdigest() == g["commitment_sha256"]
    assert len(proof.challenges) == g["n_challenges"]
    assert proof.challenges[-1].tobytes().hex() == g["last_challenge_hex"]
    assert hashlib.sha256(proof.bytes).hexdigest() == g["proof_sha256"]
