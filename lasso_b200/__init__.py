"""lasso_b200 — H100-native (sm_90a) accelerator for the a16z/Lasso prover hot path.

Host-side mirror of the reference's surface for that path (names follow the Rust items):

    DensifiedRepresentation.from_lookup_indices(ctx, indices, log_m)     src/lasso/densified.rs:22
    DensifiedRepresentation.commit(gens)                                 src/lasso/densified.rs:78
    SparsePolyCommitmentGens.new(ctx, label, c, s, num_memories, log_m)  src/lasso/surge.rs:32
    SparsePolynomialEvaluationProof.prove(ctx, strategy, dense, r, gens, ...)   src/lasso/surge.rs:119

and, for a caller that composes Lasso into a larger protocol, its own dense polynomials on its own transcript:

    Transcript(label), RandomTape(label, seed)                           src/utils/{transcript,random}.rs
    PolyCommitmentGens.new(ctx, label, num_vars)                         src/poly/dense_mlpoly.rs:38
    DensePolynomial(ctx, Z).commit(gens) / .evaluate(r)                  src/poly/dense_mlpoly.rs:152, 229
    PolyEvalProof.prove(ctx, poly, r, Zr, gens, transcript, random_tape)    src/poly/dense_mlpoly.rs:301
    DensePolynomial.eq(ctx, r)                                           src/poly/eq_poly.rs:21
    DensePolynomial.merge(ctx, polys)                                    src/poly/dense_mlpoly.rs:251
    DensePolynomial.evaluate_batch(ctx, polys, r)                        (DensePolynomial::evaluate of many, one eq table)
    DensePolynomial.new_padded(ctx, Z), .split(idx)                      src/poly/dense_mlpoly.rs:75, 101
    p.bound_top(r) / .bound_bot(r): new polynomials, p unchanged         src/poly/dense_mlpoly.rs:209, 218
    p.to_numpy() / .to_tensor() / .copy_to(tensor)                       (the evaluations Z, read back)
    CombinedTableEvalProof.prove(ctx, combined, evals, r, gens, transcript, random_tape)   src/subtables/mod.rs:284
    SumcheckInstanceProof.prove_arbitrary(ctx, polys, Comb(fn, k), transcript)   src/subprotocols/sumcheck.rs:149
    DensePolynomial.from_comb(ctx, comb, polys)                          (pointwise g(P_0, .., P_{k-1}))
    GrandProductCircuit(ctx, poly).evaluate()                            src/subprotocols/grand_product.rs:38, 60
    BatchedGrandProductArgument.prove(ctx, circuits, transcript)         src/subprotocols/grand_product.rs:100

and the memory check of a lookup proof, or of a caller's own memory, inside a caller's protocol (single GPU):

    Subtables(ctx, strategy, dense).lookup_polys / .combined_poly / .commit   src/subtables/mod.rs:116, 177
    DensifiedRepresentation.dim_poly(j) / .read_poly(j) / .final_poly(j)  src/lasso/densified.rs:8
    MemoryCheckingProof.prove(ctx, strategy, dense, (gamma, tau), gens, transcript, random_tape)
                                                                         src/subtables/memory_checking.rs:56
    GrandProducts.new(ctx, eval_table, dim, read, final, (gamma, tau))   src/subtables/memory_checking.rs:175
    Transcript.append_combined_table_commitment(commitment)              src/subtables/mod.rs:382

and zero-knowledge sumchecks over a caller's polynomials (single GPU; the commitments and dot-product proofs also sharded):

    MultiCommitGens(ctx, G, h), MultiCommitGens.new(ctx, n, label), .commit(scalars, blind)   src/poly/commitments.rs:14, 84
    DotProductProofGens.new(ctx, n, label).gens_n / .gens_1             src/subprotocols/dot_product.rs:144
    DotProductProof.prove(ctx, gens_1, gens_n, transcript, random_tape, x, blind_x, a, y, blind_y)
                                                                         src/subprotocols/dot_product.rs:31
    ZKSumcheckInstanceProof.prove(ctx, comb, polys, num_rounds, blind_claim, gens_1, gens_n, transcript, random_tape)
                                                                         src/subprotocols/sumcheck.rs:331 (its verifier)

and the Σ-protocols over committed scalars that end such a protocol (gens: a MultiCommitGens with n == 1; also sharded):

    KnowledgeProof.prove(ctx, gens, transcript, random_tape, x, r)       src/subprotocols/zk.rs:23
    EqualityProof.prove(ctx, gens, transcript, random_tape, v1, s1, v2, s2)   src/subprotocols/zk.rs:89
    ProductProof.prove(ctx, gens, transcript, random_tape, x, rX, y, rY, z, rZ)   src/subprotocols/zk.rs:169

Everything runs through the C-ABI shared library (include/lasso_b200.h); there is no CPU fallback:
importing works without a GPU, but creating a Context raises.
"""
from .api import (  # noqa: F401
    AND, LT, OR, RANGE_CHECK, XOR,
    BatchedGrandProductArgument, Comb, CombinedTableEvalProof, Context, CustomStrategy, DensePolynomial, DensifiedRepresentation, DotProductProof, DotProductProofGens, EqualityProof, GrandProductCircuit, GrandProducts, KnowledgeProof, LassoError, MemoryCheckingProof, MsmJob,
    MultiCommitGens, PolyCommitmentGens, PolyEvalProof, ProductProof, RandomTape, SparsePolyCommitmentGens, SparsePolynomialEvaluationProof, Strategy, Subtables, SumcheckInstanceProof, Transcript, ZKSumcheckInstanceProof,
    bind_bot, bind_top,
    commit_rows, eq_evals, fr_from_ints, gather_lookup_polys, gens_points_needed, lib, library_path, materialize_subtables,
    msm, poly_gens_points_needed, sample_generators, sumcheck_bind_round_arbitrary,
    sumcheck_round_arbitrary, sumcheck_round_cubic, sumcheck_round_custom, trace_combine_lookups,
)
