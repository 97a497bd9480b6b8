//! Raw declarations of include/lasso_b200.h (one per C entry point; the header cites the reference item each replaces).
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_void};

#[repr(C)]
pub struct lasso_ctx {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_gens {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_dense {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_msm_job {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_strategy {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_transcript {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_random_tape {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_poly_gens {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_poly {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_comb {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_gp_circuit {
    _p: [u8; 0],
}
#[repr(C)]
pub struct lasso_mc_gens {
    _p: [u8; 0],
}

extern "C" {
    pub fn lasso_last_error() -> *const c_char;
    pub fn lasso_ctx_create(out: *mut *mut lasso_ctx, device_id: c_int) -> c_int;
    pub fn lasso_ctx_destroy(ctx: *mut lasso_ctx);
    pub fn lasso_comm_unique_id(out: *mut u8) -> c_int;
    pub fn lasso_ctx_init_comm(ctx: *mut lasso_ctx, id: *const u8, rank: c_int, world: c_int) -> c_int;
    pub fn lasso_ctx_bind_host_threads(ctx: *mut lasso_ctx) -> c_int;
    // per-loop entry points (host buffers)
    pub fn lasso_bind_top(ctx: *mut lasso_ctx, z: *mut u64, len: usize, r: *const u64) -> c_int;
    pub fn lasso_bind_bot(ctx: *mut lasso_ctx, z: *mut u64, len: usize, r: *const u64) -> c_int;
    pub fn lasso_eq_evals(ctx: *mut lasso_ctx, r: *const u64, ell: c_int, out: *mut u64) -> c_int;
    pub fn lasso_sumcheck_round_arbitrary(ctx: *mut lasso_ctx, strategy: c_int, c: c_int, log_m: c_int, log_r: c_int,
                                          polys: *const *const u64, len: usize, evals_out: *mut u64) -> c_int;
    pub fn lasso_sumcheck_bind_round_arbitrary(ctx: *mut lasso_ctx, strategy: c_int, c: c_int, log_m: c_int, log_r: c_int,
                                               polys: *const *mut u64, len: usize, r: *const u64, evals_out: *mut u64) -> c_int;
    pub fn lasso_sumcheck_round_cubic(ctx: *mut lasso_ctx, n_circuits: c_int, a: *const *const u64, b: *const *const u64,
                                      ceq: *const u64, len: usize, e0e2e3_out: *mut u64) -> c_int;
    pub fn lasso_materialize_subtables(ctx: *mut lasso_ctx, strategy: c_int, c: c_int, log_m: c_int, log_r: c_int,
                                       tables_out: *const *mut u64) -> c_int;
    pub fn lasso_gather_lookup_polys(ctx: *mut lasso_ctx, strategy: c_int, c: c_int, log_m: c_int, log_r: c_int,
                                     nz: *const *const u64, s: usize, e_out: *const *mut u64) -> c_int;
    pub fn lasso_msm(ctx: *mut lasso_ctx, bases: *const u64, scalars: *const u64, n: usize, out_xytz: *mut u64) -> c_int;
    pub fn lasso_commit_rows(ctx: *mut lasso_ctx, gens: *const u64, z: *const u64, l_size: usize, r_size: usize,
                             out_points: *mut u64) -> c_int;
    pub fn lasso_msm_plan_info(n: usize, max_bits: u32, out: *mut c_int) -> c_int;
    pub fn lasso_msm_job_create(ctx: *mut lasso_ctx, bases: *const u64, n_pool: usize, scalars: *const u64, n: usize,
                                out: *mut *mut lasso_msm_job) -> c_int;
    pub fn lasso_msm_job_run(ctx: *mut lasso_ctx, job: *mut lasso_msm_job, iters: c_int, avg_ms: *mut f64, out_xytz: *mut u64,
                             info: *mut c_int) -> c_int;
    pub fn lasso_msm_job_naive(ctx: *mut lasso_ctx, job: *mut lasso_msm_job, out_xytz: *mut u64) -> c_int;
    pub fn lasso_msm_job_destroy(job: *mut lasso_msm_job);
    // the whole path, device resident
    pub fn lasso_gens_points_needed(c: usize, s: usize, num_memories: usize, log_m: usize) -> usize;
    pub fn lasso_sample_generators(label: *const c_char, count: usize, out_affine: *mut u64) -> c_int;
    pub fn lasso_gens_create(ctx: *mut lasso_ctx, stream: *const u64, n_points: usize, c: usize, s: usize, num_memories: usize,
                             log_m: usize, out: *mut *mut lasso_gens) -> c_int;
    pub fn lasso_gens_destroy(g: *mut lasso_gens);
    pub fn lasso_densify(ctx: *mut lasso_ctx, indices: *const u64, n_lookups: usize, c: usize, log_m: usize,
                         out: *mut *mut lasso_dense) -> c_int;
    pub fn lasso_densify_device(ctx: *mut lasso_ctx, indices: *const c_void, elem_bytes: usize, n_lookups: usize, c: usize,
                                row_stride: usize, col_stride: usize, log_m: usize, stream: *mut c_void,
                                out: *mut *mut lasso_dense) -> c_int;
    pub fn lasso_dense_destroy(d: *mut lasso_dense);
    pub fn lasso_dense_s(d: *const lasso_dense) -> usize;
    pub fn lasso_dense_read(ctx: *mut lasso_ctx, d: *const lasso_dense, which: c_int, out: *mut u64, cap_elems: usize) -> usize;
    pub fn lasso_commit(ctx: *mut lasso_ctx, d: *const lasso_dense, g: *const lasso_gens, out: *mut u8, cap: usize,
                        out_len: *mut usize) -> c_int;
    pub fn lasso_prove(ctx: *mut lasso_ctx, strategy: c_int, log_r: c_int, d: *mut lasso_dense, r: *const u64, r_len: usize,
                       g: *const lasso_gens, transcript_label: *const c_char, tape_label: *const c_char, tape_seed: *const u64,
                       proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize, challenges_out: *mut u64,
                       challenges_cap: usize, n_challenges: *mut usize) -> c_int;
    // a caller's transcript and dense polynomials (raw declarations only; not compiled: no cargo was available)
    pub fn lasso_transcript_create(label: *const c_char, out: *mut *mut lasso_transcript) -> c_int;
    pub fn lasso_transcript_destroy(t: *mut lasso_transcript);
    pub fn lasso_transcript_append_message(t: *mut lasso_transcript, label: *const c_char, msg: *const u8, len: usize) -> c_int;
    pub fn lasso_transcript_append_u64(t: *mut lasso_transcript, label: *const c_char, x: u64) -> c_int;
    pub fn lasso_transcript_append_protocol_name(t: *mut lasso_transcript, name: *const c_char) -> c_int;
    pub fn lasso_transcript_append_scalar(t: *mut lasso_transcript, label: *const c_char, s: *const u64) -> c_int;
    pub fn lasso_transcript_append_scalars(t: *mut lasso_transcript, label: *const c_char, s: *const u64, n: usize) -> c_int;
    pub fn lasso_transcript_append_point(t: *mut lasso_transcript, label: *const c_char, point: *const u8) -> c_int;
    pub fn lasso_transcript_append_points(t: *mut lasso_transcript, label: *const c_char, points: *const u8, n: usize) -> c_int;
    pub fn lasso_transcript_append_poly_commitment(t: *mut lasso_transcript, label: *const c_char, bytes: *const u8,
                                                   len: usize) -> c_int;
    pub fn lasso_transcript_challenge_scalar(t: *mut lasso_transcript, label: *const c_char, out: *mut u64) -> c_int;
    pub fn lasso_transcript_challenge_vector(t: *mut lasso_transcript, label: *const c_char, n: usize, out: *mut u64) -> c_int;
    pub fn lasso_random_tape_create(label: *const c_char, seed: *const u64, out: *mut *mut lasso_random_tape) -> c_int;
    pub fn lasso_random_tape_destroy(t: *mut lasso_random_tape);
    pub fn lasso_random_tape_random_scalar(t: *mut lasso_random_tape, label: *const c_char, out: *mut u64) -> c_int;
    pub fn lasso_random_tape_random_vector(t: *mut lasso_random_tape, label: *const c_char, n: usize, out: *mut u64) -> c_int;
    pub fn lasso_poly_gens_points_needed(num_vars: usize) -> usize;
    pub fn lasso_poly_gens_create(ctx: *mut lasso_ctx, stream: *const u64, n_points: usize, num_vars: usize,
                                  out: *mut *mut lasso_poly_gens) -> c_int;
    pub fn lasso_poly_gens_destroy(g: *mut lasso_poly_gens);
    pub fn lasso_poly_create(ctx: *mut lasso_ctx, z: *const u64, len: usize, out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_create_device(ctx: *mut lasso_ctx, z: *const u64, len: usize, row_stride: usize, stream: *mut c_void,
                                    out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_num_vars(p: *const lasso_poly) -> usize;
    pub fn lasso_poly_destroy(p: *mut lasso_poly);
    pub fn lasso_poly_commit(ctx: *mut lasso_ctx, p: *const lasso_poly, g: *const lasso_poly_gens, out: *mut u8, cap: usize,
                             out_len: *mut usize) -> c_int;
    pub fn lasso_poly_evaluate(ctx: *mut lasso_ctx, p: *const lasso_poly, r: *const u64, r_len: usize, out: *mut u64) -> c_int;
    pub fn lasso_poly_eval_prove(ctx: *mut lasso_ctx, p: *const lasso_poly, g: *const lasso_poly_gens, r: *const u64,
                                 r_len: usize, zr: *const u64, transcript: *mut lasso_transcript,
                                 random_tape: *mut lasso_random_tape, proof_out: *mut u8, proof_cap: usize,
                                 proof_len: *mut usize, c_zr_out: *mut u8) -> c_int;
    pub fn lasso_poly_create_eq(ctx: *mut lasso_ctx, r: *const u64, r_len: usize, out: *mut *mut lasso_poly) -> c_int;
    // deriving polynomials and reading them back (raw declarations only; not compiled: no cargo was available)
    pub fn lasso_poly_bind_top(ctx: *mut lasso_ctx, p: *const lasso_poly, r: *const u64, k: usize,
                               out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_bind_bot(ctx: *mut lasso_ctx, p: *const lasso_poly, r: *const u64, k: usize,
                               out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_split(ctx: *mut lasso_ctx, p: *const lasso_poly, idx: usize, lo_out: *mut *mut lasso_poly,
                            hi_out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_create_padded(ctx: *mut lasso_ctx, z: *const u64, len: usize, out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_create_padded_device(ctx: *mut lasso_ctx, z: *const u64, len: usize, row_stride: usize,
                                           stream: *mut c_void, out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_read(ctx: *mut lasso_ctx, p: *const lasso_poly, out: *mut u64, cap: usize) -> c_int;
    pub fn lasso_poly_read_device(ctx: *mut lasso_ctx, p: *const lasso_poly, dst: *mut u64, row_stride: usize,
                                  stream: *mut c_void) -> c_int;
    // many polynomials per call (raw declarations only; not compiled: no cargo was available)
    pub fn lasso_poly_create_merge(ctx: *mut lasso_ctx, polys: *const *const lasso_poly, n_polys: usize,
                                   out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_poly_evaluate_batch(ctx: *mut lasso_ctx, polys: *const *const lasso_poly, n_polys: usize, r: *const u64,
                                     r_len: usize, out: *mut u64) -> c_int;
    pub fn lasso_combined_eval_prove(ctx: *mut lasso_ctx, combined: *const lasso_poly, gens: *const lasso_poly_gens,
                                     evals: *const u64, n_evals: usize, r: *const u64, r_len: usize,
                                     transcript: *mut lasso_transcript, random_tape: *mut lasso_random_tape,
                                     proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize) -> c_int;
    // lookups inside a caller's protocol (raw declarations only; not compiled: no cargo was available)
    pub fn lasso_prove_transcript(ctx: *mut lasso_ctx, strategy: c_int, log_r: c_int, dense: *mut lasso_dense, r: *const u64,
                                  r_len: usize, gens: *const lasso_gens, transcript: *mut lasso_transcript,
                                  random_tape: *mut lasso_random_tape, proof_out: *mut u8, proof_cap: usize,
                                  proof_len: *mut usize, claimed_eval_out: *mut u64) -> c_int;
    pub fn lasso_prove_custom_transcript(ctx: *mut lasso_ctx, s: *const lasso_strategy, dense: *mut lasso_dense,
                                         r: *const u64, r_len: usize, gens: *const lasso_gens,
                                         transcript: *mut lasso_transcript, random_tape: *mut lasso_random_tape,
                                         proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize,
                                         claimed_eval_out: *mut u64) -> c_int;
    pub fn lasso_transcript_append_sparse_commitment(t: *mut lasso_transcript, bytes: *const u8, len: usize) -> c_int;
    pub fn lasso_dense_outputs(ctx: *mut lasso_ctx, strategy: c_int, log_r: c_int, dense: *const lasso_dense,
                               out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_dense_outputs_custom(ctx: *mut lasso_ctx, s: *const lasso_strategy, dense: *const lasso_dense,
                                      out: *mut *mut lasso_poly) -> c_int;
    // memory checking inside a caller's protocol (single GPU; raw declarations only)
    pub fn lasso_lookup_polys(ctx: *mut lasso_ctx, strategy: c_int, log_r: c_int, dense: *const lasso_dense,
                              out: *mut *mut lasso_poly, n_out: usize) -> c_int;
    pub fn lasso_lookup_polys_custom(ctx: *mut lasso_ctx, s: *const lasso_strategy, dense: *const lasso_dense,
                                     out: *mut *mut lasso_poly, n_out: usize) -> c_int;
    pub fn lasso_dense_poly(ctx: *mut lasso_ctx, dense: *const lasso_dense, which: c_int, j: usize,
                            out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_memory_check_prove(ctx: *mut lasso_ctx, strategy: c_int, log_r: c_int, dense: *const lasso_dense,
                                    gamma: *const u64, tau: *const u64, gens: *const lasso_gens,
                                    transcript: *mut lasso_transcript, random_tape: *mut lasso_random_tape,
                                    proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize) -> c_int;
    pub fn lasso_memory_check_prove_custom(ctx: *mut lasso_ctx, s: *const lasso_strategy, dense: *const lasso_dense,
                                           gamma: *const u64, tau: *const u64, gens: *const lasso_gens,
                                           transcript: *mut lasso_transcript, random_tape: *mut lasso_random_tape,
                                           proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize) -> c_int;
    pub fn lasso_memory_fingerprints(ctx: *mut lasso_ctx, table: *const lasso_poly, dim: *const lasso_poly,
                                     read: *const lasso_poly, final_ts: *const lasso_poly, gamma: *const u64,
                                     tau: *const u64, out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_transcript_append_combined_table_commitment(t: *mut lasso_transcript, label: *const c_char,
                                                             bytes: *const u8, len: usize) -> c_int;
    // sumchecks over a caller's polynomials (raw declarations only; not compiled: no cargo was available)
    pub fn lasso_comb_create(n_inputs: c_int, program: *const i32, n_ops: c_int, constants: *const u64, n_constants: c_int,
                             degree: c_int, out: *mut *mut lasso_comb) -> c_int;
    pub fn lasso_comb_destroy(g: *mut lasso_comb);
    pub fn lasso_sumcheck_prove(ctx: *mut lasso_ctx, comb: *const lasso_comb, polys: *const *const lasso_poly, n_polys: usize,
                                num_rounds: usize, transcript: *mut lasso_transcript, proof_out: *mut u8, proof_cap: usize,
                                proof_len: *mut usize, r_out: *mut u64, final_evals_out: *mut u64, claim_out: *mut u64)
                                -> c_int;
    pub fn lasso_mc_gens_create(ctx: *mut lasso_ctx, g_affine: *const u64, n: usize, h_affine: *const u64,
                                out: *mut *mut lasso_mc_gens) -> c_int;
    pub fn lasso_mc_gens_n(g: *const lasso_mc_gens) -> usize;
    pub fn lasso_mc_gens_destroy(g: *mut lasso_mc_gens);
    pub fn lasso_mc_commit(ctx: *mut lasso_ctx, gens: *const lasso_mc_gens, scalars: *const u64, n: usize, blind: *const u64,
                           out: *mut u8) -> c_int;
    pub fn lasso_dot_product_prove(ctx: *mut lasso_ctx, gens_1: *const lasso_mc_gens, gens_n: *const lasso_mc_gens,
                                   transcript: *mut lasso_transcript, random_tape: *mut lasso_random_tape, x: *const u64,
                                   blind_x: *const u64, a: *const u64, n: usize, y: *const u64, blind_y: *const u64,
                                   proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize, cx_out: *mut u8,
                                   cy_out: *mut u8) -> c_int;
    pub fn lasso_zk_sumcheck_prove(ctx: *mut lasso_ctx, comb: *const lasso_comb, polys: *const *const lasso_poly,
                                   n_polys: usize, num_rounds: usize, blind_claim: *const u64,
                                   gens_1: *const lasso_mc_gens, gens_n: *const lasso_mc_gens,
                                   transcript: *mut lasso_transcript, random_tape: *mut lasso_random_tape,
                                   proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize, r_out: *mut u64,
                                   final_evals_out: *mut u64, claim_out: *mut u64, comm_claim_out: *mut u8,
                                   blind_eval_out: *mut u64) -> c_int;
    pub fn lasso_knowledge_prove(ctx: *mut lasso_ctx, gens: *const lasso_mc_gens, transcript: *mut lasso_transcript,
                                 random_tape: *mut lasso_random_tape, x: *const u64, r: *const u64, proof_out: *mut u8,
                                 c_out: *mut u8) -> c_int;
    pub fn lasso_equality_prove(ctx: *mut lasso_ctx, gens: *const lasso_mc_gens, transcript: *mut lasso_transcript,
                                random_tape: *mut lasso_random_tape, v1: *const u64, s1: *const u64, v2: *const u64,
                                s2: *const u64, proof_out: *mut u8, c1_out: *mut u8, c2_out: *mut u8) -> c_int;
    pub fn lasso_product_prove(ctx: *mut lasso_ctx, gens: *const lasso_mc_gens, transcript: *mut lasso_transcript,
                               random_tape: *mut lasso_random_tape, x: *const u64, r_x: *const u64, y: *const u64,
                               r_y: *const u64, z: *const u64, r_z: *const u64, proof_out: *mut u8, x_out: *mut u8,
                               y_out: *mut u8, z_out: *mut u8) -> c_int;
    pub fn lasso_poly_create_comb(ctx: *mut lasso_ctx, comb: *const lasso_comb, polys: *const *const lasso_poly,
                                  n_polys: usize, out: *mut *mut lasso_poly) -> c_int;
    pub fn lasso_sumcheck_prove_cubic_batched(ctx: *mut lasso_ctx, a: *const *const lasso_poly, b: *const *const lasso_poly,
                                              n: usize, c: *const lasso_poly, coeffs: *const u64, claim: *const u64,
                                              num_rounds: usize, transcript: *mut lasso_transcript, proof_out: *mut u8,
                                              proof_cap: usize, proof_len: *mut usize, r_out: *mut u64,
                                              claims_a_out: *mut u64, claims_b_out: *mut u64, claim_c_out: *mut u64)
                                              -> c_int;
    // grand products over a caller's polynomials (raw declarations only; not compiled: no cargo was available)
    pub fn lasso_gp_circuit_create(ctx: *mut lasso_ctx, poly: *const lasso_poly, out: *mut *mut lasso_gp_circuit) -> c_int;
    pub fn lasso_gp_circuit_evaluate(c: *const lasso_gp_circuit, out: *mut u64) -> c_int;
    pub fn lasso_gp_circuit_num_vars(c: *const lasso_gp_circuit) -> usize;
    pub fn lasso_gp_circuit_destroy(c: *mut lasso_gp_circuit);
    pub fn lasso_gp_prove(ctx: *mut lasso_ctx, circuits: *const *const lasso_gp_circuit, n: usize,
                          transcript: *mut lasso_transcript, proof_out: *mut u8, proof_cap: usize, proof_len: *mut usize,
                          r_out: *mut u64, claims_out: *mut u64) -> c_int;
    pub fn lasso_launch_count(ctx: *const lasso_ctx) -> u64;
    pub fn lasso_last_timings(ctx: *const lasso_ctx, out_ms: *mut f64);
}
