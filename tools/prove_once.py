"""One warm-up + one measured pass of the hot path (XOR C=4 M=2^16, 2^LOG_S lookups) — a short command to put
under a profiler (launch list, per-kernel captures)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import bench
import lasso_b200 as lb

log_s = int(sys.argv[1]) if len(sys.argv) > 1 else 20
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
C, log_m = 4, 16
idx, r, seed = bench.make_inputs(log_s, C, log_m, 1)
ctx = lb.Context(0)
S = lb.Strategy(lb.XOR, C, log_m)
need = lb.gens_points_needed(C, 1 << log_s, 4, log_m)
cache = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_build", "gens_gens_sparse_poly_%d.npy" % need)
stream = np.load(cache) if os.path.exists(cache) else lb.sample_generators(b"gens_sparse_poly", need)
gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C, 1 << log_s, 4, log_m, stream=stream)
print("launches after setup", ctx.launches)
for it in range(steps):
    l0 = ctx.launches
    t = time.time()
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    com = dense.commit(gens)
    p = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    print("step %d: %.1f ms, %d launches" % (it, (time.time() - t) * 1e3, ctx.launches - l0))
