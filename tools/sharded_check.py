"""Run under torchrun with WORLD_SIZE ranks: ONE proof sharded over all ranks; rank 0 checks that commitment,
challenges and proof bytes equal the CPU oracle's (and therefore the single-GPU path's).
One GPU per rank by default (torch.distributed over NCCL carries the job id and the barriers); with
LASSO_SHARD_SAME_GPU=1 every rank uses GPU 0 (gloo for the plumbing) — the exchanges of the sharded proof (shared
host segments + CUDA IPC exchange buffers, csrc/comm.cu) do not need one device per rank, so a single-GPU box can
run this check too.
With --custom every strategy is a caller-defined one (lasso_b200.CustomStrategy): the built-in cases re-expressed as
programs plus tables that are not built in, checked against the oracle for caller-defined strategies (oracle_custom/).
With --fr the strategies are caller-defined ones over tables of arbitrary field elements (tests/field_tables.py, the
full-width commitment and openings), checked the same way.
With --device every rank passes the whole index matrix as a torch CUDA tensor on its own GPU (lasso_densify_device;
int64, and int32 for every other case) instead of a numpy array.
usage: torchrun --nproc-per-node N tools/sharded_check.py [--custom | --fr] [--device] [kind C log_m log_r lookups same]"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist
import lasso_b200 as lb
import oracle_lib as ol
import custom_builtins as cb
import oracle_custom_lib as oc
import oracle_custom_fr_lib as ocf
import field_tables as ft

rank = int(os.environ.get("RANK", 0)); local = int(os.environ.get("LOCAL_RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
same_gpu = os.environ.get("LASSO_SHARD_SAME_GPU") == "1"
if same_gpu:
    local = 0
    torch.cuda.set_device(0)
    dist.init_process_group("gloo")
else:
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
cases = [(2, 4, 16, 0, 1 << 12, 1), (3, 4, 4, 0, 128, 0), (0, 1, 16, 0, 1 << 10, 1), (4, 3, 8, 40, 256, 0), (3, 8, 8, 0, 512, 0),
         (1, 2, 8, 0, 700, 0)]
fr = "--fr" in sys.argv
custom = "--custom" in sys.argv or fr
device = "--device" in sys.argv
argv = [a for a in sys.argv if a not in ("--custom", "--fr", "--device")]
if len(argv) > 6:
    cases = [tuple(int(x) for x in argv[1:7])]
if fr:  # field-element tables: kind = -100 - their index in ft.INTS; C = 2, odd log_m, degree 2
    cases = [(-100 - i, 2, 7, 0, 600 + i, 0) for i in range(len(ft.INTS))]
elif custom:  # new tables: kind = -1 - their index in cb.NEW_TABLES
    cases += [(-1 - i, 0, 0, 0, 300 + i, 0) for i in range(len(cb.NEW_TABLES))]
ctx = lb.Context(local)
ctx.init_comm()


def indices(idx, i=0):
    """the matrix as from_lookup_indices gets it: numpy, or with --device a CUDA tensor (int32 for every other case)"""
    if not device:
        return idx
    return torch.from_numpy(idx.astype(np.int32 if i % 2 else np.int64)).to(torch.device("cuda", local))


ok = True
for i, (kind, C, log_m, log_r, n, same) in enumerate(cases):
    if kind <= -100:
        S = ft.strategy(ctx, sorted(ft.INTS)[-100 - kind], C, log_m, 2, nsub=2)
    elif kind < 0:
        S = cb.NEW_TABLES[sorted(cb.NEW_TABLES)[-1 - kind]](ctx)
        C, log_m = S.C, S.log_m
    elif custom:
        S = cb.as_custom(ctx, kind, C, log_m, log_r)
    else:
        S = lb.Strategy(kind, C, log_m, log_r)
    rng = np.random.default_rng(kind * 7 + C if kind >= 0 else 1000 - kind)
    col = rng.integers(0, 1 << log_m, size=(n, 1), dtype=np.uint64)
    idx = np.ascontiguousarray(np.repeat(col, C, axis=1) if same else rng.integers(0, 1 << log_m, size=(n, C), dtype=np.uint64))
    s = 1 << (n - 1).bit_length()
    r = ol.rand_fr(rng, s.bit_length() - 1); seed = ol.rand_fr(rng, 1)[0]
    need = lb.gens_points_needed(C, s, S.num_memories, log_m)
    stream = np.ascontiguousarray(ol.generators(max(need, 300))[:need])
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"g", C, s, S.num_memories, log_m, stream=stream)
    t0 = time.time()
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, indices(idx, i), log_m)
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
    dt = time.time() - t0
    if rank == 0:
        if custom:
            ref = (ocf if fr else oc).prove(S, idx, r, stream, seed, flags=1)
        else:
            ref = ol.prove(kind, C, log_m, log_r, idx, r, stream, seed, flags=1)
        good = ref["rc"] == 0 and com == ref["commitment"] and proof.bytes == ref["proof"]
        nch = min(len(proof.challenges), len(ref["challenges"]))
        first_bad = next((i for i in range(nch) if (proof.challenges[i] != ref["challenges"][i]).any()), None)
        print("case %s%skind=%d C=%d log_m=%d n=%d world=%d: %s (%.1f ms, commit_ok=%s, first diverging challenge=%s)" % (
            "custom " if custom else "", "device " if device else "", kind, C, log_m, n, world, "OK" if good else "MISMATCH", dt * 1e3, com == ref["commitment"], first_bad), flush=True)
        ok = ok and good
# an out-of-range index (densified.rs:46) in the LAST rank's block of rows: every rank must report it (the verdict is
# agreed through the round-message path; nobody may be left waiting in the exchange that follows)
n_bad = 1 << 12
bad = np.zeros((n_bad, 2), dtype=np.uint64)
bad[n_bad - 3, 1] = 1 << 8
try:
    lb.DensifiedRepresentation.from_lookup_indices(ctx, indices(bad), 8)
    bad_ok = False
except lb.LassoError as e:
    bad_ok = e.code == 3
flags = [None] * world
dist.all_gather_object(flags, bad_ok)
if rank == 0:
    print("out-of-range index reported on every rank: %s" % ("OK" if all(flags) else "MISMATCH %s" % flags), flush=True)
    ok = ok and all(flags)
# collective MSM: each rank holds a shard of the terms; the sum over ranks must equal the oracle's MSM of all terms
n_all = 3000
rng = np.random.default_rng(99)
bases_all = np.ascontiguousarray(ol.generators(9002)[:n_all])
sc_all = ol.rand_fr(rng, n_all)
lo, hi = n_all * rank // world, n_all * (rank + 1) // world
got = lb.msm(ctx, np.ascontiguousarray(bases_all[lo:hi]), np.ascontiguousarray(sc_all[lo:hi]))
if rank == 0:
    ref = np.zeros(16, dtype=np.uint64)
    ol.lib().orc_msm(ol.P(bases_all), ol.P(sc_all), ol.sz(n_all), 1, ol.P(ref))
    same = ol.lib().orc_point_eq(ol.P(got), ol.P(ref)) == 1
    print("collective msm over %d ranks: %s" % (world, "OK" if same else "MISMATCH"), flush=True)
    ok = ok and same
dist.barrier()
dist.destroy_process_group()
if rank == 0:
    print("SHARDED_CHECK", "PASS" if ok else "FAIL")
    sys.exit(0 if ok else 1)
