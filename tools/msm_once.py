"""One warm-up + one measured large MSM per size (a short command to put under a profiler)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import lasso_b200 as lb
import oracle_lib as ol

ctx = lb.Context(0)
pool = np.ascontiguousarray(ol.generators(8194)[:8192])
for log_n in [int(x) for x in sys.argv[1:]] or [18, 22]:
    n = 1 << log_n
    rng = np.random.default_rng(log_n)
    raw = rng.integers(0, 2**63, size=(n, 4), dtype=np.uint64)
    raw[:, 3] &= (1 << 59) - 1
    job = lb.MsmJob(ctx, pool, np.ascontiguousarray(raw))
    job.run(1)
    pt, ms, info = job.run(1)
    print("n=2^%d: %.3f ms %s" % (log_n, ms, info), flush=True)
    job.close()
