"""The bind kernel's launch shape: resident CTAs per SM the grid is sized for (each in its own process: the knob is
read once).  usage: python tools/bind_sweep.py"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
code = ("import sys; sys.path.insert(0, %r); import lasso_b200 as lb; c = lb.Context(0); "
        "ms = min(c.bench_bind(1 << 22, 5, 20) for _ in range(3)); "
        "print('%%.4f ms  %%.1f GB/s' %% (ms, 96.0 * (1 << 21) * 5 / ms / 1e6))") % ROOT
for bps in (4, 5, 6):
    env = dict(os.environ, LASSO_B200_BIND_BLOCKS=str(bps))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env)
    print("blocks/SM=%d: %s" % (bps, out.stdout.strip() or out.stderr[-300:]), flush=True)
