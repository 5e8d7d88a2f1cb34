"""Probe (not a test): device time of the eigensolver per call.  usage: python tests/probes/eigen_probe.py"""
import sys
import time
from pathlib import Path
import numpy as np
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))         # the repository: mrbayes_b200
sys.path.insert(0, str(HERE.parent))             # tests/: test_gpu_eigen
from mrbayes_b200 import abi
from test_gpu_eigen import reversible_q, make

lib = abi.engine_library()
for S, K, parts in [(4, 4, 1), (20, 4, 1), (61, 1, 1), (61, 3, 3), (64, 1, 1)]:
    rng = np.random.default_rng(S)
    Q, pi = reversible_q(rng, S, sparse=(S > 20))
    Qs = np.stack([Q * (1 + 0.3 * p) for p in range(parts)])
    with make(lib, S, K, parts) as dev:
        for _ in range(5):
            dev.set_rate_matrices(0, Qs, pi)
        dev._call("synchronize")
        n = 50
        t0 = time.perf_counter()
        for i in range(n):
            dev.set_rate_matrices(i % 3, Qs, pi)
        t1 = time.perf_counter()
        dev._call("synchronize")
        t2 = time.perf_counter()
        print(f"S={S} parts={parts}: host enqueue {1e6*(t1-t0)/n:.1f} us/call, device {1e6*(t2-t0)/n:.1f} us/call (back to back)")

# warm-started chain (what a run does): small changes, like = the other slot
for S, K, parts in [(61, 1, 1), (61, 3, 3), (20, 4, 1)]:
    rng = np.random.default_rng(S)
    Q, pi = reversible_q(rng, S, sparse=(S > 20))
    with make(lib, S, K, parts) as dev:
        dev.set_rate_matrices(0, np.stack([Q] * parts), pi)
        n = 60
        Qs = []
        for i in range(n):
            f = 1.0 + 0.1 * (rng.random() - 0.5)
            p2 = pi * np.exp(0.05 * (rng.random(S) - 0.5)); p2 /= p2.sum()
            R = Q / pi[None, :]; np.fill_diagonal(R, 0.0)
            Qn = R * p2[None, :] * f; np.fill_diagonal(Qn, -Qn.sum(1))
            Qs.append((np.stack([Qn] * parts), p2))
        dev._call("synchronize")
        t0 = time.perf_counter()
        for i, (q, p2) in enumerate(Qs):
            dev.set_rate_matrices((i + 1) % 2, q, p2, like=i % 2)
        dev._call("synchronize")
        t2 = time.perf_counter()
        print(f"warm chain S={S} parts={parts}: device {1e6*(t2-t0)/n:.1f} us/call")
