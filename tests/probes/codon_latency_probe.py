"""Dev probe: wall time per evaluation of a small codon workload (replicase-sized: 61 states, 239
patterns, 8 chains) -- the grid is far below one CTA per SM, i.e. the regime of the tensor-core kernel."""
import sys, time
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import numpy as np
from mrbayes_b200 import abi, workloads
lib = abi.engine_library()
pr = workloads.make_problem(61, 1, 239, 9, 8, seed=11)
inst = pr.create(lib, max_evaluations=8)
rng = np.random.default_rng(5)
inst.evaluate([pr.full_evaluation(ch) for ch in range(8)])
specs = [[pr.random_branch_update(ch, rng) for ch in range(8)] for _ in range(64)]
for rep in range(3):
    t0 = time.perf_counter()
    for s in specs:
        inst.evaluate(s)
    dt = time.perf_counter() - t0
    print(f"rep {rep}: {dt/len(specs)*1e6:.1f} us per 8-chain generation")
full = [pr.full_evaluation(ch) for ch in range(8)]
t0 = time.perf_counter()
for _ in range(50): inst.evaluate(full)
print(f"full-tree evaluation of 8 chains: {(time.perf_counter()-t0)/50*1e6:.1f} us")
inst.close()
