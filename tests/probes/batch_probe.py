"""Dev probe: ONE instance holding many chains of a primates-sized problem (4 states, 4 rate categories,
413 patterns, 12 tips), a generation of all of them in ONE launch.  usage: python tests/probes/batch_probe.py"""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import numpy as np, torch
from mrbayes_b200 import abi, workloads
lib = abi.engine_library()
for nch in (8, 64, 128, 256):
    pr = workloads.make_problem(4, 4, 413, 12, nch, seed=11)
    inst = pr.create(lib, max_evaluations=nch)
    inst.evaluate([pr.full_evaluation(ch) for ch in range(nch)])
    rng = np.random.default_rng(5)
    steps = [[pr.random_branch_update(ch, rng) for ch in range(nch)] for _ in range(16)]
    batches = [inst.pack(s) for s in steps]
    stream = torch.cuda.ExternalStream(inst.stream())
    upd = sum(len(e.ops) for s in steps for e in s) * pr.C * pr.K
    for rep in range(3):
        for b in batches: inst.replay(b)
    inst.synchronize()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for rep in range(20):
        for b in batches: inst.replay(b)
    e.record(stream); inst.synchronize()
    ms = a.elapsed_time(e) / (20 * len(batches))
    print(f"{nch:4d} chains in one launch: {ms*1e3:7.1f} us/step, {upd/len(batches)/(ms*1e-3):.3e} upd/s (warm L2)")
    inst.close()
