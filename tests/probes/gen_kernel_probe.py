"""GPU probe (not a test): whole-evaluation time of the generic-state kernel (doublet / covarion / protein covarion sizes).
usage: python tests/probes/gen_kernel_probe.py"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
from mrbayes_b200 import abi, workloads  # noqa: E402

lib = abi.engine_library()
for S, K, C, tips, nch in [(8, 4, 413, 12, 1), (8, 4, 413, 12, 8), (16, 1, 78, 27, 4), (40, 4, 88, 89, 2), (16, 4, 5000, 32, 1), (40, 4, 5000, 32, 1)]:
    pr = workloads.make_problem(S, K, C, tips, nch, seed=11)
    with pr.create(lib) as inst:
        inst.evaluate([pr.full_evaluation(c) for c in range(nch)])
        batch = inst.pack([pr.full_evaluation(c) for c in range(nch)])
        stream = torch.cuda.ExternalStream(inst.stream())
        for _ in range(3):
            inst.replay(batch)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(20):
            inst.replay(batch)
        b.record(stream)
        inst.synchronize()
        ms = a.elapsed_time(b) / 20
        upd = pr.n_int * pr.C * pr.K * nch
        print(json.dumps({"S": S, "K": K, "C": C, "taxa": tips, "chains": nch, "ms_per_full_evaluation": round(ms, 4),
                          "updates_per_s": upd / (ms * 1e-3), "us_per_node": 1e3 * ms / pr.n_int}), flush=True)
