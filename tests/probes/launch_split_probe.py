"""Dev probe: where a generation of the flagship workload goes -- the warm duration of the fused kernel
(event-timed replays of the bench's 128 batches, L2 not flushed, one launch each) against the
per-generation time of mb200_replay_begin / _end driven by the C generation loop.

    python tests/probes/launch_split_probe.py [--reps N]

Prints one JSON line.  The time outside the kernel is the per-generation time minus the warm kernel time."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    import bench
    from mrbayes_b200 import abi, mc3

    lib = abi.engine_library()
    hl = bench.load_host_loop()
    job = bench.Job("primates", 0, 1, lib, 0, 128)
    mc = mc3.Coordinator(rank=0, world=1, device=0, num_runs=job.runs, chains_per_run=job.chains, num_swaps=1,
                         chain_temp=0.1, swap_seed=12345)
    job.prepare(mc)
    inst = job.insts[0]
    order = list(range(128))
    # warm kernel: one launch per batch, events around each launch, nothing flushed
    inst.set_kernel_timing(True)
    for i in order:
        inst.replay(job.batches[0][i])
    inst.kernel_time()
    for _ in range(args.reps):
        for i in order:
            inst.replay(job.batches[0][i])
    ms, n = inst.kernel_time()
    inst.set_kernel_timing(False)
    kernel_us = ms * 1e3 / n
    # the same generations through replay_begin / _end with accept and swap steps (the bench's value leg, no flush)
    job.run(hl, 1, order)
    launches0 = inst.launch_count()
    wall, dev_ms, _ = job.run(hl, 1, order * args.reps)
    gens = 128 * args.reps
    gen_us = dev_ms * 1e3 / gens
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi, "warm_kernel_us": kernel_us, "kernels_timed": n, "us_per_generation": gen_us,
                      "wall_us_per_generation": wall * 1e6 / gens, "outside_kernel_us": gen_us - kernel_us,
                      "launches": inst.launch_count() - launches0, "generations": gens}), flush=True)
    job.close()
    mc.close()


if __name__ == "__main__":
    main()
