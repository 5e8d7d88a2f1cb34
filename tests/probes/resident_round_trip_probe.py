"""Dev probe: the per-generation round trip of the resident 4-state kernel against the launch path, for three
batch shapes of the primates workload (8 chains, L2 warm):

    bench     the bench's 128-generation proposal cycle (about 5 dirty nodes per evaluation)
    one_node  8 evaluations that rebuild only the interior root (branch_update of root_left): the fixed
              cost of a generation -- job pickup, staging, one node, root, packet
    full      8 full evaluations (every node of every chain)

    python tests/probes/resident_round_trip_probe.py [--reps N] [--gens N]

Resident: mb200_host_mc3_loop in mode 1 (mb200_replay_begin / _end, as bench.py's value leg), device time per
generation from the loop's events.  Launch: mb200_host_replay_loop (one mb200_replay per generation, results
in device memory), event time per generation.  The shapes and paths alternate within each repetition.
Prints one JSON line: median, min and max over the repetitions, with the card's name and power limit."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--gens", type=int, default=512, help="generations per timed run")
    args = ap.parse_args()
    import bench
    from mrbayes_b200 import abi, mc3

    lib = abi.engine_library()
    hl = bench.load_host_loop()
    hl.mb200_host_replay_loop.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int),
                                          C.c_int, C.c_void_p, C.c_size_t]
    job = bench.Job("primates", 0, 1, lib, 0, 128)
    mc = mc3.Coordinator(rank=0, world=1, device=0, num_runs=job.runs, chains_per_run=job.chains, num_swaps=1,
                         chain_temp=0.1, swap_seed=12345)
    job.prepare(mc)
    inst, pr, nl = job.insts[0], job.parts[0], job.n_local

    def batch(make):
        """pack one evaluation per chain, then undo their index flips: the batch writes only slots the cycle's
        start state does not read, so it can run between whole cycles"""
        specs = [make(ch) for ch in range(nl)]
        b = inst.pack(specs)
        for ch, sp in enumerate(specs):
            pr.reject(ch, sp)
        return b

    one_node = batch(lambda ch: pr.branch_update(ch, pr.tree[ch].root_left, float(pr.tree[ch].length[pr.tree[ch].root_left])))
    full = batch(pr.full_evaluation)
    handle = (C.c_int * 1)(inst.handle)

    def shape(batches):
        """-> (batch handles, cycle length, generation order) of a shape"""
        n = len(batches)
        return (C.c_int * n)(*batches), n, [g % n for g in range(args.gens)]

    shapes = {"bench": shape(job.batches[0]), "one_node": shape([one_node]), "full": shape([full])}

    def resident(name):
        cb, n, order = shapes[name]
        acc = np.zeros((n, nl), np.uint8)
        lnpr = np.zeros((n, nl))
        cur_lnl, cur_lnpr, sums, nacc = job.cur_lnl.copy(), job.cur_lnpr.copy(), (C.c_double * 2)(), C.c_longlong(0)
        rc = hl.mb200_host_mc3_loop(mc.handle, handle, 1, nl, 1, job.c_steps, cb, n,
                                    acc.ctypes.data_as(C.POINTER(C.c_ubyte)), lnpr.ctypes.data_as(C.POINTER(C.c_double)),
                                    (C.c_int * len(order))(*order), len(order), 1,
                                    cur_lnl.ctypes.data_as(C.POINTER(C.c_double)),
                                    cur_lnpr.ctypes.data_as(C.POINTER(C.c_double)), sums, C.byref(nacc))
        if rc != 0:
            raise RuntimeError(f"mb200_host_mc3_loop failed with code {rc}")
        return sums[1] * 1e3 / len(order)

    def launched(name):
        cb, n, order = shapes[name]
        ms = hl.mb200_host_replay_loop(handle, 1, cb, n, (C.c_int * len(order))(*order), len(order), None, 0)
        if ms < 0:
            raise RuntimeError(f"mb200_host_replay_loop failed with code {ms}")
        return ms * 1e3 / len(order)

    paths = {"resident": resident, "launch": launched}
    for name in shapes:                                   # warm-up: every shape on both paths
        for fn in paths.values():
            fn(name)
    got = {(p, s): [] for p in paths for s in shapes}
    for rep in range(args.reps):
        for s in (shapes if rep % 2 == 0 else reversed(list(shapes))):
            for p in (paths if rep % 2 == 0 else reversed(list(paths))):
                got[(p, s)].append(paths[p](s))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": smi, "reps": args.reps, "generations_per_run": args.gens, "us_per_generation": {}}
    for (p, s), v in got.items():
        out["us_per_generation"][f"{p}.{s}"] = {"median": float(np.median(v)), "min": float(np.min(v)),
                                               "max": float(np.max(v)), "runs": [round(x, 3) for x in v]}
    print(json.dumps(out), flush=True)
    job.close()
    mc.close()


if __name__ == "__main__":
    main()
