"""GPU: the generation loops bench.py times, and what it reads back from them.

  replay_begin / _end   on every kernel family (tensor core, generic, variable-state, 4-state with the ticketed device
                        sum, 4-state throughput mode), batches with and without a root: against the oracle fed the same
                        calls, bit for bit against a twin instance driven by evaluate(), the last generation against
                        the float64 reference; a bench.Job cycle replayed twice gives the same generations twice
  mb200_host_mc3_loop   modes 1 (packed batches, replay_begin / _end) and 0 (host structs, evaluate_begin / _end) on
                        every bench workload, bit for bit against bench.python_mc3_loop on an evaluate() twin: current
                        lnL and lnPrior, swaps, the coordinator's decisions and the arrays bench.dump_outputs writes
  mb200_host_generation_loop / mb200_host_replay_loop
                        every generation's lnL against the twin; 32 replicas from 1, 3 and 8 host threads
  kernel timing         mb200_set_kernel_timing / mb200_get_kernel_time: results unchanged on every family and route,
                        one timed launch per evaluation kernel, the read-out clears, the 2048-entry ring, a timed
                        instance keeps its launches instead of the resident kernel

The resident 4-state kernel serves an instance only while it is the only live engine instance on the device, so where
residency matters the twin runs before the instance under test is created, or after it is closed."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402
from engine_checks import (check_with_oracle, edge, generation_sequence, lnl_tol, nuc4_problem, ppb,  # noqa: E402
                           proposal_cycle, rel, tree_tol, via_evaluate, via_replay, via_replay_begin, written_buffers)
from f64_reference import f64_lnl, f64_std_lnl, is_variable_states  # noqa: E402
from mrbayes_b200 import abi, mc3, workloads  # noqa: E402
from std_problems import make_std_division  # noqa: E402

pytestmark = pytest.mark.gpu

KINDS = {"nuc4": abi.KERNEL_NUC4, "tensor": abi.KERNEL_TENSOR, "generic": abi.KERNEL_GENERIC, "std": abi.KERNEL_STD}


def family_of(pr):
    if is_variable_states(pr):
        return "std"
    if pr.S == 4:
        return "nuc4"
    return "tensor" if (pr.S == 20 and pr.K <= 4) or (pr.S == 61 and pr.K <= 3) else "generic"


def counters(e):
    return {f: e.kernel_launches(k) for f, k in KINDS.items()}


def final_state(e, gens):
    """every partials buffer and scaler the generations write, read back from e"""
    dests, scalers = written_buffers(gens)
    return [e.get_partials(b) for b in dests] + [e.get_scalers(s) for s in scalers]


def assert_same_state(a, b, what):
    assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b)), f"{what}: final buffers differ"


def f64_check(pr, specs, lnl, tol):
    """each evaluation of specs that reaches the root against the float64 reference of its chain as it stands now"""
    for sp, le in zip(specs, lnl):
        if sp.root < 0:
            continue
        if is_variable_states(pr):
            ref = f64_std_lnl(pr, sp.chain, rates=pr.chain_rates[sp.chain])
            assert not ref.underflow and abs(le - ref.lnl) <= ref.bound(pr), f"chain {sp.chain}: {le!r} vs {ref.lnl!r}"
        else:
            r = rel(le, f64_lnl(pr, sp.chain)[1])
            assert r < tol, f"float64 reference, chain {sp.chain}: {r:.2e}"


# ---- 1. replay_begin / _end on every family ----------------------------------------------------------------------
def std_case(seed):
    return make_std_division(150, 4, 20, 4, seed=seed, states=(2, 3, 4, 5, 7), p_poly=0.05)


REPLAY_CASES = {
    # tensor core, one pattern past a 128-row tile
    "tensor-20-1": lambda: workloads.make_problem(20, 1, 129, 24, 4, seed=101),
    "tensor-20-4": lambda: workloads.make_problem(20, 4, 129, 24, 4, seed=102, p_invar=0.1),
    "tensor-61-1": lambda: workloads.make_problem(61, 1, 129, 24, 4, seed=103),
    "tensor-61-3": lambda: workloads.make_problem(61, 3, 129, 24, 4, seed=104),
    # generic kernel: all rate categories per pass while K S (S + 1) floats fit 48 KB, else one per pass (16 states fit
    # at every category count the engine takes, up to 20)
    "generic-16-4-all": lambda: workloads.make_problem(16, 4, 150, 16, 4, seed=105),
    "generic-16-20-all": lambda: workloads.make_problem(16, 20, 90, 16, 4, seed=106),
    "generic-40-3-all": lambda: workloads.make_problem(40, 3, 150, 16, 4, seed=107, p_ambig=0.1),
    "generic-40-8-one": lambda: workloads.make_problem(40, 8, 90, 16, 4, seed=108),
    "generic-64-2-all": lambda: workloads.make_problem(64, 2, 150, 16, 4, seed=109, p_invar=0.1),
    "generic-64-3-one": lambda: workloads.make_problem(64, 3, 90, 16, 4, seed=110),
    # variable states: five state-count classes, polymorphic tips, the two constant dummy patterns
    "std": lambda: std_case(111),
    # 4 states past MB200_SEQ_SUM_TILES (16) tiles: the last CTA sums the tile partials on the device
    "nuc4-device-sum-1": lambda: nuc4_problem(1, edge(1, 20), seed=5),
    "nuc4-device-sum-4": lambda: nuc4_problem(4, edge(4, 20), seed=5),
    "nuc4-device-sum-8": lambda: nuc4_problem(8, edge(8, 20), seed=5),
    # throughput mode: one CTA per evaluation walks every tile
    "nuc4-throughput": lambda: workloads.make_problem(4, 4, edge(4, 5), 12, 4, seed=112, p_invar=0.1, p_ambig=0.05),
}


def replay_sequence(pr, seed, rootless=3, gens=6):
    """generation_sequence's run (rejections included), generation `rootless` a batch whose chain 0 does not reach the
    root (no lnL: the engine collects such a batch after a stream synchronisation, not from the result polls)"""
    seq = []
    for g, specs in generation_sequence(pr, gens, seed):
        if g == rootless:
            specs[0].root = abi.NONE
        seq.append(specs)
    return seq


@pytest.mark.parametrize("name", sorted(REPLAY_CASES))
def test_replay_begin_end_every_family(engine_lib, oracle_lib, record_property, name):
    pr = REPLAY_CASES[name]()
    flags = abi.CONFIG_THROUGHPUT if name == "nuc4-throughput" else 0
    fam = family_of(pr)
    assert name.startswith(fam)
    seq = replay_sequence(pr, seed=len(name))
    tol = lnl_tol(pr.S)
    worst = 0.0
    # the instance under test alone on the device
    with pr.create(engine_lib, flags=flags) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        batches = [e.pack(specs) for specs in seq]
        n0 = counters(e)
        got = []
        for specs, b in zip(seq, batches):
            e.replay_begin(b)
            lnl, st = e.replay_end()
            worst = max(worst, check_with_oracle(e, o, specs, lnl, st, tol, tree_tol(pr))[0])
            got.append((lnl, st))
        launched = {f: n - n0[f] for f, n in counters(e).items()}
        got_state = final_state(e, seq)
        for b in batches:
            e.free_batch(b)
    f64_check(pr, seq[-1], got[-1][0], tol)
    assert got[3][0][0] == 0.0 and got[3][1][0] == abi.EVAL_OK
    # one launch of the family's kernel per generation: no resident kernel, no other family
    assert launched == {f: (len(seq) if f == fam else 0) for f in KINDS}, launched
    # a twin driven by evaluate()
    with pr.create(engine_lib, flags=flags) as t:
        want = [t.evaluate(specs) for specs in seq]
        want_state = final_state(t, seq)
    for g, ((lg, sg), (lw, sw)) in enumerate(zip(got, want)):
        assert np.array_equal(lg, lw) and np.array_equal(sg, sw), f"generation {g}: {lg} vs evaluate() {lw}"
    assert_same_state(got_state, want_state, "replay_begin / _end vs evaluate()")
    record_property("max_rel_lnl_vs_oracle", worst)
    print(f"\nLNL_VS_ORACLE replay_begin {name} {worst:.3e}")


def shrink(monkeypatch):
    """bench's synthetic workloads at oracle size: one pattern past a tensor-core tile, 4 states past 16 tiles"""
    monkeypatch.setitem(bench.SYNTH, "aa50k", (20, 4, 129, 64))
    monkeypatch.setitem(bench.SYNTH, "codon20k", (61, 1, 129, 32))
    monkeypatch.setitem(bench.SYNTH, "nuc200k", (4, 4, 17 * ppb(4) + 1, 32))


@pytest.fixture
def shrunk(monkeypatch):
    shrink(monkeypatch)


def cycle_of(name):
    return 128 if name in ("primates", "cynmix") else 16


def replay_job_cycle(job):
    """one pass over job's cycle: per generation replay_begin on every partition, then replay_end on every partition
    -> [generation][partition] (lnL, status)"""
    batches = [[inst.pack(job.steps[p][i]) for i in range(job.cycle_len)] for p, inst in enumerate(job.insts)]
    out = []
    for i in range(job.cycle_len):
        for p, inst in enumerate(job.insts):
            inst.replay_begin(batches[p][i])
        out.append([inst.replay_end() for inst in job.insts])
    for p, inst in enumerate(job.insts):
        for b in batches[p]:
            inst.free_batch(b)
    return out


@pytest.mark.parametrize("name", ["aa50k", "codon20k", "cynmix"])
def test_job_cycle_replayed_twice(engine_lib, shrunk, name):
    """The closing step of a bench cycle returns every chain to its start state: a second pass over the cycle gives,
    bit for bit, the generations of the first, and the closing step the initial full evaluations"""
    job = bench.Job(name, 0, 1, engine_lib, 0, cycle_of(name))
    try:
        kinds0 = [counters(i) for i in job.insts]
        first, second = replay_job_cycle(job), replay_job_cycle(job)
        kinds = [{f: n - k0[f] for f, n in counters(i).items()} for i, k0 in zip(job.insts, kinds0)]
    finally:
        job.close()
    for g, (a, b) in enumerate(zip(first, second)):
        for p, ((la, sa), (lb, sb)) in enumerate(zip(a, b)):
            assert not sa.any() and np.array_equal(la, lb) and np.array_equal(sa, sb), f"generation {g}, partition {p}"
    assert np.array_equal(sum(l for l, _ in first[-1]), job.lnl0)
    for pr, k in zip(job.parts, kinds):
        assert k == {f: (2 * job.cycle_len if f == family_of(pr) else 0) for f in KINDS}, k


# ---- 2. the C loops against independent restatements ---------------------------------------------------------------
@pytest.fixture(scope="module")
def hl(engine_lib):
    return bench.load_host_loop()


def coordinator(job):
    """the coordinator bench.py gives the workload at world 1"""
    return mc3.Coordinator(rank=0, world=1, device=0, num_runs=job.runs, chains_per_run=job.chains,
                           num_swaps=job.w["swaps"], chain_temp=0.1, swap_seed=12345)


def bench_orders(name, n_steps=2):
    """bench.py's run_steps: n_steps steps of the workload's G generations, then the run back to the cycle start"""
    G, cyc = bench.WORKLOADS[name]["gens"], cycle_of(name)
    orders, g0 = [], 0
    for _ in range(n_steps):
        orders.append([(g0 + g) % cyc for g in range(G)])
        g0 = (g0 + G) % cyc
    if g0:
        orders.append([(g0 + g) % cyc for g in range(cyc - g0)])
    return orders


class CountingSwaps:
    """a coordinator that counts the swaps python_mc3_loop's attempts accept"""

    def __init__(self, mc):
        self.mc, self.accepted = mc, 0

    def exchange_begin(self, lnl, lnpr):
        self.mc.exchange_begin(lnl, lnpr)

    def exchange_end(self):
        self.mc.exchange_end()

    def attempt_swaps(self):
        n = self.mc.attempt_swaps()
        self.accepted += n
        return n


def dumped(job, out):
    """bench.dump_outputs of job's current state (per-run lnL sums reduced as bench_engine does) -> {file: array}"""
    run_sums = np.zeros(job.runs)
    for c, g in enumerate(job.globals):
        run_sums[g // job.chains] += job.cur_lnl[c]
    bench.dump_outputs(out, job, job.mc.reduce_sum(run_sums, 0), 0, 1)
    return {p.name: np.load(p) for p in sorted(out.glob("*.npy"))}


def outcome(job, accepted, out):
    return dict(lnl=job.cur_lnl.copy(), lnpr=job.cur_lnpr.copy(), accepted=accepted, hash=job.mc.decision_hash(),
                swap_info=job.mc.swap_info(), dump=dumped(job, out))


def assert_same_outcome(a, b, what):
    assert np.array_equal(a["lnl"], b["lnl"]), f"{what}: lnL {a['lnl']} vs {b['lnl']}"
    assert np.array_equal(a["lnpr"], b["lnpr"]), f"{what}: lnPrior"
    assert a["accepted"] == b["accepted"], f"{what}: swaps accepted {a['accepted']} vs {b['accepted']}"
    assert a["hash"] == b["hash"] and np.array_equal(a["swap_info"], b["swap_info"]), f"{what}: swap decisions"
    assert a["dump"].keys() == b["dump"].keys()
    for k in a["dump"]:
        assert np.array_equal(a["dump"][k], b["dump"][k]), f"{what}: {k}"


def restart(job, mc):
    """job back at its start state (its instances are, at the cycle start), driven by coordinator mc"""
    job.mc, job.cur_lnl, job.cur_lnpr = mc, job.lnl0.copy(), job.lnpr0.copy()


def accepted_prior(job, n_generations):
    lnpr = job.lnpr0.copy()
    for g in range(n_generations):
        i = g % job.cycle_len
        lnpr = np.where(job.accept[i].astype(bool), job.lnprior[i], lnpr)
    return lnpr


ORACLE_GENERATIONS = 24
MC3_CASES = [(n, False) for n in bench.WORKLOADS] + [(n, True) for n in bench.SYNTH]


@pytest.mark.parametrize("name,full", MC3_CASES, ids=[n + ("-full" if f else "") for n, f in MC3_CASES])
def test_mc3_loop(engine_lib, oracle_lib, hl, monkeypatch, tmp_path, record_property, name, full):
    """mb200_host_mc3_loop in modes 1 and 0 with bench's cycle and step pattern, against bench.python_mc3_loop on a
    twin Job driven by evaluate(); on oracle-sized shapes the first generations also against the oracle"""
    if not full:
        shrink(monkeypatch)
    orders = bench_orders(name)
    T = sum(len(o) for o in orders)
    cyc = cycle_of(name)
    assert T % cyc == 0
    runs = {}
    job = bench.Job(name, 0, 1, engine_lib, 0, cyc)          # alone on the device
    try:
        job.prepare(None)
        for mode in (1, 0):
            with coordinator(job) as mc:
                restart(job, mc)
                n0 = [counters(i) for i in job.insts]
                accepted = sum(job.run(hl, mode, order)[2] for order in orders)
                launched = [{f: n - k0[f] for f, n in counters(i).items()} for i, k0 in zip(job.insts, n0)]
                runs[mode] = outcome(job, accepted, tmp_path / f"mode{mode}")
            fams = [family_of(pr) for pr in job.parts]
            for f, k in zip(fams, launched):
                assert all(k[g] == 0 for g in KINDS if g != f), k
                if mode == 1 and name.startswith("primates"):
                    assert 1 <= k["nuc4"] <= T // 16, f"mode 1: {k['nuc4']} launches for {T} generations, not resident"
                else:
                    assert k[f] == T, f"mode {mode}: {k[f]} launches for {T} generations"
        if not full and name != "primates-sharded":
            # the first generations again from the start state, to hold against the oracle
            with coordinator(job) as mc:
                restart(job, mc)
                job.run(hl, 1, [g % cyc for g in range(ORACLE_GENERATIONS)])
                short = job.cur_lnl.copy()
    finally:
        job.close()
    assert_same_outcome(runs[1], runs[0], "mode 1 vs mode 0")
    # the twin, after the job is closed
    twin = bench.Job(name, 0, 1, engine_lib, 0, cyc)
    try:
        assert np.array_equal(twin.lnl0, job.lnl0)
        with coordinator(twin) as mc:
            counting = CountingSwaps(mc)
            twin.mc = mc
            twin.cur_lnl = bench.python_mc3_loop(twin, counting, T)
            twin.cur_lnpr = accepted_prior(twin, T)
            want = outcome(twin, counting.accepted, tmp_path / "python")
    finally:
        twin.close()
    assert_same_outcome(runs[1], want, "mb200_host_mc3_loop vs python_mc3_loop")
    if full or name == "primates-sharded":
        return
    oj = bench.Job(name, 0, 1, oracle_lib, 0, cyc)
    try:
        for i in oj.insts:
            i.set_arith(1)
        with mc3.Coordinator(num_runs=oj.runs, chains_per_run=oj.chains, num_swaps=oj.w["swaps"],
                             backend=mc3.LOOPBACK) as mc:
            ref = bench.python_mc3_loop(oj, mc, ORACLE_GENERATIONS)
    finally:
        oj.close()
    tol = max(lnl_tol(pr.S) for pr in oj.parts)
    worst = max(rel(a, b) for a, b in zip(short, ref))
    assert worst < tol, f"oracle: {worst:.2e}"
    record_property("max_rel_lnl_vs_oracle", worst)
    print(f"\nLNL_VS_ORACLE mc3 {name} {worst:.3e}")


def generation_loop(hl, ids, arrays, cycle, count, order, lnl, st, threads):
    R = len(ids)
    sec = hl.mb200_host_generation_loop((C.c_int * R)(*ids), C.c_int(R), arrays, C.c_int(cycle), C.c_int(count),
                                        (C.c_int * len(order))(*order), C.c_int(len(order)),
                                        lnl.ctypes.data_as(C.POINTER(C.c_double)), st.ctypes.data_as(C.POINTER(C.c_int)),
                                        C.c_int(threads))
    assert sec >= 0.0, f"mb200_host_generation_loop returned {sec}"


def step_pointers(arrays):
    """[replica][cycle step] host evaluation arrays -> the steps table of the host loops (replica-major)"""
    flat = [a for arr in arrays for a in arr]
    return (C.c_void_p * len(flat))(*[C.cast(a, C.c_void_p) for a in flat])


@pytest.mark.parametrize("name", ["primates", "cynmix", "aa50k", "codon20k", "nuc200k"])
def test_loops_every_generation(engine_lib, hl, shrunk, name):
    """mb200_host_generation_loop and mb200_host_replay_loop one generation per call, the partitions as replicas:
    every generation's lnL and status bit for bit what evaluate() gives on a twin"""
    cyc = cycle_of(name)
    twin = bench.Job(name, 0, 1, engine_lib, 0, cyc)
    try:
        want = [[inst.evaluate(twin.steps[p][i]) for p, inst in enumerate(twin.insts)] for i in range(cyc)]
    finally:
        twin.close()
    job = bench.Job(name, 0, 1, engine_lib, 0, cyc)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    try:
        job.prepare(None)
        nP, n = len(job.parts), job.n_local
        ids = [i.handle for i in job.insts]
        steps = step_pointers(job.host_arrays)
        for i in range(cyc):
            lnl, st = np.full(nP * n, np.nan), np.full(nP * n, -1, np.int32)
            generation_loop(hl, ids, steps, cyc, n, [i], lnl, st, threads=1)
            for p in range(nP):
                lw, sw = want[i][p]
                assert np.array_equal(lnl[p * n:(p + 1) * n], lw) and np.array_equal(st[p * n:(p + 1) * n], sw), \
                    f"generation loop, step {i}, partition {p}"
        for i in range(cyc):
            ms = hl.mb200_host_replay_loop((C.c_int * nP)(*ids), C.c_int(nP), job.c_batches, C.c_int(cyc),
                                           (C.c_int * 1)(i), C.c_int(1), C.c_void_p(flush.data_ptr()),
                                           C.c_size_t(flush.numel()))
            assert ms >= 0.0, f"mb200_host_replay_loop returned {ms}"
            for p, inst in enumerate(job.insts):
                lg, sg = inst.replay_results(job.batches[p][i], n)
                lw, sw = want[i][p]
                assert np.array_equal(lg, lw) and np.array_equal(sg, sw), f"replay loop, step {i}, partition {p}"
    finally:
        job.close()
        del flush


def threaded_last(hl, ids, steps, cycle, count, threads, k):
    """one pass over the cycle and k generations more through mb200_host_generation_loop from `threads` host threads,
    then the run back to the cycle start -> (lnL, status) of generation k - 1 of the second pass [replica * count]"""
    R = len(ids)
    lnl, st = np.full(R * count, np.nan), np.full(R * count, -1, np.int32)
    generation_loop(hl, ids, steps, cycle, count, list(range(cycle)) + list(range(k)), lnl, st, threads)
    out = lnl.copy(), st.copy()
    lnl[:] = np.nan
    generation_loop(hl, ids, steps, cycle, count, list(range(k, cycle)), lnl, st, threads)
    assert np.isfinite(lnl).all() and not st.any()
    return out


def assert_threads_agree(hl, ids, arrays, cycle, count, k):
    steps = step_pointers(arrays)
    runs = {t: threaded_last(hl, ids, steps, cycle, count, t, k) for t in (1, 3, 8)}
    lnl, st = runs[1]
    assert np.isfinite(lnl).all() and (lnl < 0).all() and not st.any()
    for t, (l, s) in runs.items():
        assert np.array_equal(l, lnl) and np.array_equal(s, st), f"{t} host threads"
    for r, h in enumerate(ids):
        l, s = threaded_last(hl, [h], step_pointers([arrays[r]]), cycle, count, 1, k)
        assert np.array_equal(l, lnl[r * count:(r + 1) * count]) and not s.any(), f"replica {r} alone"


def test_generation_loop_threads_many_analyses(engine_lib, hl):
    """many_analyses' shape: 32 primates analyses with its seeds; 1, 3 and 8 host threads, and each one alone"""
    R, cyc = 32, 32
    jobs = [bench.Job("primates", 0, 1, engine_lib, 0, cyc, seed=20260924 + 1000 * (r + 1)) for r in range(R)]
    try:
        arrays = [[abi.make_eval_array(j.steps[0][i]) for i in range(cyc)] for j in jobs]
        assert_threads_agree(hl, [j.insts[0].handle for j in jobs], arrays, cyc, 8, k=19)
        assert all(j.insts[0].kernel_launches(abi.KERNEL_NUC4) > 0 for j in jobs)
    finally:
        for j in jobs:
            j.close()


def test_generation_loop_threads_mixed_families(engine_lib, hl):
    """a primates analysis, the cynmix morphology partition, a 20-state and a 40-state division, 8 evaluations per
    step each: every family from 1, 3 and 8 host threads, and each one alone"""
    cyc, n = 24, 8
    job = bench.Job("primates", 0, 1, engine_lib, 0, cyc)
    trees = [workloads.random_tree(32, np.random.default_rng([5, ch]), mean_len=0.08) for ch in range(n)]
    std = next(p for p in bench.cynmix_partitions(n, trees) if isinstance(p, workloads.StdProblem))
    probs = [std, workloads.make_problem(20, 2, 150, 16, n, seed=31), workloads.make_problem(40, 3, 90, 16, n, seed=32)]
    insts = [p.create(engine_lib) for p in probs]
    try:
        # the evaluation arrays point into the specs' operation and matrix arrays: the cycles stay referenced
        cycles = [job.steps[0]] + [proposal_cycle(p, inst, cyc, seed=p.S) for p, inst in zip(probs, insts)]
        arrays = [[abi.make_eval_array(s) for s in steps] for steps in cycles]
        allinst = [job.insts[0]] + insts
        assert_threads_agree(hl, [i.handle for i in allinst], arrays, cyc, n, k=13)
        for pr, inst in zip([job.parts[0]] + probs, allinst):
            k = counters(inst)
            assert k[family_of(pr)] > 0 and sum(k.values()) == k[family_of(pr)], k
        assert [family_of(p) for p in [job.parts[0]] + probs] == ["nuc4", "std", "tensor", "generic"]
    finally:
        for inst in insts:
            inst.close()
        job.close()


# ---- 3. kernel timing -----------------------------------------------------------------------------------------------
TIMING_CASES = {
    "nuc4": lambda: workloads.make_problem(4, 4, edge(4, 3), 12, 3, seed=201, p_invar=0.1),
    "nuc4-device-sum": lambda: nuc4_problem(4, edge(4, 20), seed=6),
    "tensor": lambda: workloads.make_problem(20, 2, 129, 12, 3, seed=202),
    "generic": lambda: workloads.make_problem(40, 3, 90, 12, 3, seed=203),
    "std": lambda: std_case(204),
}


@pytest.mark.parametrize("name", sorted(TIMING_CASES))
def test_kernel_timing_changes_no_result(engine_lib, name):
    """A timed instance and an untimed twin fed the same calls through evaluate, replay and replay_begin / _end:
    identical lnL, status and buffers.  Generation 0 is launched untimed and timing switched on before its results are
    collected; from then on every evaluation kernel is timed, once."""
    pr = TIMING_CASES[name]()
    fam = family_of(pr)
    seq = [specs for _, specs in generation_sequence(pr, 8, seed=7)]
    routes = [via_evaluate, via_replay, via_replay_begin]
    with pr.create(engine_lib) as t, pr.create(engine_lib) as u:
        b = t.pack(seq[0])
        t.replay_begin(b)
        t.set_kernel_timing(True)
        got = [t.replay_end()]
        t.free_batch(b)
        want = [via_evaluate(u, seq[0])]
        assert t.kernel_time() == (0.0, 0)
        k0 = t.kernel_launches(KINDS[fam])
        for g, specs in enumerate(seq[1:], 1):
            got.append(routes[g % 3](t, specs))
            want.append(routes[g % 3](u, specs))
        launched = t.kernel_launches(KINDS[fam]) - k0
        ms, n = t.kernel_time()
        assert n == launched == len(seq) - 1
        assert np.isfinite(ms) and ms > 0.0
        assert t.kernel_time() == (0.0, 0)
        for g, ((lg, sg), (lw, sw)) in enumerate(zip(got, want)):
            assert not sg.any() and np.array_equal(lg, lw) and np.array_equal(sg, sw), f"generation {g}"
        assert_same_state(final_state(t, seq), final_state(u, seq), "timed vs untimed")
        t.set_kernel_timing(False)
        via_replay(t, seq[-1])
        assert t.kernel_time() == (0.0, 0)


def test_kernel_time_ring(engine_lib):
    """more timed launches than the 2048-entry ring between two reads: at most 2048 are reported"""
    pr = workloads.make_problem(4, 1, 16, 4, 1, seed=9)
    with pr.create(engine_lib) as e:
        e.set_kernel_timing(True)
        b = e.pack([pr.full_evaluation(0)])
        for _ in range(2100):
            e.replay(b)
        ms, n = e.kernel_time()
        assert n == 2048 and np.isfinite(ms) and ms > 0.0
        assert e.kernel_time() == (0.0, 0)
        for _ in range(5):
            e.replay(b)
        assert e.kernel_time()[1] == 5


def test_kernel_timing_keeps_launches_of_a_resident_instance(engine_lib):
    """A 4-state instance alone on the device is served by the resident kernel; with timing on it keeps one launch per
    generation, including timing switched on between a resident replay_begin and its replay_end; switched off, the
    resident kernel serves it again.  Every generation bit for bit what evaluate() gives."""
    pr = workloads.make_problem(4, 4, edge(4, 6), 16, 2, seed=210)
    seq = [specs for _, specs in generation_sequence(pr, 30, seed=11)]
    with pr.create(engine_lib) as twin:
        want = [twin.evaluate(specs) for specs in seq]
        want_state = final_state(twin, seq)
    with pr.create(engine_lib) as e:
        batches = [e.pack(specs) for specs in seq]
        got = []

        def gens(lo, hi):
            n0 = e.kernel_launches(abi.KERNEL_NUC4)
            for g in range(lo, hi):
                e.replay_begin(batches[g])
                got.append(e.replay_end())
            return e.kernel_launches(abi.KERNEL_NUC4) - n0

        # resident: one kernel serves the generations (a host hiccup past its idle timeout costs a relaunch)
        assert 1 <= gens(0, 12) <= 6
        e.replay_begin(batches[12])
        e.set_kernel_timing(True)
        got.append(e.replay_end())
        assert gens(13, 22) == 9                                      # timed: one launch per generation
        ms, n = e.kernel_time()
        assert n == 9 and np.isfinite(ms) and ms > 0.0
        e.set_kernel_timing(False)
        assert 1 <= gens(22, len(seq)) <= 4                           # resident again
        got_state = final_state(e, seq)
    for g, ((lg, sg), (lw, sw)) in enumerate(zip(got, want)):
        assert not sg.any() and np.array_equal(lg, lw) and np.array_equal(sg, sw), f"generation {g}"
    assert_same_state(got_state, want_state, "resident and timed vs evaluate()")
