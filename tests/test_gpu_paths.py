"""GPU: every kernel variant the engine dispatches to, against the CPU oracle and the float64
pruning reference (tests/f64_reference.py).

The engine picks its kernel from the state count, the category count, the pattern count, the
number of evaluations in a call, the entry point and the size of the packed job.  Each test here
drives one route on purpose, shows that the route was taken (a kernel counter, or the kernel's
name from a CUDA activity trace) and compares every written buffer with the oracle:

  4-state, K = 1..8   fused from the parameter block (evaluate), fused from the device blob
                      (pack + replay, ticketed device sum over more than 16 tiles), non-fused
                      (stand-alone tiprobs_kernel), resident (replay_begin / _end), throughput mode
  tensor core         S = 20 (K = 1..4) and S = 61 (K = 1..3) around the 128-pattern tile
  generic kernel      one category per pass (K S (S+1) 4 B > 48 KB) or all, tiles of 4..32 patterns
  P(t) limits         t < TIME_MIN and t > TIME_MAX on the non-fused 4-state and the Std builders
  underflow           one dead pattern in a middle or the last tile, one dead evaluation of a batch

The threshold between the fused and the non-fused 4-state path scales with the device's SM count,
so the pattern counts here are computed from it."""
import numpy as np
import pytest
import torch

from f64_reference import caterpillar_tree, f64_lnl, tree_height
from mrbayes_b200 import abi, workloads
from test_gpu_parity import SYN_RTOL, TC_RTOL, _compare_state, rel

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def ppb(K):
    """patterns per 4-state tile: 256 threads / pow2ceil(K) lanes per pattern"""
    return 256 // (1 << (K - 1).bit_length())


def edge(K, tiles):
    """a pattern count at a tile edge: exactly `tiles` tiles, or one pattern less or more (rotating with K)"""
    return tiles * ppb(K) + (K % 3) - 1


def kernel_names(fn, expect):
    """names of the CUDA kernels fn() launches (CUDA activity trace, no hardware counters), for what the
    kernel counters cannot tell: the K and parameter-block size of a 4-state instantiation.  The trace
    can miss launches, so fn -- a full evaluation, which is idempotent -- is traced up to three times
    until a kernel whose name contains `expect` shows up."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if str(e.device_type).endswith("CUDA")}
        if launched(names, expect):
            break
    return names


def launched(names, prefix):
    return any(prefix in n for n in names)


# ---- routes: how a list of evaluations reaches the engine ---------------------------------
def via_evaluate(e, specs):
    return e.evaluate(specs)


def via_replay(e, specs):
    b = e.pack(specs)
    e.replay(b)
    out = e.replay_results(b, len(specs))
    e.free_batch(b)
    return out


def compare_state(e, o, spec, pr):
    """_compare_state of the parity suite.  On the tensor-core path the 3xTF32 rounding of each level
    (up to ~1e-6 relative) adds up from the tips to the node: on H100, S = 61 and K = 3, the partials
    of a node 20 to 38 levels up differ from the oracle's by 2e-5, the parity suite's bound for its
    trees of a few levels.  So the partials and the node scalers (the log of the node's largest
    unscaled partial) get 2e-5 plus 1e-6 per level of the tree."""
    if pr.S not in (20, 61):
        return _compare_state(e, o, spec, pr.S)
    tol = 2e-5 + 1e-6 * tree_height(pr.tree[spec.chain])
    for op in spec.ops:
        a, b = e.get_partials(int(op["dest"])), o.get_partials(int(op["dest"]))
        assert np.allclose(a, b, rtol=tol, atol=1e-37), f"partials of buffer {op['dest']}"
        if op["scale_write"] >= 0:
            d = np.abs(e.get_scalers(int(op["scale_write"])) - o.get_scalers(int(op["scale_write"]))).max()
            assert d < tol, f"node scaler {op['scale_write']}: {d:.2e}"
    if spec.site_dst >= 0:
        assert np.allclose(e.get_scalers(spec.site_dst), o.get_scalers(spec.site_dst), atol=2e-5 + tol)


def tol_of(S):
    return TC_RTOL if S in (20, 61) else SYN_RTOL


def check_run(pr, e, o, route, updates, seed, chains=(0, 1)):
    """A full evaluation per chain, then `updates` branch updates over the chains with a rejection
    every third: lnL, every written partials buffer and the node and site scalers against the oracle;
    lnL against the float64 reference after the full evaluations and after the last update."""
    tol = tol_of(pr.S)
    for ch in chains:
        sp = pr.full_evaluation(ch)
        (le,), (se,) = route(e, [sp])
        (lo,), (so,) = o.evaluate(sp)
        assert se == so == abi.EVAL_OK
        assert rel(le, lo) < tol, f"full evaluation of chain {ch}"
        compare_state(e, o, sp, pr)
        r = rel(le, f64_lnl(pr, ch)[1])
        assert r < tol, f"float64 reference, chain {ch}: {r:.2e}"
    rng = np.random.default_rng(seed)
    for it in range(updates):
        ch = chains[it % len(chains)]
        old = pr.tree[ch].length.copy()
        sp = pr.random_branch_update(ch, rng)
        (le,), (se,) = route(e, [sp])
        (lo,), _ = o.evaluate(sp)
        assert se == abi.EVAL_OK and rel(le, lo) < tol, f"update {it}"
        compare_state(e, o, sp, pr)
        if it == updates - 1:
            r = rel(le, f64_lnl(pr, ch)[1])
            assert r < tol, f"float64 reference after the updates: {r:.2e}"
        elif it % 3 == 2:
            pr.reject(ch, sp, old)


def nuc4_problem(K, C, n_chains=2, seed=0, tips=40):
    """4-state problem whose chain 1 is a caterpillar (one node per level: many chunks); odd K carry
    p_invar and partial ambiguity"""
    odd = K % 2 == 1
    pr = workloads.make_problem(4, K, C, tips, n_chains, seed=1000 + 17 * K + seed,
                                p_invar=0.15 if odd else 0.0, p_ambig=0.1 if odd else 0.0)
    pr.tree[1] = caterpillar_tree(tips, np.random.default_rng(K))
    return pr


# ---- B. 4-state path matrix -------------------------------------------------------------
@pytest.mark.parametrize("K", range(1, 9))
def test_nuc4_fused_parameter_block(engine_lib, oracle_lib, K):
    pr = nuc4_problem(K, edge(K, 3))
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        sp = pr.full_evaluation(0)
        want = f"eval_nuc4_pkernel<{K}, 256, "
        names = kernel_names(lambda: e.evaluate(sp), want)
        assert launched(names, want), names
        check_run(pr, e, o, via_evaluate, 12, seed=K)
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 0


@pytest.mark.parametrize("cap,K,tips,n_eval", [(4096, 2, 12, 1), (10240, 5, 100, 1), (30720, 7, 30, 8)])
def test_nuc4_parameter_block_sizes(engine_lib, oracle_lib, cap, K, tips, n_eval):
    """The job rides in the kernel's parameter block in three sizes; a full evaluation of 100 tips
    packs to ~8 KB, eight of 30 tips to ~20 KB."""
    pr = workloads.make_problem(4, K, edge(K, 2), tips, n_eval, seed=cap)
    rng = np.random.default_rng(cap)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        for gen in range(4):
            specs = [pr.full_evaluation(ch) if gen == 0 else pr.random_branch_update(ch, rng) for ch in range(n_eval)]
            if gen == 0:
                want = f"eval_nuc4_pkernel<{K}, 256, {cap}>"
                names = kernel_names(lambda: e.evaluate(specs), want)
                assert launched(names, want), names
            lnl, st = e.evaluate(specs)
            assert not st.any()
            for i, sp in enumerate(specs):
                (lo,), _ = o.evaluate(sp)
                assert rel(lnl[i], lo) < SYN_RTOL
                _compare_state(e, o, sp, 4)
        assert rel(lnl[-1], f64_lnl(pr, n_eval - 1)[1]) < SYN_RTOL


@pytest.mark.parametrize("K", range(1, 9))
def test_nuc4_fused_device_blob(engine_lib, oracle_lib, K):
    """pack + replay: the fused kernel reads the job from device memory, and with more than 16
    tiles the last CTA sums the tile partials in parallel.  One 4-state launch per call and no
    stand-alone P(t) launch show that the fused kernel served every call."""
    pr = nuc4_problem(K, edge(K, 20), seed=1)
    assert (pr.C + ppb(K) - 1) // ppb(K) > 16
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        check_run(pr, e, o, via_replay, 12, seed=K)
        assert e.kernel_launches(abi.KERNEL_NUC4) == 14
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 0


@pytest.mark.parametrize("K", range(1, 9))
def test_nuc4_non_fused(engine_lib, oracle_lib, K):
    """more than 4 x SMs tiles in one call: stand-alone tiprobs_kernel, then the streaming kernel.
    A stand-alone P(t) launch on a 4-state instance happens only on this path."""
    tiles = 4 * num_sms() + 4
    pr = nuc4_problem(K, edge(K, tiles), seed=2)
    assert (pr.C + ppb(K) - 1) // ppb(K) > 4 * num_sms()
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        check_run(pr, e, o, via_evaluate, 10, seed=K)
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 12             # one per call
        assert e.kernel_launches(abi.KERNEL_NUC4) == 12


@pytest.mark.parametrize("K", range(1, 9))
def test_nuc4_resident_equals_launches(engine_lib, oracle_lib, K):
    """replay_begin / _end with this instance alone on the device: the resident kernel must give,
    bit for bit, what one launch per generation gives; the launches are checked against the oracle"""
    pr = nuc4_problem(K, edge(K, 12), seed=3)
    rng = np.random.default_rng(K)
    gens = [[pr.full_evaluation(0), pr.full_evaluation(1)]]
    for g in range(1, 11):
        old = [pr.tree[ch].length.copy() for ch in (0, 1)]
        gens.append([pr.random_branch_update(ch, rng) for ch in (0, 1)])
        if g % 3 == 2:
            for ch in (0, 1):
                pr.reject(ch, gens[-1][ch], old[ch])
    dests = sorted({int(op["dest"]) for s in gens for sp in s for op in sp.ops})
    scal = sorted({int(op["scale_write"]) for s in gens for sp in s for op in sp.ops if op["scale_write"] >= 0} |
                  {int(sp.site_dst) for s in gens for sp in s})

    def final_state(e):
        return [e.get_partials(b) for b in dests], [e.get_scalers(s) for s in scal]

    want = []
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        for specs in gens:
            b = e.pack(specs)
            e.replay(b)
            lnl, st = e.replay_results(b, 2)
            e.free_batch(b)
            assert not st.any()
            for i, sp in enumerate(specs):
                (lo,), _ = o.evaluate(sp)
                assert rel(lnl[i], lo) < SYN_RTOL
                _compare_state(e, o, sp, 4)
            want.append(lnl)
        assert rel(want[-1][1], f64_lnl(pr, 1)[1]) < SYN_RTOL
        want_state = final_state(e)
    with pr.create(engine_lib) as e:
        batches = [e.pack(specs) for specs in gens]
        n0 = e.launch_count()
        got = []
        for b in batches:
            assert engine_lib.fn("replay_begin")(e.handle, b) == 0
            lnl = np.zeros(2, np.float64)
            st = np.zeros(2, np.int32)
            assert engine_lib.fn("replay_end")(e.handle, lnl.ctypes.data_as(abi.C.POINTER(abi.C.c_double)),
                                              st.ctypes.data_as(abi.C.POINTER(abi.C.c_int))) == 0
            assert not st.any()
            got.append(lnl)
        launches = e.launch_count() - n0
        e.synchronize()
        got_state = final_state(e)
    assert launches < len(gens)                      # one kernel served several generations
    assert np.array_equal(np.array(got), np.array(want))
    assert all(np.array_equal(a, b) for a, b in zip(got_state[0], want_state[0]))
    assert all(np.array_equal(a, b) for a, b in zip(got_state[1], want_state[1]))


@pytest.mark.parametrize("K", range(1, 9))
def test_nuc4_throughput_mode(engine_lib, oracle_lib, K):
    """MB200_CONFIG_THROUGHPUT: one CTA per evaluation walks all its tiles"""
    nch = 4
    pr = workloads.make_problem(4, K, edge(K, 5), 10, nch, seed=2000 + K, p_invar=0.1 * (K % 2), p_ambig=0.05)
    rng = np.random.default_rng(K)
    with pr.create(engine_lib, flags=abi.CONFIG_THROUGHPUT) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        for gen in range(4):
            specs = [pr.full_evaluation(ch) if gen == 0 else pr.random_branch_update(ch, rng) for ch in range(nch)]
            lnl, st = e.evaluate(specs)
            assert not st.any()
            for i, sp in enumerate(specs):
                (lo,), _ = o.evaluate(sp)
                assert rel(lnl[i], lo) < SYN_RTOL
                _compare_state(e, o, sp, 4)
        assert rel(lnl[0], f64_lnl(pr, 0)[1]) < SYN_RTOL


# ---- C. tensor-core matrix --------------------------------------------------------------
TC_SHAPES = [(20, 1), (20, 2), (20, 3), (20, 4), (61, 1), (61, 2), (61, 3)]


@pytest.mark.parametrize("C", [127, 128, 129, 256, 385])
@pytest.mark.parametrize("S,K", TC_SHAPES)
def test_tensor_core_matrix(engine_lib, oracle_lib, S, K, C):
    """40 tips (chain 0 random, chain 1 a caterpillar); eight chains in one call whose operation
    counts differ.  C = 129 carries p_invar and 20 % ambiguity, C = 385 some all-missing columns."""
    nch = 8
    pr = workloads.make_problem(S, K, C, 40, nch, seed=3000 + S + 10 * K + C,
                                p_invar=0.1 if C == 129 else 0.0, p_ambig=0.2 if C == 129 else 0.0)
    pr.tree[1] = caterpillar_tree(40, np.random.default_rng(C))
    if C == 385:
        pr.masks[:, ::50] = np.uint64((1 << S) - 1)
    rng = np.random.default_rng(S + K + C)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        # all chains' full evaluations in one call
        specs = [pr.full_evaluation(ch) for ch in range(nch)]
        lnl, st = e.evaluate(specs)
        assert not st.any()
        for ch, sp in enumerate(specs):
            (lo,), _ = o.evaluate(sp)
            assert rel(lnl[ch], lo) < TC_RTOL, f"chain {ch}"
            if ch < 2:
                compare_state(e, o, sp, pr)
                r = rel(lnl[ch], f64_lnl(pr, ch)[1])
                assert r < TC_RTOL, f"float64 reference, chain {ch}: {r:.2e}"
        for it in range(10):
            ch = it % 2
            old = pr.tree[ch].length.copy()
            sp = pr.random_branch_update(ch, rng)
            (le,), (se,) = e.evaluate(sp)
            (lo,), _ = o.evaluate(sp)
            assert se == abi.EVAL_OK and rel(le, lo) < TC_RTOL, f"update {it}"
            compare_state(e, o, sp, pr)
            if it % 3 == 2:
                pr.reject(ch, sp, old)
        # one generation of branch updates over all chains in one call
        specs = [pr.random_branch_update(ch, rng) for ch in range(nch)]
        assert len({len(sp.ops) for sp in specs}) > 1
        lnl, st = e.evaluate(specs)
        assert not st.any()
        for ch, sp in enumerate(specs):
            (lo,), _ = o.evaluate(sp)
            assert rel(lnl[ch], lo) < TC_RTOL, f"batched update, chain {ch}"
            r = rel(lnl[ch], f64_lnl(pr, ch)[1])
            assert r < TC_RTOL, f"float64 reference, batched update, chain {ch}: {r:.2e}"
        assert e.kernel_launches(abi.KERNEL_TENSOR) == 12
        assert e.kernel_launches(abi.KERNEL_GENERIC) == 0


# ---- D. generic kernel geometry -----------------------------------------------------------
GEN_CASES = [
    # S, K, patterns per tile the instance picks (C = that x SMs; 4: small C)
    (61, 4, 32),          # K S (S+1) 4 B > 48 KB: one category per pass
    (61, 5, 8),
    (64, 3, 16),
    (64, 3, 4),
    (40, 8, 32),
    (40, 8, 4),
    (16, 4, 32),          # all categories per pass
    (16, 2, 8),
    (16, 6, 16),
    (40, 3, 32),
    (40, 7, 16),
    (64, 1, 32),
    (64, 2, 8),
]


@pytest.mark.parametrize("S,K,tp", GEN_CASES)
def test_generic_kernel_geometry(engine_lib, oracle_lib, S, K, tp):
    C = tp * num_sms() if tp > 4 else 77
    pr = workloads.make_problem(S, K, C, 8, 2, seed=4000 + S + K + tp, p_invar=0.1 if tp == 16 else 0.0,
                                p_ambig=0.1 if tp == 8 else 0.0)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        check_run(pr, e, o, via_evaluate, 4, seed=S + K)
        assert e.kernel_launches(abi.KERNEL_GENERIC) == 6
        assert e.kernel_launches(abi.KERNEL_TENSOR) == 0 and e.kernel_launches(abi.KERNEL_NUC4) == 0


# ---- E. P(t) limits ---------------------------------------------------------------------
def test_time_limits_non_fused_nuc4(engine_lib, oracle_lib):
    """t < TIME_MIN and t > TIME_MAX in the stand-alone tiprobs_kernel of the non-fused 4-state path"""
    K = 4
    pr = workloads.make_problem(4, K, edge(K, 4 * num_sms() + 4), 6, 1, seed=5)
    pr.tree[0].length[0] = 1e-13
    pr.tree[0].length[1] = 5000.0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        sp = pr.full_evaluation(0)
        (le,), _ = e.evaluate(sp)
        (lo,), _ = o.evaluate(sp)
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 1
        assert rel(le, lo) < SYN_RTOL and rel(le, f64_lnl(pr, 0)[1]) < SYN_RTOL
        P0 = e.get_transition_matrix(int(pr.chains[0].ti[0]))
        assert np.array_equal(P0, np.broadcast_to(np.eye(4, dtype=np.float32), P0.shape))
        P1 = e.get_transition_matrix(int(pr.chains[0].ti[1]))
        assert np.array_equal(P1, np.broadcast_to(pr.freqs.astype(np.float32)[None, None, :], P1.shape))


def test_time_limits_std(engine_lib, oracle_lib):
    """TiProbs_Std clamps the branch length to [BRLENS_MIN, BRLENS_MAX] instead: the matrices are the oracle's"""
    pr = workloads.make_std_problem(90, 4, 6, 1, seed=6, max_states=6, dummy=2)
    pr.tree[0].length[0] = 1e-13
    pr.tree[0].length[1] = 5000.0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        sp = pr.full_evaluation(0)
        (le,), (se,) = e.evaluate(sp)
        (lo,), (so,) = o.evaluate(sp)
        assert se == so == abi.EVAL_OK and rel(le, lo) < 1e-9
        assert e.kernel_launches(abi.KERNEL_STD) == 1
        for node in (0, 1):
            m = int(pr.chains[0].ti[node])
            assert np.allclose(e.get_transition_matrix(m), o.get_transition_matrix(m), rtol=2.5e-7, atol=1e-30)


# ---- F. underflow across tiles and evaluations -----------------------------------------------
def dead_pattern_problem(family, where, n_chains=1):
    """Every pattern compatible (all tips in one state) except pattern `dead`, where the root tip
    disagrees; with P = I (branches below TIME_MIN) that pattern's likelihood is exactly 0."""
    sms = num_sms()
    if family == "std":
        C = 64 * 5 + 1 if where == "last" else 64 * 5       # K = 2: 64 patterns per tile
        pr = workloads.make_std_problem(C, 2, 6, n_chains, seed=7, max_states=5, dummy=0)
        pr.rates = pr.rates * 1e-10          # Std clamps lengths up to BRLENS_MIN: P = I needs r t < 1e-17
        pr.masks[:] = 1
        base = np.zeros(C, np.int64)
    else:
        S, K, C, tile = {"nuc4_host": (4, 4, 10 * 64, 64), "nuc4_device": (4, 4, 40 * 64, 64),
                         "nuc4_non_fused": (4, 4, (4 * sms + 4) * 64, 64), "tensor": (20, 2, 4 * 128, 128),
                         "generic": (16, 2, 300, 4)}[family]
        if where == "last":
            C -= tile - 1                      # the last tile holds one pattern
        pr = workloads.make_problem(S, K, C, 6, n_chains, seed=8, p_missing=0.0)
        base = np.random.default_rng(1).integers(0, S, size=C)
        pr.masks[:] = (np.uint64(1) << base.astype(np.uint64))[None, :]
    # the root tip disagrees with the rest: every interior node below the root keeps a non-zero
    # (scalable) likelihood, the zero appears where the interior root combines its three children
    dead = C - 1 if where == "last" else C // 2 + 1
    pr.masks[:, dead] = np.uint64(1) << np.uint64(base[dead])
    pr.masks[pr.tree[0].root, dead] = np.uint64(1) << np.uint64((base[dead] + 1) % 2)
    return pr, dead


FAMILIES = ["nuc4_host", "nuc4_device", "nuc4_non_fused", "tensor", "generic", "std"]
KIND = {"nuc4_host": abi.KERNEL_NUC4, "nuc4_device": abi.KERNEL_NUC4, "nuc4_non_fused": abi.KERNEL_NUC4,
        "tensor": abi.KERNEL_TENSOR, "generic": abi.KERNEL_GENERIC, "std": abi.KERNEL_STD}


@pytest.mark.parametrize("where", ["middle", "last"])
@pytest.mark.parametrize("family", FAMILIES)
def test_underflow_in_one_tile(engine_lib, oracle_lib, family, where):
    pr, _ = dead_pattern_problem(family, where)
    for tr in pr.tree:
        tr.length[:] = 0.0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        sp = pr.full_evaluation(0)
        (le,), (se,) = e.evaluate(sp)
        (lo,), (so,) = o.evaluate(sp)
        assert e.kernel_launches(KIND[family]) == 1
        if family == "nuc4_non_fused":
            assert e.kernel_launches(abi.KERNEL_TIPROBS) == 1
        assert se == so == abi.EVAL_UNDERFLOW
        assert le == lo == -DBL_MAX


@pytest.mark.parametrize("family", ["nuc4_host", "nuc4_device", "tensor", "generic"])
def test_underflow_in_one_evaluation_of_a_batch(engine_lib, oracle_lib, family):
    """Only chain 2's branches are below TIME_MIN: its evaluation aborts, the others are unaffected."""
    nch = 4
    pr, _ = dead_pattern_problem(family, "middle", n_chains=nch)
    pr.tree[2].length[:] = 0.0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        specs = [pr.full_evaluation(ch) for ch in range(nch)]
        lnl, st = e.evaluate(specs)
        for ch, sp in enumerate(specs):
            (lo,), (so,) = o.evaluate(sp)
            assert st[ch] == so == (abi.EVAL_UNDERFLOW if ch == 2 else abi.EVAL_OK), f"chain {ch}"
            if ch == 2:
                assert lnl[ch] == lo == -DBL_MAX
            else:
                assert rel(lnl[ch], lo) < tol_of(pr.S), f"chain {ch}"
