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
                      (every family, and the resident and throughput 4-state routes)

The threshold between the fused and the non-fused 4-state path scales with the device's SM count,
so the pattern counts here are computed from it."""
import numpy as np
import pytest

from engine_checks import (DBL_MAX, SYN_RTOL, TC_RTOL, assert_resident_equals_launches, check_with_oracle,
                           dead_pattern_problem, edge, evaluation_sequence, kernel_names, launched, lnl_tol, num_sms,
                           nuc4_problem, parity_tol, ppb, rel, resident_generations, tree_tol, via_evaluate, via_replay)
from f64_reference import caterpillar_tree, f64_lnl
from mrbayes_b200 import abi, workloads

pytestmark = pytest.mark.gpu


def check_run(pr, e, o, route, updates, seed):
    """A full evaluation per chain, then `updates` branch updates over the chains with a rejection
    every third: lnL, every written partials buffer and the node and site scalers against the oracle;
    lnL against the float64 reference after the full evaluations and after the last update."""
    tol = lnl_tol(pr.S)
    for it, sp in evaluation_sequence(pr, updates, seed):
        lnl, st = route(e, [sp])
        check_with_oracle(e, o, [sp], lnl, st, tol, tree_tol(pr))
        if it < 0 or it == updates - 1:
            r = rel(lnl[0], f64_lnl(pr, sp.chain)[1])
            assert r < tol, f"float64 reference after evaluation {it} (chain {sp.chain}): {r:.2e}"


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
            check_with_oracle(e, o, specs, lnl, st, SYN_RTOL, parity_tol(4))
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
    assert_resident_equals_launches(engine_lib, oracle_lib, pr, gens, SYN_RTOL, parity_tol(4))


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
            check_with_oracle(e, o, specs, lnl, st, SYN_RTOL, parity_tol(4))
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
        check_with_oracle(e, o, specs, lnl, st, TC_RTOL, tree_tol(pr))
        for ch in range(2):
            r = rel(lnl[ch], f64_lnl(pr, ch)[1])
            assert r < TC_RTOL, f"float64 reference, chain {ch}: {r:.2e}"
        for it in range(10):
            ch = it % 2
            old = pr.tree[ch].length.copy()
            sp = pr.random_branch_update(ch, rng)
            check_with_oracle(e, o, [sp], *e.evaluate(sp), TC_RTOL, tree_tol(pr))
            if it % 3 == 2:
                pr.reject(ch, sp, old)
        # one generation of branch updates over all chains in one call
        specs = [pr.random_branch_update(ch, rng) for ch in range(nch)]
        assert len({len(sp.ops) for sp in specs}) > 1
        lnl, st = e.evaluate(specs)
        check_with_oracle(e, o, specs, lnl, st, TC_RTOL, tree_tol(pr))
        for ch in range(nch):
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
FAMILIES = ["nuc4_host", "nuc4_device", "nuc4_non_fused", "nuc4_resident", "nuc4_throughput", "tensor", "generic", "std"]
KIND = {"nuc4_host": abi.KERNEL_NUC4, "nuc4_device": abi.KERNEL_NUC4, "nuc4_non_fused": abi.KERNEL_NUC4,
        "nuc4_resident": abi.KERNEL_NUC4, "nuc4_throughput": abi.KERNEL_NUC4,
        "tensor": abi.KERNEL_TENSOR, "generic": abi.KERNEL_GENERIC, "std": abi.KERNEL_STD}


def family_instance(pr, lib, family):
    return pr.create(lib, flags=abi.CONFIG_THROUGHPUT if family == "nuc4_throughput" else 0)


def family_evaluate(e, family, specs):
    """e.evaluate, or for nuc4_resident one generation through replay_begin / _end"""
    if family != "nuc4_resident":
        return e.evaluate(specs)
    return resident_generations(e, [specs])[0]


@pytest.mark.parametrize("where", ["middle", "last"])
@pytest.mark.parametrize("family", FAMILIES)
def test_underflow_in_one_tile(engine_lib, oracle_lib, family, where):
    """On the resident route the dead generation is followed by one that is not (the interior root's
    branch, to the root tip, gets a length): the same resident kernel serves it -- a dead
    generation does not end residency."""
    pr, _ = dead_pattern_problem(family, where)
    for tr in pr.tree:
        tr.length[:] = 0.0
    with family_instance(pr, engine_lib, family) as e, pr.create(oracle_lib) as o:
        sp = pr.full_evaluation(0)
        if family == "nuc4_resident":
            alive = pr.branch_update(0, pr.tree[0].root_left, 0.1)
            ((le,), (se,)), ((la,), (sa,)) = resident_generations(e, [[sp], [alive]])
        else:
            (le,), (se,) = e.evaluate(sp)
        (lo,), (so,) = o.evaluate(sp)
        assert e.kernel_launches(KIND[family]) == 1               # resident: one kernel for both generations
        if family == "nuc4_non_fused":
            assert e.kernel_launches(abi.KERNEL_TIPROBS) == 1
        assert se == so == abi.EVAL_UNDERFLOW
        assert le == lo == -DBL_MAX
        if family == "nuc4_resident":
            (lo,), (so,) = o.evaluate(alive)
            assert sa == so == abi.EVAL_OK and rel(la, lo) < SYN_RTOL


@pytest.mark.parametrize("family", ["nuc4_host", "nuc4_device", "nuc4_resident", "nuc4_throughput", "tensor", "generic"])
def test_underflow_in_one_evaluation_of_a_batch(engine_lib, oracle_lib, family):
    """Only chain 2's branches are below TIME_MIN: its evaluation aborts, the others are unaffected."""
    nch = 4
    pr, _ = dead_pattern_problem(family, "middle", n_chains=nch)
    pr.tree[2].length[:] = 0.0
    with family_instance(pr, engine_lib, family) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        specs = [pr.full_evaluation(ch) for ch in range(nch)]
        lnl, st = family_evaluate(e, family, specs)
        assert e.kernel_launches(KIND[family]) == 1
        for ch, sp in enumerate(specs):
            (lo,), (so,) = o.evaluate(sp)
            assert st[ch] == so == (abi.EVAL_UNDERFLOW if ch == 2 else abi.EVAL_OK), f"chain {ch}"
            if ch == 2:
                assert lnl[ch] == lo == -DBL_MAX
            else:
                assert rel(lnl[ch], lo) < lnl_tol(pr.S), f"chain {ch}"
