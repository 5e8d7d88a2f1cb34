"""GPU: the CUDA engine through the C-ABI against (1) the reference's recorded lnL, (2) the
CPU oracle on identical inputs, (3) size-independent properties at BASELINE.json's full sizes.

Tolerances (tests/engine_checks.py): lnL 1e-8 relative, 100x tighter than the north-star bar, on the
recorded cases; conditional likelihoods 2e-6 relative, node scalers 1e-6 absolute (parity_tol)."""
import numpy as np
import pytest

from conftest import GOLDEN, GOLDEN_FILES
from engine_checks import LNL_RTOL, SYN_RTOL, check_with_oracle, compare_written, evaluation_sequence, lnl_tol, \
    parity_tol, rel
from mrbayes_b200 import abi, records, workloads

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("stem,arith", GOLDEN_FILES)
def test_engine_matches_reference_records(engine_lib, oracle_lib, stem, arith):
    got = records.replay(engine_lib, GOLDEN / f"{stem}.gold.gz")
    assert len(got) >= 40
    worst = max(rel(l, s.lnl_ref) for s, l, _ in got)
    assert all(st == abi.EVAL_OK for _, _, st in got)
    tol = lnl_tol(len(got[0][0].freqs), LNL_RTOL)
    assert worst < tol, f"{stem}: max relative lnL error vs reference {worst:.3e}"


def test_transition_matrices_match_oracle(engine_lib, oracle_lib):
    for stem in ("primates_gtr_g4_fma", "ovomucoids_wag_g4_sse", "replicase_m0_sse"):
        divs, events = records.load(GOLDEN / f"{stem}.gold.gz")
        d = divs[0]
        with records.make_instance(engine_lib, d) as e, records.make_instance(oracle_lib, d) as o:
            n = 0
            for ev in events:
                if ev.kind != "eval":
                    records.apply_event(e, ev); records.apply_event(o, ev)
                    continue
                e.evaluate(ev.spec); o.evaluate(ev.spec)
                for m in ev.spec.mats["matrix"][:6]:
                    Pe, Po = e.get_transition_matrix(int(m)), o.get_transition_matrix(int(m))
                    # double exp() may differ in the last bit between glibc and CUDA: <= 1 float ulp
                    assert np.allclose(Pe, Po, rtol=2.5e-7, atol=1e-30), stem
                    assert np.allclose(Pe.sum(-1), 1.0, atol=1e-5)
                n += 1
                if n >= 3:
                    break


CASES = [
    # S, K, C, tips, p_invar, p_ambig
    (4, 4, 413, 12, 0.0, 0.0),
    (4, 4, 1, 4, 0.0, 0.0),
    (4, 4, 31, 5, 0.2, 0.1),
    (4, 4, 33, 6, 0.0, 0.3),
    (4, 1, 128, 7, 0.0, 0.0),
    (4, 2, 129, 7, 0.1, 0.0),
    (4, 3, 500, 8, 0.0, 0.05),
    (4, 5, 77, 5, 0.0, 0.0),
    (4, 8, 260, 6, 0.3, 0.0),
    (4, 6, 97, 7, 0.1, 0.05),
    (4, 7, 64, 9, 0.0, 0.0),
    (4, 10, 60, 5, 0.0, 0.0),      # K > 8: generic kernel on 4 states
    (20, 4, 88, 9, 0.0, 0.0),
    (20, 4, 33, 6, 0.1, 0.2),
    (20, 1, 70, 5, 0.0, 0.0),
    (20, 2, 129, 8, 0.0, 0.1),
    (20, 3, 128, 7, 0.15, 0.0),
    (61, 1, 239, 9, 0.0, 0.0),
    (61, 1, 20, 4, 0.0, 0.1),
    (61, 2, 31, 5, 0.0, 0.0),
    (61, 3, 130, 6, 0.0, 0.0),     # the NY98 / M3 shape: three omega categories
    (2, 4, 50, 6, 0.0, 0.0),
    (16, 2, 45, 6, 0.0, 0.0),
    (64, 1, 19, 5, 0.0, 0.0),
]


@pytest.mark.parametrize("S,K,C,tips,pinv,pamb", CASES)
def test_engine_matches_oracle_synthetic(engine_lib, oracle_lib, S, K, C, tips, pinv, pamb):
    """Full evaluations, then a run of partial updates with rejections, engine and oracle fed
    the same calls; every written buffer compared."""
    nch = 2
    pr = workloads.make_problem(S, K, C, tips, nch, seed=100 + S + K + C, p_invar=pinv, p_ambig=pamb)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        for _, sp in evaluation_sequence(pr, 10, seed=7):
            check_with_oracle(e, o, [sp], *e.evaluate(sp), lnl_tol(S), parity_tol(S))


@pytest.mark.parametrize("S,K,C,tips", [(4, 4, 413, 12), (20, 4, 64, 6), (61, 1, 40, 5)])
def test_chain_batched_launch_equals_serial(engine_lib, S, K, C, tips):
    """All chains of a generation in ONE mb200_evaluate call == one call per chain."""
    nch = 8
    a = workloads.make_problem(S, K, C, tips, nch, seed=5)
    b = workloads.make_problem(S, K, C, tips, nch, seed=5)
    rng_a, rng_b = np.random.default_rng(1), np.random.default_rng(1)
    with a.create(engine_lib) as ia, b.create(engine_lib) as ib:
        la, _ = ia.evaluate([a.full_evaluation(ch) for ch in range(nch)])
        lb = np.array([ib.evaluate(b.full_evaluation(ch))[0][0] for ch in range(nch)])
        assert np.array_equal(la, lb)          # same kernels, same order: bit-identical
        for gen in range(3):
            la, _ = ia.evaluate([a.random_branch_update(ch, rng_a) for ch in range(nch)])
            lb = np.array([ib.evaluate(b.random_branch_update(ch, rng_b))[0][0] for ch in range(nch)])
            assert np.array_equal(la, lb)


def test_partition_batched_begin_end_equals_evaluate(engine_lib):
    """The divisions of a chain (separate instances) launched together with evaluate_begin and
    collected with evaluate_end give exactly what one evaluate() per division gives
    (LaunchBEAGLELogLikeMultiPartition semantics, reference src/likelihood.c:7792)."""
    shapes = [(4, 4, 537, 32), (4, 4, 125, 32), (4, 4, 205, 32), (20, 4, 90, 10)]
    probs_a = [workloads.make_problem(S, K, C, tips, 1, seed=40 + i) for i, (S, K, C, tips) in enumerate(shapes)]
    probs_b = [workloads.make_problem(S, K, C, tips, 1, seed=40 + i) for i, (S, K, C, tips) in enumerate(shapes)]
    insts_a = [p.create(engine_lib) for p in probs_a]
    insts_b = [p.create(engine_lib) for p in probs_b]
    try:
        rng_a, rng_b = np.random.default_rng(3), np.random.default_rng(3)
        for gen in range(4):
            specs_a = [p.full_evaluation(0) if gen == 0 else p.random_branch_update(0, rng_a) for p in probs_a]
            specs_b = [p.full_evaluation(0) if gen == 0 else p.random_branch_update(0, rng_b) for p in probs_b]
            for inst, sp in zip(insts_a, specs_a):
                inst.evaluate_begin(sp)                       # all divisions in flight
            got = [inst.evaluate_end() for inst in insts_a]
            want = [inst.evaluate(sp) for inst, sp in zip(insts_b, specs_b)]
            for (lg, sg), (lw, sw) in zip(got, want):
                assert np.array_equal(lg, lw) and np.array_equal(sg, sw)
        # protocol errors: a second begin before end, an end without begin
        insts_a[0].evaluate_begin(probs_a[0].full_evaluation(0))
        with pytest.raises(abi.AbiError):
            insts_a[0].evaluate_begin(probs_a[0].full_evaluation(0))
        insts_a[0].evaluate_end()
        with pytest.raises(abi.AbiError):
            insts_a[0].evaluate_end()
    finally:
        for inst in insts_a + insts_b:
            inst.close()


@pytest.mark.parametrize("K,C", [(4, 413), (1, 700), (3, 65)])
def test_throughput_mode_equals_latency_mode(engine_lib, K, C):
    """MB200_CONFIG_THROUGHPUT: one CTA per evaluation walks all pattern tiles (P(t) built once).  Every
    buffer must come out bit-identical to the default tiling; lnL only differs in the order of the final sum."""
    nch = 4
    a = workloads.make_problem(4, K, C, 12, nch, seed=77)
    b = workloads.make_problem(4, K, C, 12, nch, seed=77)
    rng_a, rng_b = np.random.default_rng(2), np.random.default_rng(2)
    with a.create(engine_lib) as ia, b.create(engine_lib, flags=abi.CONFIG_THROUGHPUT) as ib:
        for gen in range(4):
            sa = [a.full_evaluation(ch) if gen == 0 else a.random_branch_update(ch, rng_a) for ch in range(nch)]
            sb = [b.full_evaluation(ch) if gen == 0 else b.random_branch_update(ch, rng_b) for ch in range(nch)]
            la, sta = ia.evaluate(sa)
            lb, stb = ib.evaluate(sb)
            assert not sta.any() and not stb.any()
            assert np.allclose(la, lb, rtol=1e-13, atol=0.0)
            for spa, spb in zip(sa, sb):
                for opa, opb in zip(spa.ops, spb.ops):
                    assert np.array_equal(ia.get_partials(int(opa["dest"])), ib.get_partials(int(opb["dest"])))
                    if opa["scale_write"] >= 0:
                        assert np.array_equal(ia.get_scalers(int(opa["scale_write"])), ib.get_scalers(int(opb["scale_write"])))
                assert np.array_equal(ia.get_scalers(spa.site_dst), ib.get_scalers(spb.site_dst))


def test_resident_replay_equals_host_call(engine_lib):
    pr = workloads.make_problem(4, 4, 413, 12, 8, seed=9)
    with pr.create(engine_lib) as inst:
        specs = [pr.full_evaluation(ch) for ch in range(8)]
        want, _ = inst.evaluate(specs)
        # same evaluations again from a device-resident packed batch (full evaluations are idempotent)
        batch = inst.pack(specs)
        n0 = inst.launch_count()
        inst.replay(batch)
        got, st = inst.replay_results(batch, 8)
        assert inst.launch_count() - n0 == 1     # P(t) rebuild is fused into the pruning kernel for small launches
        assert np.array_equal(got, want) and not st.any()
        inst.free_batch(batch)


def test_node_granular_verbs_equal_fused_evaluation(engine_lib):
    """TiProbs / CondLikeDown+Scaler / Likelihood as separate calls (the reference's
    function-pointer granularity) give the fused result."""
    pr = workloads.make_problem(4, 4, 200, 8, 1, seed=21, p_invar=0.1)
    pr2 = workloads.make_problem(4, 4, 200, 8, 1, seed=21, p_invar=0.1)
    with pr.create(engine_lib) as a, pr2.create(engine_lib) as b:
        sp = pr.full_evaluation(0)
        (want,), _ = a.evaluate(sp)
        sp2 = pr2.full_evaluation(0)
        b.update_transition_matrices(sp2.mats, sp2.rates, sp2.freqs)
        b.reset_scalers(sp2.site_dst)
        for i in range(len(sp2.ops)):
            b.update_partials(sp2.ops[i:i + 1], sp2.site_dst)
        got, st = b.root_log_likelihood(sp2.root, sp2.site_dst, 0, sp2.freqs, sp2.cat_weights, 1, sp2.p_invar, sp2.flags)
        assert st == abi.EVAL_OK
        assert got == want


def test_time_min_and_time_max_branches(engine_lib, oracle_lib):
    """t < TIME_MIN -> identity, t > TIME_MAX -> stationary rows (src/likelihood.c:9503-9525)."""
    pr = workloads.make_problem(4, 4, 50, 6, 1, seed=3)
    pr.tree[0].length[0] = 1e-13
    pr.tree[0].length[1] = 5000.0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        sp = pr.full_evaluation(0)
        (le,), _ = e.evaluate(sp); (lo,), _ = o.evaluate(sp)
        assert rel(le, lo) < LNL_RTOL
        P0 = e.get_transition_matrix(int(pr.chains[0].ti[0]))
        assert np.array_equal(P0, np.broadcast_to(np.eye(4, dtype=np.float32), P0.shape))
        P1 = e.get_transition_matrix(int(pr.chains[0].ti[1]))
        assert np.array_equal(P1, np.broadcast_to(pr.freqs.astype(np.float32)[None, None, :], P1.shape))


@pytest.mark.parametrize("S,K", [(16, 4), (20, 4), (61, 3), (61, 4), (64, 2)])
def test_time_min_and_time_max_branches_other_state_counts(engine_lib, oracle_lib, S, K):
    """The same limits in the other P(t) builders: tiprobs_kernel (16 states; 20 states, then the
    tensor-core split images) and tiprobs_mm_kernel (61 and 64 states)."""
    pr = workloads.make_problem(S, K, 50, 6, 1, seed=3)
    pr.tree[0].length[0] = 1e-13
    pr.tree[0].length[1] = 5000.0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        sp = pr.full_evaluation(0)
        (le,), _ = e.evaluate(sp); (lo,), _ = o.evaluate(sp)
        assert rel(le, lo) < lnl_tol(S)
        P0 = e.get_transition_matrix(int(pr.chains[0].ti[0]))
        assert np.array_equal(P0, np.broadcast_to(np.eye(S, dtype=np.float32), P0.shape))
        P1 = e.get_transition_matrix(int(pr.chains[0].ti[1]))
        assert np.array_equal(P1, np.broadcast_to(pr.freqs.astype(np.float32)[None, None, :], P1.shape))


def test_underflow_sets_abort_status(engine_lib, oracle_lib):
    """like < LIKE_EPSILON at some pattern -> lnL = -DBL_MAX + status (abortMove protocol)."""
    pr = workloads.make_problem(4, 1, 8, 3, 1, seed=1, p_missing=0.0)
    pr.tree[0].length[:] = 0.0          # identity matrices everywhere
    pr.masks[0, :] = 1; pr.masks[1, :] = 2; pr.masks[2, :] = 1   # incompatible tips
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        sp = pr.full_evaluation(0)
        (le,), (se,) = e.evaluate(sp); (lo,), (so,) = o.evaluate(sp)
        assert se == so == abi.EVAL_UNDERFLOW
        assert le == lo == -np.finfo(np.float64).max


def test_repeatability(engine_lib):
    """Same inputs -> bit-identical lnL (fixed-order tile reduction, no float atomics)."""
    vals = []
    for _ in range(3):
        pr = workloads.make_problem(4, 4, 5000, 16, 2, seed=77)
        with pr.create(engine_lib) as inst:
            vals.append(inst.evaluate([pr.full_evaluation(0), pr.full_evaluation(1)])[0])
    assert np.array_equal(vals[0], vals[1]) and np.array_equal(vals[0], vals[2])


# ---- BASELINE.json full sizes: size-independent properties --------------------------------
FULL = [
    ("aa_50k", 20, 4, 50_000, 64),
    ("codon_20k", 61, 1, 20_000, 32),
    ("nuc_200k", 4, 4, 200_000, 32),
]


@pytest.mark.parametrize("name,S,K,C,tips", FULL)
def test_full_size_subset_equals_oracle_on_subset(engine_lib, oracle_lib, name, S, K, C, tips):
    """Site patterns are independent: with the pattern weights of the full-size instance zeroed
    outside a random subset, lnL must equal the oracle's lnL of the sub-alignment."""
    pr = workloads.make_problem(S, K, C, tips, 1, seed=2026, same_tree=True)
    rng = np.random.default_rng(5)
    sub = np.sort(rng.choice(C, size=300, replace=False))
    w_sub = np.zeros(C, np.float32); w_sub[sub] = pr.weights[sub]
    with pr.create(engine_lib) as e:
        (l_all,), (st,) = e.evaluate(pr.full_evaluation(0))
        assert st == abi.EVAL_OK and np.isfinite(l_all)
        # additivity over a partition of the patterns
        half = np.zeros(C, np.float32); half[: C // 2] = pr.weights[: C // 2]
        e.set_pattern_weights(0, half)
        (l_a,), _ = e.evaluate(pr.full_evaluation(0))
        e.set_pattern_weights(0, pr.weights - half)
        (l_b,), _ = e.evaluate(pr.full_evaluation(0))
        assert rel(l_a + l_b, l_all) < 1e-11
        e.set_pattern_weights(0, w_sub)
        (l_sub,), _ = e.evaluate(pr.full_evaluation(0))
    small = workloads.make_problem(S, K, C, tips, 1, seed=2026, same_tree=True)
    small.masks = np.ascontiguousarray(small.masks[:, sub]); small.weights = small.weights[sub]; small.C = len(sub)
    with small.create(oracle_lib) as o:
        (l_o,), _ = o.evaluate(small.full_evaluation(0))
    assert rel(l_sub, l_o) < lnl_tol(S, LNL_RTOL)


@pytest.mark.parametrize("tips,K", [(40, 4), (90, 4), (150, 1), (70, 8)])
def test_large_trees_span_several_chunks(engine_lib, oracle_lib, tips, K):
    """Operation lists longer than one shared-memory chunk (more nodes / more branches than the
    kernel's P(t) slots): full evaluations and partial updates against the oracle."""
    pr = workloads.make_problem(4, K, 150, tips, 1, seed=tips)
    rng = np.random.default_rng(3)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        sp = pr.full_evaluation(0)
        (le,), _ = e.evaluate(sp); (lo,), _ = o.evaluate(sp)
        assert rel(le, lo) < SYN_RTOL
        compare_written(e, o, sp, parity_tol(4))
        for it in range(6):
            sp = pr.random_branch_update(0, rng)
            (le,), _ = e.evaluate(sp); (lo,), _ = o.evaluate(sp)
            assert rel(le, lo) < SYN_RTOL


def test_api_edge_cases(engine_lib, oracle_lib):
    """Degenerate and invalid inputs at the C-ABI: a single site pattern, an evaluation that only
    integrates at the root, an evaluation without a root, out-of-range indices, protocol misuse."""
    # one pattern, one category, four states: the smallest instance
    pr_e = workloads.make_problem(4, 1, 1, 3, 1, seed=3)
    pr_o = workloads.make_problem(4, 1, 1, 3, 1, seed=3)
    with pr_e.create(engine_lib) as e, pr_o.create(oracle_lib) as o:
        le, se = e.evaluate(pr_e.full_evaluation(0))
        lo, so = o.evaluate(pr_o.full_evaluation(0))
        assert not se.any() and abs(le[0] - lo[0]) <= 2e-7 * abs(lo[0])

    pr_e = workloads.make_problem(4, 4, 97, 7, 2, seed=8)
    with pr_e.create(engine_lib, max_evaluations=2) as e:
        full = pr_e.full_evaluation(0)
        want, _ = e.evaluate(full)
        # root integration only: no matrix updates, no node updates, same buffers -> same lnL, bit for bit
        root_only = abi.EvalSpec(mats=full.mats[:0], ops=full.ops[:0], site_dst=abi.NONE, site_src=full.site_dst,
                                 root=full.root, weights_row=full.weights_row, flags=full.flags, p_invar=full.p_invar,
                                 has_p_invar=full.has_p_invar, rates=full.rates, cat_weights=full.cat_weights, freqs=full.freqs)
        got, st = e.evaluate(root_only)
        assert not st.any() and np.array_equal(got, want)
        # no root: buffers are updated, lnL comes back as 0 / OK
        other = pr_e.full_evaluation(1)
        no_root = abi.EvalSpec(mats=other.mats, ops=other.ops, site_dst=other.site_dst, site_src=other.site_src,
                               root=abi.NONE, weights_row=0, flags=other.flags, p_invar=other.p_invar,
                               has_p_invar=other.has_p_invar, rates=other.rates, cat_weights=other.cat_weights, freqs=other.freqs)
        l0, s0 = e.evaluate(no_root)
        assert l0[0] == 0.0 and s0[0] == 0
        # ... and a root-only pass over them gives what a fused evaluation gives
        pr_f = workloads.make_problem(4, 4, 97, 7, 2, seed=8)
        with pr_f.create(engine_lib, max_evaluations=2) as f:
            f.evaluate(pr_f.full_evaluation(0))
            wantf, _ = f.evaluate(pr_f.full_evaluation(1))
        root_only1 = abi.EvalSpec(mats=other.mats[:0], ops=other.ops[:0], site_dst=abi.NONE, site_src=other.site_dst,
                                  root=other.root, weights_row=other.weights_row, flags=other.flags, p_invar=other.p_invar,
                                  has_p_invar=other.has_p_invar, rates=other.rates, cat_weights=other.cat_weights, freqs=other.freqs)
        l1, s1 = e.evaluate(root_only1)
        assert not s1.any() and np.array_equal(l1, wantf)

        # invalid indices are refused before anything is launched
        bad = pr_e.full_evaluation(0)
        bad.ops = bad.ops.copy(); bad.ops[0]["dest"] = 10 ** 6
        with pytest.raises(abi.AbiError):
            e.evaluate(bad)
        bad = pr_e.full_evaluation(0)
        bad.mats = bad.mats.copy(); bad.mats[0]["matrix"] = -5
        with pytest.raises(abi.AbiError):
            e.evaluate(bad)
        with pytest.raises(abi.AbiError):
            e.evaluate([pr_e.full_evaluation(0)] * 3)          # more evaluations than max_evaluations
        # the instance is still usable afterwards
        again, st = e.evaluate(pr_e.full_evaluation(0))
        assert not st.any() and np.isfinite(again).all()


# ---------------------------------------------------------------------------------------------
# variable-state (STANDARD data) divisions: the *_Std kernel family
# ---------------------------------------------------------------------------------------------
STD_CASES = [
    # C, K, tips, max states, dummy patterns
    (162, 4, 32, 8, 2),       # cynmix's morphology partition: size and shape
    (1, 4, 4, 2, 0),
    (33, 1, 5, 3, 2),
    (70, 5, 6, 10, 2),        # L = 8 lanes per pattern
    (129, 2, 7, 4, 4),
    (40, 10, 5, 6, 0),        # L = 16
    (37, 4, 6, 16, 2),
    (25, 3, 5, 24, 2),        # MAX_STD_STATES
]


@pytest.mark.parametrize("C,K,tips,smax,dummy", STD_CASES)
def test_variable_state_engine_matches_oracle(engine_lib, oracle_lib, C, K, tips, smax, dummy):
    """Mk + gamma on patterns with their own state counts: P(t), every written conditional-likelihood
    buffer (ragged host layout), node and site scalers, and lnL with the coding-bias correction."""
    nch = 2
    pr = workloads.make_std_problem(C, K, tips, nch, seed=900 + C + K + smax, max_states=smax, dummy=dummy)
    rng = np.random.default_rng(11)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        for it, sp in evaluation_sequence(pr, 12, seed=rng):
            check_with_oracle(e, o, [sp], *e.evaluate(sp), 1e-9, parity_tol(smax))
            if it < 0:
                for m in sp.mats["matrix"][:5]:
                    assert np.allclose(e.get_transition_matrix(int(m)), o.get_transition_matrix(int(m)), rtol=2.5e-7,
                                       atol=1e-30)
        assert e.kernel_launches(abi.KERNEL_STD) == nch + 12        # the variable-state kernel served every call
        # all chains of a generation in one launch == one call per chain
        sps = [pr.random_branch_update(ch, rng) for ch in range(nch)]
        lb, _ = e.evaluate(sps)
        lo2 = np.array([o.evaluate(sp)[0][0] for sp in sps])
        assert np.allclose(lb, lo2, rtol=1e-9)


def test_variable_state_general_matrices(engine_lib, oracle_lib):
    """Caller-supplied transition matrices (mb200_set_transition_matrix) need not have the Mk form:
    the kernel then reads every entry."""
    pr = workloads.make_std_problem(60, 2, 5, 1, seed=77, max_states=5, dummy=2)
    rng = np.random.default_rng(3)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        sp = pr.full_evaluation(0)
        (l0,), _ = e.evaluate(sp)
        (o0,), _ = o.evaluate(sp)
        assert rel(l0, o0) < 1e-9
        # re-load one matrix unchanged: same lnL through the general path
        m = int(sp.mats["matrix"][0])
        e.set_transition_matrix(m, e.get_transition_matrix(m))
        sp2 = abi.EvalSpec(ops=sp.ops[-1:].copy(), site_dst=sp.site_dst, site_src=sp.site_dst, root=sp.root, rates=sp.rates,
                           cat_weights=sp.cat_weights, freqs=sp.freqs)
        sp2.ops["scale_remove"] = abi.NONE
        (l1,), _ = e.evaluate(sp2)
        (o1,), _ = o.evaluate(sp2)
        assert rel(l1, o1) < 1e-9


def test_tensor_core_kernel_serves_20_and_61_states(engine_lib):
    """S = 20 and S = 61 must run on the wgmma kernel, not on the CUDA-core correctness path
    (which would pass the same parity tolerance)."""
    for S, K in ((20, 4), (20, 1), (61, 1), (61, 3)):          # (61, 3): omega categories (NY98 / M3)
        pr = workloads.make_problem(S, K, 300, 8, 1, seed=3)
        with pr.create(engine_lib) as e:
            e.evaluate(pr.full_evaluation(0))
            assert e.kernel_launches(abi.KERNEL_TENSOR) == 1
            assert e.kernel_launches(abi.KERNEL_GENERIC) == 0
    pr = workloads.make_problem(4, 4, 300, 8, 1, seed=3)
    with pr.create(engine_lib) as e:
        e.evaluate(pr.full_evaluation(0))
        assert e.kernel_launches(abi.KERNEL_NUC4) == 1 and e.kernel_launches(abi.KERNEL_TENSOR) == 0
