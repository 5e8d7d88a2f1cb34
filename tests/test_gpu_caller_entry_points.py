"""GPU: the caller-facing entry points of include/mb200.h beyond mb200_evaluate, on every kernel family -- the node-
granular verbs (update_transition_matrices, reset / copy_scalers, update_partials, root_log_likelihood), caller-set P(t)
(set_transition_matrix: the pinned ring, and on the tensor cores tc_split_kernel's operand images) and seeded partials and
scalers (set_partials / set_scalers), on the launch paths and between resident 4-state generations.

Each call is checked on its own inputs against the float64 reference of one evaluation (f64_reference.f64_evaluation,
bars in engine_checks.f64_call_check); each evaluation against the CPU oracle; and the verbs against the fused evaluation
bit for bit, since they run the same kernels in the same float order."""
import numpy as np
import pytest

from engine_checks import (FLT_MIN, SYN_RTOL, ULP, check_with_oracle, edge, evaluation_sequence, f64_call_check, f64_inputs,
                           foreign_matrix, generation_sequence, lnl_tol, num_sms, resident_generations,
                           rel, seed_chain, seeded_partials, seeded_scalers, tree_tol, via_evaluate, via_replay)
from f64_reference import std_mk_block, transition_matrices
from mrbayes_b200 import abi, workloads

pytestmark = pytest.mark.gpu

ERROR_OUT_OF_RANGE, ERROR_UNSUPPORTED = -3, -5
PART_SCALE = (0.5, 1.0, 2.0)          # three eigen parts: part k is the problem's rate matrix times PART_SCALE[k]


# ---- the instances ------------------------------------------------------------------------------------------------
class Case:
    """A problem, how its instances are created, the kernel family that must serve it and the route its fused
    evaluations take"""

    def __init__(self, pr, kind, route=via_evaluate, flags=0, parts=1):
        self.pr, self.kind, self.route, self.flags, self.parts = pr, kind, route, flags, parts

    @property
    def tensor(self):
        return self.kind == abi.KERNEL_TENSOR

    def create(self, lib):
        pr = self.pr
        if self.parts == 1:
            return pr.create(lib, flags=self.flags)
        cfg = pr.config()
        inst = abi.Instance(lib, flags=self.flags | (self.parts << 8), **cfg)
        for t in range(pr.n_tips):
            inst.set_tip_states(t, pr.masks[t])
        inst.set_pattern_weights(0, pr.weights)
        S = pr.S
        cijk = np.einsum("is,sj->ijs", pr.V, pr.Vinv).ravel()
        inst.set_cijk(0, np.concatenate([np.concatenate([pr.lam * f, np.zeros(S), cijk]) for f in PART_SCALE]))
        return inst

    @property
    def Q(self):
        """per-category rate matrices of a case with eigen parts, else None (the problem's eigensystem)"""
        if self.parts == 1:
            return None
        Q = (self.pr.V * self.pr.lam) @ self.pr.Vinv
        return np.stack([f * Q for f in PART_SCALE])

    def pmat(self, length, rates, freqs):
        """float64 P(t) of a matrix update"""
        pr = self.pr
        if isinstance(pr, workloads.StdProblem):
            return std_mk_block(pr, length, rates)
        scale = np.asarray(PART_SCALE) if self.parts > 1 else 1.0
        return transition_matrices(pr, length, np.asarray(rates) * scale, freqs=freqs)


NUC4_TILES = {"host": 3, "device": 20, "non_fused": None, "throughput": 5}


def nuc4_case(K, route):
    tiles = NUC4_TILES[route] or 4 * num_sms() + 4
    pr = workloads.make_problem(4, K, edge(K, tiles), 12 if route in ("throughput", "non_fused") else 16, 2,
                                seed=900 + 7 * K, p_invar=0.15 if K % 2 else 0.0, p_ambig=0.1 if K % 2 else 0.0)
    return Case(pr, abi.KERNEL_NUC4, via_replay if route == "device" else via_evaluate,
                abi.CONFIG_THROUGHPUT if route == "throughput" else 0)


def other_case(name):
    if name == "std":
        pr = workloads.make_std_problem(150, 3, 10, 2, seed=41)          # state counts {2, 3, 4, 6}: 15 frequencies, S = 6
        return Case(pr, abi.KERNEL_STD)
    S, K, C, tips, pinv, parts = {"nuc4-K10": (4, 10, 60, 9, 0.1, 1), "tensor20-K1": (20, 1, 129, 9, 0.0, 1),
                                  "tensor20-K4": (20, 4, 100, 8, 0.1, 1), "tensor61-K1": (61, 1, 130, 7, 0.0, 1),
                                  "tensor61-K3-parts3": (61, 3, 70, 6, 0.0, 3), "generic16": (16, 4, 90, 9, 0.1, 1),
                                  "generic40": (40, 2, 50, 7, 0.0, 1), "generic64": (64, 2, 40, 6, 0.0, 1)}[name]
    pr = workloads.make_problem(S, K, C, tips, 2, seed=950 + S + K, p_invar=pinv, p_ambig=0.05)
    kind = abi.KERNEL_TENSOR if (S, K) in ((20, 1), (20, 4), (61, 1), (61, 3)) else abi.KERNEL_GENERIC
    return Case(pr, kind, parts=parts)


OTHER = ["nuc4-K10", "tensor20-K1", "tensor20-K4", "tensor61-K1", "tensor61-K3-parts3", "generic16", "generic40",
         "generic64", "std"]
ALL_CASES = [f"nuc4-K{K}-{r}" for K in range(1, 9) for r in NUC4_TILES] + OTHER
# Where the verbs' lnL is not the fused evaluation's bit for bit (every buffer still is).  Throughput mode serves an
# evaluation with one CTA only when its operations fit one chunk; at K = 1 a chunk holds 8 nodes, so the fused full
# evaluation of 12 tips (10 nodes) runs tiled with its tile sums added on the host, while root_log_likelihood (no
# nodes) runs on one CTA that adds the tiles itself: the same terms, summed in another order.
LNL_ORDER_DIFFERS = {"nuc4-K1-throughput"}
ONE_PER_FAMILY = ["nuc4-K4-host", "nuc4-K5-device", "nuc4-K10", "tensor20-K4", "tensor61-K3-parts3", "generic16", "std"]


def make_case(name):
    if name.startswith("nuc4-K") and name.count("-") == 2:
        _, k, route = name.split("-")
        return nuc4_case(int(k[1:]), route)
    return other_case(name)


def assert_family(e, case, tiprobs=None):
    """the instance's launches went to case's family, and to no other evaluation kernel"""
    for kind in (abi.KERNEL_NUC4, abi.KERNEL_TENSOR, abi.KERNEL_GENERIC, abi.KERNEL_STD):
        n = e.kernel_launches(kind)
        assert (n > 0) if kind == case.kind else (n == 0), f"kernel kind {kind}: {n} launches"
    if tiprobs is not None:
        assert (e.kernel_launches(abi.KERNEL_TIPROBS) > 0) == tiprobs


def oracle_tol(case):
    """tree_tol; on the tensor cores with a floor of three flushed products (below FLT_MIN each) per term of each
    operation, for the foreign matrices' tiny entries and the seeded partials just above FLT_MIN"""
    base = tree_tol(case.pr)
    if not case.tensor:
        return base

    def tol(sp):
        from dataclasses import replace
        return replace(base(sp), partials_atol=3 * case.pr.S * FLT_MIN * len(sp.ops))
    return tol


def without_updates(sp):
    """sp with no matrix updates: the branches keep what the matrix buffers hold"""
    out = abi.EvalSpec(ops=sp.ops, site_dst=sp.site_dst, site_src=sp.site_src, root=sp.root, weights_row=sp.weights_row,
                       flags=sp.flags, p_invar=sp.p_invar, has_p_invar=sp.has_p_invar, rates=sp.rates,
                       cat_weights=sp.cat_weights, freqs=sp.freqs, chain=sp.chain)
    return out


def written_state(e, sp):
    """every buffer sp wrote on e"""
    parts = [e.get_partials(int(op["dest"])) for op in sp.ops]
    scal = [e.get_scalers(int(op["scale_write"])) for op in sp.ops if op["scale_write"] >= 0]
    if sp.site_dst >= 0:
        scal.append(e.get_scalers(sp.site_dst))
    return parts, scal


def same_state(a, b, sp):
    pa, sa = written_state(a, sp)
    pb, sb = written_state(b, sp)
    return all(np.array_equal(x, y) for x, y in zip(pa + sa, pb + sb))


def assert_same_state(a, b, sp, what):
    pa, sa = written_state(a, sp)
    pb, sb = written_state(b, sp)
    for op, x, y in zip(sp.ops, pa, pb):
        assert np.array_equal(x, y), f"{what}: partials of buffer {op['dest']} differ"
    for i, (x, y) in enumerate(zip(sa, sb)):
        assert np.array_equal(x, y), f"{what}: scaler {i} of the evaluation differs"


# ---- the node-granular verbs --------------------------------------------------------------------------------------
def verbs(e, case, sp, per_op, used):
    """sp as LaunchLogLikeForDivision decomposes it: P(t), reset / copy of the site scaler, the node updates (one call
    per operation, or all in one), the root.  Every call is checked against f64_evaluation on the inputs it read.
    -> (lnL, status); used[0] takes the largest fraction of a float64 bar."""
    pr = case.pr
    if len(sp.mats):
        e.update_transition_matrices(sp.mats, sp.rates, sp.freqs)
        for mu in sp.mats:
            want = case.pmat(float(mu["length"]), sp.rates, sp.freqs[:pr.S])
            got = e.get_transition_matrix(int(mu["matrix"])).astype(np.float64)
            # float rounding of a double eigen-sum of S terms
            bar = ULP * np.abs(want) + pr.S * 1e-15
            used[0] = max(used[0], float((np.abs(got - want) / bar).max()))
            assert (np.abs(got - want) <= bar).all(), f"P(t) of matrix {mu['matrix']}"
    if sp.site_src == abi.NONE:
        e.reset_scalers(sp.site_dst)
    else:
        e.copy_scalers(sp.site_dst, sp.site_src)
    groups = [sp.ops[i:i + 1] for i in range(len(sp.ops))] if per_op else [sp.ops]
    for ops in groups:
        # update_partials carries no evaluation flags: no tip shortcuts (include/mb200.h)
        call = abi.EvalSpec(ops=ops, site_dst=sp.site_dst, site_src=sp.site_dst, rates=sp.rates, freqs=sp.freqs,
                            flags=0)
        inputs = f64_inputs(e, call)
        e.update_partials(ops, sp.site_dst)
        used[0] = max(used[0], f64_call_check(e, pr, call, _f64(pr, call, inputs), case.tensor))
    root = abi.EvalSpec(site_src=sp.site_dst, root=sp.root, weights_row=sp.weights_row, flags=sp.flags,
                        p_invar=sp.p_invar, has_p_invar=sp.has_p_invar, rates=sp.rates, cat_weights=sp.cat_weights,
                        freqs=sp.freqs)
    inputs = f64_inputs(e, root)
    lnl, st = e.root_log_likelihood(sp.root, sp.site_dst, sp.weights_row, sp.freqs, sp.cat_weights, sp.has_p_invar,
                                    sp.p_invar, sp.flags)
    used[0] = max(used[0], f64_call_check(e, pr, root, _f64(pr, root, inputs), case.tensor, st, lnl))
    return lnl, st


def _f64(pr, sp, inputs, Q=None):
    from f64_reference import f64_evaluation
    return f64_evaluation(pr, sp, *inputs, Q=Q)


@pytest.mark.parametrize("name", ALL_CASES)
def test_verbs_equal_fused_evaluation(engine_lib, oracle_lib, name, record_property):
    """Full evaluations, then branch updates with every third rejected (scale_remove and copy_scalers at work): the
    verbs -- one update_partials call per operation on one instance, all operations in one call on another -- give
    the fused evaluation's lnL, status, partials and node and site scalers bit for bit (LNL_ORDER_DIFFERS: lnL within
    lnl_tol, and it does differ).  The fused twin and the oracle take the flags the verbs carry, without tip
    shortcuts.  Every verb call is within the float64 bars of its own inputs, every decomposed evaluation within
    tree_tol of the oracle, and the kernel counters show the family that served it."""
    case = make_case(name)
    pr = case.pr
    used, worst = [0.0], np.zeros(3)
    lnl_differs = False
    with case.create(engine_lib) as each, case.create(engine_lib) as whole, case.create(engine_lib) as fused, \
            case.create(oracle_lib) as o:
        o.set_arith(1)
        for it, sp in evaluation_sequence(pr, 6, seed=3):
            sp.flags &= ~abi.FLAG_TIP_SHORTCUTS
            (lf,), (sf,) = case.route(fused, [sp])
            le, se = verbs(each, case, sp, True, used)
            lw, sw = verbs(whole, case, sp, False, used)
            for e, l, st, how in ((each, le, se, "one operation per call"), (whole, lw, sw, "all operations in one call")):
                assert st == sf, f"evaluation {it}, {how}: status {st}, fused {sf}"
                what = f"evaluation {it}, {how}"
                assert_same_state(e, fused, sp, what)
                if name in LNL_ORDER_DIFFERS:
                    lnl_differs |= l != lf
                    assert rel(l, lf) < lnl_tol(pr.S), f"{what}: {l!r}, fused {lf!r}"
                else:
                    assert l == lf, f"{what}: {l!r}, fused {lf!r}"
            worst = np.maximum(worst, check_with_oracle(each, o, [sp], [le], [se], lnl_tol(pr.S), tree_tol(pr)))
        tiprobs = None if case.kind != abi.KERNEL_NUC4 else name.endswith("non_fused")
        for e in (each, whole, fused):
            assert_family(e, case, tiprobs)
        # the eigensystem of an evaluation cannot travel with a verb
        mats = sp.mats.copy() if len(sp.mats) else np.array([(0, 0, 0.1)], abi.MAT_DTYPE)
        mats["eigen"] = abi.EIGEN_INLINE
        with pytest.raises(abi.AbiError) as err:
            each.update_transition_matrices(mats, sp.rates, sp.freqs)
        assert err.value.code == ERROR_UNSUPPORTED
    assert lnl_differs == (name in LNL_ORDER_DIFFERS), "LNL_ORDER_DIFFERS no longer describes this case"
    record_property("oracle_lnl_rel", float(worst[0]))
    record_property("f64_bar_used", used[0])


@pytest.mark.parametrize("S,K", [(4, 4), (16, 4), (20, 4)])
def test_update_partials_takes_no_tip_shortcuts(engine_lib, oracle_lib, S, K):
    """Tips without partial ambiguity but with missing observations, where MB200_FLAG_TIP_SHORTCUTS makes a missing
    observation contribute exactly 1: update_partials, which carries no flags, sums the P(t) row instead.  The verbs
    equal, bit for bit, the fused evaluation without the flag, and differ from it with the flag"""
    short = abi.FLAG_TIP_SHORTCUTS | (abi.FLAG_NUC4_PINVAR_QUIRK if S == 4 else 0)
    pr = workloads.make_problem(S, K, 90, 10, 2, seed=970 + S, p_missing=0.1, p_ambig=0.0, flags=short)
    full = np.uint64((1 << S) - 1)
    single = (pr.masks & (pr.masks - np.uint64(1))) == 0
    assert ((pr.masks == full) | single).all() and (pr.masks == full).any(axis=1).all()
    case = Case(pr, abi.KERNEL_NUC4 if S == 4 else abi.KERNEL_TENSOR if S == 20 else abi.KERNEL_GENERIC)
    used, with_flag_differs = [0.0], False
    with case.create(engine_lib) as each, case.create(engine_lib) as plain, case.create(engine_lib) as flagged, \
            case.create(oracle_lib) as o:
        o.set_arith(1)
        for it, sp in evaluation_sequence(pr, 4, seed=1):
            assert sp.flags & abi.FLAG_TIP_SHORTCUTS
            (ls,), _ = flagged.evaluate(sp)
            bare = without_updates(sp)
            bare.mats, bare.flags = sp.mats, sp.flags & ~abi.FLAG_TIP_SHORTCUTS
            (lp,), (sp_st,) = plain.evaluate(bare)
            le, se = verbs(each, case, bare, True, used)
            assert le == lp and se == sp_st, f"evaluation {it}: verbs {le!r}, fused without shortcuts {lp!r}"
            assert_same_state(each, plain, bare, f"evaluation {it}")
            with_flag_differs |= ls != le or not same_state(flagged, each, bare)
            check_with_oracle(each, o, [bare], [le], [se], lnl_tol(S), tree_tol(pr))
        assert with_flag_differs, "no evaluation took a tip shortcut"


def test_update_transition_matrices_needs_frequencies(engine_lib):
    """NULL state_freqs: refused where P(t) has stationary rows, accepted on a variable-state instance"""
    for name, ok in (("nuc4-K4-host", False), ("generic16", False), ("tensor20-K1", False), ("std", True)):
        case = make_case(name)
        pr = case.pr
        with case.create(engine_lib) as e:
            sp = pr.full_evaluation(0)
            if ok:
                e.update_transition_matrices(sp.mats, sp.rates, None)
            else:
                with pytest.raises(abi.AbiError) as err:
                    e.update_transition_matrices(sp.mats, sp.rates, None)
                assert err.value.code == ERROR_OUT_OF_RANGE, name


def test_std_root_log_likelihood_reads_whole_frequency_table(engine_lib, oracle_lib):
    """A variable-state division whose frequency table (15 entries: classes 2, 3, 4 and 6) is longer than its state
    count (6): root_log_likelihood over the buffers a fused evaluation wrote gives that evaluation's lnL bit for bit"""
    case = other_case("std")
    pr = case.pr
    assert len(pr.freqs) > pr.S and (pr.freq_offsets + pr.state_counts).max() == len(pr.freqs)
    with case.create(engine_lib) as e, case.create(oracle_lib) as o:
        for ch in range(pr.n_chains):
            sp = pr.full_evaluation(ch)
            (want,), (ws,) = e.evaluate(sp)
            (lo,), _ = o.evaluate(sp)
            got, st = e.root_log_likelihood(sp.root, sp.site_dst, 0, sp.freqs, sp.cat_weights)
            assert ws == st == abi.EVAL_OK, f"chain {ch}: status {st}"
            assert got == want, f"chain {ch}: root_log_likelihood {got!r}, evaluate {want!r}"
            assert abs(got - lo) < SYN_RTOL * abs(lo)


# ---- caller-set P(t) ----------------------------------------------------------------------------------------------
MATRIX_CASES = ["nuc4-K4-host", "nuc4-K3-non_fused", "nuc4-K10", "tensor20-K1", "tensor20-K4", "tensor61-K1",
                "tensor61-K3-parts3", "generic16", "generic40", "std"]


@pytest.mark.parametrize("name", MATRIX_CASES)
def test_set_transition_matrix_round_trip(engine_lib, name):
    """get_transition_matrix -> set_transition_matrix of every branch of an engine-built evaluation, then the same
    evaluation without matrix updates: bit for bit the engine-built result.  At 61 states this pins tc_split_kernel's
    operand images against the ones tiprobs_mm_kernel writes; at 20 states the engine-built images come from
    tc_split_kernel too (after tiprobs_kernel), so there the round trip pins the ring and the copy only, and
    test_foreign_transition_matrices holds tc_split_kernel to the oracle."""
    case = make_case(name)
    pr = case.pr
    with case.create(engine_lib) as a, case.create(engine_lib) as b:
        for ch in range(pr.n_chains):
            sp = pr.full_evaluation(ch)
            (la,), (sa,) = case.route(a, [sp])
            setup = b.kernel_launches(abi.KERNEL_SETUP)
            for m in sp.mats["matrix"]:
                b.set_transition_matrix(int(m), a.get_transition_matrix(int(m)))
            if case.tensor:
                assert b.kernel_launches(abi.KERNEL_SETUP) - setup == len(sp.mats)      # one tc_split_kernel each
            (lb,), (sb,) = case.route(b, [without_updates(sp)])
            assert lb == la and sb == sa == abi.EVAL_OK, f"chain {ch}: {lb!r} vs {la!r}"
            assert_same_state(a, b, sp, f"chain {ch}")
        assert b.kernel_launches(abi.KERNEL_TIPROBS) == 0
        assert_family(b, case)


@pytest.mark.parametrize("name", MATRIX_CASES)
def test_foreign_transition_matrices(engine_lib, oracle_lib, name, record_property):
    """Stochastic, non-reversible matrices with exact zeros, entries of 1e-30 and subnormal ones, and identity rows on
    every branch (full evaluations), then on the branch of each update: against the oracle given the same matrices
    and against f64_evaluation over the matrices read back"""
    case = make_case(name)
    pr = case.pr
    rng = np.random.default_rng(11)
    used, worst = 0.0, np.zeros(3)
    with case.create(engine_lib) as e, case.create(oracle_lib) as o:
        o.set_arith(1)
        for it, sp in evaluation_sequence(pr, 4, seed=rng):
            for m in sp.mats["matrix"]:
                P = foreign_matrix(pr, rng)
                e.set_transition_matrix(int(m), P)
                o.set_transition_matrix(int(m), P)
            sp = without_updates(sp)
            inputs = f64_inputs(e, sp)
            lnl, st = case.route(e, [sp])
            worst = np.maximum(worst, check_with_oracle(e, o, [sp], lnl, st, lnl_tol(pr.S), oracle_tol(case)))
            used = max(used, f64_call_check(e, pr, sp, _f64(pr, sp, inputs), case.tensor, st[0], lnl[0]))
        assert_family(e, case)
    record_property("oracle_lnl_rel", float(worst[0]))
    record_property("f64_bar_used", used)


@pytest.mark.parametrize("name", ["nuc4-K4-host", "generic16", "std"])
def test_set_transition_matrix_ring_wrap(engine_lib, oracle_lib, name):
    """More than 64 set_transition_matrix calls between two evaluations -- the pinned ring wraps -- with some matrices
    written twice: the last write wins, on every branch, against the oracle"""
    case = make_case(name)                              # 40 tips: 77 branches
    pr = case.pr = (workloads.make_std_problem(150, 3, 40, 2, seed=41) if name == "std" else
                    workloads.make_problem(case.pr.S, case.pr.K, case.pr.C, 40, 2, seed=77))
    if name == "generic16":
        assert (pr.S, pr.K) == (16, 4)
    rng = np.random.default_rng(5)
    with case.create(engine_lib) as e, case.create(oracle_lib) as o:
        o.set_arith(1)
        sp = pr.full_evaluation(0)
        check_with_oracle(e, o, [sp], *e.evaluate(sp), lnl_tol(pr.S), tree_tol(pr))
        sp = pr.full_evaluation(0)
        mats = [int(m) for m in sp.mats["matrix"]]
        twice = set(rng.choice(mats, 8, replace=False).tolist())
        last = {}
        calls = 0
        for m in mats + sorted(twice):
            P = foreign_matrix(pr, rng)
            e.set_transition_matrix(m, P)
            o.set_transition_matrix(m, P)
            last[m] = P
            calls += 1
        assert calls > 64
        sp = without_updates(sp)
        check_with_oracle(e, o, [sp], *e.evaluate(sp), lnl_tol(pr.S), tree_tol(pr))
        for m, P in last.items():
            assert np.array_equal(e.get_transition_matrix(m), P), f"matrix {m}"


# ---- seeded partials and scalers ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ONE_PER_FAMILY)
def test_seeded_partials_and_scalers(engine_lib, oracle_lib, name, record_property):
    """set_partials / set_scalers on each chain's interior partials, node scalers and site scaler -- zeros, values just
    above FLT_MIN, patterns peaking in different categories -- then branch updates whose clean operands, scale_remove
    buffers and site_scaler_src are the seeded ones: against the oracle seeded the same way and f64_evaluation"""
    case = make_case(name)
    pr = case.pr
    rng = np.random.default_rng(13)
    used, removed, worst = 0.0, 0, np.zeros(3)
    with case.create(engine_lib) as e, case.create(oracle_lib) as o:
        o.set_arith(1)
        for ch in range(pr.n_chains):
            sp = pr.full_evaluation(ch)
            case.route(e, [sp]); o.evaluate(sp)
            seed_chain([e, o], pr, ch, rng)
            x = seeded_partials(pr, rng)
            assert (x == 0).any() and ((x > 0) & (x < 4 * FLT_MIN)).any()
        for it in range(8):
            ch = it % pr.n_chains
            sp = pr.random_branch_update(ch, rng)
            removed += int((sp.ops["scale_remove"] >= 0).sum())
            assert sp.site_src >= 0
            inputs = f64_inputs(e, sp)
            lnl, st = case.route(e, [sp])
            worst = np.maximum(worst, check_with_oracle(e, o, [sp], lnl, st, lnl_tol(pr.S), oracle_tol(case)))
            used = max(used, f64_call_check(e, pr, sp, _f64(pr, sp, inputs, case.Q), case.tensor, st[0], lnl[0]))
        assert removed > 0
        assert_family(e, case)
    record_property("oracle_lnl_rel", float(worst[0]))
    record_property("f64_bar_used", used)


# ---- between resident 4-state generations -------------------------------------------------------------------------
def test_set_calls_between_resident_generations(engine_lib, oracle_lib):
    """set_transition_matrix, set_partials and set_scalers before every third resident generation, on data that
    generation reads (a clean operand, a matrix it does not rebuild, its site_scaler_src): the generation sees the new
    data -- the oracle given the same calls agrees, and the lnL differs from the run without them -- and the resident
    kernel gives, bit for bit, what one launch per generation with the same calls gives"""
    pr = workloads.make_problem(4, 4, edge(4, 12), 16, 2, seed=17)
    gens = [specs for _, specs in generation_sequence(pr, 9, 5)]
    rng = np.random.default_rng(19)
    calls = {}
    for g in range(3, len(gens), 3):
        calls[g] = []
        for sp in gens[g]:
            dests = {int(op["dest"]) for op in sp.ops}
            rebuilt = {int(m) for m in sp.mats["matrix"]}
            clean = [int(op[f]) for op in sp.ops for f in ("child1", "child2")
                     if int(op[f]) >= pr.n_tips and int(op[f]) not in dests]
            m = next(int(op[f]) for op in sp.ops for f in ("matrix1", "matrix2") if int(op[f]) not in rebuilt)
            calls[g].append((clean[:1], seeded_partials(pr, rng), m, foreign_matrix(pr, rng), sp.site_src,
                             seeded_scalers(pr, rng, 100.0)))
        assert any(c for c, *_ in calls[g])

    def before(g, inst):
        for clean, x, m, P, site, v in calls.get(g, ()):
            for b in clean:
                inst.set_partials(b, x)
            inst.set_transition_matrix(m, P)
            inst.set_scalers(site, v)

    dests = sorted({int(op["dest"]) for specs in gens for sp in specs for op in sp.ops})
    with pr.create(engine_lib) as e:
        n0 = e.launch_count()
        got = resident_generations(e, gens, before)
        launches = e.launch_count() - n0
        e.synchronize()
        got_parts = [e.get_partials(b) for b in dests]
    assert launches < len(gens)
    with pr.create(engine_lib) as e, pr.create(engine_lib) as plain, pr.create(oracle_lib) as o:
        o.set_arith(1)
        for g, specs in enumerate(gens):
            before(g, e)
            before(g, o)
            lnl, st = via_replay(e, specs)
            lp, _ = via_replay(plain, specs)
            assert np.array_equal(lnl, got[g][0]) and np.array_equal(st, got[g][1]), f"generation {g}"
            check_with_oracle(e, o, specs, lnl, st, lnl_tol(4), tree_tol(pr))
            if g in calls:
                assert not np.array_equal(lnl, lp), f"generation {g} did not see the set calls"
        assert all(np.array_equal(a, e.get_partials(b)) for a, b in zip(got_parts, dests))
