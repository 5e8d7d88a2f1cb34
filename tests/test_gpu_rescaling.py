"""GPU: sparse rescaling and the float-range guard (MB200_FLAG_RANGE_GUARD) on every kernel route.

With rescaling at every node, an operation never leaves a node unscaled and never removes an old
scaler without writing a new one.  The dynamic rescaling scheme does both (tests/sparse_rescaling.py
builds its operation lists), and asks for the guard on 4-state divisions.  Each test here shows the
route it took (kernel counters) and compares with the CPU oracle (set_arith(1)) and with the float64
reference.  Partials can be tiny when nodes go unscaled, so they are compared with a relative
tolerance and an absolute floor of 1e-44 (the subnormal range), not the parity suite's 1e-37
(engine_checks.sparse_tol).

  sparse parity      f in {1, 2, 3, 7, inf} on the 4-state routes, tensor core, generic kernel, Std
  deep subtrees      an 80-tip caterpillar with the guard off: scale4's division branch (a maximum
                     <= 1e-30) and log_of_max's library branch (a subnormal maximum)
  guard contract     flag set, 4-state K = 1..20: the oracle's status; lnL within 1e-6 of float64 when OK
  guard threshold    a node maximum / root likelihood of exactly 1e-24f, the float below and 1.00003e-24f
  other families     the flag is ignored for S != 4 and Std"""
import numpy as np
import pytest

from engine_checks import (DBL_MAX, SYN_RTOL, assert_resident_equals_launches, check_with_oracle, compare_written,
                           edge, evaluation_sequence, lnl_tol, num_sms, nuc4_problem, ppb, rel, sparse_tol,
                           via_evaluate, via_replay)
from f64_reference import caterpillar_tree, f64_lnl
from mrbayes_b200 import abi, workloads
from sparse_rescaling import (GUARD_MIN, deep_problem, run_threshold, sparse_rescaling, step_frequency,
                              threshold_instance, threshold_setup, threshold_spec, unscaled_maxima)

pytestmark = pytest.mark.gpu

FREQS = [1, 2, 3, 7, np.inf]


def remove_only(sp):
    return int(((sp.ops["scale_remove"] >= 0) & (sp.ops["scale_write"] < 0)).sum())


def sparse_run(pr, e, o, route, f, updates=10, seed=0):
    """A full evaluation per chain, then `updates` branch updates (the frequency stepping between f
    and f + 1) with every third rejected: status, lnL and every written buffer against the oracle,
    lnL against float64 (not for Std) after each full evaluation and the last update.  -> calls made"""
    tol = lnl_tol(pr.S)
    calls = n_remove_only = 0
    for it, sp in evaluation_sequence(pr, updates, seed, before_update=lambda it: step_frequency(pr, f, it)):
        lnl, st = route(e, [sp])
        calls += 1
        n_remove_only += remove_only(sp)
        check_with_oracle(e, o, [sp], lnl, st, tol, sparse_tol(pr))
        if (it < 0 or it == updates - 1) and not isinstance(pr, workloads.StdProblem):
            r = rel(lnl[0], f64_lnl(pr, sp.chain)[1])
            assert r < tol, f"float64 reference, evaluation {it}: {r:.2e}"
    assert (n_remove_only > 0) == (1 < f < np.inf)           # the lists hold remove-only operations
    return calls


# ---- sparse parity -------------------------------------------------------------------------------
NUC4_C = {"host": lambda K: edge(K, 3), "device": lambda K: edge(K, 20),
          "non_fused": lambda K: edge(K, 4 * num_sms() + 4), "throughput": lambda K: edge(K, 5),
          "resident": lambda K: edge(K, 12)}


@pytest.mark.parametrize("f", FREQS)
@pytest.mark.parametrize("K", [1, 4, 5, 8])
@pytest.mark.parametrize("route", ["host", "device", "non_fused", "throughput"])
def test_sparse_nuc4(engine_lib, oracle_lib, route, K, f):
    """4-state routes; chain 1 is a caterpillar, odd K carry p_invar and ambiguity (nuc4_problem).
    Throughput mode serves single-chunk evaluations only: 12 tips there, 32 elsewhere.  The counters
    tell the non-fused path (a stand-alone P(t) launch per call) from the fused ones; evaluate() at
    these sizes is the parameter-block kernel test_nuc4_fused_parameter_block traces, and pack +
    replay the device blob with its sum over more than 16 tiles."""
    pr = sparse_rescaling(nuc4_problem(K, NUC4_C[route](K), seed=7, tips=12 if route == "throughput" else 32), f)
    flags = abi.CONFIG_THROUGHPUT if route == "throughput" else 0
    with pr.create(engine_lib, flags=flags) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        calls = sparse_run(pr, e, o, via_replay if route == "device" else via_evaluate, f, seed=K)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == (calls if route == "non_fused" else 0)
        if route == "device":
            assert (pr.C + ppb(K) - 1) // ppb(K) > 16          # the device sum over more than 16 tiles


@pytest.mark.parametrize("f", FREQS)
@pytest.mark.parametrize("K", [1, 4, 5, 8])
def test_sparse_nuc4_resident_equals_launches(engine_lib, oracle_lib, K, f):
    """replay_begin / _end: bit for bit what one launch per generation gives; the launches against the oracle"""
    pr = sparse_rescaling(nuc4_problem(K, NUC4_C["resident"](K), seed=8, tips=32), f)
    rng = np.random.default_rng(K)
    gens = [[pr.full_evaluation(0), pr.full_evaluation(1)]]
    for g in range(1, 11):
        old = [pr.tree[ch].length.copy() for ch in (0, 1)]
        step_frequency(pr, f, g)
        gens.append([pr.random_branch_update(ch, rng) for ch in (0, 1)])
        if g % 3 == 2:
            for ch in (0, 1):
                pr.reject(ch, gens[-1][ch], old[ch])
    assert (sum(remove_only(sp) for s in gens for sp in s) > 0) == (1 < f < np.inf)
    assert_resident_equals_launches(engine_lib, oracle_lib, pr, gens, SYN_RTOL, sparse_tol(pr))


@pytest.mark.parametrize("f", FREQS)
@pytest.mark.parametrize("family,S,K", [("tensor", 20, 2), ("tensor", 61, 1), ("tensor", 61, 3),
                                        ("generic", 16, 2), ("generic", 4, 10), ("std", 6, 4)])
def test_sparse_other_families(engine_lib, oracle_lib, family, S, K, f):
    """tensor core (the doScale == false copy-out, the closing item's -old / +new replay), generic
    kernel (m = 1, the remove-only site update; S = 4 with K > 8 runs here) and Std, on 24-tip trees"""
    if family == "std":
        pr = workloads.make_std_problem(90, K, 24, 2, seed=11, max_states=S, dummy=2)
    else:
        pr = workloads.make_problem(S, K, 129, 24, 2, seed=5000 + S + K, p_invar=0.1, p_ambig=0.1)
    pr.tree[1] = caterpillar_tree(24, np.random.default_rng(S + K))
    sparse_rescaling(pr, f)
    kind = {"tensor": abi.KERNEL_TENSOR, "generic": abi.KERNEL_GENERIC, "std": abi.KERNEL_STD}[family]
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        calls = sparse_run(pr, e, o, via_evaluate, f, seed=S + K)
        assert e.kernel_launches(kind) == calls
        assert sum(e.kernel_launches(k) for k in (abi.KERNEL_NUC4, abi.KERNEL_TENSOR, abi.KERNEL_GENERIC,
                                                  abi.KERNEL_STD)) == calls


# ---- deep unscaled subtrees, guard off -------------------------------------------------------------
@pytest.mark.parametrize("f", [40, 50, 68, np.inf])
@pytest.mark.parametrize("route", ["host", "device"])
def test_deep_unscaled_subtrees(engine_lib, oracle_lib, route, f):
    """f = 50 rescales a maximum below 1e-30 (scale4's plain division), f = 68 a subnormal one
    (log_of_max's library log), f = inf leaves 78 levels unscaled.  Status is the oracle's; lnL is
    the float64 reference's while rescaling keeps the values normal (f <= 50), the oracle's beyond"""
    pr = sparse_rescaling(deep_problem(), f)
    fn = via_replay if route == "device" else via_evaluate
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        rng = np.random.default_rng(3)
        lowest = 0.0
        for it in range(-1, 6):
            old = pr.tree[0].length.copy()
            sp = pr.full_evaluation(0) if it < 0 else pr.random_branch_update(0, rng)
            (le,), (se,) = fn(e, [sp])
            (lo,), (so,) = o.evaluate(sp)
            assert se == so, f"evaluation {it}"
            assert rel(le, lo) < SYN_RTOL, f"evaluation {it}: {rel(le, lo):.2e}"
            compare_written(e, o, sp, sparse_tol(pr))
            if f <= 50:
                r = rel(le, f64_lnl(pr, 0)[1])
                assert r < SYN_RTOL, f"float64 reference, evaluation {it}: {r:.2e}"
            for s in sp.ops["scale_write"][sp.ops["scale_write"] >= 0]:
                lowest = min(lowest, float(o.get_scalers(int(s)).min()))
            if it >= 0 and it % 3 == 2:
                pr.reject(0, sp, old)
        assert e.kernel_launches(abi.KERNEL_NUC4) == 7 and e.kernel_launches(abi.KERNEL_TIPROBS) == 0
    # which branches of scale4 / log_of_max the oracle's node scalers say were reached
    assert (lowest < np.log(1e-30)) == (f in (50, 68))
    assert (lowest < np.log(2.0 ** -126)) == (f == 68)


# ---- guard contract ----------------------------------------------------------------------------------
def trips(o, sp, pr):
    """(a rescaler maximum < 1e-24, an unscaled root likelihood < 1e-24) per the oracle's buffers"""
    node = any((o.get_scalers(int(s)) < np.log(1e-24)).any() for s in sp.ops["scale_write"] if s >= 0)
    cl = o.get_partials(sp.root).astype(np.float64)
    like = np.einsum("kcs,s,k->c", cl, np.asarray(pr.freqs, float), sp.cat_weights)
    return node, bool((like < 1e-24).any())


@pytest.mark.parametrize("tips,f", [(60, 8), (60, 20), (60, 48), (60, np.inf), (30, np.inf)])
@pytest.mark.parametrize("K", [1, 4, 5, 8, 10, 20])
def test_guard_contract(engine_lib, oracle_lib, record_property, K, tips, f):
    """Flag set, both chains caterpillars: the engine's status is the oracle's, and an OK lnL is
    within 1e-6 of float64 -- the bar dynamic rescaling is held to.  On 60 tips, f = 48 trips only
    through a rescaler maximum (level 48), f = inf only through the root likelihood (level 58)."""
    pr = nuc4_problem(K, 150, seed=9, tips=tips)
    pr.tree[0] = caterpillar_tree(tips, np.random.default_rng(100 + K))
    pr.flags |= abi.FLAG_RANGE_GUARD
    sparse_rescaling(pr, f)
    rng = np.random.default_rng(K)
    worst, kinds = 0.0, set()
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        for it in range(-2, 10):
            ch = it % 2
            old = pr.tree[ch].length.copy()
            sp = pr.full_evaluation(ch) if it < 0 else pr.random_branch_update(ch, rng)
            (le,), (se,) = e.evaluate(sp)
            (lo,), (so,) = o.evaluate(sp)
            node, root = trips(o, sp, pr)
            kinds.add((node, root))
            assert so == (abi.EVAL_UNDERFLOW if node or root else abi.EVAL_OK), f"oracle, evaluation {it}"
            assert se == so, f"evaluation {it}"
            if se == abi.EVAL_OK:
                r = rel(le, f64_lnl(pr, ch)[1])
                worst = max(worst, r)
                assert r < 1e-6, f"float64 reference, evaluation {it}: {r:.2e}"
            else:
                assert le == lo == -DBL_MAX
            if it >= 0 and it % 3 == 2:
                pr.reject(ch, sp, old)
        assert e.kernel_launches(abi.KERNEL_GENERIC if K > 8 else abi.KERNEL_NUC4) == 12
    record_property("max_rel_err_vs_f64", worst)
    if tips == 60 and f == 48:
        assert (True, False) in kinds
    if tips == 60 and f == np.inf:
        assert (False, True) in kinds


# ---- guard threshold, exact ------------------------------------------------------------------------
THRESHOLD_VALUES = [(GUARD_MIN, abi.EVAL_OK), (np.nextafter(GUARD_MIN, np.float32(0)), abi.EVAL_UNDERFLOW),
                    (np.float32(1.00003e-24), abi.EVAL_OK)]
ROUTES = ["host", "device", "non_fused", "throughput", "resident"]


@pytest.mark.parametrize("where", ["middle", "last"])
@pytest.mark.parametrize("kind", ["node", "root"])
@pytest.mark.parametrize("route", ROUTES)
def test_guard_threshold(engine_lib, oracle_lib, route, kind, where):
    """1e-24f passes, the float below trips, 1.00003e-24f passes: a rescaler maximum (K = 4) and an
    unscaled root likelihood (K = 1), in a middle tile and in the last, partial tile.  One call per
    value; on the resident route one kernel serves all three, the tripping one included"""
    K = 4 if kind == "node" else 1
    pr, C, c = threshold_setup(route, K, where, len(THRESHOLD_VALUES))
    values = [x for x, _ in THRESHOLD_VALUES]
    with threshold_instance(pr, engine_lib, route, values, kind, c) as e, \
         threshold_instance(pr, oracle_lib, route, values, kind, c) as o:
        o.set_arith(1)
        res = run_threshold(e, o, route, [[threshold_spec(pr, i, kind)] for i in range(len(values))])
        for ((le, se, lo, so),), (x, want) in zip(res, THRESHOLD_VALUES):
            assert so == want, f"oracle, x = {x:.9g}"
            assert se == want, f"x = {x:.9g}: status {se}"
            if want == abi.EVAL_OK:
                assert rel(le, lo) < SYN_RTOL, f"x = {x:.9g}"
            else:
                assert le == lo == -DBL_MAX
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == (3 if route == "non_fused" else 0)
        assert e.kernel_launches(abi.KERNEL_NUC4) == (1 if route == "resident" else 3)
        if route == "device":
            assert (C + ppb(K) - 1) // ppb(K) > 16


@pytest.mark.parametrize("kind", ["node", "root"])
@pytest.mark.parametrize("route", ROUTES)
def test_guard_threshold_in_one_evaluation_of_a_batch(engine_lib, oracle_lib, route, kind):
    """four evaluations in one call, the float below 1e-24f in evaluation 2: only it trips"""
    K = 4 if kind == "node" else 1
    pr, C, c = threshold_setup(route, K, "middle", 4)
    values = [None, GUARD_MIN, np.nextafter(GUARD_MIN, np.float32(0)), np.float32(1.00003e-24)]
    with threshold_instance(pr, engine_lib, route, values, kind, c) as e, \
         threshold_instance(pr, oracle_lib, route, values, kind, c) as o:
        o.set_arith(1)
        (res,) = run_threshold(e, o, route, [[threshold_spec(pr, i, kind) for i in range(4)]])
        for i, (le, se, lo, so) in enumerate(res):
            want = abi.EVAL_UNDERFLOW if i == 2 else abi.EVAL_OK
            assert se == so == want, f"evaluation {i}"
            assert (le == lo == -DBL_MAX) if i == 2 else rel(le, lo) < SYN_RTOL, f"evaluation {i}"


# ---- the flag on other families ------------------------------------------------------------------------
def first_level_below(pr, x):
    """the lowest caterpillar level at which, unscaled, some pattern's float64 maximum is below x"""
    m = unscaled_maxima(pr, 0)
    return next(i + 1 for i, p in enumerate(pr.tree[0].post) if m[p].min() < x)


@pytest.mark.parametrize("trip", ["rescaler", "root"])
@pytest.mark.parametrize("family,S,K", [("generic", 16, 2), ("tensor", 20, 2), ("tensor", 61, 1), ("std", 6, 2)])
def test_guard_flag_ignored_for_other_families(engine_lib, oracle_lib, family, S, K, trip):
    """Caterpillars on which the 4-state guard would trip: a rescaler maximum (40 tips, rescaled every
    L levels) or the unscaled root likelihood (L + 2 tips, never rescaled) falls below 1e-24 but stays
    a normal float, L being the first level at which some pattern's maximum falls below 1e-26.  With
    and without the flag, the engine and the oracle give identical status and lnL.  (Std: fixed
    depths; its float64 maxima are not computed here.)"""
    def problem(tips):
        if family == "std":
            pr = workloads.make_std_problem(90, K, tips, 1, seed=13, max_states=S, dummy=2)
        else:
            pr = workloads.make_problem(S, K, 130, tips, 1, seed=5)
        pr.tree[0] = caterpillar_tree(tips, np.random.default_rng(5))
        return pr
    L = 14 if family == "std" else first_level_below(problem(40), 1e-26)
    pr = sparse_rescaling(problem(40) if trip == "rescaler" else problem(L + 2), L if trip == "rescaler" else np.inf)
    sp = pr.full_evaluation(0)
    flagged = abi.EvalSpec(mats=sp.mats, ops=sp.ops, site_dst=sp.site_dst, site_src=sp.site_src, root=sp.root,
                           flags=sp.flags | abi.FLAG_RANGE_GUARD, p_invar=sp.p_invar, has_p_invar=sp.has_p_invar,
                           rates=sp.rates, cat_weights=sp.cat_weights, freqs=sp.freqs)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        res = {}
        for name, inst in (("engine", e), ("oracle", o)):
            for tag, s in (("plain", sp), ("flagged", flagged)):
                (l,), (st,) = inst.evaluate(s)
                res[name, tag] = (l, st)
            assert res[name, "plain"] == res[name, "flagged"], (name, res)
        assert res["engine", "plain"][1] == res["oracle", "plain"][1] == abi.EVAL_OK
        assert rel(res["engine", "plain"][0], res["oracle", "plain"][0]) < lnl_tol(S)
        if family != "std":
            assert trips(o, sp, pr) == ((True, False) if trip == "rescaler" else (False, True))
        kind = {"tensor": abi.KERNEL_TENSOR, "generic": abi.KERNEL_GENERIC, "std": abi.KERNEL_STD}[family]
        assert e.kernel_launches(kind) == 2
