"""GPU: evaluations on trees of 300 to 1000 tips on every kernel route, against the CPU oracle and the float64 pruning
reference (tests/f64_reference.py).

Several parts of the engine depend on the tree's size: the 4-state job is cut into chunks of operations, branches
and tip operands; the tensor-core work queue hands out one item per node and level, and a caterpillar has one level
per node; the resident kernel takes operation lists of any length; float site scalers add up hundreds of node
scalers and every branch update removes and re-adds some.  Each test drives one route on purpose, shows that it was
taken (kernel counters, the 4-state parameter-block and one-CTA-per-evaluation sub-counts among them) and sends several chains per call --
a random tree, a caterpillar and a balanced tree, whose operation counts differ -- a full evaluation and then branch
updates with every third generation rejected.  Every written buffer and lnL is checked against the oracle with the
small-tree bars, and lnL against float64 within the small-tree bar plus the drift that float site scalers carry
(f64_reference.ScalerLedger).

The +I tests put the constant patterns' site scalers past -200, where MrBayes stops exponentiating the scaler, on
every route with invariable sites, under the quirk flag and without it, and show that each branch of the root rule
was taken.  The largest differences each test measured are printed and recorded as test properties."""
import numpy as np
import pytest

from engine_checks import (SYN_RTOL, Checker, StdChecker, assert_resident_equals_launches, edge, generation_sequence,
                           num_sms, parity_tol, ppb, resident_generations, switch_problem, variant_root, via_evaluate,
                           via_replay, with_root_variant)
from f64_reference import ABOVE_SWITCH, INVAR_DOMINATES, INVAR_TINY, INVAR_ZERO, balanced_tree, caterpillar_tree
from mrbayes_b200 import abi, workloads

pytestmark = pytest.mark.gpu


def install_trees(pr, mean_len=0.1, kinds=None):
    """chain 0 keeps its random tree, then caterpillar, balanced, random, ... (or the tree builders `kinds` names)"""
    builders = {"caterpillar": caterpillar_tree, "balanced": balanced_tree}
    for ch in range(pr.n_chains):
        kind = kinds[ch % len(kinds)] if kinds else ("random", "caterpillar", "balanced")[ch % 3]
        if kind in builders:
            pr.tree[ch] = builders[kind](pr.n_tips, np.random.default_rng(100 + ch), mean_len)
    return pr


def run(pr, e, o, route, gens, seed, checker, variant=None, before=None):
    """generation_sequence through route(e, specs), each generation checked; before(g, specs) may evaluate it itself
    (returning (lnl, status)) -> number of calls"""
    calls = 0
    for g, specs in generation_sequence(pr, gens, seed):
        if variant:
            specs = [variant(pr, sp) for sp in specs]
        out = before(g, specs) if before else None
        lnl, st = out if out is not None else route(e, specs)
        calls += 1
        checker(specs, lnl, st)
    return calls


# ---- 4-state routes ------------------------------------------------------------------------------------------------
def test_nuc4_parameter_block_large(engine_lib, oracle_lib, record_property):
    """300 tips, K = 4, three chains, evaluate(): at least every branch update's job rides in the kernel's parameter
    block (KERNEL_NUC4_PARAMS)"""
    pr = install_trees(workloads.make_problem(4, 4, edge(4, 3), 300, 3, seed=41, p_ambig=0.05))
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = Checker(pr, e, o)
        gens = 9
        calls = run(pr, e, o, via_evaluate, gens, 1, chk)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls
        assert gens <= e.kernel_launches(abi.KERNEL_NUC4_PARAMS) <= calls
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 0
    chk.report(record_property, "nuc4 parameter block")


def test_nuc4_device_blob_large(engine_lib, oracle_lib, record_property):
    """1000 tips, K = 2, more than 16 tiles: pack + replay, the fused kernel reads the job from device memory"""
    pr = install_trees(workloads.make_problem(4, 2, edge(2, 20), 1000, 3, seed=42, p_ambig=0.05))
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = Checker(pr, e, o)
        calls = run(pr, e, o, via_replay, 9, 2, chk)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls
        assert e.kernel_launches(abi.KERNEL_NUC4_PARAMS) == 0
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 0
    chk.report(record_property, "nuc4 device blob")


def test_nuc4_non_fused_large(engine_lib, oracle_lib, record_property):
    """300 tips, K = 3, four chains per call over more than 4 x SMs tiles: stand-alone P(t), then the streaming kernel"""
    nch = 4
    tiles = num_sms() + 2
    pr = install_trees(workloads.make_problem(4, 3, edge(3, tiles), 300, nch, seed=43, p_invar=0.1))
    assert tiles * nch > 4 * num_sms()
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = Checker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 4, 3, chk)
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == calls == e.kernel_launches(abi.KERNEL_NUC4)
    chk.report(record_property, "nuc4 non-fused")


def test_nuc4_throughput_large(engine_lib, oracle_lib, record_property):
    """MB200_CONFIG_THROUGHPUT, 600 tips, balanced trees: a full evaluation spans several chunks and runs one CTA per
    tile; a branch update fits one chunk and runs one CTA per evaluation (KERNEL_NUC4_PER_EVAL)"""
    nch, K = 4, 2
    tiles = 5
    pr = install_trees(workloads.make_problem(4, K, tiles * ppb(K), 600, nch, seed=44, p_ambig=0.05),
                       kinds=["balanced"])
    with pr.create(engine_lib, flags=abi.CONFIG_THROUGHPUT) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = Checker(pr, e, o)
        gens = 6
        calls = run(pr, e, o, via_evaluate, gens, 4, chk)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls
        assert e.kernel_launches(abi.KERNEL_NUC4_PER_EVAL) == gens       # the updates; not the multi-chunk full ones
    chk.report(record_property, "nuc4 throughput")


def test_nuc4_resident_large(engine_lib, oracle_lib):
    """replay_begin / _end on two 600-tip chains (random and caterpillar): bit for bit what one launch per generation
    gives, the launches against the oracle and float64"""
    K = 4
    pr = install_trees(workloads.make_problem(4, K, edge(K, 12), 600, 2, seed=45, p_invar=0.1, p_ambig=0.05))
    gens = [specs for _, specs in generation_sequence(pr, 10, 5)]
    assert_resident_equals_launches(engine_lib, oracle_lib, pr, gens, SYN_RTOL, parity_tol(4), drift=True)


# ---- tensor core and generic kernel ----------------------------------------------------------------------------------
def relative_partials_error(e, o, pr, ch, levels):
    """-> {level: largest relative difference engine vs oracle of the partials above 1e-6 of their pattern's largest}
    of caterpillar chain ch's nodes `levels` levels above the tips"""
    tr = pr.tree[ch]
    out = {}
    for lv in levels:
        buf = int(pr.chains[ch].cl[tr.n_tips + lv - 1])
        a, b = e.get_partials(buf).astype(np.float64), o.get_partials(buf).astype(np.float64)
        peak = np.abs(b).max(axis=(0, 2), keepdims=True)
        big = np.abs(b) > 1e-6 * peak
        out[lv] = float((np.abs(a - b)[big] / np.abs(b[big])).max(initial=0.0))
    return out


@pytest.mark.parametrize("S,K", [(20, 1), (20, 4), (61, 1), (61, 3)])
def test_tensor_core_large(engine_lib, oracle_lib, record_property, S, K):
    """300 tips (a caterpillar: 298 levels), three chains per call, C one pattern past a tile.  Partials within
    subtree_tol (2e-5 plus 1e-6 per interior node below); the caterpillar's error by level is recorded."""
    C = 129
    pr = install_trees(workloads.make_problem(S, K, C, 300, 3, seed=46 + S + K, p_ambig=0.05))
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = Checker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 4, 6, chk)
        measured = relative_partials_error(e, o, pr, 1, (10, 40, 100, 200, 298))
        assert e.kernel_launches(abi.KERNEL_TENSOR) == calls
        assert e.kernel_launches(abi.KERNEL_GENERIC) == 0
    for lv, r in measured.items():
        record_property(f"partials_rel_level_{lv}", r)
    print("\npartials relative error by level: " + ", ".join(f"{lv}: {r:.1e}" for lv, r in measured.items()))
    chk.report(record_property, f"tensor core S={S} K={K}")


@pytest.mark.parametrize("S", [16, 40, 64])
def test_generic_large(engine_lib, oracle_lib, record_property, S):
    pr = install_trees(workloads.make_problem(S, 2, 77, 300, 3, seed=47 + S, p_invar=0.1, p_ambig=0.05))
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = Checker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 4, 7, chk)
        assert e.kernel_launches(abi.KERNEL_GENERIC) == calls
        assert e.kernel_launches(abi.KERNEL_TENSOR) == 0 and e.kernel_launches(abi.KERNEL_NUC4) == 0
    chk.report(record_property, f"generic S={S}")


# ---- variable-state (Std) ----------------------------------------------------------------------------------------------
def test_std_large(engine_lib, oracle_lib, record_property):
    pr = install_trees(workloads.make_std_problem(150, 2, 400, 3, seed=48, max_states=6, dummy=2))
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        chk = StdChecker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 4, 8, chk)
        assert e.kernel_launches(abi.KERNEL_STD) == calls
    chk.report(record_property, "std")


# ---- invariable sites past the -200 site-scaler switch ------------------------------------------------------------------
# route: (S, K, patterns, tips, mean branch length, kernel counter).  K = 1, except on the resident and throughput
# routes: at K = 1 and 1000 tips neither the resident kernel nor the one-CTA-per-evaluation mode served these
# evaluations (their counters stayed at one launch per generation and 0), so those two routes run at K = 2 with the
# same flat rates, where they do.
PINVAR_ROUTES = {
    "nuc4_parameter_block": (4, 1, 256, 1000, 0.15, abi.KERNEL_NUC4),
    "nuc4_device_blob": (4, 1, 256 * 17, 1000, 0.15, abi.KERNEL_NUC4),
    "nuc4_non_fused": (4, 1, None, 300, 0.5, abi.KERNEL_NUC4),
    "nuc4_resident": (4, 2, 128 * 3, 1000, 0.15, abi.KERNEL_NUC4),
    "nuc4_throughput": (4, 2, 128 * 2, 1000, 0.15, abi.KERNEL_NUC4),
    "tensor_20": (20, 1, 129, 300, 0.4, abi.KERNEL_TENSOR),
    "tensor_61": (61, 1, 129, 300, 0.5, abi.KERNEL_TENSOR),
    "generic_16": (16, 1, 64, 300, 0.4, abi.KERNEL_GENERIC),
    "generic_40": (40, 1, 32, 300, 0.5, abi.KERNEL_GENERIC),
    "generic_64": (64, 1, 32, 300, 0.5, abi.KERNEL_GENERIC),
}


@pytest.mark.parametrize("route", list(PINVAR_ROUTES))
def test_pinvar_past_scaler_switch(engine_lib, oracle_lib, record_property, route):
    """Four chains, K = 1, +I with constant patterns whose site scalers pass -200: chain ch evaluates under
    root_variants[ch] (quirk flag on and off, p_invar 0.2 and 1e-80).  lnL against the oracle and against the float64
    rule the flags ask for, its decision read from the engine's site scalers; every branch of the rule occurs --
    on 4 states all but INVAR_TINY, which cannot occur there (p_invar is a float, 1e-80 is 0)."""
    S, K, C, tips, mean, kind = PINVAR_ROUTES[route]
    nch = 4
    if C is None:                                        # more than 4 x SMs tiles in a call of four evaluations
        C = 256 * (num_sms() + 2)
    pr = switch_problem(S, K, C, tips, nch, seed=60 + S, mean_len=mean)
    trees = ["balanced"] if route == "nuc4_throughput" else None
    install_trees(pr, mean, kinds=trees)
    flags = abi.CONFIG_THROUGHPUT if route == "nuc4_throughput" else 0
    with pr.create(engine_lib, flags=flags) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = Checker(pr, e, o, ref=lambda sp, sc: variant_root(pr, sp, sc))

        played = []

        def route_fn(e, specs):
            out = (via_replay if route in ("nuc4_device_blob", "nuc4_resident") else via_evaluate)(e, specs)
            played.append((specs, out[0].copy()))
            return out
        gens = 6 if route == "nuc4_resident" else 3
        calls = run(pr, e, o, route_fn, gens, 9, chk, variant=with_root_variant)
        assert e.kernel_launches(kind) == calls
        if route == "nuc4_non_fused":
            assert e.kernel_launches(abi.KERNEL_TIPROBS) == calls
        elif S == 4:
            assert e.kernel_launches(abi.KERNEL_TIPROBS) == 0
        if route == "nuc4_parameter_block":
            # the full evaluations, and updates that climb a long caterpillar path, exceed the block's 30 KB
            assert 1 <= e.kernel_launches(abi.KERNEL_NUC4_PARAMS) < calls
        if route == "nuc4_throughput":
            assert e.kernel_launches(abi.KERNEL_NUC4_PER_EVAL) == gens
    if route == "nuc4_resident":
        # the same generations through one resident kernel, this instance alone on the device: bit for bit the lnL
        # the checked launches gave
        with pr.create(engine_lib) as e:
            got = resident_generations(e, [specs for specs, _ in played])
            assert e.kernel_launches(abi.KERNEL_NUC4) < len(played)      # one kernel served several generations
        assert all(np.array_equal(lnl, want) and not st.any() for (lnl, st), (_, want) in zip(got, played))
    want = {ABOVE_SWITCH, INVAR_DOMINATES, INVAR_ZERO} | ({INVAR_TINY} if S != 4 else set())
    assert chk.branches == want, chk.branches
    chk.report(record_property, f"+I past -200, {route}")
