"""GPU: the operation lists of tree moves (tests/tree_moves.py) on every kernel route -- whole-tree updates that keep
their site scalers, NNI and SPR moves whose dirty set is two or more paths and may change the interior root, and rooted
clock trees whose root multiplies two children.  Each call sends several chains, and in one generation the chains make
different moves, so the operation counts and shapes differ inside a launch; every third generation is rejected.

Each evaluation is checked three ways: lnL and every written buffer against the CPU oracle (check_with_oracle with
large_tree_tol, or sparse_tol under sparse rescaling); every written buffer and lnL against f64_evaluation of the same
call over the inputs it read (f64_call_check, lnL with the rounding of the site scalers the call adds to); and lnL
against the float64 likelihood of the chain's tree, recomputed from scratch, within lnl_tol(S) |lnL| plus the float site
scalers' drift (ScalerLedger).  A stale buffer or a wrong
dirty set shows up in the last.  Each test shows its route taken by the kernel counters and records the largest
differences it measured as test properties."""
import numpy as np
import pytest

import tree_moves as tm
from engine_checks import (SYN_RTOL, Checker, StdChecker, assert_resident_equals_launches, edge, f64_call_check,
                           f64_inputs, num_sms, parity_tol, sparse_tol, via_evaluate, via_replay)
from f64_reference import balanced_tree, caterpillar_tree, f64_evaluation
from mrbayes_b200 import abi, workloads

pytestmark = pytest.mark.gpu

# chain ch cycles through PLAN[ch]: in each generation the chains make different moves
PLAN = [["spr_far", "whole_length", "nni", "branch"],
        ["spr_root_out", "whole_model", "nni_root", "spr_root_in"],
        ["spr_across_root", "branch", "whole_model", "spr_random"],
        ["whole_length", "spr_far", "branch", "nni"]]


def plan_for(pr, model_moves=True):
    plan = [p + ["node_age"] if tm.rooted(pr) else p for p in PLAN]
    if not model_moves:          # the whole-tree update that keeps the problem's model
        plan = [[k.replace("whole_model", "whole_length") for k in p] for p in plan]
    return plan


def move_problem(S, K, C, tips, n_chains, seed, is_rooted, p_invar=0.0, std=False, p_ambig=0.05):
    """chains: a comb, a random tree, a balanced tree, a caterpillar, ...; rooted: `tips` tips and the dummy root tip"""
    n = tips + 1 if is_rooted else tips
    if std:
        pr = workloads.make_std_problem(C, K, n, n_chains, seed=seed, max_states=6, dummy=2)
    else:
        pr = workloads.make_problem(S, K, C, n, n_chains, seed=seed, p_invar=p_invar, p_ambig=p_ambig)
    build = [tm.comb_tree, None, balanced_tree, caterpillar_tree]
    for ch in range(n_chains):
        if build[ch % 4]:
            pr.tree[ch] = build[ch % 4](n, np.random.default_rng(seed + ch))
    if is_rooted:
        tm.make_rooted(pr, np.random.default_rng(seed + 7))
    return pr


class MoveChecker:
    """Checker (or StdChecker) against the chain's own model on its current tree, plus f64_call_check of every
    evaluation over the inputs it read; records which shapes were sent"""

    def __init__(self, pr, e, o, tol=None):
        self.pr, self.e = pr, e
        std = isinstance(pr, workloads.StdProblem)
        self.chk = (StdChecker(pr, e, o, ref=lambda sp, sc: tm.f64(pr, sp.chain), tol=tol) if std else
                    Checker(pr, e, o, ref=lambda sp, sc: tm.f64(pr, sp.chain, sc), tol=tol))
        self.tensor = pr.S in (20, 61) and not std
        self.worst_call = 0.0
        self.shapes = set()

    def inputs(self, specs):
        return [f64_inputs(self.e, sp) for sp in specs]

    def __call__(self, specs, inputs, lnl, st):
        self.chk(specs, lnl, st)
        for i, sp in enumerate(specs):
            ref = f64_evaluation(self.pr, sp, *inputs[i])
            self.worst_call = max(self.worst_call, f64_call_check(self.e, self.pr, sp, ref, self.tensor, st[i], lnl[i],
                                                                  site_drift=True))
            lengths, meets = tm.arms(sp, self.pr.n_tips)
            if meets:
                self.shapes.add("arms")
            if sp.site_src >= 0 and len(sp.ops) == self.pr.n_int:
                self.shapes.add("whole")

    def report(self, record_property, what):
        self.chk.worst["f64_call_of_bar"] = self.worst_call
        self.chk.report(record_property, what)


def run(pr, e, o, route, gens, seed, chk, plan=None):
    """move_sequence through route(e, specs), each generation checked -> number of calls"""
    calls = 0
    for g, mvs, specs in tm.move_sequence(pr, gens, seed, plan or plan_for(pr)):
        inputs = chk.inputs(specs)
        lnl, st = route(e, specs)
        calls += 1
        chk(specs, inputs, lnl, st)
    return calls


ROOTED = pytest.mark.parametrize("is_rooted", [False, True], ids=["unrooted", "rooted"])


# ---- 4-state routes ----------------------------------------------------------------------------------------------
@ROOTED
@pytest.mark.parametrize("K", [1, 4, 5])
def test_nuc4_parameter_block_moves(engine_lib, oracle_lib, record_property, K, is_rooted):
    """evaluate(): the jobs ride in the kernel's parameter block (KERNEL_NUC4_PARAMS)"""
    pr = move_problem(4, K, edge(K, 3), 80, 4, 100 + K, is_rooted, p_invar=0.15 if K % 2 else 0.0)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = MoveChecker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 8, K, chk)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls
        assert e.kernel_launches(abi.KERNEL_NUC4_PARAMS) >= calls // 2
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 0
    assert chk.shapes == {"arms", "whole"}
    chk.report(record_property, f"nuc4 parameter block K={K} {'rooted' if is_rooted else 'unrooted'}")


@pytest.mark.parametrize("f", [1, 4])
@ROOTED
def test_nuc4_sparse_rescaling_moves(engine_lib, oracle_lib, record_property, f, is_rooted):
    """the host route with sparse rescaling: moves change the unscaled counts, so some nodes remove a scaler and write
    none without any change of frequency"""
    from sparse_rescaling import sparse_rescaling
    pr = sparse_rescaling(move_problem(4, 4, edge(4, 3), 80, 4, 110 + f, is_rooted, p_invar=0.1), f)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = MoveChecker(pr, e, o, tol=sparse_tol(pr))
        removes_only = 0

        def route(e, specs):
            nonlocal removes_only
            removes_only += sum(int(((sp.ops["scale_remove"] >= 0) & (sp.ops["scale_write"] < 0)).sum()) for sp in specs)
            return via_evaluate(e, specs)
        calls = run(pr, e, o, route, 8, f, chk)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls and e.kernel_launches(abi.KERNEL_TIPROBS) == 0
    assert removes_only > 0
    chk.report(record_property, f"nuc4 sparse rescaling f={f} {'rooted' if is_rooted else 'unrooted'}")


@ROOTED
@pytest.mark.parametrize("K", [1, 4, 5])
def test_nuc4_device_blob_moves(engine_lib, oracle_lib, record_property, K, is_rooted):
    """pack + replay over more than 16 tiles: the fused kernel reads the job from device memory"""
    pr = move_problem(4, K, edge(K, 17), 80, 4, 120 + K, is_rooted, p_invar=0.15 if K % 2 else 0.0)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = MoveChecker(pr, e, o)
        calls = run(pr, e, o, via_replay, 6, K, chk)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls
        assert e.kernel_launches(abi.KERNEL_NUC4_PARAMS) == 0 and e.kernel_launches(abi.KERNEL_TIPROBS) == 0
    chk.report(record_property, f"nuc4 device blob K={K} {'rooted' if is_rooted else 'unrooted'}")


@ROOTED
@pytest.mark.parametrize("K", [1, 4, 5])
def test_nuc4_non_fused_moves(engine_lib, oracle_lib, record_property, K, is_rooted):
    """four chains per call over more than 4 x SMs tiles: stand-alone P(t), then the streaming kernel"""
    tiles = num_sms() + 2
    pr = move_problem(4, K, edge(K, tiles), 40, 4, 130 + K, is_rooted, p_invar=0.15 if K % 2 else 0.0)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = MoveChecker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 4, K, chk)
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == calls == e.kernel_launches(abi.KERNEL_NUC4)
    chk.report(record_property, f"nuc4 non-fused K={K} {'rooted' if is_rooted else 'unrooted'}")


# trees small enough that every evaluation, the full ones included, fits one chunk (nodes, P(t) slots and tip
# tables of mb200_device.cuh at each K)
THROUGHPUT_TIPS = {1: 10, 4: 20, 5: 16}


@ROOTED
@pytest.mark.parametrize("K", [1, 4, 5])
def test_nuc4_throughput_moves(engine_lib, oracle_lib, record_property, K, is_rooted):
    """MB200_CONFIG_THROUGHPUT: single-chunk evaluations run one CTA per evaluation (KERNEL_NUC4_PER_EVAL), and that
    includes multi-arm topology moves and whole-tree updates"""
    tips = THROUGHPUT_TIPS[K] - (1 if is_rooted else 0)
    pr = move_problem(4, K, edge(K, 5), tips, 4, 140 + K, is_rooted, p_invar=0.15 if K % 2 else 0.0)
    with pr.create(engine_lib, flags=abi.CONFIG_THROUGHPUT) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = MoveChecker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 8, K, chk)
        assert e.kernel_launches(abi.KERNEL_NUC4) == calls
        assert e.kernel_launches(abi.KERNEL_NUC4_PER_EVAL) == calls
    assert chk.shapes == {"arms", "whole"}
    chk.report(record_property, f"nuc4 throughput K={K} {'rooted' if is_rooted else 'unrooted'}")


@ROOTED
@pytest.mark.parametrize("K", [1, 4, 5])
def test_nuc4_resident_moves(engine_lib, oracle_lib, K, is_rooted):
    """replay_begin / _end: bit for bit what one launch per generation gives, the launches against the oracle and the
    last evaluation against the float64 likelihood of its tree (the problem's model: no model moves here)"""
    pr = move_problem(4, K, edge(K, 12), 120, 4, 150 + K, is_rooted, p_invar=0.15 if K % 2 else 0.0)
    gens = [specs for _, _, specs in tm.move_sequence(pr, 9, K, plan_for(pr, model_moves=False))]
    assert_resident_equals_launches(engine_lib, oracle_lib, pr, gens, SYN_RTOL, parity_tol(4), drift=True)


# ---- tensor core, generic kernel, Std ---------------------------------------------------------------------------------
@ROOTED
@pytest.mark.parametrize("S,K", [(20, 1), (20, 4), (61, 1), (61, 3)])
def test_tensor_core_moves(engine_lib, oracle_lib, record_property, S, K, is_rooted):
    pr = move_problem(S, K, 129, 100, 4, 160 + S + K, is_rooted, p_invar=0.1 if K > 1 else 0.0)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = MoveChecker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 5, S + K, chk)
        assert e.kernel_launches(abi.KERNEL_TENSOR) == calls and e.kernel_launches(abi.KERNEL_GENERIC) == 0
    assert chk.shapes == {"arms", "whole"}
    chk.report(record_property, f"tensor core S={S} K={K} {'rooted' if is_rooted else 'unrooted'}")


@ROOTED
@pytest.mark.parametrize("S", [16, 40, 64])
def test_generic_moves(engine_lib, oracle_lib, record_property, S, is_rooted):
    pr = move_problem(S, 2, 45, 60, 3, 170 + S, is_rooted, p_invar=0.1)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        chk = MoveChecker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 5, S, chk)
        assert e.kernel_launches(abi.KERNEL_GENERIC) == calls
        assert e.kernel_launches(abi.KERNEL_TENSOR) == 0 and e.kernel_launches(abi.KERNEL_NUC4) == 0
    chk.report(record_property, f"generic S={S} {'rooted' if is_rooted else 'unrooted'}")


@ROOTED
def test_std_moves(engine_lib, oracle_lib, record_property, is_rooted):
    pr = move_problem(None, 2, 120, 80, 3, 180, is_rooted, std=True)
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        chk = MoveChecker(pr, e, o)
        calls = run(pr, e, o, via_evaluate, 5, 8, chk)
        assert e.kernel_launches(abi.KERNEL_STD) == calls
    chk.report(record_property, f"std {'rooted' if is_rooted else 'unrooted'}")
