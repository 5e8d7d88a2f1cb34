"""CPU: the tree-move builders of tests/tree_moves.py -- whole-tree updates that keep their site scalers, NNI and SPR
moves, rooted clock trees with node-age moves -- pinned before any GPU test relies on them.  Trees stay valid through
moves and rejections; the CPU oracle's lnL after every move is the float64 likelihood of the chain's current tree,
recomputed from scratch, at 4, 16, 20 and 61 states and on Std divisions, unrooted and rooted; the operation lists
have the shapes the GPU tests are there to send; and each way a builder could go wrong moves the oracle's lnL outside
the bar, so that these checks can tell."""
import numpy as np
import pytest

import tree_moves as tm
from f64_reference import ScalerLedger, balanced_tree, caterpillar_tree
from mrbayes_b200 import abi, workloads

RTOL = 2e-7                      # float oracle vs float64 (test_f64_reference.py)
NUC_MAXPRE = 8                   # clean operands the 4-state kernel prefetches per chunk (mb200_device.cuh)
CHUNK = 32                       # operations per 4-state chunk at K >= 3

# chain ch of a problem cycles through PLAN[ch]: every move kind, each on a tree it suits
PLAN = [["spr_far", "whole_length", "nni", "branch"],
        ["spr_root_out", "spr_root_in", "whole_model", "nni_root"],
        ["spr_across_root", "spr_random", "branch", "whole_model"]]


def move_problem(S, K, C, tips, seed, is_rooted, p_invar=0.0, std=False):
    """three chains: a comb, a random tree and a balanced tree; rooted: `tips` tips and the dummy root tip"""
    n = tips + 1 if is_rooted else tips
    if std:
        pr = workloads.make_std_problem(C, K, n, 3, seed=seed, max_states=5, dummy=2)
    else:
        pr = workloads.make_problem(S, K, C, n, 3, seed=seed, p_invar=p_invar, p_ambig=0.05)
    pr.tree[0] = tm.comb_tree(n, np.random.default_rng(seed))
    pr.tree[2] = balanced_tree(n, np.random.default_rng(seed + 1))
    if is_rooted:
        tm.make_rooted(pr, np.random.default_rng(seed + 2))
    return pr


# ---- the trees ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("is_rooted", [False, True])
def test_moves_keep_trees_valid(is_rooted):
    """After every move and every rejection the tree is valid (a rooted root has two children and a clock tree's lengths
    are its age differences); a rejection restores the tree, its ages and the chain's index tables exactly; clock trees
    have branches of length exactly 0"""
    pr = move_problem(4, 2, 4, 40, 3, is_rooted)
    pr.tree[1] = caterpillar_tree(pr.n_tips, np.random.default_rng(9)) if not is_rooted else pr.tree[1]
    rng = np.random.default_rng(1)
    for ch in range(3):
        tm.full(pr, ch)
    if is_rooted:
        for tr in pr.tree:
            zero = tr.length == 0
            zero[[tr.root, tr.root_left]] = False
            assert zero[:tr.n_tips].any() and zero[tr.n_tips:].any()
    kinds = sorted({k for plan in PLAN for k in plan} | {"node_age"} if is_rooted else {k for plan in PLAN for k in plan})
    roots_changed = 0
    for it in range(60):
        ch, kind = it % 3, kinds[it % len(kinds)]
        tr, st = pr.tree[ch], pr.chains[ch]
        before = [a.copy() for a in (tr.left, tr.right, tr.anc, tr.length, st.cl, st.ti, st.ns, st.scaled)]
        post, site = list(tr.post), st.site
        mv = tm.make_move(pr, ch, kind, rng)
        tm.check_tree(tr, is_rooted)
        roots_changed += mv.info.get("root_changed", False)
        if it % 3 == 2:
            tm.reject(pr, mv)
            tm.check_tree(tr, is_rooted)
            after = (tr.left, tr.right, tr.anc, tr.length, st.cl, st.ti, st.ns, st.scaled)
            assert all(np.array_equal(a, b) for a, b in zip(before, after)) and tr.post == post and st.site == site
    assert roots_changed >= 4


# ---- against the float64 likelihood of the tree ------------------------------------------------------------------------
SEQ_CASES = [
    # S, K, C, tips, p_invar, Std
    (4, 4, 60, 40, 0.15, False),
    (4, 1, 50, 33, 0.0, False),
    (16, 2, 30, 24, 0.0, False),
    (20, 3, 30, 24, 0.1, False),
    (61, 2, 12, 20, 0.0, False),
    (None, 3, 50, 24, 0.0, True),
]


def oracle_run(oracle_lib, pr, gens, seed, plan=PLAN):
    """move_sequence on the oracle: every lnL within RTOL |lnL| plus the ScalerLedger drift of the float64 lnL of the
    chain's current tree -> the move kinds taken"""
    ledger, kinds = ScalerLedger(), set()
    std = isinstance(pr, workloads.StdProblem)
    w = np.asarray(pr.weights, np.float64).copy()
    if std:
        w[:pr.dummy] = 0.0
    with pr.create(oracle_lib) as o:
        o.set_arith(1)
        for g, mvs, specs in tm.move_sequence(pr, gens, seed, plan):
            lnl, st = o.evaluate(specs)
            for i, sp in enumerate(specs):
                assert st[i] == abi.EVAL_OK
                sc = o.get_scalers(sp.site_dst)
                ledger.record(sp, sc)
                ref = tm.f64(pr, sp.chain, sc)
                bar = (ref.bound(pr) if std else RTOL * abs(ref.lnl)) + ledger.drift(sp, w)
                what = mvs[i].kind if mvs[i] else "full"
                assert abs(lnl[i] - ref.lnl) <= bar, f"generation {g}, chain {sp.chain}, {what}: {lnl[i]!r} vs {ref.lnl!r}"
                kinds.add(what)
    return kinds


@pytest.mark.parametrize("is_rooted", [False, True], ids=["unrooted", "rooted"])
@pytest.mark.parametrize("S,K,C,tips,pinv,std", SEQ_CASES)
def test_move_sequence_matches_f64(oracle_lib, S, K, C, tips, pinv, std, is_rooted):
    """Every move kind, every third generation rejected: the oracle against the float64 likelihood of the tree after
    each move"""
    pr = move_problem(S, K, C, tips, 70 + K, is_rooted, pinv, std)
    plan = PLAN if not is_rooted else [p + ["node_age"] for p in PLAN]
    kinds = oracle_run(oracle_lib, pr, 12, 5, plan)
    assert kinds >= {"spr_far", "whole_length", "whole_model", "nni", "nni_root", "spr_root_out", "spr_root_in",
                     "spr_across_root", "spr_random"}


@pytest.mark.parametrize("f", [1, 4])
def test_move_sequence_sparse_rescaling(oracle_lib, f):
    """The moves composed with sparse rescaling (tests/sparse_rescaling.py): topology moves change the unscaled counts,
    so nodes come out of a move without the scaler they held"""
    from sparse_rescaling import sparse_rescaling
    for is_rooted in (False, True):
        pr = sparse_rescaling(move_problem(4, 4, 60, 40, 80 + f, is_rooted, 0.1), f)
        removes_only = []
        orig = pr._spec

        def spy(ch, b, d, full, orig=orig):
            sp = orig(ch, b, d, full)
            removes_only.append(int(((sp.ops["scale_remove"] >= 0) & (sp.ops["scale_write"] < 0)).sum()))
            return sp
        pr._spec = spy
        oracle_run(oracle_lib, pr, 9, 6)
        assert sum(removes_only) > (3 if f > 1 else 0)        # at f = 1, only a new interior root removes only


# ---- the shapes of the operation lists ------------------------------------------------------------------------------
@pytest.mark.parametrize("is_rooted", [False, True], ids=["unrooted", "rooted"])
def test_move_operation_lists(is_rooted):
    """What the GPU tests rely on the builders to send: two arms, one longer than a chunk, and more than NUC_MAXPRE
    clean operands in one chunk (a regraft far up a comb); two arms that meet only at the interior root; a change of
    the interior root in both directions, with its scaler bookkeeping; a scale_remove on every rescaled operation of a
    whole-tree update; no child3, matrix3 or scaler at a rooted root, whose branch is never rebuilt"""
    pr = move_problem(4, 4, 8, 150, 11, is_rooted)
    for ch in range(3):
        tm.full(pr, ch)
    rng = np.random.default_rng(2)
    n = pr.n_tips

    def root_op(sp):
        (i,) = np.flatnonzero(sp.ops["dest"] == sp.root)
        assert i == len(sp.ops) - 1
        return sp.ops[i]

    def check_root(mv):
        op, tr, st = root_op(mv.spec), pr.tree[mv.ch], pr.chains[mv.ch]
        assert op["scale_write"] == abi.NONE
        if is_rooted:
            assert op["child3"] == abi.NONE and op["matrix3"] == abi.NONE
            assert not set(mv.spec.mats["matrix"].tolist()) & {int(st.ti[tr.root_left]), int(st.ti_scratch[tr.root_left])}
        else:
            assert op["child3"] == tr.root

    mv = tm.spr(pr, 0, rng, "far")
    lengths, meets = tm.arms(mv.spec, n)
    assert len(lengths) >= 2 and max(lengths) > CHUNK and meets
    assert max(tm.clean_operands_per_chunk(mv.spec, n, CHUNK)) > NUC_MAXPRE
    check_root(mv)
    mv = tm.spr(pr, 2, rng, "across_root")
    lengths, meets = tm.arms(mv.spec, n)
    assert len(lengths) == 3 and min(lengths[:2]) >= 3 and meets == [mv.spec.root]
    check_root(mv)
    for kind in ("root_out", "root_in"):
        old_root = pr.tree[1].root_left
        mv = tm.spr(pr, 1, rng, kind)
        tr, st, ops = pr.tree[1], pr.chains[1], mv.spec.ops
        assert tr.root_left != old_root and mv.info["root_changed"]
        new, former = ops[-1], ops[np.flatnonzero(ops["dest"] == st.cl[old_root])[0]]
        # the new root held a scaler as an ordinary node and writes none; the former one writes one, removing none
        assert new["scale_remove"] >= 0 and new["scale_write"] == abi.NONE
        assert former["scale_remove"] == abi.NONE and former["scale_write"] >= 0
        check_root(mv)
    for kind in ("length", "model"):
        mv = tm.whole_tree_update(pr, 0, rng, kind)
        ops = mv.spec.ops
        assert len(ops) == n - 2 and mv.spec.site_src >= 0
        assert ((ops["scale_write"] >= 0) == (ops["scale_remove"] >= 0)).all() and (ops["scale_write"] >= 0).sum() == n - 3
        check_root(mv)
    for kind in ("nni", "nni_root", "branch"):
        check_root(tm.make_move(pr, 2, kind, rng))


# ---- sensitivity: each way a builder could go wrong shows in lnL -----------------------------------------------------
def sensitivity_pair(oracle_lib, is_rooted, build):
    """the same state twice; build(pr, mutated) makes one move on each -> (correct, mutated) |lnL - lnL64| / bar"""
    out = []
    for mutated in (False, True):
        pr = move_problem(4, 4, 60, 60, 21, is_rooted, 0.1)
        with pr.create(oracle_lib) as o:
            o.set_arith(1)
            ledger = ScalerLedger()
            for ch in range(3):
                sp = tm.full(pr, ch)
                o.evaluate([sp])
                ledger.record(sp, o.get_scalers(sp.site_dst))
            sp = build(pr, mutated, np.random.default_rng(4)).spec
            (lnl,), _ = o.evaluate([sp])
            sc = o.get_scalers(sp.site_dst)
            ledger.record(sp, sc)
            ref = tm.f64(pr, sp.chain, sc).lnl
            out.append(abs(lnl - ref) / (RTOL * abs(ref) + ledger.drift(sp, pr.weights)))
    return out


@pytest.mark.parametrize("is_rooted", [False, True], ids=["unrooted", "rooted"])
def test_sensitivity_whole_tree_without_removes(oracle_lib, is_rooted):
    good, bad = sensitivity_pair(oracle_lib, is_rooted,
                                 lambda pr, m, rng: tm.whole_tree_update(pr, 1, rng, "length", drop_removes=m))
    assert good <= 1.0 < bad


@pytest.mark.parametrize("is_rooted", [False, True], ids=["unrooted", "rooted"])
def test_sensitivity_second_arm_node_left_out(oracle_lib, is_rooted):
    """a regraft far up the comb with p, where the second arm starts, left out of the dirty set"""
    drop = lambda tr, dirty, info: info["parent"]
    good, bad = sensitivity_pair(oracle_lib, is_rooted,
                                 lambda pr, m, rng: tm.spr(pr, 0, rng, "far", drop=drop if m else None))
    assert good <= 1.0 < bad


def test_sensitivity_rooted_root_reads_pre_move_buffer(oracle_lib):
    """an NNI at the rooted root, the root's operation reading its rebuilt child's pre-move buffer"""
    def build(pr, mutated, rng):
        tr, st = pr.tree[2], pr.chains[2]
        mv = tm.nni(pr, 2, rng, at_root=True)
        op = mv.spec.ops[-1]
        (col,) = [c for c in ("child1", "child2") if op[c] in mv.spec.ops["dest"][:-1]]
        if mutated:
            child = int(np.flatnonzero(st.cl == op[col])[0])
            mv.spec.ops[col][-1] = st.cl_scratch[child]
        return mv
    good, bad = sensitivity_pair(oracle_lib, True, build)
    assert good <= 1.0 < bad
