"""CPU: the float64 pruning reference against the CPU oracle, on the synthetic configurations the
recorded reference runs (tests/golden) do not cover -- 2, 16, 40 and 64 states, 6 and 7 rate
categories, and variable-state (Std) divisions at the shapes of test_gpu_std.py -- so that the oracle, the
only judge of the engine there, is itself checked; and the tree builders the GPU path tests use."""
import numpy as np
import pytest

from f64_reference import balanced_tree, caterpillar_tree, f64_lnl, f64_root, transition_matrices, tree_height
from mrbayes_b200 import abi, workloads

# float oracle vs double reference: float rounding in P(t), in the node products and in the scalers
RTOL = 2e-7


@pytest.mark.parametrize("build,n,height", [(caterpillar_tree, 3, 1), (caterpillar_tree, 40, 38),
                                            (balanced_tree, 40, 6), (balanced_tree, 5, 2)])
def test_tree_builders(build, n, height):
    tr = build(n, np.random.default_rng(1))
    assert tr.n_nodes == 2 * n - 2 and tr.root == n - 1 and tr.left[tr.root] == tr.root_left
    assert sorted(tr.post) == list(range(n, 2 * n - 2))
    seen = set(range(n))
    for p in tr.post:                                   # post-order: children before parents
        assert int(tr.left[p]) in seen and int(tr.right[p]) in seen
        assert tr.anc[tr.left[p]] == p and tr.anc[tr.right[p]] == p
        seen.add(p)
    assert tr.anc[tr.root_left] == tr.root
    assert tree_height(tr) == height
    assert tr.path_to_root(0)[-1] == tr.root_left


CASES = [
    # S, K, C, tips, p_invar, p_ambig, tree
    (2, 4, 90, 9, 0.0, 0.0, "random"),
    (2, 6, 61, 12, 0.2, 0.0, "caterpillar"),
    (16, 2, 45, 6, 0.0, 0.1, "random"),
    (16, 7, 33, 24, 0.1, 0.0, "balanced"),
    (40, 3, 20, 7, 0.0, 0.0, "random"),
    (40, 8, 17, 5, 0.0, 0.2, "caterpillar"),
    (64, 1, 19, 5, 0.0, 0.0, "random"),
    (64, 3, 12, 9, 0.15, 0.0, "balanced"),
    (4, 6, 150, 40, 0.0, 0.05, "caterpillar"),
    (4, 7, 131, 16, 0.25, 0.0, "random"),
    (20, 7, 40, 8, 0.0, 0.0, "random"),
    (61, 6, 15, 6, 0.0, 0.0, "random"),
]


def install(pr, ch, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "caterpillar":
        pr.tree[ch] = caterpillar_tree(pr.n_tips, rng)
    elif kind == "balanced":
        pr.tree[ch] = balanced_tree(pr.n_tips, rng)


@pytest.mark.parametrize("S,K,C,tips,pinv,pamb,tree", CASES)
def test_f64_reference_matches_oracle(oracle_lib, S, K, C, tips, pinv, pamb, tree):
    pr = workloads.make_problem(S, K, C, tips, 1, seed=300 + S + K, p_invar=pinv, p_ambig=pamb)
    install(pr, 0, tree, S * K)
    rng = np.random.default_rng(4)
    with pr.create(oracle_lib) as o:
        o.set_arith(1)
        (lo,), (so,) = o.evaluate(pr.full_evaluation(0))
        assert so == abi.EVAL_OK
        _, lf = f64_lnl(pr, 0)
        assert abs(lo - lf) < RTOL * abs(lf)
        for it in range(4):                              # partial updates: the oracle's scaler bookkeeping
            old = pr.tree[0].length.copy()
            sp = pr.random_branch_update(0, rng)
            (lo,), _ = o.evaluate(sp)
            _, lf = f64_lnl(pr, 0)
            assert abs(lo - lf) < RTOL * abs(lf), f"update {it}"
            if it == 1:
                pr.reject(0, sp, old)


@pytest.mark.parametrize("S", [4, 20, 61])
def test_f64_transition_matrix_limits(S):
    pr = workloads.make_problem(S, 3, 5, 4, 1, seed=1)
    rates = np.array([0.5, 1.0, 2.0])
    assert np.array_equal(transition_matrices(pr, 1e-13, rates), np.broadcast_to(np.eye(S), (3, S, S)))
    assert np.array_equal(transition_matrices(pr, 5000.0, rates), np.broadcast_to(pr.freqs[None, None, :], (3, S, S)))
    P = transition_matrices(pr, 0.3, rates)
    assert np.allclose(P.sum(-1), 1.0, atol=1e-12)
    from scipy.linalg import expm
    Q = (pr.V * pr.lam) @ pr.Vinv
    assert np.allclose(P[1], expm(Q * 0.3), atol=1e-12)


# ---- per-chain models (tests/chain_models.py): the oracle paths the shared-model cases never take -----------
MIXED_CASES = [
    # S, K, parts, C, tips, chains
    (4, 4, 1, 150, 12, 4),          # unequal category weights at S = 4 (the oracle's non-`equal` root), inline
    (4, 7, 1, 97, 9, 4),            # eigensystems next to slot ones, weights rows 1..3
    (61, 3, 3, 15, 6, 3),           # one Q per omega category (MB200_CONFIG_CIJK_PARTS(3))
    (20, 2, 1, 40, 7, 3),
    (16, 5, 1, 33, 8, 3),
]


@pytest.mark.parametrize("S,K,parts,C,tips,nch", MIXED_CASES)
def test_f64_reference_per_chain_models(oracle_lib, S, K, parts, C, tips, nch):
    """Every chain with its own slot (slot 0 a decoy), frequencies, rates, category weights, p_invar, flags and
    weights row (row 0 a decoy): the float64 reference with the evaluation's own model against the oracle, after
    a full evaluation and after branch updates; and the models differ enough to tell an index mix-up."""
    from chain_models import MixedModels
    pr = workloads.make_problem(S, K, C, tips, nch, seed=500 + S + K, p_ambig=0.0)
    pr.tree[0] = caterpillar_tree(tips, np.random.default_rng(S))
    mm = MixedModels(pr, seed=S * K)
    ms = mm.models
    assert {m.slot for m in ms} == set(range(1, nch + 1)) and all(m.row > 0 for m in ms)
    assert len({m.row for m in ms}) > 1 and any(m.p_invar > 0 for m in ms) and any(m.p_invar == 0 for m in ms)
    if K > 1:
        assert any(np.ptp(m.cat_weights) > 0 for m in ms) and any(np.ptp(m.cat_weights) == 0 for m in ms)
    if S == 4:
        assert any(m.inline for m in ms) and not all(m.inline for m in ms)
    rng = np.random.default_rng(S)
    with mm.create(oracle_lib) as o, mm.create(oracle_lib) as scratch:
        o.set_arith(1)
        scratch.set_arith(1)
        mm.assert_models_differ(scratch, range(nch))
        for ch in range(nch):
            (lo,), (so,) = o.evaluate(mm.full(ch))
            assert so == abi.EVAL_OK
            lf = mm.f64(ch)
            assert abs(lo - lf) < RTOL * abs(lf), f"chain {ch}"
        for it in range(2 * nch):
            ch = it % nch
            old = pr.tree[ch].length.copy()
            sp = mm.update(ch, rng)
            (lo,), _ = o.evaluate(sp)
            lf = mm.f64(ch)
            assert abs(lo - lf) < RTOL * abs(lf), f"update {it}"
            if it % 3 == 2:
                pr.reject(ch, sp, old)
        # root integration alone under another weights row and p_invar: the same buffers, other sums
        m = ms[1].with_p_invar(0.2).replace(row=1 + ms[1].row % (mm.rows - 1))
        (lo,), _ = o.evaluate(mm.apply(mm.root_only(1), m))
        lf = mm.f64(1, m)
        assert abs(lo - lf) < RTOL * abs(lf)


def test_f64_reference_matrix_exponential_matches_eigensystem():
    """the Q override builds P(t) by expm: the same matrices as the problem's eigensystem, limits included"""
    pr = workloads.make_problem(4, 3, 5, 4, 1, seed=2)
    Q = (pr.V * pr.lam) @ pr.Vinv
    rates = np.array([0.3, 1.0, 2.5])
    for t in (1e-13, 0.05, 0.7, 5000.0):
        assert np.allclose(transition_matrices(pr, t, rates, Q=Q), transition_matrices(pr, t, rates), atol=1e-12)
    Qs = np.stack([Q, 2 * Q, 3 * Q])
    assert np.allclose(transition_matrices(pr, 0.2, np.ones(3), Q=Qs), transition_matrices(pr, 0.2, [1.0, 2.0, 3.0]), atol=1e-12)


# ---- variable-state (Std) divisions: the float64 reference against the oracle at the shapes of test_gpu_std.py ----
def std_oracle_run(oracle_lib, name, updates=6):
    """-> [(evaluation, oracle lnL, oracle status, float64 StdLnl)] of a full evaluation per chain and branch updates"""
    from engine_checks import evaluation_sequence
    from f64_reference import f64_std_lnl
    from std_problems import make_case
    pr, supplier = make_case(name)
    out = []
    with pr.create(oracle_lib) as o:
        for _, sp in evaluation_sequence(pr, updates, seed=1):
            if supplier:
                supplier(sp, [o])
            (lo,), (so,) = o.evaluate(sp)
            ref = f64_std_lnl(pr, sp.chain, rates=pr.chain_rates[sp.chain],
                              matrices=supplier.matrices(sp.chain) if supplier else None)
            out.append((sp, lo, so, ref))
    return pr, out


def _std_case_names():
    from std_problems import CASES
    return list(CASES)


@pytest.mark.parametrize("name", _std_case_names())
def test_f64_std_reference_matches_oracle(oracle_lib, name):
    """Mk (or caller-supplied) matrices per state-count class, per-chain rates, the coding-bias correction: lnL within
    2e-7 relative; the clamp case is -U log(1e-300) on both; nothing underflows"""
    pr, out = std_oracle_run(oracle_lib, name)
    for i, (sp, lo, so, ref) in enumerate(out):
        assert so == abi.EVAL_OK and not ref.underflow, f"evaluation {i}"
        # near-degenerate: the float partials' ulps in pUn ~ 1 become relative errors of pObserved ~ 1e-4
        assert abs(lo - ref.lnl) < RTOL * abs(ref.lnl) + ref.conditioning(pr), f"evaluation {i}: {lo!r} vs {ref.lnl!r}"
    if name == "clamp":
        assert ref.p_un > 1.9
    if name == "near-degenerate":
        assert all(1e-5 < 1.0 - r.p_un < 1e-3 for *_, r in out)
    if name.startswith("informative"):
        assert pr.dummy == 66


def test_f64_std_reference_orientation(oracle_lib):
    """The non-symmetric matrices decide the result: reading them transposed moves lnL far outside the tolerance"""
    from f64_reference import f64_std_lnl, std_pattern_classes
    from std_problems import make_case
    pr, supplier = make_case("supplied-nonsymmetric-K3")
    with pr.create(oracle_lib) as o:
        sp = supplier(pr.full_evaluation(0), [o])
        (lo,), _ = o.evaluate(sp)
    mats = supplier.matrices(0)
    ref = f64_std_lnl(pr, 0, rates=pr.chain_rates[0], matrices=mats)
    transposed = {}
    for node, blk in mats.items():
        t = blk.copy()
        for n, ti, _ in std_pattern_classes(pr):
            for k in range(pr.K):
                s = slice(ti + k * n * n, ti + (k + 1) * n * n)
                t[s] = blk[s].reshape(n, n).T.ravel()
        transposed[node] = t
    wrong = f64_std_lnl(pr, 0, rates=pr.chain_rates[0], matrices=transposed)
    assert abs(lo - ref.lnl) < RTOL * abs(ref.lnl)
    assert abs(wrong.lnl - ref.lnl) > 1e3 * RTOL * abs(ref.lnl)


def test_f64_std_reference_matrices_and_layout():
    """Mk by expm against its closed form (TiProbs_Std); ordered matrices symmetric birth-death chains; the tables
    of an ordered, informative division in the reference's layout"""
    from scipy.linalg import expm
    from f64_reference import mk_rate_matrix
    from std_problems import dummy_masks, make_std_division, ordered_rate_matrix
    for n in (2, 3, 7, 24):
        v = 0.37
        e = np.exp(-n / (n - 1) * v)
        P = expm(mk_rate_matrix(n) * v)
        assert np.allclose(np.diag(P), 1 / n + (n - 1) / n * e, atol=1e-14)
        assert np.allclose(P[0, 1:], 1 / n - e / n, atol=1e-14)
        Q = ordered_rate_matrix(n)
        assert np.allclose(Q.sum(1), 0) and np.isclose(-np.diag(Q).mean(), 1.0) and np.allclose(Q, Q.T)
        assert np.count_nonzero(np.triu(Q, 2)) == 0
    dm = dummy_masks(4, "informative")
    assert dm.shape == (4, 10) and list(dm[:, 0]) == [2, 1, 1, 1] and list(dm[:, 4]) == [1, 2, 2, 2]
    assert list(dm[:, 8]) == [1] * 4 and list(dm[:, 9]) == [2] * 4
    pr = make_std_division(60, 3, 5, 1, seed=1, states=(2, 3, 5), ordered=(3, 5), coding="informative")
    assert pr.dummy == 12 and pr.weights[:12].sum() == 0 and pr.uncompressed == int(pr.weights.sum())
    blocks = [(2, False), (3, False), (5, False), (3, True), (5, True)]
    ti = np.cumsum([0] + [n * n * 3 for n, _ in blocks])
    bs = np.cumsum([0] + [n for n, _ in blocks])
    for c in range(pr.C):
        j = blocks.index((int(pr.state_counts[c]), bool(pr.ordered[c])))
        assert pr.matrix_offsets[c] == ti[j] and pr.freq_offsets[c] == bs[j]
    assert pr.matrix_length == ti[-1] and len(pr.freqs) == bs[-1]


def tree_from_evaluation(sp, n_tips):
    """The tree of a full evaluation (every branch's matrix update, every interior node's operation), in MrBayes'
    numbering: interior node n_tips + i is the destination of operation i, the root tip is the last one's third child"""
    length = {int(m["matrix"]): float(m["length"]) for m in sp.mats}
    n_nodes = 2 * n_tips - 2
    left, right, anc, lens = np.full(n_nodes, -1), np.full(n_nodes, -1), np.full(n_nodes, -1), np.zeros(n_nodes)
    node = {}
    for i, op in enumerate(sp.ops):
        p = n_tips + i
        node[int(op["dest"])] = p
        for side, (c, m) in enumerate(((op["child1"], op["matrix1"]), (op["child2"], op["matrix2"]))):
            cn = int(c) if c < n_tips else node[int(c)]
            (left if side == 0 else right)[p] = cn
            anc[cn], lens[cn] = p, length[int(m)]
        if op["child3"] >= 0:
            root = int(op["child3"])
            anc[p], left[root], lens[p] = root, p, length[int(op["matrix3"])]
    assert len(sp.ops) == n_tips - 2 and len(sp.mats) == n_nodes - 1
    return workloads.Tree(n_tips, left, right, anc, lens, root, list(range(n_tips, n_nodes)))


def test_f64_std_reference_matches_cynmix_golden():
    """cynmix's morphology partition (Mk + G4, coding=variable): every full evaluation of the recorded reference
    run, rebuilt as a tree, against the lnL the reference's own Likelihood_Std returned"""
    from types import SimpleNamespace
    from conftest import GOLDEN
    from f64_reference import f64_std_lnl
    from mrbayes_b200 import records
    divs, events = records.load(GOLDEN / "cynmix_full_fma.gold.gz")
    (div,) = [d for d in divs.values() if d.pattern_states is not None]
    ps, n_tips = div.pattern_states, div.cfg["tip_count"]
    fulls = [ev.spec for ev in events if ev.kind == "eval" and ev.division == div.division
             and ev.spec.site_src == abi.NONE and len(ev.spec.ops) == n_tips - 2]
    assert len(fulls) >= 4
    masks = np.stack([div.tips[t] for t in range(n_tips)])
    for sp in fulls:
        pr = SimpleNamespace(C=div.cfg["pattern_count"], masks=masks, freqs=sp.freqs, weights=div.weights[sp.weights_row],
                             state_counts=ps["state_counts"], matrix_offsets=ps["matrix_offsets"],
                             freq_offsets=ps["freq_offsets"], dummy=ps["dummy_patterns"],
                             uncompressed=ps["uncompressed_sites"])
        ref = f64_std_lnl(pr, sp.chain, tree_from_evaluation(sp, n_tips), rates=sp.rates)
        assert not ref.underflow and 0.0 < ref.p_un < 1.0
        assert abs(ref.lnl - sp.lnl_ref) < RTOL * abs(sp.lnl_ref), f"chain {sp.chain}: {ref.lnl!r} vs {sp.lnl_ref!r}"


# ---- the root with invariable sites past the -200 site-scaler switch, at a few hundred to a thousand tips -------------
SWITCH_CASES = [
    # S, K, C, tips, mean branch length
    (4, 1, 256, 1000, 0.15),
    (4, 4, 256, 600, 0.25),
    (20, 1, 64, 300, 0.4),
    (20, 4, 64, 400, 0.4),
    (61, 1, 32, 300, 0.5),
    (61, 4, 32, 300, 0.5),
]


@pytest.mark.parametrize("S,K,C,tips,mean", SWITCH_CASES)
def test_root_rules_past_scaler_switch(oracle_lib, S, K, C, tips, mean):
    """Each chain evaluates under one of root_variants (quirk flag on or off, p_invar 0.2 or 1e-80).  The oracle's lnL
    is the float64 reference's under the rule its flags ask for, the decision at -200 read from the oracle's site
    scalers, within the small-tree bar plus the scaler drift.  The quirk moves lnL by thousands of log units and ROOT_GEN
    is ROOT_EXACT except where it drops a tiny likeI.  Every branch of the rule occurs, except INVAR_TINY on 4 states,
    where p_invar is a float and 1e-80 is 0."""
    from engine_checks import root_variants, switch_problem, variant_root, with_root_variant
    from f64_reference import (ABOVE_SWITCH, INVAR_DOMINATES, INVAR_TINY, INVAR_ZERO, ROOT_EXACT, ROOT_GEN, ROOT_QUIRK,
                               ScalerLedger, root_site_terms)
    pr = switch_problem(S, K, C, tips, 4, seed=10 + S + K, mean_len=mean)
    pr.tree[1] = caterpillar_tree(tips, np.random.default_rng(S), mean_len=mean)
    pr.tree[2] = balanced_tree(tips, np.random.default_rng(K), mean_len=mean)
    seen = set()
    with pr.create(oracle_lib) as o:
        o.set_arith(1)
        for ch in range(4):
            sp = with_root_variant(pr, pr.full_evaluation(ch))
            (lo,), (so,) = o.evaluate(sp)
            assert so == abi.EVAL_OK
            sc = o.get_scalers(sp.site_dst)
            ledger = ScalerLedger()
            ledger.record(sp, sc)
            ref = variant_root(pr, sp, sc)
            bar = RTOL * abs(ref.lnl) + ledger.drift(sp, pr.weights)
            assert abs(lo - ref.lnl) <= bar, f"chain {ch}: oracle {lo!r}, float64 {ref.lnl!r}, bar {bar:.2e}"
            seen |= set(ref.branch.tolist())
            # the other rules on the same terms, and where they part
            args = (ref.lnscale, ref.like, ref.like_i)
            exact, _ = root_site_terms(*args, ROOT_EXACT, sc)
            gen, _ = root_site_terms(*args, ROOT_GEN, sc)
            quirk, _ = root_site_terms(*args, ROOT_QUIRK, sc)
            tiny = ref.branch == INVAR_TINY
            assert np.allclose(gen[~tiny], exact[~tiny], rtol=1e-12, atol=1e-12)
            assert (gen[tiny] < exact[tiny] - 1.0).all()                        # the dropped likeI dominated
            dom = ref.branch == INVAR_DOMINATES
            assert np.array_equal(quirk[~dom], gen[~dom])
            assert np.allclose(quirk[dom], gen[dom] + ref.lnscale[dom], rtol=1e-12)
            if dom.any():
                assert abs(float((quirk - gen) @ pr.weights)) > 1e3
            flags, _ = root_variants(pr)[ch]
            assert np.array_equal(ref.site, quirk if flags & abi.FLAG_NUC4_PINVAR_QUIRK else gen)
    want = {ABOVE_SWITCH, INVAR_DOMINATES, INVAR_ZERO} | ({INVAR_TINY} if S != 4 else set())
    assert seen == want, seen


@pytest.mark.parametrize("S,K,C,tips,updates", [(4, 4, 256, 1000, 60), (61, 2, 32, 300, 60)])
def test_scaler_drift_bar_long_run(oracle_lib, S, K, C, tips, updates):
    """A full evaluation per chain (a random tree and a caterpillar), then branch updates with every third rejected: the
    oracle stays within the small-tree bar plus the site-scaler drift (f64_reference.ScalerLedger) of float64 at every
    step, and each chain's drift term grows with its updates.  At the end a fresh full evaluation of each chain's tree
    shows the drift itself: the updated float site scalers differ from the fresh ones, and by no more than the two
    vectors' per-pattern bounds."""
    from engine_checks import evaluation_sequence
    from f64_reference import ScalerLedger
    pr = workloads.make_problem(S, K, C, tips, 2, seed=20 + S, p_ambig=0.05)
    pr.tree[1] = caterpillar_tree(tips, np.random.default_rng(S))
    ledger = ScalerLedger()
    drifts = {0: [], 1: []}
    last = {}
    cache = {}
    with pr.create(oracle_lib) as o:
        o.set_arith(1)
        for it, sp in evaluation_sequence(pr, updates, seed=S):
            (lo,), (so,) = o.evaluate(sp)
            assert so == abi.EVAL_OK
            ledger.record(sp, o.get_scalers(sp.site_dst))
            lf = f64_root(pr, sp.chain, pmat_cache=cache).lnl
            drift = ledger.drift(sp, pr.weights)
            drifts[sp.chain].append(drift)
            assert abs(lo - lf) <= RTOL * abs(lf) + drift, f"evaluation {it}: {lo!r} vs {lf!r}, drift {drift:.2e}"
            if it % 3 != 2:                               # the state the chain keeps
                last[sp.chain] = sp
        assert all(d[-1] > d[0] for d in drifts.values())
        for ch in range(2):
            # the last kept update's site scalers against a fresh full evaluation of the same tree
            kept = last[ch] if last[ch].site_dst == pr.chains[ch].site else None
            assert kept is not None
            updated = o.get_scalers(kept.site_dst).astype(np.float64)
            bound = ledger.pattern_bound(kept)
            fresh_sp = pr.full_evaluation(ch)
            o.evaluate(fresh_sp)
            fresh = o.get_scalers(fresh_sp.site_dst).astype(np.float64)
            ledger.record(fresh_sp, fresh)
            d = np.abs(updated - fresh)
            assert d.max() > 0.0, f"chain {ch}"
            assert (d <= bound + ledger.pattern_bound(fresh_sp)).all(), f"chain {ch}: {d.max():.2e}"
