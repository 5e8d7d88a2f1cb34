"""CPU: the float64 pruning reference against the CPU oracle, on the synthetic configurations the
recorded reference runs (tests/golden) do not cover -- 2, 16, 40 and 64 states, 6 and 7 rate
categories -- so that the oracle, the only judge of the engine there, is itself checked; and the
tree builders the GPU path tests use."""
import numpy as np
import pytest

from f64_reference import balanced_tree, caterpillar_tree, f64_lnl, transition_matrices, tree_height
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
