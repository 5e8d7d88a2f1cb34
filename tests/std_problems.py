"""Variable-state (STANDARD data) divisions for the Std kernel tests, at shapes make_std_problem does not make:
chosen state counts, ordered classes, polymorphic tips, fossil-like taxa, coding=informative and per-chain rates.

The tables follow the reference's layout for equal state frequencies (src/model.c:16562-16677): one [K][n][n]
run of matrices per state count of unordered patterns, in increasing n, then one per state count of ordered
patterns; the frequency table likewise, one run of n entries per block.  The dummy patterns come first, as
AddDummyChars writes them (src/model.c:176-300): for coding=informative the singletons -- all taxa in state 0
but one in state 1, for each taxon, then the reverse -- then the two constant patterns.

The engine builds only Mk matrices (one per block, from the evaluation's matrix updates).  Ordered classes need
the caller's matrices on every branch, as the seam sends them (set_transition_matrix per dirty branch and no
matrix updates): `supply` does that for an evaluation, on every instance given."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from f64_reference import BRLENS_MAX, BRLENS_MIN, caterpillar_tree, mk_rate_matrix, std_pattern_classes
from mrbayes_b200 import abi, workloads


@dataclass
class StdDivision(workloads.StdProblem):
    ordered: np.ndarray = None          # [C] the pattern's matrices are the ordered block of its state count
    chain_rates: list = None            # per chain: the category rates its evaluations send

    def _spec(self, ch, dirty_branches, dirty_nodes, full):
        sp = super()._spec(ch, dirty_branches, dirty_nodes, full)
        sp.rates = self.chain_rates[ch].copy()
        return sp

    def node_of_matrix(self, ch):
        return {int(m): node for node, m in enumerate(self.chains[ch].ti)}


def dummy_masks(n_tips, coding):
    """[n_tips, dummies] state sets of the unobservable patterns AddDummyChars adds: coding=variable the constant
    patterns (all taxa in state 0, all in state 1); coding=informative also, first, the 2 * n_tips singletons"""
    cols = []
    if coding == "informative":
        for k in (0, 1):
            for i in range(n_tips):
                col = np.full(n_tips, 1 << k, np.uint64)
                col[i] = (1 << k) ^ 3
                cols.append(col)
    cols += [np.full(n_tips, 1, np.uint64), np.full(n_tips, 2, np.uint64)]
    return np.stack(cols, axis=1)


def make_std_division(C, K, n_tips, n_chains, seed, states=(2, 3, 4), ordered=(), coding="variable",
                      p_missing=0.05, p_poly=0.0, fossils=0, tree="random", alpha=0.8, mean_len=0.1) -> StdDivision:
    """C patterns in all, dummies included; every state count in `states` occurs among the observed patterns, and
    for each n in `ordered` (n >= 3) about half of its patterns are ordered.  p_poly: share of tip entries with 2 or 3
    states (polymorphic); fossils: taxa with 70-95 % of their entries missing.  Chain ch's rates are discrete-gamma
    rates times its own multiplier in [0.5, 2]."""
    rng = np.random.default_rng(seed)
    dm = dummy_masks(n_tips, coding)
    dummy = dm.shape[1]
    assert C > dummy + len(states) + len(ordered)
    obs = C - dummy
    ns = rng.choice(np.array(states, np.int32), size=obs)
    ns[:len(states)] = states                            # every state count occurs
    is_ord = np.zeros(obs, bool)
    for i, n in enumerate(ordered):
        assert n >= 3 and n in states
        ns[len(states) + i] = n
        is_ord |= (ns == n) & (rng.random(obs) < 0.5)
        is_ord[len(states) + i] = True
    ns = np.concatenate([np.full(dummy, 2, np.int32), ns]).astype(np.int32)
    is_ord = np.concatenate([np.zeros(dummy, bool), is_ord])
    # blocks: unordered state counts in increasing n, then ordered ones
    blocks = [(int(n), False) for n in sorted(set(ns[~is_ord].tolist()))] + \
             [(int(n), True) for n in sorted(set(ns[is_ord].tolist()))]
    ti_of, bs_of, ti, bs = {}, {}, 0, 0
    for b in blocks:
        ti_of[b], bs_of[b] = ti, bs
        ti += b[0] * b[0] * K
        bs += b[0]
    assert bs <= abi.MAX_STATES, "the frequency table holds 64 entries"
    freqs = np.concatenate([np.full(n, 1.0 / n) for n, _ in blocks])
    key = [(int(n), bool(o)) for n, o in zip(ns, is_ord)]

    # observed patterns: a base state per pattern, mutated on 30 % of the taxa
    masks = np.zeros((n_tips, C), np.uint64)
    full = (np.uint64(1) << ns.astype(np.uint64)) - np.uint64(1)
    base = rng.integers(0, 1 << 30, size=C)
    fossil = np.zeros(n_tips, bool)
    fossil[rng.choice(n_tips, size=fossils, replace=False)] = True
    for t in range(n_tips):
        st = np.where(rng.random(C) < 0.3, rng.integers(0, 1 << 30, size=C), base) % ns
        m = np.uint64(1) << st.astype(np.uint64)
        if p_poly > 0:                                   # 2 or 3 states: one or two more (fewer where draws coincide)
            poly = rng.random(C) < p_poly
            for more in (poly, poly & (rng.random(C) < 0.5)):
                add = np.uint64(1) << ((st + 1 + rng.integers(0, 1 << 30, size=C) % (ns - 1)) % ns).astype(np.uint64)
                m = np.where(more, m | add, m)
        miss = rng.random(C) < (rng.uniform(0.7, 0.95) if fossil[t] else p_missing)
        masks[t] = np.where(miss, full, m)
    masks[:, :dummy] = dm
    weights = rng.integers(1, 4, size=C).astype(np.float32)
    weights[:dummy] = 0.0
    make_tree = {"random": lambda r: workloads.random_tree(n_tips, r, mean_len),
                 "caterpillar": lambda r: caterpillar_tree(n_tips, r, mean_len)}[tree]
    trees = [make_tree(rng) for _ in range(n_chains)]
    gamma = workloads.discrete_gamma_rates(alpha, K)
    chain_rates = [gamma * rng.uniform(0.5, 2.0) for _ in range(n_chains)]
    S = int(ns.max())
    pr = StdDivision(S, K, C, n_chains, trees, masks, weights, freqs, np.zeros((S, S)), np.zeros((S, S)), np.zeros(S),
                     chain_rates[0], 0.0, flags=0,
                     state_counts=ns, matrix_offsets=np.array([ti_of[k] for k in key], np.int32),
                     freq_offsets=np.array([bs_of[k] for k in key], np.int32), matrix_length=ti,
                     dummy=dummy, uncompressed=int(weights.sum()), ordered=is_ord, chain_rates=chain_rates)
    pr.allocate()
    return pr


# ----------------------------------------------------------------------------- caller-supplied matrices
def ordered_rate_matrix(n):
    """Q of an ordered character with equal frequencies: a birth-death chain, state i to i +- 1 only, at one
    change per unit time on average"""
    Q = np.zeros((n, n))
    i = np.arange(n - 1)
    Q[i, i + 1] = Q[i + 1, i] = n / (2.0 * (n - 1))
    np.fill_diagonal(Q, -Q.sum(1))
    return Q


def model_block(pr, length, rates):
    """A branch's block (matrix_length floats): expm(Q v) for every class and category, Q the Mk or the ordered
    rate matrix of the class, v = clamp(length, BRLENS_MIN, BRLENS_MAX) * r_k"""
    from scipy.linalg import expm
    blk = np.zeros(pr.matrix_length, np.float32)
    v = min(max(float(length), BRLENS_MIN), BRLENS_MAX) * np.asarray(rates, float)
    for n, ti, idx in std_pattern_classes(pr):
        Q = ordered_rate_matrix(n) if pr.ordered[idx[0]] else mk_rate_matrix(n)
        for k, vk in enumerate(v):
            blk[ti + k * n * n: ti + (k + 1) * n * n] = np.maximum(expm(Q * vk), 0.0).ravel()
    return blk


def random_block(pr, rng):
    """A branch's block of non-symmetric row-stochastic matrices, one per class and category: a heavy diagonal
    plus Dirichlet rows, so that P[a][i] != P[i][a]"""
    blk = np.zeros(pr.matrix_length, np.float32)
    for n, ti, _ in std_pattern_classes(pr):
        for k in range(pr.K):
            P = 0.5 * np.eye(n) + 0.5 * rng.dirichlet(np.full(n, 0.7), size=n)
            blk[ti + k * n * n: ti + (k + 1) * n * n] = P.ravel()
    return blk


class MatrixSupplier:
    """Caller-supplied P(t) the way the seam sends them: for every matrix update of an evaluation on a branch in
    `nodes(chain)`, the block goes to every instance through set_transition_matrix and the update leaves the
    evaluation.  `make(pr, ch, node)` builds the block.  The blocks are kept by matrix index, so that after a
    rejection the float64 reference reads what the instances hold."""

    def __init__(self, pr, make, nodes):
        self.pr, self.make, self.nodes, self.blocks = pr, make, nodes, {}

    def __call__(self, sp, insts):
        pr, ch = self.pr, sp.chain
        node_of = pr.node_of_matrix(ch)
        keep = []
        for j, mu in enumerate(sp.mats):
            node = node_of[int(mu["matrix"])]
            if node not in self.nodes(ch):
                keep.append(j)
                continue
            blk = np.ascontiguousarray(self.make(pr, ch, node), np.float32)
            self.blocks[ch, int(mu["matrix"])] = blk
            for inst in insts:
                inst.set_transition_matrix(int(mu["matrix"]), blk)
        sp.mats = sp.mats[keep].copy()
        return sp

    def matrices(self, ch):
        """node -> the block the instances hold for chain ch's current matrix of that branch"""
        ti = self.pr.chains[ch].ti
        return {node: self.blocks[ch, int(ti[node])] for node in self.nodes(ch) if (ch, int(ti[node])) in self.blocks}


# ----------------------------------------------------------------------------- the shapes the Std tests run
def lanes(K):
    """lanes per pattern of the Std kernel: pow2ceil(K); a 128-thread CTA holds 128 / lanes patterns"""
    return 1 << (K - 1).bit_length()


def _cases():
    cases = {}
    for K in (1, 2, 3, 4, 5, 8, 9, 16, 17, 19, 20):               # lane widths 1 ... 32, tile edges
        tp = 128 // lanes(K)
        t = 2 if tp >= 16 else 3
        for d in (-1, 0, 1):
            cases[f"lanes-K{K}-C{tp * t + d}"] = dict(C=tp * t + d, K=K, n_tips=6, n_chains=2, states=(2, 3, 4),
                                                      p_poly=0.1)
    for i, smax in enumerate((4, 5, 8, 9, 12, 13, 16, 17, 24)):    # both sides of each SMAX boundary
        cases[f"smax-{smax}"] = dict(C=61, K=(4, 2, 3, 5, 1, 4, 2, 6, 3)[i], n_tips=7, n_chains=2,
                                     states=(2, 3, smax), p_poly=0.1)
    cases["classes-2to10-K20"] = dict(C=120, K=20, n_tips=8, n_chains=2, states=tuple(range(2, 11)))
    cases["informative-K4"] = dict(C=126, K=4, n_tips=32, n_chains=1, states=(2, 3, 4), coding="informative")
    cases["informative-K17"] = dict(C=100, K=17, n_tips=32, n_chains=1, states=(2, 3, 4), coding="informative")
    cases["near-degenerate"] = dict(C=80, K=4, n_tips=12, n_chains=2, states=(2, 3, 4), mean_len=5e-6)
    cases["clamp"] = dict(C=60, K=4, n_tips=8, n_chains=2, states=(2, 3, 4), missing_dummies=True)
    cases["supplied-nonsymmetric-K3"] = dict(C=90, K=3, n_tips=8, n_chains=2, states=(2, 3, 5), supply="random")
    cases["supplied-nonsymmetric-K17"] = dict(C=40, K=17, n_tips=8, n_chains=2, states=(2, 3, 5), supply="random")
    cases["supplied-ordered"] = dict(C=120, K=4, n_tips=8, n_chains=2, states=(2, 3, 4, 5, 6), ordered=(3, 4, 5, 6),
                                     supply="model")
    cases["hymfossil"] = dict(C=150, K=4, n_tips=114, n_chains=1, states=(2, 3, 4, 5, 6, 7), fossils=45, p_poly=0.05,
                              tree="caterpillar")
    return cases


CASES = _cases()


def make_case(name, seed=0):
    """-> (StdDivision, MatrixSupplier or None) of a named shape.  supply="random": the branches of even node index
    get non-symmetric matrices, the others keep the engine's Mk; supply="model": every branch gets the Mk or ordered
    expm matrices of its class, as the seam sends them for ordered characters."""
    kw = dict(CASES[name])
    supply = kw.pop("supply", None)
    missing_dummies = kw.pop("missing_dummies", False)
    pr = make_std_division(seed=sum(map(ord, name)) + seed, **kw)
    if missing_dummies:                                 # sum L_c over the dummies ~ 2: the pObserved clamp
        pr.masks[:, :pr.dummy] = np.uint64(3)
    if supply is None:
        return pr, None
    if supply == "random":
        rng = np.random.default_rng(len(name) + seed)
        return pr, MatrixSupplier(pr, lambda pr, ch, node: random_block(pr, rng),
                                  lambda ch: {n for n in range(pr.n_nodes) if n % 2 == 0 and n != pr.tree[ch].root})
    return pr, MatrixSupplier(pr, lambda pr, ch, node: model_block(pr, pr.tree[ch].length[node], pr.chain_rates[ch]),
                              lambda ch: {n for n in range(pr.n_nodes) if n != pr.tree[ch].root})
