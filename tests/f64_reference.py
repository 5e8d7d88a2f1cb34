"""Float64 tree pruning, written from the model's definition and independent of the engine and the
oracle: the reference the GPU kernels and the CPU oracle are both checked against.  Also tree
builders for the shapes random_tree rarely makes (a caterpillar, one interior node per level, and a
balanced tree), in MrBayes' numbering so that workloads.Problem can drive them unchanged."""
import numpy as np

from mrbayes_b200 import workloads

TIME_MIN = float(np.float32(1.0e-11))       # P(t) = I below, stationary rows above (TiProbs_Gen)
TIME_MAX = float(np.float32(100.0))


def transition_matrices(pr, length, rates):
    """[K, S, S] P(t) = V diag(exp(lambda r_k t)) V^-1 in double, negative entries clamped to 0."""
    out = []
    for r in rates:
        t = length * r
        if t < TIME_MIN:
            out.append(np.eye(pr.S))
        elif t > TIME_MAX:
            out.append(np.tile(np.asarray(pr.freqs, float), (pr.S, 1)))
        else:
            out.append(np.maximum((pr.V * np.exp(pr.lam * t)) @ pr.Vinv, 0.0))
    return np.array(out)


def tip_partials(pr, tip):
    """[C, S] 1.0 for every state in the tip's state set."""
    bits = (pr.masks[tip][:, None] >> np.arange(pr.S, dtype=np.uint64)[None, :]) & np.uint64(1)
    return bits.astype(np.float64)


def f64_lnl(pr, ch, tree=None):
    """-> (per-pattern log likelihoods [C], lnL) of chain `ch` on its current tree."""
    tr = pr.tree[ch] if tree is None else tree
    rates = np.asarray(pr.rates, float) / (1.0 - pr.p_invar)
    catw = (1.0 - pr.p_invar) / pr.K
    cl, lnscale = {}, np.zeros(pr.C)

    def child(node):
        x = np.broadcast_to(tip_partials(pr, node), (pr.K, pr.C, pr.S)) if node < tr.n_tips else cl[node]
        P = transition_matrices(pr, tr.length[node], rates)
        return np.einsum("kij,kcj->kci", P, x)

    for p in tr.post:
        x = child(int(tr.left[p])) * child(int(tr.right[p]))
        if tr.anc[p] == tr.root:                       # the interior root also takes the root tip
            rt = tip_partials(pr, tr.root)[None]
            x = x * np.einsum("kij,kcj->kci", transition_matrices(pr, tr.length[p], rates), np.broadcast_to(rt, x.shape))
        m = x.max(axis=(0, 2))
        m = np.where(m > 0, m, 1.0)
        cl[p] = x / m[None, :, None]
        lnscale += np.log(m)
    like = catw * np.einsum("kcs,s->c", cl[tr.root_left], np.asarray(pr.freqs, float))
    if pr.p_invar > 0:
        inv = np.bitwise_and.reduce(pr.masks, axis=0)
        bits = (inv[:, None] >> np.arange(pr.S, dtype=np.uint64)[None, :]) & np.uint64(1)
        like_i = pr.p_invar * (bits * np.asarray(pr.freqs, float)[None, :]).sum(1)
        # Likelihood_Gen's formula; below a scaler of -200 the reference switches to an approximation
        assert lnscale.min() >= -200.0, "site scaler below -200: the reference approximates there"
        site = lnscale + np.log(like + like_i * np.exp(-lnscale))
    else:
        with np.errstate(divide="ignore"):
            site = lnscale + np.log(like)
    return site, float(site @ np.asarray(pr.weights, float))


# ----------------------------------------------------------------------------- trees
def tree_height(tr, node=None):
    """interior levels from the tips up to `node` (default: the interior root)"""
    node = tr.root_left if node is None else node
    if node < tr.n_tips:
        return 0
    return 1 + max(tree_height(tr, int(tr.left[node])), tree_height(tr, int(tr.right[node])))


def _tree(n, left, right, rng, mean_len):
    """Tree from child tables; interior nodes are numbered n..2n-3 in post-order, 2n-3 is the
    interior root and tip n-1 hangs above it."""
    n_nodes = 2 * n - 2
    anc = np.full(n_nodes, -1)
    for p in range(n, n_nodes):
        anc[left[p]] = anc[right[p]] = p
    root = n - 1
    anc[n_nodes - 1] = root
    left[root] = n_nodes - 1
    length = rng.exponential(mean_len, n_nodes)
    length[root] = 0.0
    return workloads.Tree(n, left, right, anc, length, root, list(range(n, n_nodes)))


def caterpillar_tree(n, rng, mean_len=0.1):
    """Every interior node has a tip child: height n - 2, one node per level."""
    assert n >= 3
    left, right = np.full(2 * n - 2, -1), np.full(2 * n - 2, -1)
    left[n], right[n] = 0, 1
    for i in range(1, n - 2):
        left[n + i], right[n + i] = n + i - 1, i + 1
    return _tree(n, left, right, rng, mean_len)


def balanced_tree(n, rng, mean_len=0.1):
    """Tips 0..n-2 split in halves recursively below the interior root: height ~log2(n)."""
    assert n >= 3
    left, right = np.full(2 * n - 2, -1), np.full(2 * n - 2, -1)
    nxt = [n]

    def build(lo, hi):                     # subtree over tips [lo, hi); returns its node
        if hi - lo == 1:
            return lo
        mid = (lo + hi) // 2
        a, b = build(lo, mid), build(mid, hi)
        p = nxt[0]; nxt[0] += 1
        left[p], right[p] = a, b
        return p

    build(0, n - 1)
    return _tree(n, left, right, rng, mean_len)
