"""Float64 tree pruning, written from the model's definition and independent of the engine and the
oracle: the reference the GPU kernels and the CPU oracle are both checked against.  Also tree
builders for the shapes random_tree rarely makes (a caterpillar, one interior node per level, and a
balanced tree), in MrBayes' numbering so that workloads.Problem can drive them unchanged."""
import numpy as np

from mrbayes_b200 import workloads

TIME_MIN = float(np.float32(1.0e-11))       # P(t) = I below, stationary rows above (TiProbs_Gen)
TIME_MAX = float(np.float32(100.0))


def transition_matrices(pr, length, rates, Q=None, freqs=None):
    """[K, S, S] P(t) in double, negative entries clamped to 0: V diag(exp(lambda r_k t)) V^-1 from the
    problem's eigensystem, or with Q -- [S, S], or [K, S, S], one rate matrix per category -- the matrix
    exponential expm(Q_k r_k t), independent of any eigensystem.  Stationary rows are `freqs` (default
    the problem's)."""
    from scipy.linalg import expm
    freqs = np.asarray(pr.freqs if freqs is None else freqs, float)
    Qk = None if Q is None else np.broadcast_to(np.asarray(Q, float).reshape(-1, pr.S, pr.S), (len(rates), pr.S, pr.S))
    out = []
    for k, r in enumerate(rates):
        t = length * r
        if t < TIME_MIN:
            out.append(np.eye(pr.S))
        elif t > TIME_MAX:
            out.append(np.tile(freqs, (pr.S, 1)))
        elif Qk is not None:
            out.append(np.maximum(expm(Qk[k] * t), 0.0))
        else:
            out.append(np.maximum((pr.V * np.exp(pr.lam * t)) @ pr.Vinv, 0.0))
    return np.array(out)


def tip_partials(pr, tip):
    """[C, S] 1.0 for every state in the tip's state set."""
    bits = (pr.masks[tip][:, None] >> np.arange(pr.S, dtype=np.uint64)[None, :]) & np.uint64(1)
    return bits.astype(np.float64)


def f64_lnl(pr, ch, tree=None, *, Q=None, freqs=None, rates=None, cat_weights=None, p_invar=None, weights=None):
    """-> (per-pattern log likelihoods [C], lnL) of chain `ch` on its current tree.

    Without overrides the model is the problem's: its eigensystem, frequencies, rates / (1 - p_invar) and
    equal category weights (1 - p_invar) / K.  Overrides describe one evaluation's own model: Q (per-category
    rate matrices, see transition_matrices), freqs, rates and cat_weights exactly as the evaluation sends
    them, p_invar (0: none) and the pattern weights of its weights row."""
    tr = pr.tree[ch] if tree is None else tree
    pinv = pr.p_invar if p_invar is None else float(p_invar)
    freqs = np.asarray(pr.freqs if freqs is None else freqs, float)
    rates = np.asarray(pr.rates, float) / (1.0 - pinv) if rates is None else np.asarray(rates, float)
    catw = np.full(pr.K, (1.0 - pinv) / pr.K) if cat_weights is None else np.asarray(cat_weights, float)
    weights = np.asarray(pr.weights if weights is None else weights, float)
    cl, lnscale = {}, np.zeros(pr.C)

    def pmat(node):
        return transition_matrices(pr, tr.length[node], rates, Q, freqs)

    def child(node):
        x = np.broadcast_to(tip_partials(pr, node), (pr.K, pr.C, pr.S)) if node < tr.n_tips else cl[node]
        return np.einsum("kij,kcj->kci", pmat(node), x)

    for p in tr.post:
        x = child(int(tr.left[p])) * child(int(tr.right[p]))
        if tr.anc[p] == tr.root:                       # the interior root also takes the root tip
            rt = tip_partials(pr, tr.root)[None]
            x = x * np.einsum("kij,kcj->kci", pmat(p), np.broadcast_to(rt, x.shape))
        m = x.max(axis=(0, 2))
        m = np.where(m > 0, m, 1.0)
        cl[p] = x / m[None, :, None]
        lnscale += np.log(m)
    like = np.einsum("k,kcs,s->c", catw, cl[tr.root_left], freqs)
    if pinv > 0:
        inv = np.bitwise_and.reduce(pr.masks, axis=0)
        bits = (inv[:, None] >> np.arange(pr.S, dtype=np.uint64)[None, :]) & np.uint64(1)
        like_i = pinv * (bits * freqs[None, :]).sum(1)
        # Likelihood_Gen's formula; below a scaler of -200 the reference switches to an approximation
        assert lnscale.min() >= -200.0, "site scaler below -200: the reference approximates there"
        site = lnscale + np.log(like + like_i * np.exp(-lnscale))
    else:
        with np.errstate(divide="ignore"):
            site = lnscale + np.log(like)
    return site, float(site @ weights)


# ----------------------------------------------------------------------------- variable-state (Std) divisions
BRLENS_MIN = float(np.float32(1e-8))        # TiProbs_Std clamps the branch length to [BRLENS_MIN, BRLENS_MAX]
BRLENS_MAX = float(np.float32(100.0))
LIKE_EPSILON = 1e-300


def mk_rate_matrix(n):
    """Q of the equal-frequency Mk model on n states: 1/(n-1) off the diagonal, -1 on it (one change per unit time)"""
    Q = np.full((n, n), 1.0 / (n - 1))
    np.fill_diagonal(Q, -1.0)
    return Q


def std_pattern_classes(pr):
    """-> [(n, tiIndex, pattern indices)], one entry per (state count, matrix offset) pair"""
    keys = sorted(set(zip(pr.state_counts.tolist(), pr.matrix_offsets.tolist())))
    return [(n, ti, np.flatnonzero((pr.state_counts == n) & (pr.matrix_offsets == ti))) for n, ti in keys]


class StdLnl:
    """f64_std_lnl's result: per-pattern log likelihoods (site), lnL, the probability of the unobservable
    (dummy) patterns p_un, and whether a non-dummy pattern's likelihood fell below LIKE_EPSILON"""

    def __init__(self, site, lnl, p_un, underflow):
        self.site, self.lnl, self.p_un, self.underflow = site, lnl, p_un, underflow

    def bound(self, pr, weights=None):
        """|lnL - lnL64| allowed for a float evaluation: 2e-7 relative on every observed pattern's log term, plus the
        conditioning of the coding-bias correction, U * 2e-6 * pUn / pObserved (float partials carry a few ulps into
        pUn; the log divides by pObserved).  When 1 - pUn is below LIKE_EPSILON the correction is the clamped
        constant on every side and adds nothing."""
        w = np.asarray(pr.weights if weights is None else weights, float)[pr.dummy:]
        return 2e-7 * float(np.abs(self.site[pr.dummy:]) @ w) + self.conditioning(pr)

    def conditioning(self, pr):
        """U * 2e-6 * pUn / pObserved, or 0 without dummies or when the correction is clamped"""
        p_obs = 1.0 - self.p_un
        return pr.uncompressed * 2e-6 * self.p_un / p_obs if pr.dummy and p_obs >= LIKE_EPSILON else 0.0


def f64_std_lnl(pr, ch, tree=None, *, rates=None, matrices=None, weights=None):
    """Float64 likelihood of a variable-state (STANDARD data) division, from the model's definition.

    Pattern c has n = state_counts[c] states.  P(t) of category k is expm(Q_n v) with v = clamp(length, BRLENS_MIN,
    BRLENS_MAX) * r_k, or, for a branch in `matrices` (node -> the branch's block of matrix_length floats in the host
    layout), the block's [n][n] matrix at matrix_offsets[c] + k n^2, read as row a (parent state), column i (child
    state).  Pruning with the interior root's three neighbours and per-pattern rescaling by the max over categories
    and states.  At the root L_c = 1/K sum_k sum_j pi_j cl[k][c][j], pi = freqs[freq_offsets[c]:] (category weights
    are not used), and lnL = sum_{c >= dummy} w_c log L_c - U log(max(1 - sum_{c < dummy} L_c, LIKE_EPSILON)).
    -> StdLnl"""
    from scipy.linalg import expm
    tr = pr.tree[ch] if tree is None else tree
    rates = np.asarray(pr.rates if rates is None else rates, float)
    weights = np.asarray(pr.weights if weights is None else weights, float)
    matrices = matrices or {}
    K = len(rates)
    classes = std_pattern_classes(pr)
    lnscale = np.zeros(pr.C)
    cl = {}                                              # (node, class) -> [K, patterns, n]

    def pmat(node, n, ti):
        if node in matrices:
            blk = np.asarray(matrices[node], np.float64)
            return blk[ti:ti + K * n * n].reshape(K, n, n)
        v = min(max(float(tr.length[node]), BRLENS_MIN), BRLENS_MAX) * rates
        return np.array([expm(mk_rate_matrix(n) * vk) for vk in v])

    def tip(node, idx, n):
        m = pr.masks[node][idx]
        return ((m[:, None] >> np.arange(n, dtype=np.uint64)[None, :]) & np.uint64(1)).astype(np.float64)

    def child(node, j, n, ti, idx):
        x = np.broadcast_to(tip(node, idx, n), (K, len(idx), n)) if node < tr.n_tips else cl[node, j]
        return np.einsum("kai,kci->kca", pmat(node, n, ti), x)

    for p in tr.post:
        l, r = int(tr.left[p]), int(tr.right[p])
        for j, (n, ti, idx) in enumerate(classes):
            x = child(l, j, n, ti, idx) * child(r, j, n, ti, idx)
            if tr.anc[p] == tr.root:                     # the interior root also takes the root tip
                x = x * np.einsum("kai,kci->kca", pmat(p, n, ti), np.broadcast_to(tip(tr.root, idx, n), x.shape))
            m = x.max(axis=(0, 2))
            m = np.where(m > 0, m, 1.0)
            cl[p, j] = x / m[None, :, None]
            lnscale[idx] += np.log(m)
    like = np.zeros(pr.C)
    for j, (n, ti, idx) in enumerate(classes):
        pi = pr.freqs[pr.freq_offsets[idx][:, None] + np.arange(n)[None, :]]      # [patterns, n]
        like[idx] = np.einsum("kcj,cj->c", cl[tr.root_left, j], pi) / K
    d = pr.dummy
    underflow = bool((like[d:] < LIKE_EPSILON).any())
    with np.errstate(divide="ignore"):
        site = lnscale + np.log(like)
    p_un = float((like[:d] * np.exp(lnscale[:d])).sum())
    lnl = float(site[d:] @ weights[d:]) - pr.uncompressed * np.log(max(1.0 - p_un, LIKE_EPSILON))
    return StdLnl(site, lnl, p_un, underflow)


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
