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


# ---- the root with an invariable-sites category ------------------------------------------------------------------
# A pattern's likelihood is (1 - p) L + p L_I, with L = exp(lnScaler) like the rescaled root sum.  MrBayes cannot
# exponentiate a site scaler below SCALER_SWITCH, so there it approximates, and two of its likelihood families do so
# differently.  Three rules, per pattern, with s the site scaler the decision reads:
#   ROOT_EXACT  logaddexp(lnScaler + log like, log likeI), the mixture itself;
#   ROOT_GEN    Likelihood_Gen / _Gen_SSE: s >= -200: log(like + likeI / exp(lnScaler)) + lnScaler;
#               s < -200: log likeI if likeI > LIKE_I_MIN (like is negligible beside it), else lnScaler + log like
#               (likeI is dropped, even where it dominates);
#   ROOT_QUIRK  Likelihood_NUC4_* (MB200_FLAG_NUC4_PINVAR_QUIRK): as ROOT_GEN, except that for s < -200 and
#               likeI > LIKE_I_MIN the term is lnScaler + log likeI -- the scaler is added to a likelihood that was
#               never scaled.
# ROOT_GEN equals ROOT_EXACT except where s < -200 and 0 < likeI <= LIKE_I_MIN (it is lower there); ROOT_QUIRK equals
# ROOT_GEN except where s < -200 and likeI > LIKE_I_MIN (lower by |lnScaler|).
ROOT_EXACT, ROOT_GEN, ROOT_QUIRK = "exact", "gen", "quirk"
SCALER_SWITCH = -200.0
LIKE_I_MIN = 1e-70
FLAG_NUC4_PINVAR_QUIRK = 1                    # MB200_FLAG_NUC4_PINVAR_QUIRK (include/mb200.h)
# which side of the switch a pattern is on (RootTerms.branch)
ABOVE_SWITCH, INVAR_DOMINATES, INVAR_TINY, INVAR_ZERO = 0, 1, 2, 3


class RootTerms:
    """f64_root's result: per-pattern log likelihoods (site) and lnL; the float64 site scalers (lnscale), the rescaled
    root sums (like) and the invariable-site likelihoods p L_I (like_i); with p_invar, per pattern which branch of the
    rule it took (branch: ABOVE_SWITCH, or below the switch INVAR_DOMINATES (likeI > LIKE_I_MIN), INVAR_TINY
    (0 < likeI <= LIKE_I_MIN) or INVAR_ZERO), else None"""

    def __init__(self, site, lnl, lnscale, like, like_i, branch):
        self.site, self.lnl, self.lnscale, self.like, self.like_i, self.branch = site, lnl, lnscale, like, like_i, branch


def root_rule_of(flags):
    """the rule an evaluation with these flags asks for: ROOT_QUIRK with MB200_FLAG_NUC4_PINVAR_QUIRK, else ROOT_GEN"""
    return ROOT_QUIRK if int(flags) & FLAG_NUC4_PINVAR_QUIRK else ROOT_GEN


def root_site_terms(lnscale, like, like_i, rule, scalers=None):
    """-> (per-pattern log likelihoods, branch) under `rule`.  The terms use the float64 lnscale; the decision at
    SCALER_SWITCH reads `scalers` if given (a float site-scaler vector read back from an engine or the oracle, so
    that a pattern near -200 branches as it did there), else lnscale."""
    s = np.asarray(lnscale if scalers is None else scalers, np.float64)
    below_switch = s < SCALER_SWITCH
    branch = np.where(~below_switch, ABOVE_SWITCH,
                      np.where(like_i > LIKE_I_MIN, INVAR_DOMINATES, np.where(like_i > 0, INVAR_TINY, INVAR_ZERO)))
    with np.errstate(divide="ignore", over="ignore"):
        log_like_i = np.log(like_i)
        exact = np.logaddexp(lnscale + np.log(like), log_like_i)
        if rule == ROOT_EXACT:
            return exact, branch
        mixed = lnscale + np.log(like + like_i * np.exp(np.minimum(-lnscale, 700.0)))
        dominated = log_like_i + (lnscale if rule == ROOT_QUIRK else 0.0)
    assert rule in (ROOT_GEN, ROOT_QUIRK), rule
    site = np.where(branch == ABOVE_SWITCH, mixed,
                    np.where(branch == INVAR_DOMINATES, dominated, lnscale + np.log(like)))
    return site, branch


def f64_lnl(pr, ch, tree=None, **kw):
    """-> (per-pattern log likelihoods [C], lnL) of chain `ch` on its current tree: f64_root's"""
    r = f64_root(pr, ch, tree, **kw)
    return r.site, r.lnl


def f64_root(pr, ch, tree=None, *, Q=None, freqs=None, rates=None, cat_weights=None, p_invar=None, weights=None,
             flags=None, rule=None, scalers=None, pmat_cache=None):
    """Float64 pruning of chain `ch` on its current tree -> RootTerms.

    Without overrides the model is the problem's: its eigensystem, frequencies, rates / (1 - p_invar) and
    equal category weights (1 - p_invar) / K.  Overrides describe one evaluation's own model: Q (per-category
    rate matrices, see transition_matrices), freqs, rates and cat_weights exactly as the evaluation sends
    them, p_invar (0: none) and the pattern weights of its weights row.  With p_invar the root follows `rule`
    (ROOT_EXACT, ROOT_GEN or ROOT_QUIRK; default the one `flags` ask for, default the problem's flags), its
    decision at the switch read from `scalers` if given (root_site_terms).  pmat_cache, a dict the caller keeps
    across calls with the same model, holds P(t) by branch length, for long runs of branch updates."""
    tr = pr.tree[ch] if tree is None else tree
    pinv = pr.p_invar if p_invar is None else float(p_invar)
    freqs = np.asarray(pr.freqs if freqs is None else freqs, float)
    rates = np.asarray(pr.rates, float) / (1.0 - pinv) if rates is None else np.asarray(rates, float)
    catw = np.full(pr.K, (1.0 - pinv) / pr.K) if cat_weights is None else np.asarray(cat_weights, float)
    weights = np.asarray(pr.weights if weights is None else weights, float)
    cl, lnscale = {}, np.zeros(pr.C)

    def pmat(node):
        t = float(tr.length[node])
        if pmat_cache is None:
            return transition_matrices(pr, t, rates, Q, freqs)
        if t not in pmat_cache:
            pmat_cache[t] = transition_matrices(pr, t, rates, Q, freqs)
        return pmat_cache[t]

    def child(node):
        x = np.broadcast_to(tip_partials(pr, node), (pr.K, pr.C, pr.S)) if node < tr.n_tips else cl[node]
        return np.einsum("kij,kcj->kci", pmat(node), x)

    for p in tr.post:
        x = child(int(tr.left[p])) * child(int(tr.right[p]))
        if tr.anc[p] == tr.root:                       # the interior root also takes the root tip
            rt = tip_partials(pr, tr.root)[None]
            x = x * np.einsum("kij,kcj->kci", pmat(p), np.broadcast_to(rt, x.shape))
            # ...and is not rescaled, as in MrBayes: the site scaler holds the other nodes' scalers only, which
            # matters where a root rule adds it to a likelihood it did not scale (ROOT_QUIRK)
            cl[p] = x
            continue
        m = x.max(axis=(0, 2))
        m = np.where(m > 0, m, 1.0)
        cl[p] = x / m[None, :, None]
        lnscale += np.log(m)
    like = np.einsum("k,kcs,s->c", catw, cl[tr.root_left], freqs)
    like_i, branch = np.zeros(pr.C), None
    if pinv > 0:
        inv = np.bitwise_and.reduce(pr.masks, axis=0)
        bits = (inv[:, None] >> np.arange(pr.S, dtype=np.uint64)[None, :]) & np.uint64(1)
        # the 4-state family takes p_invar as a float (Likelihood_NUC4_*: (CLFlt) pInvar), so below FLT_TRUE_MIN it
        # is 0 and likeI with it: 0 < likeI <= LIKE_I_MIN (INVAR_TINY) cannot occur on 4 states
        p = float(np.float32(pinv)) if pr.S == 4 else pinv
        like_i = p * (bits * freqs[None, :]).sum(1)
        rule = root_rule_of(pr.flags if flags is None else flags) if rule is None else rule
        site, branch = root_site_terms(lnscale, like, like_i, rule, scalers)
    else:
        with np.errstate(divide="ignore"):
            site = lnscale + np.log(like)
    return RootTerms(site, float(site @ weights), lnscale, like, like_i, branch)


# ---- how far float site scalers may drift from float64 ------------------------------------------------------------
# An engine (and MrBayes) keeps a pattern's site scaler as a float sum: a full evaluation resets it and adds one node
# scaler per rescaled node, each branch update removes the replaced nodes' scalers and adds the new ones, a rejected
# update flips back to the previous vector.  Each addition or removal rounds to the nearest float, an error of at most
# half an ulp of the value it lands on; each node scaler is itself log(max) rounded to float, half an ulp of the node
# scaler.  Node scalers are logs of maxima <= 1, so all of them are <= 0: a node scaler is no larger than the site
# scaler it is part of, and every partial sum on the way from a vector s_src to its update s_dst is bounded by
# |s_src| + |s_dst| (removals move towards 0; the additions are a subset of s_dst's terms).  With M_c the largest
# such bound since the last reset, n the additions and removals since then and m the node scalers in the sum, the
# site scaler of pattern c is off by at most (n + m) ulp(M_c) / 2, and lnL, which adds each site scaler w_c times, by
#     drift = sum_c w_c (n + m) ulp(M_c) / 2.
# At a thousand tips this is far above a few float ulps of lnL: a 4-state full evaluation at 1000 tips rounds ~1000
# times into values of a few hundred.  The bar a float evaluation meets against float64 is the small-tree relative
# bar for everything else (P(t), partials, the root sum) plus this drift.
def half_ulp(x):
    """half the float32 ulp of |x|, elementwise, in double"""
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64) / 2


class ScalerLedger:
    """Per site-scaler buffer: the additions and removals (n) and node scalers (m) its float sum has taken since its
    last reset, and M_c of every pattern -- the drift bound above.  record() each evaluation with the site scalers it
    wrote (read back, float); a rejection needs nothing, since the restored buffer's entry is still here."""

    def __init__(self):
        self.book = {}                                   # site buffer -> (n, m, M [C], s [C])

    def record(self, sp, site_scalers):
        s = np.abs(np.asarray(site_scalers, np.float64))
        writes = int((sp.ops["scale_write"] >= 0).sum())
        removes = int((sp.ops["scale_remove"] >= 0).sum())
        if sp.site_src < 0:
            n, m, M = writes, writes, s
        else:
            n0, m, M0, s0 = self.book[int(sp.site_src)]
            n, M = n0 + writes + removes, np.maximum(M0, s0 + s)
            m += writes - removes
        self.book[int(sp.site_dst)] = (n, m, M, s)

    def pattern_bound(self, sp):
        """[C] how far each float site scaler of sp's destination may be from float64: (n + m) ulp(M_c) / 2"""
        n, m, M, _ = self.book[int(sp.site_dst)]
        return (n + m) * half_ulp(M)

    def drift(self, sp, weights):
        """the bound on |lnL - lnL64| the float site scalers of sp's destination may carry"""
        return float(np.asarray(weights, np.float64) @ self.pattern_bound(sp))


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


# ----------------------------------------------------------------------------- one evaluation over explicit buffers
FLAG_TIP_SHORTCUTS = 2                        # MB200_FLAG_TIP_SHORTCUTS (include/mb200.h)
NONE = -1


def is_variable_states(pr):
    return getattr(pr, "state_counts", None) is not None


def ragged_to_padded(pr, a):
    """Std partials: the ragged host layout [K, sum nStates] -> [K, C, S], zeros past each pattern's state count"""
    off = np.concatenate([[0], np.cumsum(pr.state_counts)])
    out = np.zeros((pr.K, pr.C, pr.S))
    for c in range(pr.C):
        out[:, c, :pr.state_counts[c]] = a[:, off[c]:off[c + 1]]
    return out


def padded_to_ragged(pr, x):
    return np.concatenate([x[:, c, :pr.state_counts[c]] for c in range(pr.C)], axis=1)


def std_mk_block(pr, length, rates):
    """a variable-state branch's block in float64: expm of each class's Mk rate matrix times clamp(length) r_k, as the
    engine builds it for a matrix update"""
    from scipy.linalg import expm
    blk = np.zeros(pr.matrix_length)
    v = min(max(float(length), BRLENS_MIN), BRLENS_MAX) * np.asarray(rates, float)
    for n, ti, _ in std_pattern_classes(pr):
        for k, vk in enumerate(v):
            blk[ti + k * n * n: ti + (k + 1) * n * n] = np.maximum(expm(mk_rate_matrix(n) * vk), 0.0).ravel()
    return blk


class Evaluation64:
    """f64_evaluation's result: every partials buffer the operations wrote (host layout: [K, C, S], ragged for Std),
    every node scaler they wrote, the site scaler (None without site_dst) and the one it started from, lnL and whether a pattern underflowed (None
    without a root), and per destination the operations of the call in its subtree, itself included (below) and the
    largest product before rescaling, per pattern (peak; 1 where the node is not rescaled)"""

    def __init__(self):
        self.partials, self.scalers, self.below, self.peak = {}, {}, {}, {}
        self.site = self.site_src = self.lnl = self.underflow = None
        self.p_un = 0.0


def f64_evaluation(pr, sp, partials=None, matrices=None, scalers=None, weights=None, Q=None):
    """Float64 restatement of one mb200_evaluation over the exact operation list of sp -> Evaluation64.

    The inputs are the buffers the operations read, as the caller holds them: tips from pr.masks; interior partials
    (partials: buffer -> host layout), P(t) (matrices: matrix -> [K, S, S] or a Std block) and node and site scalers
    (scalers: buffer -> [C]).  sp's matrix updates are rebuilt here in float64 from the problem's eigensystem, or with Q
    (per-category rate matrices) by the matrix exponential (transition_matrices; Std: the Mk model), with sp's rates and
    frequencies, and replace the given ones.  Operations run in order: each child term is
    P x (a tip's state set as 0/1; with MB200_FLAG_TIP_SHORTCUTS a missing observation on a tip without partial
    ambiguity is exactly 1), the children multiply, scale_remove leaves the site scaler first, then with scale_write
    the node is divided by its largest entry per pattern, whose log is the node scaler and joins the site scaler.  A
    node without scale_write -- the interior root -- is not rescaled.  The site scaler starts from site_scaler_src
    (zeros without).  The root follows f64_root: ROOT_QUIRK or ROOT_GEN by sp's flags with p_invar, Std's coding-bias
    correction, weights row `weights` (default the problem's)."""
    std = is_variable_states(pr)
    K, C, S = pr.K, pr.C, pr.S
    weights = np.asarray(pr.weights if weights is None else weights, float)
    rates, freqs = np.asarray(sp.rates, float), np.asarray(sp.freqs, float)
    mats = {int(m): np.asarray(v, np.float64) for m, v in (matrices or {}).items()}
    for mu in sp.mats:
        m, t = int(mu["matrix"]), float(mu["length"])
        mats[m] = std_mk_block(pr, t, rates) if std else transition_matrices(pr, t, rates, Q, freqs[:S])
    given = {int(b): (ragged_to_padded(pr, np.asarray(a, np.float64)) if std else np.asarray(a, np.float64))
             for b, a in (partials or {}).items()}
    scal = {int(s): np.asarray(v, np.float64) for s, v in (scalers or {}).items()}
    n_tips = pr.masks.shape[0]
    full = np.uint64((1 << S) - 1) if S < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
    classes = std_pattern_classes(pr) if std else None
    out = Evaluation64()
    cl = {}

    def tip(node):
        if std:
            n = pr.state_counts.astype(np.uint64)
            bits = (pr.masks[node][:, None] >> np.arange(S, dtype=np.uint64)[None, :]) & np.uint64(1)
            return np.where(np.arange(S)[None, :] < n[:, None], bits, 0).astype(np.float64)
        return tip_partials(pr, node)

    def ambiguous(node):
        m = pr.masks[node]
        return bool(((m != full) & ((m & (m - np.uint64(1))) != 0)).any())

    def term(child, matrix):
        x = cl[child] if child in cl else given[child] if child >= n_tips else np.broadcast_to(tip(child), (K, C, S))
        P = mats[matrix]
        if not std:
            y = np.einsum("kij,kcj->kci", P, x)
            if child < n_tips and sp.flags & FLAG_TIP_SHORTCUTS and not ambiguous(child):
                y[:, pr.masks[child] == full, :] = 1.0
            return y
        y = np.zeros((K, C, S))
        for n, ti, idx in classes:
            Pk = P[ti:ti + K * n * n].reshape(K, n, n)
            y[:, idx, :n] = np.einsum("kai,kci->kca", Pk, x[:, idx, :n])
        return y

    site = scal[sp.site_src].copy() if sp.site_src >= 0 else np.zeros(C)
    out.site_src = site.copy()
    for op in sp.ops:
        dest = int(op["dest"])
        x = term(int(op["child1"]), int(op["matrix1"])) * term(int(op["child2"]), int(op["matrix2"]))
        if op["child3"] >= 0:
            x = x * term(int(op["child3"]), int(op["matrix3"]))
        if op["scale_remove"] >= 0:
            r = int(op["scale_remove"])
            site -= out.scalers[r] if r in out.scalers else scal[r]
        peak = np.ones(C)
        if op["scale_write"] >= 0:
            peak = x.max(axis=(0, 2))
            peak = np.where(peak > 0, peak, 1.0)
            x = x / peak[None, :, None]
            with np.errstate(divide="ignore"):
                out.scalers[int(op["scale_write"])] = np.log(peak)
            site += np.log(peak)
        cl[dest] = x
        out.peak[dest] = peak
        out.below[dest] = 1 + sum(out.below.get(int(op[f]), 0) for f in ("child1", "child2", "child3") if op[f] >= n_tips)
    for dest, x in cl.items():
        out.partials[dest] = padded_to_ragged(pr, x) if std else x
    if sp.site_dst >= 0:
        out.site = site
    if sp.root < 0:
        return out
    root = cl[sp.root] if sp.root in cl else given[sp.root]
    with np.errstate(divide="ignore", invalid="ignore"):
        if std:
            like = np.zeros(C)
            for n, ti, idx in classes:
                pi = freqs[pr.freq_offsets[idx][:, None] + np.arange(n)[None, :]]
                like[idx] = np.einsum("kcj,cj->c", root[:, idx, :n], pi) / K
            d = pr.dummy
            out.p_un = float((like[:d] * np.exp(site[:d])).sum())
            out.underflow = bool((like[d:] < LIKE_EPSILON).any())
            out.lnl = float((site[d:] + np.log(like[d:])) @ weights[d:]) - \
                pr.uncompressed * np.log(max(1.0 - out.p_un, LIKE_EPSILON))
            return out
        like = np.einsum("k,kcs,s->c", np.asarray(sp.cat_weights, float), root, freqs[:S])
        if not sp.has_p_invar:
            out.underflow = bool((like < LIKE_EPSILON).any())
            out.lnl = float((site + np.log(like)) @ weights)
            return out
        inv = np.bitwise_and.reduce(pr.masks, axis=0)
        bits = (inv[:, None] >> np.arange(S, dtype=np.uint64)[None, :]) & np.uint64(1)
        p = float(np.float32(sp.p_invar)) if S == 4 else float(sp.p_invar)
        like_i = p * (bits * freqs[None, :S]).sum(1)
        rule = root_rule_of(sp.flags)
        terms, _ = root_site_terms(site, like, like_i, rule)
        if rule == ROOT_QUIRK:        # the quirk tests the likelihood it takes the log of
            tested = np.where(site < SCALER_SWITCH, np.where(like_i > LIKE_I_MIN, like_i, like),
                              like + like_i * np.exp(np.minimum(-site, 700.0)))
        else:
            tested = like
        out.underflow = bool((tested < LIKE_EPSILON).any())
        out.lnl = float(terms @ weights)
    return out
