"""Sparse rescaling for workloads.Problem: the reference's rescale-frequency bookkeeping
(src/likelihood.c:7938-7965, restated by the seam's SeamBuildOps), so that tests can send the
engine operation lists in which some interior nodes write no scaler and some remove an old
scaler without writing a new one -- what the dynamic rescaling scheme produces.

Per chain, a table counts the unscaled interior levels below each node (tips count 0):

  unscaled[p] = 1 + unscaled[left] + unscaled[right]
  remove p's old scaler   iff unscaled[p] == 0 before the update and the evaluation is not a full one
  write a new scaler      iff unscaled[p] reaches f and p is not the interior root; unscaled[p] = 0 then

A copy of the table is kept with each evaluation and put back when it is rejected
(unscaledNodesScratch, src/likelihood.c:5645).  f = 1 gives Problem's own lists; f = inf never
rescales.

The threshold_* builders at the end set up one-node evaluations whose rescaler maximum or root
likelihood sits exactly at the float-range guard's threshold (MB200_FLAG_RANGE_GUARD)."""
import types

import numpy as np

from engine_checks import num_sms, ppb, resident_generations, via_evaluate, via_replay
from mrbayes_b200 import abi, workloads


def _spec(self, ch, dirty_branches, dirty_nodes, full):
    sp = type(self)._spec(self, ch, dirty_branches, dirty_nodes, full)
    st, tr, u = self.chains[ch], self.tree[ch], self.unscaled[ch]
    self.unscaled_scratch[ch] = u.copy()
    ops = sp.ops
    for i, p in enumerate([p for p in tr.post if p in dirty_nodes]):
        assert ops["dest"][i] == st.cl[p]
        # Problem's _spec has flipped the scaler slots: the old scaler is the scratch slot now
        ops["scale_remove"][i] = st.ns_scratch[p] if (u[p] == 0 and not full) else abi.NONE
        u[p] = 1 + u[int(tr.left[p])] + u[int(tr.right[p])]
        if u[p] >= self.rescale_freq and tr.anc[p] != tr.root:
            ops["scale_write"][i] = st.ns[p]
            u[p] = 0
        else:
            ops["scale_write"][i] = abi.NONE
    return sp


def _reject(self, ch, spec, old_lengths=None):
    self.unscaled[ch][:] = self.unscaled_scratch[ch]
    type(self).reject(self, ch, spec, old_lengths)


def sparse_rescaling(pr, f):
    """Switch pr's evaluation builders (full_evaluation, branch_update, reject) to rescale every
    f-th unscaled level; call before the first evaluation."""
    pr.rescale_freq = f
    pr.unscaled = [np.zeros(pr.n_nodes, np.int64) for _ in range(pr.n_chains)]
    pr.unscaled_scratch = [u.copy() for u in pr.unscaled]
    pr._spec = types.MethodType(_spec, pr)
    pr.reject = types.MethodType(_reject, pr)
    return pr


def step_frequency(pr, f, it):
    """Frequency of update `it` of a run at f: f and f + 1 in turn for 1 < f < inf.  A dynamic scheme
    changes a chain's frequency between evaluations; only then does a node that held a scaler come
    out of an update without one -- the remove-only operation -- since a branch-length update leaves
    the counts below each node as they were."""
    pr.rescale_freq = f if f in (1, np.inf) else f + it % 2


def deep_problem():
    """4-state, K = 4, 192 patterns (three 64-pattern tiles), an 80-tip caterpillar with mean branch
    length 0.1.  Unscaled, the float64 node maxima of some pattern fall below 1e-24 at level 36,
    1e-30 at level 46 and the normal float range at level 65 (tests/test_sparse_rescaling.py checks)"""
    from f64_reference import caterpillar_tree
    pr = workloads.make_problem(4, 4, 192, 80, 1, seed=5)
    pr.tree[0] = caterpillar_tree(80, np.random.default_rng(5))
    return pr


def unscaled_maxima(pr, ch):
    """{interior node: float64 largest entry of its conditional likelihoods over categories and
    states, per pattern [C]} with no node rescaled: how far sparse rescaling lets a subtree fall"""
    from f64_reference import tip_partials, transition_matrices
    tr = pr.tree[ch]
    rates = np.asarray(pr.rates, float) / (1.0 - pr.p_invar)
    cl, out = {}, {}

    def child(node, length):
        x = np.broadcast_to(tip_partials(pr, node), (pr.K, pr.C, pr.S)) if node < tr.n_tips else cl[node]
        return np.einsum("kij,kcj->kci", transition_matrices(pr, length, rates), x)

    for p in tr.post:
        x = child(int(tr.left[p]), tr.length[tr.left[p]]) * child(int(tr.right[p]), tr.length[tr.right[p]])
        if tr.anc[p] == tr.root:                       # the root tip hangs on the interior root's branch
            x = x * child(tr.root, tr.length[p])
        cl[p] = x
        out[p] = x.max(axis=(0, 2))
    return out


# ---- the float-range guard at its threshold -------------------------------------------------------------------------
GUARD_MIN = np.float32(1e-24)
THRESHOLD_C = {"host": 10, "device": 40, "non_fused": None, "throughput": 10, "resident": 12}   # resident: <= 16 tiles


def threshold_setup(route, K, where, n_eval):
    """n_eval evaluations of one node each over 4 tips (buffers and slots of chain e for evaluation e):
    the node multiplies interior buffers x and 1.0 through P = I (branch length 0).  -> problem, C,
    the pattern that will carry the value"""
    tiles = THRESHOLD_C[route] or 4 * num_sms() + 4
    C = tiles * ppb(K) - (ppb(K) - 1 if where == "last" else 0)
    pr = workloads.make_problem(4, K, C, 4, n_eval, seed=12, flags=abi.FLAG_NUC4_PINVAR_QUIRK | abi.FLAG_RANGE_GUARD)
    pr.freqs = np.full(4, 0.25)
    return pr, C, (C - 1 if where == "last" else C // 2 + 1)


def threshold_spec(pr, e_idx, kind):
    """kind 'node': buffer a -> rescaled node d1 -> unscaled root d2; kind 'root': a -> unscaled root d1"""
    nI = pr.n_int
    a, ones, d1, d2 = (pr.n_tips + 2 * e_idx * nI + j for j in range(4))
    mat = 2 * e_idx * pr.n_nodes
    base = 2 * e_idx * (nI + 1)
    op = lambda dest, c1, sw: (dest, c1, mat, ones, mat, abi.NONE, abi.NONE, sw, abi.NONE)
    ops = [op(d1, a, base), op(d2, d1, abi.NONE)] if kind == "node" else [op(d1, a, abi.NONE)]
    return abi.EvalSpec(mats=np.array([(mat, 0, 0.0)], abi.MAT_DTYPE), ops=np.array(ops, abi.OP_DTYPE),
                        site_dst=base + 1, site_src=abi.NONE, root=ops[-1][0], flags=pr.flags,
                        rates=pr.rates, cat_weights=np.full(pr.K, 1.0 / pr.K), freqs=pr.freqs, chain=e_idx)


def threshold_partials(pr, kind, c, x):
    """'node': 0.5 everywhere but x at pattern c -- its maximum; 'root' (K = 1, frequencies 1/4):
    1.0 everywhere but x in every state of c, so that likeF = 4 (x / 4) = x exactly"""
    a = np.full((pr.K, pr.C, 4), 0.5 if kind == "node" else 1.0, np.float32)
    if x is not None:
        a[:, c, :] = x
    return a


def run_threshold(e, o, route, gens):
    """each generation (a list of evaluations) on the route and on the oracle -> [(lnL, status, oracle
    lnL, oracle status)] per evaluation, per generation.  The resident route packs every generation
    first, so that one kernel can serve them all."""
    if route == "resident":
        got = resident_generations(e, gens)
    else:
        got = [(via_replay if route == "device" else via_evaluate)(e, specs) for specs in gens]
    out = []
    for (lnl, st), specs in zip(got, gens):
        out.append([(lnl[i], st[i]) + tuple(x[0] for x in o.evaluate(sp)) for i, sp in enumerate(specs)])
    return out


def threshold_instance(pr, lib, route, values, kind, c):
    e = pr.create(lib, flags=abi.CONFIG_THROUGHPUT if route == "throughput" else 0)
    ones = np.ones((pr.K, pr.C, 4), np.float32)
    for i, x in enumerate(values):
        base = pr.n_tips + 2 * i * pr.n_int
        e.set_partials(base, threshold_partials(pr, kind, c, x))
        e.set_partials(base + 1, ones)
    return e
