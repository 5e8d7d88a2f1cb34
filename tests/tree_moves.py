"""Tree moves for workloads.Problem: the operation lists MrBayes sends after moves other than a branch-length change,
built through the problem's own _spec (so sparse_rescaling composes with them), and rooted clock trees.

- Whole-tree updates that keep their site scalers (TouchAllTreeNodes, reference src/proposal.c; upDateAll is set only
  after UpDateCijk, src/likelihood.c:7864-7872): every branch rebuilt and every interior node dirty with
  site_scaler_src copied, not reset, so every rescaled node removes its old scaler.  Two kinds: tree length (every
  length times a factor; on a clock tree, every age) and the chain's model (new rates, and with invariable sites a new
  p_invar and category weights), lengths unchanged.
- Topology moves (NNI, SPR): children, ancestors and lengths change, post is recomputed as a down pass.  A node is
  dirty when its children changed, a branch below it changed length, or it becomes or stops being the interior root,
  and so is every node above one; the branches whose length changed are rebuilt, and on unrooted trees the interior
  root's own branch (as branch_update does).  So the dirty set is the union of two or more paths to the root, a clean
  interior buffer can be read by a new parent, and the interior root can change: the new one removes its old scaler
  and writes none, the former one writes a scaler with nothing to remove.
- Rooted trees (clock analyses): tip n_tips - 1, the Tree's root tip, is a dummy with an all-missing mask that no
  operation reads, so the interior root has two children: its operation has no child3 / matrix3 and writes no scaler,
  and its own branch is never rebuilt (src/likelihood.c:7910-7936).  Branch lengths are age differences, some exactly
  0 (sampled ancestors, and interior nodes as old as a child); a node-age move changes the three branches at a node.

Every builder returns a Move; reject(pr, mv) puts topology, post, lengths, ages, the chain's model and which nodes hold
a scaler back and undoes the index flips with the problem's reject (ResetFlips).  Each chain carries its own model
(rates, category weights, p_invar), which every evaluation built here sends; f64(pr, ch) is the float64 likelihood
of the chain's current tree under it."""
from dataclasses import dataclass, field

import numpy as np

from f64_reference import f64_root, f64_std_lnl
from mrbayes_b200 import abi, workloads


# ---- rooted problems ------------------------------------------------------------------------------------------------
class RootedSpec:
    """_spec for rooted trees: the interior root's branch is never rebuilt, its operation multiplies two children"""

    def _spec(self, ch, dirty_branches, dirty_nodes, full):
        tr = self.tree[ch]
        sp = super()._spec(ch, [b for b in dirty_branches if b != tr.root_left], dirty_nodes, full)
        if sp.ops is not None and len(sp.ops):
            at = sp.ops["dest"] == self.chains[ch].cl[tr.root_left]
            sp.ops["child3"][at] = abi.NONE
            sp.ops["matrix3"][at] = abi.NONE
        return sp


class RootedProblem(RootedSpec, workloads.Problem):
    pass


class RootedStdProblem(RootedSpec, workloads.StdProblem):
    pass


def make_rooted(pr, rng, p_zero=0.15, mean_gap=0.05):
    """pr (a Problem or StdProblem with one tip more than the rooted tree has) as a rooted problem: the root tip is the
    dummy, every chain's tree a clock tree (clock_ages).  Call before the first evaluation."""
    pr.__class__ = RootedStdProblem if isinstance(pr, workloads.StdProblem) else RootedProblem
    pr.rooted = True
    for tr in pr.tree:
        assert tr.root == pr.n_tips - 1
    if isinstance(pr, workloads.StdProblem):
        full = (np.uint64(1) << pr.state_counts.astype(np.uint64)) - np.uint64(1)
    else:
        full = np.full(pr.C, np.uint64((1 << pr.S) - 1) if pr.S < 64 else np.uint64(0xFFFFFFFFFFFFFFFF))
    pr.masks[pr.tree[0].root] = full
    for tr in pr.tree:
        clock_ages(tr, rng, p_zero, mean_gap)
    return pr


def clock_ages(tr, rng, p_zero=0.15, mean_gap=0.05):
    """Ultrametric lengths from node ages (tr.age): an interior node is older than its older child by an exponential
    gap, or, with probability p_zero where its children differ in age, exactly as old as the older one; a few tips are
    fossils (older than 0) and a few sampled ancestors (as old as their parent, where no other branch at the parent
    has length 0).  So some branches, tip and interior, have length exactly 0, and no two tips are joined by a path
    of them (that would make a pattern where they differ impossible)."""
    age = np.zeros(tr.n_nodes)
    for p in tr.post:
        a, b = age[tr.left[p]], age[tr.right[p]]
        age[p] = max(a, b) + (0.0 if a != b and rng.random() < p_zero else rng.exponential(mean_gap))
    for t in range(tr.n_tips):
        if t == tr.root:
            continue
        q, u = int(tr.anc[t]), rng.random()
        alone = q != tr.root_left and age[sibling(tr, t)] < age[q] < age[tr.anc[q]]
        if u < 0.12 and alone:
            age[t] = age[q]                              # sampled ancestor
        elif u < 0.25:
            age[t] = rng.uniform(0.0, age[q])            # fossil
    tr.age = age
    lengths_from_ages(tr)


def lengths_from_ages(tr):
    for c in range(tr.n_nodes):
        tr.length[c] = 0.0 if c in (tr.root, tr.root_left) else tr.age[tr.anc[c]] - tr.age[c]


def rooted(pr):
    return getattr(pr, "rooted", False)


# ---- trees --------------------------------------------------------------------------------------------------------
def down_pass(tr):
    """interior nodes below the root tip in post-order (intDownPass)"""
    out, stack = [], [(int(tr.left[tr.root]), 0)]
    while stack:
        node, st = stack.pop()
        if node < tr.n_tips:
            continue
        if st == 0:
            stack += [(node, 1), (int(tr.right[node]), 0), (int(tr.left[node]), 0)]
        else:
            out.append(node)
    return out


def comb_tree(n, rng, mean_len=0.1):
    """A spine whose every node has a cherry (two tips) beside it: a path up the spine reads one clean interior
    operand per node.  Tips 0..n-2 below the interior root, n-1 the root tip; interior nodes numbered in post-order."""
    from f64_reference import _tree
    left, right = np.full(2 * n - 2, -1), np.full(2 * n - 2, -1)
    nxt = [n]

    def node(a, b):
        p = nxt[0]; nxt[0] += 1
        left[p], right[p] = a, b
        return p
    spine, t = node(0, 1), 2
    while t < n - 1:
        if t + 1 < n - 1:
            side = node(t, t + 1); t += 2
        else:
            side = t; t += 1
        spine = node(spine, side)
    return _tree(n, left, right, rng, mean_len)


def subtree(tr, v):
    out, stack = set(), [v]
    while stack:
        x = stack.pop()
        out.add(x)
        if x >= tr.n_tips and x != tr.root:
            stack += [int(tr.left[x]), int(tr.right[x])]
    return out


def depth(tr, v):
    return len(tr.path_to_root(v))


def sibling(tr, v):
    p = tr.anc[v]
    return int(tr.right[p]) if tr.left[p] == v else int(tr.left[p])


def check_tree(tr, is_rooted=False):
    """the invariants of a tree in MrBayes' numbering; a clock tree's lengths are its age differences"""
    n = tr.n_tips
    assert tr.left[tr.root] == tr.root_left and tr.anc[tr.root_left] == tr.root and tr.anc[tr.root] == -1
    assert sorted(tr.post) == list(range(n, 2 * n - 2)) and tr.post == down_pass(tr)
    seen = set(range(n))
    for p in tr.post:
        assert int(tr.left[p]) in seen and int(tr.right[p]) in seen and tr.left[p] != tr.right[p]
        assert tr.anc[tr.left[p]] == p and tr.anc[tr.right[p]] == p
        seen.add(p)
    assert (tr.length >= 0).all()
    if is_rooted:
        assert tr.root_left >= n and tr.left[tr.root_left] >= 0 and tr.right[tr.root_left] >= 0
        for c in range(tr.n_nodes):
            if c not in (tr.root, tr.root_left):
                assert tr.length[c] == tr.age[tr.anc[c]] - tr.age[c]


# ---- per-chain models ---------------------------------------------------------------------------------------------
@dataclass
class Model:
    rates: np.ndarray            # before the 1 / (1 - p_invar) the evaluation sends
    p_invar: float
    weights: np.ndarray          # category weights before the (1 - p_invar)


def models(pr):
    if not hasattr(pr, "chain_model"):
        pr.chain_model = [Model(np.asarray(pr.rates, float).copy(), pr.p_invar, np.full(pr.K, 1.0 / pr.K))
                          for _ in range(pr.n_chains)]
    return pr.chain_model


def with_model(pr, sp):
    """sp under its chain's model"""
    m = models(pr)[sp.chain]
    sp.rates = m.rates / (1.0 - m.p_invar)
    sp.cat_weights = m.weights * (1.0 - m.p_invar)
    sp.p_invar, sp.has_p_invar = m.p_invar, int(m.p_invar > 0)
    return sp


def f64(pr, ch, scalers=None):
    """float64 likelihood of chain ch's current tree under its model: RootTerms (StdLnl for Std)"""
    m = models(pr)[ch]
    if isinstance(pr, workloads.StdProblem):
        return f64_std_lnl(pr, ch, rates=m.rates)
    return f64_root(pr, ch, rates=m.rates / (1.0 - m.p_invar), cat_weights=m.weights * (1.0 - m.p_invar),
                    p_invar=m.p_invar, scalers=scalers)


# ---- moves ----------------------------------------------------------------------------------------------------------
@dataclass
class Move:
    kind: str
    ch: int
    spec: object
    saved: tuple
    mats: object = None
    info: dict = field(default_factory=dict)


def _save(pr, ch):
    tr, st = pr.tree[ch], pr.chains[ch]
    m = models(pr)[ch]
    return (tr.left.copy(), tr.right.copy(), tr.anc.copy(), tr.length.copy(), list(tr.post),
            getattr(tr, "age", np.zeros(0)).copy(), st.scaled.copy(), Model(m.rates.copy(), m.p_invar, m.weights.copy()))


def _spec(pr, ch, kind, saved, branches, dirty, info=None):
    sp = with_model(pr, pr._spec(ch, branches, dirty, False))
    return Move(kind, ch, sp, saved, sp.mats.copy(), info or {})


def full(pr, ch):
    """the chain's full evaluation under its model"""
    return with_model(pr, pr.full_evaluation(ch))


def reject(pr, mv):
    tr = pr.tree[mv.ch]
    left, right, anc, length, post, age, scaled, model = mv.saved
    tr.left[:], tr.right[:], tr.anc[:], tr.length[:] = left, right, anc, length
    tr.post = list(post)
    if len(age):
        tr.age = age.copy()
    pr.chains[mv.ch].scaled[:] = scaled
    models(pr)[mv.ch] = model
    mv.spec.mats = mv.mats                      # a MatrixSupplier may have taken its updates out of the spec
    pr.reject(mv.ch, mv.spec)


def branch_update(pr, ch, rng):
    """a branch-length move: one branch and the path above it (rooted: a node-age move)"""
    if rooted(pr):
        return node_age(pr, ch, rng)
    saved = _save(pr, ch)
    tr = pr.tree[ch]
    node = int(rng.integers(0, tr.n_nodes - 1))
    node += node >= tr.root
    length = float(tr.length[node] * np.exp(0.5 * (rng.random() - 0.5)))
    sp = with_model(pr, pr.branch_update(ch, node, length))
    return Move("branch", ch, sp, saved, sp.mats.copy())


def node_age(pr, ch, rng, node=None):
    """clock trees: a new age for an interior node other than the root, between its older child and its parent --
    three branches, then the path above"""
    tr = pr.tree[ch]
    saved = _save(pr, ch)
    if node is None:
        node = int(rng.choice([p for p in tr.post if p != tr.root_left]))
    lo, hi = max(tr.age[tr.left[node]], tr.age[tr.right[node]]), tr.age[tr.anc[node]]
    tr.age[node] = rng.uniform(lo, hi)
    lengths_from_ages(tr)
    branches = [node, int(tr.left[node]), int(tr.right[node])]
    return _spec(pr, ch, "node_age", saved, branches, {node} | set(tr.path_to_root(node)))


def whole_tree_update(pr, ch, rng, kind="length", factor=None, drop_removes=False):
    """Every branch rebuilt, every interior node dirty, the site scalers copied.  kind 'length': every length (clock:
    every age) times factor; 'model': the chain gets new rates (gamma shape and rate multiplier) and, with invariable
    sites, a new p_invar and so new category weights.  drop_removes (a mutation for the sensitivity checks): the
    operations remove no old scaler."""
    tr = pr.tree[ch]
    saved = _save(pr, ch)
    if kind == "length":
        f = float(np.exp(rng.uniform(-0.3, 0.3))) if factor is None else factor
        if rooted(pr):
            tr.age *= f
            lengths_from_ages(tr)
        else:
            tr.length *= f
    else:
        m = models(pr)[ch]
        alpha = float(np.exp(rng.uniform(-1.0, 1.5)))
        m.rates = workloads.discrete_gamma_rates(alpha, pr.K) * float(np.exp(rng.uniform(-0.3, 0.3)))
        if m.p_invar > 0:
            m.p_invar = float(rng.uniform(0.05, 0.4))
    branches = [n for n in range(tr.n_nodes) if n != tr.root]
    mv = _spec(pr, ch, "whole_" + kind, saved, branches, set(tr.post))
    if drop_removes:
        mv.spec.ops["scale_remove"] = abi.NONE
    return mv


def _topology(pr, ch, kind, saved, drop=None, info=None):
    """after tree arrays changed: post, the dirty nodes and branches (see the module's docstring), the evaluation"""
    tr = pr.tree[ch]
    left, right, anc, length, post, age = saved[:6]
    old_root = post[-1]
    tr.post = down_pass(tr)
    if rooted(pr):
        lengths_from_ages(tr)
    seeds = {p for p in tr.post if (tr.left[p], tr.right[p]) != (left[p], right[p])}
    changed = [c for c in range(tr.n_nodes) if c != tr.root and tr.length[c] != length[c]]
    for c in changed:
        if c != tr.root_left:
            seeds.add(int(tr.anc[c]))
        elif not rooted(pr):
            seeds.add(c)
    if tr.root_left != old_root:
        seeds |= {old_root, tr.root_left}
    dirty = set()
    for s in seeds:
        dirty |= {s} | set(tr.path_to_root(s))
    branches = set(changed)
    if not rooted(pr):
        branches.add(tr.root_left)
    elif tr.root_left != old_root:
        branches.add(old_root)                      # its matrix was never built while it was the root
    info = dict(info or {}, seeds=seeds, root_changed=tr.root_left != old_root)
    if drop is not None:
        dirty.discard(drop(tr, dirty, info))
    return _spec(pr, ch, kind, saved, sorted(branches), dirty, info)


def nni(pr, ch, rng, at_root=False, drop=None):
    """Swap the sibling of an interior node c with one of c's children.  at_root: c is a child of the interior root
    (the root's children change).  Unrooted: c's branch length changes too; clock: c gets a new age."""
    tr = pr.tree[ch]
    saved = _save(pr, ch)
    cands = [c for c in tr.post if c != tr.root_left and (tr.anc[c] == tr.root_left) == at_root]
    c = int(rng.choice(cands))
    p, s = int(tr.anc[c]), sibling(tr, c)
    x_left = rng.random() < 0.5
    x, y = (int(tr.left[c]), int(tr.right[c])) if x_left else (int(tr.right[c]), int(tr.left[c]))
    if tr.left[p] == s:
        tr.left[p] = x
    else:
        tr.right[p] = x
    if x_left:
        tr.left[c] = s
    else:
        tr.right[c] = s
    tr.anc[x], tr.anc[s] = p, c
    if rooted(pr):
        tr.age[c] = rng.uniform(max(tr.age[s], tr.age[y]), tr.age[p])
    else:
        tr.length[c] *= float(np.exp(0.5 * (rng.random() - 0.5)))
    return _topology(pr, ch, "nni_root" if at_root else "nni", saved, drop)


def _detach(tr, v):
    """take v and its parent p out: p's other child s takes p's place -> (p, s)"""
    p, s = int(tr.anc[v]), sibling(tr, v)
    g = int(tr.anc[p])
    if g == tr.root:
        tr.left[g] = s
    elif tr.left[g] == p:
        tr.left[g] = s
    else:
        tr.right[g] = s
    tr.anc[s] = g
    tr.length[s] += tr.length[p]
    return p, s


def spr_targets(tr, v, is_rooted):
    """the branches (by lower node) v can be regrafted onto: outside v's subtree, not its parent's or its sibling's
    (which would give the same tree); on a clock tree only where the branch's upper end is older than v"""
    p, s = int(tr.anc[v]), sibling(tr, v)
    if p == tr.root_left and s < tr.n_tips:
        return []                                        # the root tip cannot hang on a tip
    inside = subtree(tr, v)
    out = []
    for t in range(tr.n_nodes):
        if t in inside or t in (p, s, tr.root):
            continue
        a = int(tr.anc[t])
        if is_rooted and a != tr.root and tr.age[a] <= tr.age[v]:
            continue
        out.append(t)
    return out


def spr(pr, ch, rng, kind="random", prune=None, target=None, drop=None):
    """Subtree prune and regraft: v (with its parent p) leaves its place, p's other child takes p's place, and p is
    inserted on the branch above t.  kind picks v and t:
      'random'       any valid pair;
      'far'          v among the deepest nodes, t the valid target farthest from it below the interior root: on a
                     caterpillar or a comb, one arm climbs the whole spine and the other starts near the top;
      'across_root'  v deep below one child of the interior root, t deep below the other: two arms that meet only at
                     the interior root;
      'root_out'     v is a child of the interior root: its other child becomes the interior root;
      'root_in'      t is the interior root: p becomes the interior root, the former one an ordinary node.
    prune / target give v and t explicitly.  Unrooted: the two branches at s merge, t's branch is split at random;
    clock: p gets an age between t (and v) and t's parent (above t at the root)."""
    tr = pr.tree[ch]
    saved = _save(pr, ch)
    rl = tr.root_left
    deep = lambda nodes: max(nodes, key=lambda x: (depth(tr, x), -x))
    if prune is not None:
        v = prune
    elif kind == "root_out":
        kids = [k for k in (int(tr.left[rl]), int(tr.right[rl])) if spr_targets(tr, k, rooted(pr))]
        assert kids, "neither child of the interior root can move"
        v = min(kids, key=lambda k: len(subtree(tr, k)))
    elif kind in ("far", "across_root"):
        side = subtree(tr, int(tr.left[rl])) if kind == "across_root" else set(range(tr.n_nodes))
        v = deep([x for x in side if x != tr.root and x != rl])
    else:
        cands = [x for x in range(tr.n_nodes) if x not in (tr.root, rl) and (kind != "root_in" or tr.anc[x] != rl)]
        v = int(rng.choice(cands))
        while not spr_targets(tr, v, rooted(pr)):
            v = int(rng.choice(cands))
    targets = spr_targets(tr, v, rooted(pr))
    if target is not None:
        t = target
    elif kind == "root_in":
        t = rl
    elif kind == "far":
        pv = set(tr.path_to_root(v))
        t = max([x for x in targets if x != rl], key=lambda x: (len(pv ^ set(tr.path_to_root(x))), -x))
    elif kind == "across_root":
        right_side = subtree(tr, int(tr.right[rl]))
        t = deep([x for x in targets if x in right_side])
    else:
        t = int(rng.choice(targets))
    assert t in targets, (v, t)
    p, s = _detach(tr, v)
    a = int(tr.anc[t])
    if a == tr.root:
        tr.left[a] = p
    elif tr.left[a] == t:
        tr.left[a] = p
    else:
        tr.right[a] = p
    tr.anc[p] = a
    if tr.left[p] == v:
        tr.right[p] = t
    else:
        tr.left[p] = t
    tr.anc[t] = p
    if rooted(pr):
        lo = max(tr.age[t], tr.age[v])
        tr.age[p] = lo + rng.exponential(0.05) if a == tr.root else rng.uniform(lo, tr.age[a])
    else:
        u = rng.uniform(0.1, 0.9)
        tr.length[p], tr.length[t] = u * tr.length[t], (1 - u) * tr.length[t]
    return _topology(pr, ch, "spr_" + kind, saved, drop, info=dict(prune=v, target=t, parent=p, sibling=s))


# ---- runs -----------------------------------------------------------------------------------------------------------
def make_move(pr, ch, kind, rng):
    """one move of `kind`: 'branch', 'node_age', 'whole_length', 'whole_model', 'nni', 'nni_root', or 'spr_<kind>'"""
    if kind == "branch":
        return branch_update(pr, ch, rng)
    if kind == "node_age":
        return node_age(pr, ch, rng)
    if kind.startswith("whole_"):
        return whole_tree_update(pr, ch, rng, kind[6:])
    if kind in ("nni", "nni_root"):
        return nni(pr, ch, rng, at_root=kind == "nni_root")
    assert kind.startswith("spr_"), kind
    return spr(pr, ch, rng, kind[4:])


def move_sequence(pr, gens, seed, plan):
    """Generation 0: every chain's full evaluation; then `gens` generations of one move per chain, chain ch cycling
    through plan[ch] (a list of make_move kinds), every third generation rejected once the caller has evaluated it.
    Yields (g, [Move or None for the full evaluations], specs)."""
    rng = np.random.default_rng(seed)
    yield 0, [None] * pr.n_chains, [full(pr, ch) for ch in range(pr.n_chains)]
    for g in range(1, gens + 1):
        mvs = [make_move(pr, ch, plan[ch % len(plan)][(g - 1) % len(plan[ch % len(plan)])], rng)
               for ch in range(pr.n_chains)]
        yield g, mvs, [mv.spec for mv in mvs]
        if g % 3 == 2:
            for mv in mvs:
                reject(pr, mv)


# ---- what the operation lists hold --------------------------------------------------------------------------------
def arms(sp, n_tips):
    """the chains of operations the evaluation walks: an arm starts at an operation that reads no buffer written
    earlier in the evaluation and grows by each operation that reads one; an operation that reads two or more is where
    arms meet, and starts the next arm -> (arm lengths, the destinations where arms meet)"""
    written, arm_of, length, meets = set(), {}, [], []
    for op in sp.ops:
        ins = [int(op[f]) for f in ("child1", "child2", "child3") if op[f] >= n_tips and int(op[f]) in written]
        if len(ins) == 1:
            a = arm_of[ins[0]]
            length[a] += 1
        else:
            a = len(length)
            length.append(1)
            if ins:
                meets.append(int(op["dest"]))
        arm_of[int(op["dest"])] = a
        written.add(int(op["dest"]))
    return length, meets


def clean_operands_per_chunk(sp, n_tips, chunk=32):
    """interior operands read from buffers not written earlier in the evaluation, per run of `chunk` operations"""
    written, out = set(), []
    for i, op in enumerate(sp.ops):
        if i % chunk == 0:
            out.append(0)
        out[-1] += sum(1 for f in ("child1", "child2", "child3") if op[f] >= n_tips and int(op[f]) not in written)
        written.add(int(op["dest"]))
    return out
