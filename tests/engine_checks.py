"""What the GPU test modules share: the tolerance bars, the device geometry, the routes by which a list of evaluations
reaches the engine, the comparison of every buffer an evaluation wrote with the CPU oracle, and the run of evaluations
most tests send.  Test modules import these from here, never from each other."""

from dataclasses import dataclass

import numpy as np
import torch

from f64_reference import FLAG_NUC4_PINVAR_QUIRK, caterpillar_tree, f64_lnl, f64_root, tree_height
from mrbayes_b200 import abi, workloads

DBL_MAX = np.finfo(np.float64).max
FLT_MIN = float(np.finfo(np.float32).tiny)

# ---- lnL bars ---------------------------------------------------------------------------------------------------
# 1e-6 relative is the north-star bar (BASELINE.json); what the recorded cases require is 100x tighter, because the
# engine reproduces the reference's float operation order.  What is left (observed ~1e-9) is the last-bit difference
# between glibc's and CUDA's log/exp in the node scalers and in P(t), the same size as the reference's own SSE-vs-FMA
# spread.
LNL_RTOL = 1e-8
# synthetic cases have |lnL| of a few hundred and, for S != 4, fused-vs-separate multiply-add
# differences against the oracle's *_Gen_SSE arithmetic: still 5x inside the north-star bar
SYN_RTOL = 2e-7
# 20- and 61-state divisions run on the tensor cores with 3xTF32 operand splitting: each matvec
# carries ~7e-7 relative error, mostly the tensor core's truncating FP32 accumulation (a small
# negative bias), which shows up as ~1e-7 relative in lnL -- 5x inside the north-star bar of 1e-6
TC_RTOL = 5e-7


def lnl_tol(S, base=SYN_RTOL):
    """the lnL bar of an S-state division: TC_RTOL for the tensor-core state counts, else base"""
    return TC_RTOL if S in (20, 61) else base


def rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


# ---- bars of the buffers an evaluation writes -------------------------------------------------------------------
def below(x):
    """the largest float below x: |d| <= below(x) is |d| < x for a float d"""
    return np.nextafter(np.float32(x), np.float32(0))


@dataclass(frozen=True)
class Tol:
    """|engine - oracle| <= atol + rtol |oracle| per entry, in float as numpy's isclose computes it; partials may also
    differ by partials_of_peak times the largest entry of their pattern in the buffer (then in double)"""
    partials_rtol: float
    partials_atol: float
    node_rtol: float
    node_atol: float
    site_rtol: float
    site_atol: float
    partials_of_peak: float = 0.0
    partials_rtol_of: object = None          # dest -> partials_rtol of that buffer, in place of partials_rtol


def parity_tol(S):
    """Conditional likelihoods 2e-6 relative (a few float ulps: FMA contraction and summation order are the only
    differences allowed; 2e-5 on the tensor cores), node scalers 1e-6 and site scalers 2e-5 absolute"""
    return Tol(2e-5 if S in (20, 61) else 2e-6, 1e-37, 1e-5, 1e-6, 1e-5, 2e-5)


def tree_tol(pr):
    """-> tol(sp): parity_tol(pr.S); on the tensor-core path the 3xTF32 rounding of each level (up to ~1e-6
    relative) adds up from the tips to the node: on H100, S = 61 and K = 3, the partials of a node 20 to 38 levels up
    differ from the oracle's by 2e-5, parity_tol's bound for trees of a few levels.  So the partials and the node
    scalers (the log of the node's largest unscaled partial) get 2e-5 plus 1e-6 per level of sp's tree."""
    def tol(sp):
        if pr.S not in (20, 61):
            return parity_tol(pr.S)
        t = 2e-5 + 1e-6 * tree_height(pr.tree[sp.chain])
        return Tol(t, 1e-37, 0.0, below(t), 1e-5, 2e-5 + t)
    return tol


def interior_below(tr):
    """[n_nodes] interior nodes in each node's subtree, itself included: the nodes whose partials its own are
    computed from"""
    n = np.zeros(tr.n_nodes, np.int64)
    for p in tr.post:                                    # children before parents
        n[p] = 1 + n[int(tr.left[p])] + n[int(tr.right[p])]
    return n


def subtree_tol(pr):
    """-> tol(sp): tree_tol with its per-level term counted per node.  The 3xTF32 rounding of one node (up to ~1e-6
    relative) reaches its parent through either child, so a node's partials carry the rounding of every interior
    node below it, not only of one path: 2e-5 plus 1e-6 per interior node in the node's subtree, which is tree_tol's
    per-level term on a caterpillar.  Measured on H100, S = 61 at 300 tips: a balanced tree's interior root (9 levels,
    298 nodes below) differed from the oracle by 1.1e-4 at K = 3 -- 3.7 x tree_tol, 0.34 x this bound -- with P(t)
    bit-identical to the oracle's and the slowest category (P close to I) exact; at most 0.39 x this bound at K = 1 to
    3 on random, caterpillar and balanced trees.  Node scalers get the largest bound of the nodes sp writes."""
    def tol(sp):
        base = parity_tol(pr.S)
        if pr.S not in (20, 61):
            return base
        tr, cl = pr.tree[sp.chain], pr.chains[sp.chain].cl
        node_of = {int(cl[n]): n for n in range(tr.n_tips, tr.n_nodes)}
        below_n = interior_below(tr)
        per_dest = {int(op["dest"]): 2e-5 + 1e-6 * float(below_n[node_of[int(op["dest"])]]) for op in sp.ops}
        t = max(per_dest.values(), default=base.partials_rtol)
        return Tol(t, 1e-37, 0.0, below(t), 1e-5, 2e-5 + t, partials_rtol_of=per_dest.get)
    return tol


def sparse_tol(pr):
    """-> tol(sp) for sparse rescaling.  Partials relative (tensor core: 2e-5 plus 1e-6 per tree level, as
    tree_tol) with an absolute floor of 1e-44 -- the subnormal range, since partials can be tiny when nodes go
    unscaled; on the tensor core the smallest normal float, because its products flush subnormals: an entry just
    above 1e-38 loses the terms below (on H100, 5.7e-38 differed by 8e-5 relative); node scalers to 1e-6 plus two
    float ulps of their size (a sparse scaler is the log of a small maximum: -55 has an ulp of 4e-6); site scalers
    to 2e-5 plus two ulps"""
    def tol(sp):
        if pr.S not in (20, 61):
            return Tol(2e-6, 1e-44, 2.5e-7, 1e-6, 2.5e-7, 2e-5 + 1e-6)
        t = 2e-5 + 1e-6 * tree_height(pr.tree[sp.chain])
        return Tol(t, FLT_MIN, 2.5e-7, t, 2.5e-7, 2e-5 + t)
    return tol


# The generic kernel's parity_tol (S = 20 and 61 run there too, not on the tensor cores) at the shapes production
# models send (tests/model_shapes.py), except that a partial may also differ by 2e-7 times the largest entry of its
# pattern in the buffer.  That term is the error P(t) brings in: an entry summed from an eigensystem in double is
# good to ~1e-14 absolute (P_EPS bounds the device eigensolver's), and at these shapes P(t) has entries of 1e-12 and
# far below (rare codons, short branches, 20 gamma categories).  Where the children of a node disagree, the
# pattern's largest product is small and the rescaling amplifies such absolute errors.  Measured on an H100 (700 W):
# partials of 1e-16 to 1e-25 of their pattern's largest differ from the oracle's by up to 7e-3 relative; what exceeds
# 2e-6 relative reaches 5.8e-8 of the pattern's largest with device eigensystems (60 and 63 codons, one Q; 7e-9 at
# K = 4) and stays below 2e-12 with host eigensystems; entries above 1e-6 of the largest differ by up to 2e-4
# relative (63 codons, device).  lnL agrees to 1e-8 throughout.  The dense models with Dirichlet(5) frequencies of
# the other tests have no such entries.
# Node scalers get the site scalers' 2e-5 instead of 1e-6: a child's partials carry that error of up to 2e-7 of their
# largest entry, and a parent whose largest product rests on such entries of the child moves its scaler by their
# relative error (measured: 7.2e-6 at one pattern of a 60-codon node, device eigensystems, the node's partials and
# lnL within their bounds).
SHAPES_TOL = Tol(2e-6, 0.0, 0.0, below(2e-5), 0.0, below(2e-5), partials_of_peak=2e-7)


def compare_written(e, o, sp, tol):
    """Every partials buffer and node scaler sp wrote, and its site scalers, engine e against oracle o within tol (a
    Tol, or tol(sp) -> Tol).  -> (largest relative difference over the partials above 1e-6 of their pattern's
    largest, largest excess over partials_rtol relative as a fraction of the pattern's largest); both 0 unless tol
    has a partials_of_peak term"""
    if callable(tol):
        tol = tol(sp)
    rel_big = rel_peak = 0.0
    for op in sp.ops:
        a, b = e.get_partials(int(op["dest"])), o.get_partials(int(op["dest"]))
        atol = tol.partials_atol
        rtol = tol.partials_rtol if tol.partials_rtol_of is None else tol.partials_rtol_of(int(op["dest"]))
        if tol.partials_of_peak:
            a, b = a.astype(np.float64), b.astype(np.float64)
            peak = np.abs(b).max(axis=(0, 2), keepdims=True)
            atol = atol + tol.partials_of_peak * peak
            d = np.abs(a - b)
            big = np.abs(b) > 1e-6 * peak
            rel_big = max(rel_big, float((d[big] / np.abs(b[big])).max(initial=0.0)))
            rel_peak = max(rel_peak, float(((d - rtol * np.abs(b)) / np.where(peak > 0, peak, 1.0)).max()))
        bad = ~np.isclose(a, b, rtol=rtol, atol=atol)
        if bad.any():
            ratio = (np.abs(a - b) / (atol + rtol * np.abs(b)))[bad].max()
            maxima = b.max(axis=(0, 2))[np.nonzero(bad)[1][:3]] if b.ndim == 3 else None
            raise AssertionError(f"partials of buffer {op['dest']}: {bad.sum()} entries, e.g. {a[bad][:3]} vs "
                                 f"{b[bad][:3]}, {ratio:.2f} x the bound; pattern maxima {maxima}")
        if op["scale_write"] >= 0:
            a, b = e.get_scalers(int(op["scale_write"])), o.get_scalers(int(op["scale_write"]))
            assert np.allclose(a, b, rtol=tol.node_rtol, atol=tol.node_atol), \
                f"node scaler {op['scale_write']}: {np.abs(a - b).max():.2e}"
    if sp.site_dst >= 0:
        a, b = e.get_scalers(sp.site_dst), o.get_scalers(sp.site_dst)
        assert np.allclose(a, b, rtol=tol.site_rtol, atol=tol.site_atol), \
            f"site scaler {sp.site_dst}: {np.abs(a - b).max():.2e}"
    return rel_big, rel_peak


def check_with_oracle(e, o, specs, lnl, status, rtol, tol):
    """Each of specs, which gave (lnl, status) on engine e, on the oracle o: status the oracle's and EVAL_OK, lnL
    within rtol relative, every buffer it wrote within tol (compare_written).  -> (largest lnL difference relative,
    and the largest values compare_written returned)"""
    worst = np.zeros(3)
    for i, sp in enumerate(specs):
        (lo,), (so,) = o.evaluate(sp)
        what = f"evaluation {i} (chain {sp.chain})"
        assert status[i] == so == abi.EVAL_OK, f"{what}: status {status[i]}, oracle {so}"
        r = rel(lnl[i], lo)
        assert r < rtol, f"{what}: {r:.2e}"
        worst = np.maximum(worst, (r,) + compare_written(e, o, sp, tol))
    return tuple(float(x) for x in worst)


# ---- geometry and traces ----------------------------------------------------------------------------------------
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def ppb(K):
    """patterns per 4-state tile: 256 threads / pow2ceil(K) lanes per pattern"""
    return 256 // (1 << (K - 1).bit_length())


def edge(K, tiles):
    """a pattern count at a tile edge: exactly `tiles` tiles, or one pattern less or more (rotating with K)"""
    return tiles * ppb(K) + (K % 3) - 1


def kernel_names(fn, expect):
    """names of the CUDA kernels fn() launches (CUDA activity trace, no hardware counters), for what the
    kernel counters cannot tell: the K and parameter-block size of a 4-state instantiation.  The trace
    can miss launches, so fn -- a full evaluation, which is idempotent -- is traced up to three times
    until a kernel whose name contains `expect` shows up."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if str(e.device_type).endswith("CUDA")}
        if launched(names, expect):
            break
    return names


def launched(names, prefix):
    return any(prefix in n for n in names)


# ---- routes: how a list of evaluations reaches the engine ---------------------------------------------------------
def via_evaluate(e, specs):
    return e.evaluate(specs)


def via_replay(e, specs):
    b = e.pack(specs)
    e.replay(b)
    out = e.replay_results(b, len(specs))
    e.free_batch(b)
    return out


def resident_generations(e, gens, before=None):
    """generations through replay_begin / _end, all packed first (packing retires a resident kernel); before(g, e),
    if given, runs just before generation g's replay_begin -> [(lnL, status)] per generation"""
    batches = [e.pack(specs) for specs in gens]
    out = []
    for g, b in enumerate(batches):
        if before:
            before(g, e)
        e.replay_begin(b)
        out.append(e.replay_end())
    for b in batches:
        e.free_batch(b)
    return out


def written_buffers(gens):
    """-> (partials buffers, scalers) the evaluations of generations gens write"""
    specs = [sp for s in gens for sp in s]
    dests = sorted({int(op["dest"]) for sp in specs for op in sp.ops})
    scalers = sorted({int(op["scale_write"]) for sp in specs for op in sp.ops if op["scale_write"] >= 0} |
                     {int(sp.site_dst) for sp in specs if sp.site_dst >= 0})
    return dests, scalers


# ---- runs ---------------------------------------------------------------------------------------------------------
def evaluation_sequence(pr, updates, seed, before_update=None):
    """A full evaluation per chain, then `updates` branch updates over the chains in turn; every third update, the
    last one included, is rejected once the caller has evaluated it.  seed is anything np.random.default_rng takes:
    a Generator is drawn from as it is, so that the caller can go on drawing from it.  before_update(it) runs before
    update it is drawn.  Yields (it, evaluation), it < 0 for the full evaluations."""
    rng = np.random.default_rng(seed)
    n = pr.n_chains
    for ch in range(n):
        yield ch - n, pr.full_evaluation(ch)
    for it in range(updates):
        ch = it % n
        if before_update:
            before_update(it)
        old = pr.tree[ch].length.copy()
        sp = pr.random_branch_update(ch, rng)
        mats = sp.mats.copy()                            # a MatrixSupplier takes its updates out of sp
        yield it, sp
        if it % 3 == 2:
            sp.mats = mats                               # every branch whose matrix index flipped flips back
            pr.reject(ch, sp, old)


def generation_sequence(pr, gens, seed):
    """Generation 0: every chain's full evaluation; then `gens` generations of one branch update per chain, every third
    generation rejected once the caller has evaluated it.  The chains' operation counts differ wherever their trees
    do.  Yields (g, specs)."""
    rng = np.random.default_rng(seed)
    yield 0, [pr.full_evaluation(ch) for ch in range(pr.n_chains)]
    for g in range(1, gens + 1):
        old = [tr.length.copy() for tr in pr.tree]
        specs = [pr.random_branch_update(ch, rng) for ch in range(pr.n_chains)]
        mats = [sp.mats.copy() for sp in specs]
        yield g, specs
        if g % 3 == 2:
            for ch, sp in enumerate(specs):
                sp.mats = mats[ch]
                pr.reject(ch, sp, old[ch])


def assert_resident_equals_launches(engine_lib, oracle_lib, pr, gens, rtol, tol, drift=False):
    """replay_begin / _end with this instance alone on the device: the resident kernel must give, bit for bit, the
    lnL and the final buffers that one launch per generation (pack + replay) gives; the launches are checked against
    the oracle, and the last evaluation against the float64 reference: within rtol relative, plus with `drift` the
    float site scalers' drift (f64_reference.ScalerLedger) for large trees"""
    from f64_reference import ScalerLedger
    dests, scalers = written_buffers(gens)
    ledger = ScalerLedger()

    def final_state(e):
        return [e.get_partials(b) for b in dests], [e.get_scalers(s) for s in scalers]

    want = []
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        o.set_arith(1)
        for specs in gens:
            lnl, st = via_replay(e, specs)
            check_with_oracle(e, o, specs, lnl, st, rtol, tol)
            for sp in specs:
                ledger.record(sp, e.get_scalers(sp.site_dst))
            want.append(lnl)
        last = gens[-1][-1]
        lf = f64_lnl(pr, last.chain)[1]
        bar = rtol * abs(lf) + (ledger.drift(last, pr.weights) if drift else 0.0)
        assert abs(want[-1][-1] - lf) < bar, f"float64 reference: {want[-1][-1]!r} vs {lf!r}, bar {bar:.2e}"
        want_state = final_state(e)
    with pr.create(engine_lib) as e:
        n0 = e.launch_count()
        got = resident_generations(e, gens)
        launches = e.launch_count() - n0
        e.synchronize()
        got_state = final_state(e)
    assert not any(st.any() for _, st in got)
    assert launches < len(gens)                      # one kernel served several generations
    assert np.array_equal(np.array([lnl for lnl, _ in got]), np.array(want))
    assert all(np.array_equal(a, b) for a, b in zip(got_state[0], want_state[0]))
    assert all(np.array_equal(a, b) for a, b in zip(got_state[1], want_state[1]))


# ---- problem builders -------------------------------------------------------------------------------------------
def nuc4_problem(K, C, n_chains=2, seed=0, tips=40):
    """4-state problem whose chain 1 is a caterpillar (one node per level: many chunks); odd K carry
    p_invar and partial ambiguity"""
    odd = K % 2 == 1
    pr = workloads.make_problem(4, K, C, tips, n_chains, seed=1000 + 17 * K + seed,
                                p_invar=0.15 if odd else 0.0, p_ambig=0.1 if odd else 0.0)
    pr.tree[1] = caterpillar_tree(tips, np.random.default_rng(K))
    return pr


def dead_pattern_problem(family, where, n_chains=1):
    """Every pattern compatible (all tips in one state) except pattern `dead`, where the root tip
    disagrees; with P = I (branches below TIME_MIN) that pattern's likelihood is exactly 0."""
    sms = num_sms()
    if family == "std":
        C = 64 * 5 + 1 if where == "last" else 64 * 5       # K = 2: 64 patterns per tile
        pr = workloads.make_std_problem(C, 2, 6, n_chains, seed=7, max_states=5, dummy=0)
        pr.rates = pr.rates * 1e-10          # Std clamps lengths up to BRLENS_MIN: P = I needs r t < 1e-17
        pr.masks[:] = 1
        base = np.zeros(C, np.int64)
    else:
        S, K, C, tile = {"nuc4_host": (4, 4, 10 * 64, 64), "nuc4_device": (4, 4, 40 * 64, 64),
                         "nuc4_non_fused": (4, 4, (4 * sms + 4) * 64, 64), "nuc4_resident": (4, 4, 12 * 64, 64),
                         "nuc4_throughput": (4, 4, 10 * 64, 64), "tensor": (20, 2, 4 * 128, 128),
                         "generic": (16, 2, 300, 4)}[family]
        if where == "last":
            C -= tile - 1                      # the last tile holds one pattern
        pr = workloads.make_problem(S, K, C, 6, n_chains, seed=8, p_missing=0.0)
        base = np.random.default_rng(1).integers(0, S, size=C)
        pr.masks[:] = (np.uint64(1) << base.astype(np.uint64))[None, :]
    # the root tip disagrees with the rest: every interior node below the root keeps a non-zero
    # (scalable) likelihood, the zero appears where the interior root combines its three children
    dead = C - 1 if where == "last" else C // 2 + 1
    pr.masks[:, dead] = np.uint64(1) << np.uint64(base[dead])
    pr.masks[pr.tree[0].root, dead] = np.uint64(1) << np.uint64((base[dead] + 1) % 2)
    return pr, dead


def switch_problem(S, K, C, tips, n_chains, seed, mean_len):
    """+I problem (p_invar 0.2, rates flat: gamma shape 50) whose branches average mean_len: every 8th pattern constant
    (state c mod S), every 29th from 3 on all-missing (site scaler 0, above the switch), the others random.  At a few
    hundred tips and the lengths the callers pick, the constant patterns' site scalers fall between -200 and -300 and
    the random ones far below: every branch of the root rule (f64_reference.root_site_terms) is taken somewhere."""
    pr = workloads.make_problem(S, K, C, tips, n_chains, seed=seed, alpha=50.0, p_invar=0.2)
    rng = np.random.default_rng(seed)
    for tr in pr.tree:
        tr.length[:] = rng.exponential(mean_len, tr.n_nodes)
        tr.length[tr.root] = 0.0
    const = np.arange(0, C, 8)
    pr.masks[:, const] = np.uint64(1) << (const % S).astype(np.uint64)[None, :]
    pr.masks[:, 3::29] = np.uint64((1 << S) - 1)
    return pr


# (flags, p_invar) of the evaluations switch_problem's chains send, chain ch the entry ch mod 4: the quirk flag on and
# off; p_invar = 0.2 puts the constant patterns' likeI far above LIKE_I_MIN, p_invar = 1e-80 below it (0 on 4 states)
def root_variants(pr):
    quirk, gen = pr.flags | FLAG_NUC4_PINVAR_QUIRK, pr.flags & ~FLAG_NUC4_PINVAR_QUIRK
    return [(quirk, 0.2), (quirk, 1e-80), (gen, 0.2), (gen, 1e-80)]


def with_root_variant(pr, sp):
    """sp under its chain's root_variants entry: flags, p_invar and the rates and category weights that go with it"""
    flags, p = root_variants(pr)[sp.chain % 4]
    sp.flags, sp.p_invar, sp.has_p_invar = flags, p, 1
    sp.rates = np.asarray(pr.rates, np.float64) / (1.0 - p)
    sp.cat_weights = np.full(pr.K, (1.0 - p) / pr.K)
    return sp


def variant_root(pr, sp, scalers):
    """f64_root of sp's chain under its root variant, the decision at the switch read from `scalers`"""
    flags, p = root_variants(pr)[sp.chain % 4]
    return f64_root(pr, sp.chain, p_invar=p, flags=flags, scalers=scalers)


def reversible_q(rng, S, sparse=False, skew=False, equal=False):
    R = rng.gamma(1.0, 1.0, (S, S)) + 0.05
    if equal:
        R[:] = 1.0
    if sparse:                                   # codon-like: most exchanges impossible, chain graph keeps it connected
        keep = rng.random((S, S)) < 0.15
        for i in range(S - 1):
            keep[i, i + 1] = True
        R = np.where(keep, R, 0.0)
    R = np.triu(R, 1); R = R + R.T
    pi = rng.dirichlet(np.full(S, 0.3 if skew else 5.0))
    pi = np.maximum(pi, 1e-7); pi /= pi.sum()
    Q = R * pi[None, :]
    np.fill_diagonal(Q, 0.0)
    np.fill_diagonal(Q, -Q.sum(1))
    Q /= -(pi * np.diag(Q)).sum()                # one expected substitution per unit time
    return Q, pi


def eigen_instance(lib, S, K, parts):
    """a small instance whose slots and matrices the eigensolver tests fill: 16 patterns, 6 matrices, 3 eigen slots,
    parts rate matrices per slot"""
    flags = (parts << 8) if parts > 1 else 0
    return abi.Instance(lib, tip_count=2, partials_count=4, state_count=S, pattern_count=16, category_count=K,
                        matrix_count=6, scaler_count=2, eigen_count=3, flags=flags)


# ---- one call against the float64 reference over the buffers it read (f64_reference.f64_evaluation) ---------------
ULP = 2.0 ** -23                                 # float ulp of 1


def f64_inputs(inst, sp):
    """-> (partials, matrices, scalers) sp reads, read back from inst (engine or oracle) now: its interior operands and
    root buffer, the matrices of its operations and the scalers it removes and copies"""
    tips = inst.cfg.tip_count
    parts, mats, scal = {}, {}, {}
    for op in sp.ops:
        for c, m in ((op["child1"], op["matrix1"]), (op["child2"], op["matrix2"]), (op["child3"], op["matrix3"])):
            if c < 0:
                continue
            if c >= tips and int(c) not in parts:
                parts[int(c)] = inst.get_partials(int(c))
            mats.setdefault(int(m), inst.get_transition_matrix(int(m)))
        if op["scale_remove"] >= 0:
            scal[int(op["scale_remove"])] = inst.get_scalers(int(op["scale_remove"]))
    if sp.site_src >= 0:
        scal[sp.site_src] = inst.get_scalers(sp.site_src)
    if sp.root >= 0:
        parts.setdefault(sp.root, inst.get_partials(sp.root))
    return parts, mats, scal


def f64_call_check(inst, pr, sp, ref, tensor, status=None, lnl=None):
    """Every buffer sp wrote on inst, and its lnL, against ref = f64_evaluation of the same call on the same inputs.

    Off the tensor cores every term is non-negative, so a node carries at most about S + 3 roundings (the S-term dot
    product, the products of its children, the division by its peak) on top of its children's error: the partials bar
    is (S + 3) float ulps relative per operation of the call in the node's subtree (Evaluation64.below), with an absolute
    floor of as many flushed subnormal results (FLT_MIN each) divided by the node's peak.  On the tensor cores
    subtree_tol's per-node term counted within the call, 2e-5 + 1e-6 per operation below, with a floor of three flushed
    products per term (the 3xTF32 split) of each operation below, divided by the peak.  A node scaler is the log of the peak: the node's bar before rescaling plus half a float
    ulp of the scaler; a site scaler adds its node scalers' bars and half an ulp of its running size per addition and
    removal.  lnL: lnl_tol(S) relative (plus, for Std, the coding-bias conditioning).  -> the largest fraction of a bar
    used."""
    from f64_reference import half_ulp
    S = pr.S
    used = 0.0
    node_bar = {}
    for op in sp.ops:
        dest = int(op["dest"])
        n = ref.below[dest]
        want = ref.partials[dest]
        got = inst.get_partials(dest).astype(np.float64)
        # the floor: a product below FLT_MIN may be flushed to zero (the tensor cores flush subnormals, and so may the
        # other kernels), an error below FLT_MIN per product -- three per term with the 3xTF32 split -- which the
        # division by the node's peak enlarges
        if tensor:
            rtol, floor = 2e-5 + 1e-6 * n, n * 3 * S * FLT_MIN / ref.peak[dest]
        else:
            rtol, floor = n * (S + 3) * ULP, n * (S + 3) * FLT_MIN / ref.peak[dest]
        atol = floor[None, :, None] if want.ndim == 3 else np.repeat(floor, pr.state_counts)[None, :]
        bar = atol + rtol * np.abs(want)
        frac = np.abs(got - want) / bar
        worst = float(frac.max())
        assert worst <= 1.0, f"partials of buffer {dest}: {worst:.2f} x the float64 bar (rtol {rtol:.2e}, {n} below)"
        used = max(used, worst)
        if op["scale_write"] >= 0:
            w = int(op["scale_write"])
            node_bar[w] = rtol + half_ulp(ref.scalers[w])
            d = np.abs(inst.get_scalers(w).astype(np.float64) - ref.scalers[w])
            worst = float((d / node_bar[w]).max())
            assert worst <= 1.0, f"node scaler {w}: {worst:.2f} x the float64 bar"
            used = max(used, worst)
    if ref.site is not None:
        steps = int((sp.ops["scale_write"] >= 0).sum() + (sp.ops["scale_remove"] >= 0).sum())
        bar = sum(node_bar.values(), np.zeros(pr.C)) + steps * half_ulp(np.abs(ref.site_src) + np.abs(ref.site))
        d = np.abs(inst.get_scalers(sp.site_dst).astype(np.float64) - ref.site)
        worst = float((d / np.maximum(bar, 1e-300)).max())
        assert worst <= 1.0, f"site scaler {sp.site_dst}: {worst:.2f} x the float64 bar"
        used = max(used, worst)
    if ref.lnl is not None and lnl is not None:
        assert status == (abi.EVAL_UNDERFLOW if ref.underflow else abi.EVAL_OK), f"status {status}"
        if not ref.underflow:
            cond = pr.uncompressed * 2e-6 * ref.p_un / (1.0 - ref.p_un) if ref.p_un else 0.0
            bar = lnl_tol(S) * abs(ref.lnl) + cond
            worst = abs(lnl - ref.lnl) / bar
            assert worst <= 1.0, f"lnL {lnl!r} vs float64 {ref.lnl!r}: {worst:.2f} x the bar"
            used = max(used, worst)
    return used


# ---- caller data: seeded buffers and foreign matrices -------------------------------------------------------------
def _host_layout(pr, x):
    """[K, C, S] -> the host layout of pr's partials (ragged for variable-state divisions)"""
    from f64_reference import is_variable_states, padded_to_ragged
    return padded_to_ragged(pr, x).astype(np.float32) if is_variable_states(pr) else x.astype(np.float32)


def seeded_partials(pr, rng):
    """Interior partials a caller might hold, in pr's host layout: every pattern peaks (0.5 to 1) in a category of its
    own, the other categories lie 1 to 1e-6 below; about 15 % of the entries are exact zeros and 5 % sit just above
    FLT_MIN.  Every pattern keeps its peak, so no pattern is zero throughout."""
    from f64_reference import is_variable_states
    K, C, S = pr.K, pr.C, pr.S
    x = rng.uniform(0.0, 1.0, (K, C, S)) ** 2
    top = rng.integers(0, K, C)
    x *= np.where(np.arange(K)[:, None] == top[None, :], 1.0, 10.0 ** -rng.uniform(0, 6, (K, C)))[:, :, None]
    x[rng.random(x.shape) < 0.15] = 0.0
    tiny = rng.random(x.shape) < 0.05
    x[tiny] = FLT_MIN * rng.uniform(1.0, 4.0, int(tiny.sum()))
    n = pr.state_counts if is_variable_states(pr) else np.full(C, S)
    x[:, np.arange(S)[None, :] >= n[:, None]] = 0.0
    x[top, np.arange(C), rng.integers(0, 1 << 30, C) % n] = rng.uniform(0.5, 1.0, C)
    return _host_layout(pr, x)


def seeded_scalers(pr, rng, depth):
    """a scaler buffer: log-peaks down to -depth, some exactly 0"""
    v = -rng.uniform(0.0, depth, pr.C)
    v[rng.random(pr.C) < 0.1] = 0.0
    return v.astype(np.float32)


def foreign_rows(n, rng):
    """[n, n] row-stochastic, non-reversible: a diagonal of 0.3 to 0.9 and Dirichlet rows off it; some rows have
    exact zeros, some entries of 1e-30 or subnormal, some rows are identity rows.  Row 0 is positive throughout, so that
    every node keeps a positive entry in state 0 of every category and no pattern's product vanishes."""
    P = np.zeros((n, n))
    for i in range(n):
        d = rng.uniform(0.3, 0.9)
        off = rng.dirichlet(np.full(n - 1, 0.5)) * (1.0 - d)
        u = rng.random() if i > 0 else 1.0
        if u < 0.1:
            d, off = 1.0, np.zeros(n - 1)                        # identity row
        elif u < 0.3:
            off[rng.random(n - 1) < 0.5] = 0.0                   # exact zeros
        elif u < 0.5:
            j = rng.integers(0, n - 1, 2)
            off[j[0]] = 1e-30 * rng.uniform(0.5, 2.0)
            off[j[1]] = 1e-40 * rng.uniform(0.5, 2.0)            # subnormal in float
        P[i] = np.insert(off, i, d)
    return P


def foreign_matrix(pr, rng):
    """a transition-matrix buffer of foreign_rows in pr's host layout: [K, S, S], or a variable-state block with one
    such matrix per state-count class and category"""
    from f64_reference import is_variable_states, std_pattern_classes
    if not is_variable_states(pr):
        return np.stack([foreign_rows(pr.S, rng) for _ in range(pr.K)]).astype(np.float32)
    blk = np.zeros(pr.matrix_length, np.float32)
    for n, ti, _ in std_pattern_classes(pr):
        for k in range(pr.K):
            blk[ti + k * n * n: ti + (k + 1) * n * n] = foreign_rows(n, rng).ravel()
    return blk


def seed_chain(insts, pr, ch, rng, depth=30.0):
    """set_partials / set_scalers, identically on every instance, of chain ch's current interior partials, node scalers
    and site scaler: the clean operands, removed scalers and site_scaler_src of its next branch update"""
    st, tr = pr.chains[ch], pr.tree[ch]
    for p in tr.post:
        x = seeded_partials(pr, rng)
        for inst in insts:
            inst.set_partials(int(st.cl[p]), x)
        if st.scaled[p]:
            v = seeded_scalers(pr, rng, depth)
            for inst in insts:
                inst.set_scalers(int(st.ns[p]), v)
    v = seeded_scalers(pr, rng, depth * 5)
    for inst in insts:
        inst.set_scalers(int(st.site), v)
