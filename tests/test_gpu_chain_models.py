"""GPU: chain-batched calls whose evaluations carry different models, on every kernel route.

Per-evaluation values reach the kernels by several independent paths: the job index in the parameter block
(at most 16 fused evaluations), the DevEval headers of the blob (more evaluations, non-fused batches, every
other family), the resident job rows with the weight the resident kernel keeps from job to job, and the search
of the stand-alone P(t) kernels for the evaluation that owns a matrix update.  Here every chain has its own
eigen slot or inline eigensystem, frequencies, rates, category weights, p_invar, flags and weights row
(tests/chain_models.py; slot 0 and row 0 are decoys), so an evaluation handed another one's values fails.

Every batch mixes root-only evaluations and evaluations without matrix updates (first, last and between
evaluations with updates) with a full evaluation and branch updates, rejections included.  Every evaluation
is checked against the oracle (lnL, status, written partials, node and site scalers), against the float64
reference under its own model (after the full evaluations and after the last batch; Std excepted, which the
reference does not model), and against the same evaluation sent alone to a twin instance: bit for bit on the
fused 4-state evaluate() routes (job index and headers), the tensor cores, the generic kernel and Std; within the route's
tolerance on the device blob, non-fused, throughput and resident routes, where the evaluation alone takes
another route or another reduction.  A batch of full evaluations sent reversed and rotated gives every
evaluation the same lnL bit for bit."""
import numpy as np
import pytest

from chain_models import MixedModels
from engine_checks import (DBL_MAX, SYN_RTOL, check_with_oracle, compare_written, edge, lnl_tol, num_sms, ppb, rel,
                           resident_generations, tree_tol, via_evaluate, via_replay)
from f64_reference import caterpillar_tree, transition_matrices
from mrbayes_b200 import abi, workloads
from sparse_rescaling import GUARD_MIN, run_threshold, threshold_instance, threshold_setup, threshold_spec

pytestmark = pytest.mark.gpu
ROLES = ["upd", "root", "upd", "nomat", "upd", "full"]


def batch(mm, g, rng, counts, full=()):
    """Generation g: all full evaluations at g = 0; afterwards a root-only evaluation first, one without matrix
    updates last and both again between branch updates, with a full evaluation among them; the chain of each
    position rotates with g.  Every third update of a chain is rejected after the batch.
    -> (specs, rejections [(chain, spec, old lengths)])"""
    pr = mm.pr
    n = pr.n_chains
    if g == 0:
        return [mm.full(ch) for ch in range(n)], []
    roles = ["root"] + [ROLES[i % len(ROLES)] for i in range(n - 2)] + ["nomat"]
    specs, rejects = [], []
    for i, role in enumerate(roles):
        ch = (i + g) % n
        role = "full" if ch in full else role
        if role == "root":
            specs.append(mm.root_only(ch))
        elif role == "nomat":
            specs.append(mm.no_matrix_update(ch, rng))
        elif role == "full":
            specs.append(mm.full(ch))
        else:
            old = pr.tree[ch].length.copy()
            specs.append(mm.update(ch, rng))
            counts[ch] += 1
            if counts[ch] % 3 == 0:
                rejects.append((ch, specs[-1], old))
    return specs, rejects


def check_against_f64(mm, specs, lnl, tol):
    if mm.std:
        return
    for i, sp in enumerate(specs):
        r = rel(lnl[i], mm.f64(sp.chain))
        assert r < tol, f"float64 reference, evaluation {i} (chain {sp.chain}): {r:.2e}"


def check_alone(got, lnl, bitwise, tol):
    for i, ((la,), (sa,)) in enumerate(got):
        assert sa == abi.EVAL_OK
        if bitwise:
            assert la == lnl[i], f"evaluation {i}: alone {la!r}, batched {lnl[i]!r}"
        else:
            assert rel(la, lnl[i]) < tol, f"evaluation {i}: alone vs batched {rel(la, lnl[i]):.2e}"


def mixed_run(mm, e, o, twin, oracle_lib, route, bitwise, gens=5, seed=0):
    """gens mixed batches on `route`, then the permutation check -> number of calls made on e"""
    pr, tol = mm.pr, lnl_tol(mm.pr.S)
    n = pr.n_chains
    with mm.create(oracle_lib) as scratch:
        scratch.set_arith(1)
        mm.assert_models_differ(scratch, range(n))
    rng = np.random.default_rng(seed)
    counts = [0] * n
    for g in range(gens):
        specs, rejects = batch(mm, g, rng, counts)
        lnl, st = route(e, specs)
        check_alone([twin.evaluate(sp) for sp in specs], lnl, bitwise, tol)
        check_with_oracle(e, o, specs, lnl, st, tol, tree_tol(pr))
        if g in (0, gens - 1):
            check_against_f64(mm, specs, lnl, tol)
        for ch, sp, old in rejects:
            pr.reject(ch, sp, old)
    # full evaluations are idempotent: the same batch reversed and rotated
    fulls = [mm.full(ch) for ch in range(n)]
    want, st = route(e, fulls)
    assert not st.any()
    for order in (list(range(n))[::-1], [(i + 3) % n for i in range(n)]):
        got, st = route(e, [fulls[i] for i in order])
        assert not st.any()
        for pos, i in enumerate(order):
            assert got[pos] == want[i], f"chain {i} at position {pos}: {got[pos]!r} != {want[i]!r}"
    return gens + 3


def nuc4_models(K, C, n=8, tips=40, seed=0, caterpillar=True):
    """4-state chains with mixed models; chain 1 a caterpillar (one node per level: many chunks)"""
    pr = workloads.make_problem(4, K, C, tips, n, seed=7000 + 31 * K + seed)
    if caterpillar:
        pr.tree[1] = caterpillar_tree(tips, np.random.default_rng(K + seed))
    return MixedModels(pr, seed=K + 100 * seed)


def run_route(engine_lib, oracle_lib, mm, route, bitwise, flags=0):
    with mm.create(engine_lib, flags=flags) as e, mm.create(engine_lib, flags=flags) as twin, \
         mm.create(oracle_lib) as o:
        o.set_arith(1)
        calls = mixed_run(mm, e, o, twin, oracle_lib, route, bitwise)
        counters = {k: e.kernel_launches(k) for k in (abi.KERNEL_NUC4, abi.KERNEL_TIPROBS, abi.KERNEL_GENERIC,
                                                       abi.KERNEL_TENSOR, abi.KERNEL_STD)}
    return calls, counters


# ---- 4-state routes ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 4, 5, 8])
def test_nuc4_job_index(engine_lib, oracle_lib, K):
    """8 evaluations over 3 tiles: fused (no stand-alone P(t) launch), and with at most MB200_JOB_INDEX_MAX = 16
    evaluations each one's doubles and eigen0 come from the job index"""
    mm = nuc4_models(K, edge(K, 3))
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_evaluate, bitwise=True)
    assert cnt[abi.KERNEL_NUC4] == calls and cnt[abi.KERNEL_TIPROBS] == 0


@pytest.mark.parametrize("K", [2, 5])
def test_nuc4_header_path(engine_lib, oracle_lib, K):
    """18 evaluations (more than MB200_JOB_INDEX_MAX = 16): the job index is empty and every CTA reads its
    evaluation's DevEval header (on an H100, eval_nuc4_kernel<K, 256, true> reading the copied blob: a job this
    large does not fit the parameter block)"""
    mm = nuc4_models(K, edge(K, 3), n=18, tips=20)
    assert mm.config()["max_evaluations"] >= 17
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_evaluate, bitwise=True)
    assert cnt[abi.KERNEL_NUC4] == calls and cnt[abi.KERNEL_TIPROBS] == 0


@pytest.mark.parametrize("K", [3, 4])
def test_nuc4_device_blob(engine_lib, oracle_lib, K):
    """pack + replay over more than 16 tiles: the fused kernel reads the headers from device memory"""
    mm = nuc4_models(K, edge(K, 20), seed=1)
    assert (mm.pr.C + ppb(K) - 1) // ppb(K) > 16
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_replay, bitwise=False)
    assert cnt[abi.KERNEL_NUC4] == calls and cnt[abi.KERNEL_TIPROBS] == 0


@pytest.mark.parametrize("K", [2, 4])
def test_nuc4_non_fused(engine_lib, oracle_lib, K):
    """tiles x evaluations > 4 x SMs and tiles > 16: the stand-alone tiprobs_kernel finds the evaluation of each
    matrix update, then the streaming kernel"""
    tiles = 4 * num_sms() // 8 + 8
    mm = nuc4_models(K, edge(K, tiles), seed=2)
    assert tiles * 8 > 4 * num_sms() and tiles > 16
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_evaluate, bitwise=False)
    assert cnt[abi.KERNEL_TIPROBS] == calls and cnt[abi.KERNEL_NUC4] == calls


@pytest.mark.parametrize("K", [2, 4])
def test_nuc4_throughput(engine_lib, oracle_lib, K):
    """MB200_CONFIG_THROUGHPUT, single-chunk evaluations: one CTA per evaluation walks all its tiles"""
    mm = nuc4_models(K, edge(K, 5), tips=10, seed=3, caterpillar=False)
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_evaluate, bitwise=False, flags=abi.CONFIG_THROUGHPUT)
    assert cnt[abi.KERNEL_NUC4] == calls and cnt[abi.KERNEL_TIPROBS] == 0


# ---- other families -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,K,C", [(16, 4, 150), (64, 2, 60), (4, 10, 97)])
def test_generic(engine_lib, oracle_lib, S, K, C):
    pr = workloads.make_problem(S, K, C, 10, 8, seed=7100 + S + K)
    mm = MixedModels(pr, seed=S + K, inline=False)
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_evaluate, bitwise=True)
    assert cnt[abi.KERNEL_GENERIC] == calls and cnt[abi.KERNEL_NUC4] == cnt[abi.KERNEL_TENSOR] == 0


@pytest.mark.parametrize("S,K,parts,device", [(20, 4, 1, True), (61, 1, 1, False), (61, 3, 3, False)])
def test_tensor_core(engine_lib, oracle_lib, S, K, parts, device):
    """S = 20 with the device eigensolver (the oracle gets the host eigensystem of the same Q's); S = 61 with
    one Q per omega category in three cijk parts"""
    pr = workloads.make_problem(S, K, 129, 10, 8, seed=7200 + S + K)
    pr.tree[1] = caterpillar_tree(10, np.random.default_rng(S))
    mm = MixedModels(pr, seed=S * K, parts=parts, device_eigen=device)
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_evaluate, bitwise=True)
    assert cnt[abi.KERNEL_TENSOR] == calls and cnt[abi.KERNEL_GENERIC] == 0


def test_std(engine_lib, oracle_lib):
    """per-chain rates and weights rows (the Mk frequencies stay equal, Std ignores category weights)"""
    pr = workloads.make_std_problem(90, 4, 8, 8, seed=7300)
    mm = MixedModels(pr, seed=73)
    calls, cnt = run_route(engine_lib, oracle_lib, mm, via_evaluate, bitwise=True)
    assert cnt[abi.KERNEL_STD] == calls


# ---- resident ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 4, 5])
def test_nuc4_resident(engine_lib, oracle_lib, K):
    """replay_begin / _end with the instance alone on the device.  Generation g gives chain ch weights row
    1 + (ch + g) % 3, so the weight each CTA keeps must be reloaded; other generations change only p_invar or
    the frequencies.  Before generation X, set_pattern_weights rewrites a row in use and set_eigen_decomposition
    the slot of chain c, whose full evaluation in the already packed generation X reads it.  Each generation
    against the oracle (which gets the same calls), the final buffers too, and against the evaluations sent
    alone to a twin instance afterwards, within tolerance."""
    n, G, X, c = 6, 10, 5, 3
    mm = nuc4_models(K, edge(K, 12), n=n, seed=4)
    assert not mm.models[c].inline
    R = mm.rows
    rng, mrng = np.random.default_rng(K), np.random.default_rng(100 + K)
    counts = [0] * n
    gens, expect = [], {}
    for g in range(G):
        for ch in range(n):
            m = mm.models[ch].replace(row=1 + (ch + g) % (R - 1))
            if g % 3 == 1 and ch % 2 == g % 2:
                m = m.with_p_invar(0.0 if ch % 3 == 0 else float(mrng.uniform(0.05, 0.3)))
            if g % 3 == 2 and ch % 2 != g % 2:
                m = m.replace(freqs=mrng.dirichlet(np.full(4, 5.0)))
            mm.models[ch] = m
        if g == X:
            row = mm.models[0].row
            old_w, new_w = mm.weights[row].copy(), mm.weights[row][::-1].copy()
            mm.weights[row] = new_w
            mm.models[c] = mm.new_eigensystem(c, seed=K)
            new_model = mm.models[c]
        specs, rejects = batch(mm, g, rng, counts, full={c} if g == X else ())
        if g in (0, G - 1):
            expect[g] = [mm.f64(sp.chain) for sp in specs]
        for ch, sp, old in rejects:
            mm.pr.reject(ch, sp, old)
        gens.append(specs)
        if g == 0:
            models0 = list(mm.models)
    # the instances start from generation 0's slots and rows
    mm.models, mm.weights[row] = models0, old_w

    def set_calls(g, inst):
        if g == X:
            inst.set_pattern_weights(row, new_w)
            mm.load(inst, new_model.slot, new_model)

    with mm.create(oracle_lib) as scratch:
        scratch.set_arith(1)
        mm.assert_models_differ(scratch, range(n))
    with mm.create(engine_lib) as e, mm.create(oracle_lib) as o:
        o.set_arith(1)
        n0 = e.kernel_launches(abi.KERNEL_NUC4)
        got = resident_generations(e, gens, set_calls)
        launches = e.kernel_launches(abi.KERNEL_NUC4) - n0
        e.synchronize()
        assert launches <= G // 2          # one kernel served several generations (the set calls retire it)
        for g, specs in enumerate(gens):
            set_calls(g, o)
            lnl, st = got[g]
            if g == G - 1:                 # the engine holds the last generation's buffers: compare them too
                check_with_oracle(e, o, specs, lnl, st, SYN_RTOL, tree_tol(mm.pr))
            else:
                for i, sp in enumerate(specs):
                    (lo,), (so,) = o.evaluate(sp)
                    assert st[i] == so == abi.EVAL_OK, f"generation {g}, evaluation {i}"
                    assert rel(lnl[i], lo) < SYN_RTOL, f"generation {g}, evaluation {i}: {rel(lnl[i], lo):.2e}"
            if g in expect:
                for i, want in enumerate(expect[g]):
                    assert rel(lnl[i], want) < SYN_RTOL, f"float64 reference, generation {g}, evaluation {i}"
    with mm.create(engine_lib) as twin:
        for g, specs in enumerate(gens):
            set_calls(g, twin)
            check_alone([twin.evaluate(sp) for sp in specs], got[g][0], False, SYN_RTOL)


# ---- two eigen slots in one evaluation ---------------------------------------------------------------------------------
TWO_SLOT = {"fused": (4, 4, 300, 12), "fused_caterpillar": (4, 4, 300, 40), "non_fused": (4, 4, None, 12),
            "generic": (16, 3, 90, 10), "tensor": (20, 2, 129, 10)}


@pytest.mark.parametrize("route", list(TWO_SLOT))
def test_two_slots_in_one_evaluation(engine_lib, oracle_lib, route):
    """The first matrix update reads slot a, the others slot b (validate() accepts it): every rebuilt P(t) against
    expm of its slot's Q, and the evaluation against the oracle.  On the caterpillar the slot-b branches are
    rebuilt in later chunks than the first; the branch update puts slot a on tip 0 and slot b on the interior
    root's branch, whose node is the last."""
    S, K, C, tips = TWO_SLOT[route]
    C = C or edge(K, 4 * num_sms() + 4)
    pr = workloads.make_problem(S, K, C, tips, 2, seed=7400 + S + tips)
    if route == "fused_caterpillar":
        pr.tree[0] = caterpillar_tree(tips, np.random.default_rng(1))
    mm = MixedModels(pr, seed=74, inline=False)
    a, b = mm.models[0], mm.models[1]
    with mm.create(engine_lib) as e, mm.create(oracle_lib) as o:
        o.set_arith(1)
        node = 0 if pr.tree[0].root != 0 else 1
        for step in ("full", "update"):
            if step == "full":
                sp = mm.full(0)
            else:
                sp = mm.apply(pr.branch_update(0, node, pr.tree[0].length[node] * 1.7))
                assert len(sp.mats) == 2
            sp.mats["eigen"][0] = a.slot
            sp.mats["eigen"][1:] = b.slot
            (le,), (se,) = e.evaluate(sp)
            (lo,), (so,) = o.evaluate(sp)
            assert se == so == abi.EVAL_OK and rel(le, lo) < lnl_tol(S), step
            compare_written(e, o, sp, tree_tol(pr))
            node_of = {int(v): i for i, v in enumerate(pr.chains[0].ti)}
            for j, mu in enumerate(sp.mats):
                m = a if j == 0 else b
                want = transition_matrices(pr, pr.tree[0].length[node_of[int(mu["matrix"])]], a.rates, Q=m.Q, freqs=a.freqs)
                got = e.get_transition_matrix(int(mu["matrix"])).astype(np.float64)
                assert np.abs(got - want).max() < 2e-7, f"{step}, matrix update {j}: {np.abs(got - want).max():.2e}"
                assert np.allclose(got, o.get_transition_matrix(int(mu["matrix"])), rtol=2.5e-7, atol=1e-30)
        kind = {"fused": abi.KERNEL_NUC4, "fused_caterpillar": abi.KERNEL_NUC4, "non_fused": abi.KERNEL_TIPROBS,
                "generic": abi.KERNEL_GENERIC, "tensor": abi.KERNEL_TENSOR}[route]
        assert e.kernel_launches(kind) == 2
        if route.startswith("fused"):
            assert e.kernel_launches(abi.KERNEL_TIPROBS) == 0


# ---- the float-range guard flag differs within one batch -----------------------------------------------------------------
@pytest.mark.parametrize("kind", ["node", "root"])
@pytest.mark.parametrize("route", ["host", "device", "non_fused", "throughput", "resident"])
def test_guard_flag_in_one_evaluation_of_a_batch(engine_lib, oracle_lib, route, kind):
    """Evaluations 1 and 2 carry the same values, the float below 1e-24f; only 1 has MB200_FLAG_RANGE_GUARD, and
    only 1 reports EVAL_UNDERFLOW"""
    K = 4 if kind == "node" else 1
    pr, C, c = threshold_setup(route, K, "middle", 4)
    x = np.nextafter(GUARD_MIN, np.float32(0))
    values = [None, x, x, None]
    specs = [threshold_spec(pr, i, kind) for i in range(4)]
    specs[2].flags &= ~abi.FLAG_RANGE_GUARD
    with threshold_instance(pr, engine_lib, route, values, kind, c) as e, \
         threshold_instance(pr, oracle_lib, route, values, kind, c) as o:
        o.set_arith(1)
        (res,) = run_threshold(e, o, route, [specs])
        for i, (le, se, lo, so) in enumerate(res):
            want = abi.EVAL_UNDERFLOW if i == 1 else abi.EVAL_OK
            assert se == so == want, f"evaluation {i}"
            assert (le == lo == -DBL_MAX) if i == 1 else rel(le, lo) < SYN_RTOL, f"evaluation {i}"


# ---- API --------------------------------------------------------------------------------------------------------------------
def test_api_per_evaluation_checks(engine_lib, oracle_lib):
    """weights_row == weight_rows with a root -> OUT_OF_RANGE; an inline eigensystem on S != 4, or inline and slot
    updates in one evaluation -> UNSUPPORTED; nothing is launched, and the instance works afterwards"""
    pr = workloads.make_problem(4, 4, 97, 8, 3, seed=7500)
    mm = MixedModels(pr, seed=75)
    rng = np.random.default_rng(5)
    with mm.create(engine_lib) as e, mm.create(oracle_lib) as o:
        o.set_arith(1)
        specs = [mm.full(ch) for ch in range(3)]
        lnl, st = e.evaluate(specs)
        for sp in specs:
            o.evaluate(sp)
        n0 = e.launch_count()
        bad = mm.root_only(0)
        bad.weights_row = mm.rows
        with pytest.raises(abi.AbiError) as err:
            e.evaluate([mm.root_only(1), bad])
        assert err.value.code == -3                         # MB200_ERROR_OUT_OF_RANGE
        slot_ch = next(ch for ch in range(3) if not mm.models[ch].inline)
        old = pr.tree[slot_ch].length.copy()
        mixed = mm.update(slot_ch, rng)
        mixed.mats["eigen"][0] = abi.EIGEN_INLINE
        mixed.inline_eigen = mm.models[slot_ch].block()
        with pytest.raises(abi.AbiError) as err:
            e.evaluate(mixed)
        assert err.value.code == -5                         # MB200_ERROR_UNSUPPORTED
        pr.reject(slot_ch, mixed, old)
        assert e.launch_count() == n0
        got, st = e.evaluate([mm.root_only(ch) for ch in range(3)])
        assert not st.any() and np.array_equal(got, lnl)
        sp = mm.update(1, rng)
        (le,), _ = e.evaluate(sp)
        (lo,), _ = o.evaluate(sp)
        assert rel(le, lo) < SYN_RTOL
    pr = workloads.make_problem(16, 2, 40, 6, 1, seed=7501)
    mm = MixedModels(pr, seed=76, inline=False)
    with mm.create(engine_lib) as e:
        sp = mm.full(0)
        sp.mats["eigen"] = abi.EIGEN_INLINE
        sp.inline_eigen = mm.models[0].block()
        with pytest.raises(abi.AbiError) as err:
            e.evaluate(sp)
        assert err.value.code == -5
        (l,), (s,) = e.evaluate(mm.full(0))
        assert s == abi.EVAL_OK and rel(l, mm.f64(0)) < SYN_RTOL
