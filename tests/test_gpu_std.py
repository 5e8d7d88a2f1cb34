"""GPU: the variable-state (STANDARD data) kernel family -- tiprobs_std_kernel and eval_std_kernel<SMAX> -- against
the CPU oracle and the float64 reference (f64_std_lnl), at the shapes where it can go wrong: every lane width
L = pow2ceil(K) = 1 ... 32 at tile edges, every SMAX instantiation from both sides, nine state-count classes at
K = 20, coding=informative dummies over several tiles, a near-degenerate and a clamped coding-bias correction,
caller-supplied non-symmetric and ordered matrices, a hymfossil-sized division with fossil taxa on a caterpillar,
and chain batches (tests/std_problems.py builds the divisions).

Each evaluation is compared with the oracle (lnL within 1e-9, status, every written partials buffer, node and site
scalers, the first engine-built P(t)) and with float64: |lnL - lnL64| <= 2e-7 sum_c w_c |log L_c| + U 2e-6 pUn /
pObserved (StdLnl.bound).  The largest ratio of the error to that bound is recorded per case as
max_error_to_bound."""
import numpy as np
import pytest

from engine_checks import DBL_MAX, check_with_oracle, dead_pattern_problem, evaluation_sequence, rel, tree_tol
from f64_reference import f64_std_lnl, tree_height
from std_problems import CASES, lanes, make_case, make_std_division
from mrbayes_b200 import abi, workloads

pytestmark = pytest.mark.gpu


def smax_instantiation(S):
    """eval_std_kernel<SMAX> the engine launches for a division whose largest state count is S: the row padded to a
    multiple of 4 against 4, 8, 12 and 16, else 24 (the kernel counters cannot tell the instantiations apart)"""
    Sp = (S + 3) & ~3
    return next((m for m in (4, 8, 12, 16) if Sp <= m), 24)


def check_run(engine_lib, oracle_lib, pr, supplier, record_property, updates=6):
    """A full evaluation per chain, then branch updates with a rejection every third, on the engine and the oracle
    (caller-supplied matrices to both); every evaluation on KERNEL_STD"""
    worst, calls = 0.0, 0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        for _, sp in evaluation_sequence(pr, updates, seed=3):
            if supplier:
                supplier(sp, [e, o])
            lnl, st = e.evaluate(sp)
            calls += 1
            what = f"evaluation {calls} (chain {sp.chain})"
            check_with_oracle(e, o, [sp], lnl, st, 1e-9, tree_tol(pr))
            le = lnl[0]
            for m in sp.mats["matrix"][:3]:
                assert np.allclose(e.get_transition_matrix(int(m)), o.get_transition_matrix(int(m)), rtol=2.5e-7,
                                   atol=1e-30), what
            ref = f64_std_lnl(pr, sp.chain, rates=pr.chain_rates[sp.chain],
                              matrices=supplier.matrices(sp.chain) if supplier else None)
            assert not ref.underflow
            ratio = abs(le - ref.lnl) / ref.bound(pr)
            worst = max(worst, ratio)
            assert ratio <= 1.0, f"{what}: engine {le!r}, float64 {ref.lnl!r}, {ratio:.2f} x the bound"
        assert e.kernel_launches(abi.KERNEL_STD) == calls          # the variable-state kernel served every call
    record_property("max_error_to_bound", float(worst))
    return ref


def names(prefix):
    return [n for n in CASES if n.startswith(prefix)]


@pytest.mark.parametrize("name", names("lanes-"))
def test_lane_widths(engine_lib, oracle_lib, record_property, name):
    """L = 1 ... 32 lanes per pattern (K = 17 ... 20: one pattern per warp, the shuffles span all 32 lanes); the
    pattern count one less than, equal to and one more than a whole number of 128 / L-pattern tiles"""
    pr, _ = make_case(name)
    tp = 128 // lanes(pr.K)
    assert (pr.C + 1) % tp in (0, 1, 2) and pr.C >= 2 * tp - 1
    check_run(engine_lib, oracle_lib, pr, None, record_property)


SMAX = {"smax-4": 4, "smax-5": 8, "smax-8": 8, "smax-9": 12, "smax-12": 12, "smax-13": 16, "smax-16": 16,
        "smax-17": 24, "smax-24": 24}


@pytest.mark.parametrize("name", names("smax-"))
def test_smax_instantiations(engine_lib, oracle_lib, record_property, name):
    """the largest state count on both sides of each eval_std_kernel<4|8|12|16|24> boundary"""
    pr, _ = make_case(name)
    assert pr.S == int(name.split("-")[1]) and smax_instantiation(pr.S) == SMAX[name]
    check_run(engine_lib, oracle_lib, pr, None, record_property)


def test_many_classes(engine_lib, oracle_lib, record_property):
    """state counts 2 ... 10 at K = 20: 180 (class, category) matrices for tiprobs_std_kernel's 64 threads"""
    pr, _ = make_case("classes-2to10-K20")
    assert len(set(pr.state_counts.tolist())) * pr.K == 180
    check_run(engine_lib, oracle_lib, pr, None, record_property)


@pytest.mark.parametrize("name,tiles", [("informative-K4", 3), ("informative-K17", 17)])
def test_coding_informative(engine_lib, oracle_lib, record_property, name, tiles):
    """2 + 2 x 32 dummy patterns spread over several tiles: the unobserved probability summed across them"""
    pr, _ = make_case(name)
    tp = 128 // lanes(pr.K)
    assert pr.dummy == 66 and (pr.dummy + tp - 1) // tp == tiles
    check_run(engine_lib, oracle_lib, pr, None, record_property, updates=4)


def test_coding_near_degenerate(engine_lib, oracle_lib, record_property):
    """short branches: pObserved ~ 1e-4, the correction amplifies the partials' rounding by 1 / pObserved"""
    pr, _ = make_case("near-degenerate")
    ref = check_run(engine_lib, oracle_lib, pr, None, record_property)
    assert 1e-5 < 1.0 - ref.p_un < 1e-3


def test_coding_clamp(engine_lib, oracle_lib, record_property):
    """two dummy patterns with every tip missing: sum L_c ~ 2, pObserved clamps to 1e-300 and the correction is
    -U log(1e-300) on the engine, the oracle and float64 alike"""
    pr, _ = make_case("clamp")
    ref = check_run(engine_lib, oracle_lib, pr, None, record_property)
    assert ref.p_un > 1.9


@pytest.mark.parametrize("name", ["supplied-nonsymmetric-K3", "supplied-nonsymmetric-K17"])
def test_supplied_nonsymmetric_matrices(engine_lib, oracle_lib, record_property, name):
    """non-symmetric row-stochastic matrices on the even branches, the engine's own Mk on the others, in one
    evaluation: the general path reads P[a * n + i], parent state a, child state i"""
    pr, supplier = make_case(name)
    check_run(engine_lib, oracle_lib, pr, supplier, record_property)
    assert supplier.blocks


def test_supplied_ordered_matrices(engine_lib, oracle_lib, record_property):
    """an ordered block per state count 3 ... 6 after the unordered ones, every matrix supplied by the caller (Mk for
    the unordered blocks, expm of a birth-death Q for the ordered ones), no matrix updates in the evaluations"""
    pr, supplier = make_case("supplied-ordered")
    assert sorted(set(pr.state_counts[pr.ordered].tolist())) == [3, 4, 5, 6]
    check_run(engine_lib, oracle_lib, pr, supplier, record_property)


def test_hymfossil_sized(engine_lib, oracle_lib, record_property):
    """114 taxa, 45 of them fossils with 70-95 % missing, up to 7 states, K = 4, on a caterpillar: 112 levels of
    node scalers add up in the site scalers"""
    pr, _ = make_case("hymfossil")
    assert tree_height(pr.tree[0]) == 112
    check_run(engine_lib, oracle_lib, pr, None, record_property)


# ---- batches -------------------------------------------------------------------------------------------------------
def test_underflow_in_one_evaluation_of_a_batch(engine_lib, oracle_lib):
    """Four chains in one launch; only chain 2's branches give P = I, so only its root, where the root tip
    disagrees with the others, has a zero-likelihood pattern: it alone reports EVAL_UNDERFLOW.  (The live chains'
    partials are not compared: at r t ~ 1e-11 TiProbs_Std's 1/n - e/n cancels, and the last-bit difference between
    CUDA's and glibc's exp becomes ~1e-5 relative in pChange.)"""
    nch = 4
    pr, _ = dead_pattern_problem("std", "middle", n_chains=nch)
    pr.tree[2].length[:] = 0.0
    with pr.create(engine_lib) as e, pr.create(oracle_lib) as o:
        specs = [pr.full_evaluation(ch) for ch in range(nch)]
        lnl, st = e.evaluate(specs)
        assert e.kernel_launches(abi.KERNEL_STD) == 1
        for ch, sp in enumerate(specs):
            (lo,), (so,) = o.evaluate(sp)
            assert st[ch] == so == (abi.EVAL_UNDERFLOW if ch == 2 else abi.EVAL_OK), f"chain {ch}"
            if ch == 2:
                assert lnl[ch] == lo == -DBL_MAX
            else:
                assert rel(lnl[ch], lo) < 1e-9, f"chain {ch}"


def cynmix_like(seed):
    """cynmix's shape: four 4-state GTR + G4 partitions and a morphology partition, 32 taxa, one chain"""
    dna = [workloads.make_problem(4, 4, C, 32, 1, seed=seed + i) for i, C in enumerate((537, 125, 205, 332))]
    return dna + [make_std_division(162, 4, 32, 1, seed=seed, states=(2, 3, 4, 5, 6, 8), p_poly=0.05)]


def test_cynmix_generation_begin_end(engine_lib):
    """All five divisions of a generation in flight through evaluate_begin ... evaluate_end: bit for bit what one
    evaluate() per division gives"""
    probs_a, probs_b = cynmix_like(80), cynmix_like(80)
    insts_a = [p.create(engine_lib) for p in probs_a]
    insts_b = [p.create(engine_lib) for p in probs_b]
    try:
        rng_a, rng_b = np.random.default_rng(5), np.random.default_rng(5)
        gens = 5
        for gen in range(gens):
            specs_a = [p.full_evaluation(0) if gen == 0 else p.random_branch_update(0, rng_a) for p in probs_a]
            specs_b = [p.full_evaluation(0) if gen == 0 else p.random_branch_update(0, rng_b) for p in probs_b]
            for inst, sp in zip(insts_a, specs_a):
                inst.evaluate_begin(sp)
            got = [inst.evaluate_end() for inst in insts_a]
            want = [inst.evaluate(sp) for inst, sp in zip(insts_b, specs_b)]
            for d, ((lg, sg), (lw, sw)) in enumerate(zip(got, want)):
                assert not sg.any() and np.array_equal(lg, lw) and np.array_equal(sg, sw), f"generation {gen}, division {d}"
        assert insts_a[-1].kernel_launches(abi.KERNEL_STD) == gens
        assert all(inst.kernel_launches(abi.KERNEL_STD) == 0 for inst in insts_a[:4])
    finally:
        for inst in insts_a + insts_b:
            inst.close()
