"""CPU: the model builders of tests/model_shapes.py, and the oracle against the float64 reference at every shape
test_gpu_model_shapes.py runs, so that the oracle is a sound judge there; plus the checks that make a failure of
those GPU tests mean something (wrong eigen parts change lnL, the last states are observed, P_EPS is not loose)."""
import numpy as np
import pytest
from scipy.linalg import expm

from f64_reference import f64_lnl
from model_shapes import (CODE_OF_STATES, CODES, P_EPS, P_TIMES, SHAPES, ShapeModels, codon_model, covarion_masks,
                          covarion_model, eig_of_reversible, sense_codons, shape_problem, solver_cases)
from mrbayes_b200 import abi

RTOL = 2e-7          # float oracle vs double reference (test_f64_reference.py)


def assert_reversible(Q, pi):
    assert np.allclose(Q.sum(1), 0.0, atol=1e-12)
    assert (Q - np.diag(np.diag(Q)) >= 0).all()
    F = pi[:, None] * Q
    assert np.allclose(F, F.T, rtol=1e-12, atol=1e-15)
    assert np.isclose(pi.sum(), 1.0)


@pytest.mark.parametrize("code", list(CODES))
def test_codon_builder(code):
    """sense-codon counts of the NCBI tables; q_ij = 0 unless one nucleotide differs, otherwise pi_j times kappa for a
    transition and omega for a nonsynonymous change, up to the common scale; one substitution per unit time; F3x4
    frequencies down to ~1e-4"""
    want = {"universal": 61, "vertmt": 60, "ciliate": 63}.get(code, 62)
    sc = sense_codons(code)
    assert len(sc) == want
    kappa, omegas = 3.5, [0.07, 0.8, 4.0]
    Qs, pi = codon_model(code, np.random.default_rng(1), kappa, omegas, 1.0)
    assert Qs.shape == (3, want, want)
    assert 1e-5 < pi.min() < 1e-3
    for Q, w in zip(Qs, omegas):
        assert_reversible(Q, pi)
        assert np.isclose(-(pi * np.diag(Q)).sum(), 1.0)
        R = Q / pi[None, :]
        unit = None
        for i, (a, x) in enumerate(sc):
            for j, (b, y) in enumerate(sc):
                diff = [p for p in range(3) if a[p] != b[p]]
                if i == j:
                    continue
                if len(diff) != 1:
                    assert Q[i, j] == 0.0
                    continue
                ts = {a[diff[0]], b[diff[0]]} in ({"T", "C"}, {"A", "G"})
                f = (kappa if ts else 1.0) * (1.0 if x == y else w)
                unit = R[i, j] / f if unit is None else unit
                assert np.isclose(R[i, j], unit * f, rtol=1e-12)
    assert sorted(CODE_OF_STATES) == [60, 61, 62, 63]


@pytest.mark.parametrize("S0,K,s01,s10", [(4, 4, 0.3, 0.8), (20, 8, 0.01, 0.013)])
def test_covarion_builder(S0, K, s01, s10):
    """rows sum to 0, detailed balance, the switching entries, no substitutions in the off block, category k's on
    block = the same model times its gamma rate, pi = pi0 (x) (s10, s01) / (s01 + s10)"""
    Qs, pi = covarion_model(S0, K, np.random.default_rng(S0), s01, s10, 0.5)
    assert Qs.shape == (K, 2 * S0, 2 * S0)
    on, off = slice(0, S0), slice(S0, 2 * S0)
    assert np.isclose(pi[on].sum() / pi[off].sum(), s10 / s01)
    assert np.allclose(pi[on] / pi[on].sum(), pi[off] / pi[off].sum())
    for Q in Qs:
        assert_reversible(Q, pi)
        assert np.allclose(np.diag(Q[on, off]), s01) and np.allclose(np.diag(Q[off, on]), s10)
        assert np.count_nonzero(Q[on, off] - np.diag(np.diag(Q[on, off]))) == 0
        assert np.count_nonzero(Q[off, off] - np.diag(np.diag(Q[off, off]))) == 0
    ratio = Qs[:, 0, 1] / Qs[0, 0, 1]
    assert np.ptp(ratio) > 0.5 and np.allclose(Qs[:, on, on][:, 1:, 0] / Qs[0, on, on][1:, 0], ratio[:, None])


def test_covarion_masks():
    """every observed bit lands in both hidden blocks, and nothing else: bit i and bit i + S0"""
    rng = np.random.default_rng(3)
    for S0 in (4, 20):
        m0 = rng.integers(0, 1 << S0, size=200).astype(np.uint64)
        m0[:3] = [1, 1 << (S0 - 1), (1 << S0) - 1]
        m = covarion_masks(m0, S0)
        for a, b in zip(m0, m):
            for i in range(S0):
                bit = (int(a) >> i) & 1
                assert (int(b) >> i) & 1 == bit and (int(b) >> (i + S0)) & 1 == bit
            assert int(b) >> (2 * S0) == 0
    sh = SHAPES["covarion40_g4"]
    pr = shape_problem(sh, 50, 6, 1, seed=2)
    assert np.array_equal(pr.masks, covarion_masks(pr.masks & np.uint64((1 << 20) - 1), 20))


def test_eig_of_reversible():
    for Qs, pi in solver_cases().values():
        for Q in Qs:
            V, Vi, lam = eig_of_reversible(Q, pi)
            assert np.allclose((V * lam) @ Vi, Q, atol=1e-12) and np.allclose(Vi @ V, np.eye(len(pi)), atol=1e-10)


def test_p_eps_covers_float64_eigen_products():
    """P_EPS: numpy's eigh-based P(t) in double against expm on the solver's matrices.  Measured: 1.3e-14 at most
    (codon), 3e-15 (covarion); P_EPS = 1e-12 leaves a factor of 50 for the device's Jacobi tolerance (off-diagonal
    entries below 1e-14 of the largest diagonal one)."""
    worst = 0.0
    for Qs, pi in solver_cases().values():
        for Q in Qs:
            V, Vi, lam = eig_of_reversible(Q, pi)
            for t in P_TIMES:
                worst = max(worst, np.abs((V * np.exp(lam * t)) @ Vi - expm(Q * t)).max())
    assert worst < P_EPS / 50, worst
    # the bound is not loose where it matters: the shortest codon branch has entries far below float's ulp at 1
    Qs, _ = solver_cases()["codon63_p3"]
    P = expm(Qs[0] * P_TIMES[0])
    small = P[(P > 1e-7) & (P < 1e-5)]
    assert small.size > 50
    bound = 2 * np.spacing(small.astype(np.float32)).astype(float) + P_EPS
    assert (bound < 1e-4 * small).all()          # a 0.01 % error of such an entry is outside the bound


@pytest.mark.parametrize("name", list(SHAPES))
def test_oracle_matches_f64_at_gpu_shapes(oracle_lib, name):
    """Three chains with their own models (host eigensystems for the oracle, as the GPU tests give it), full
    evaluations and branch updates with a rejection: oracle within 2e-7 of the float64 reference.  Where a slot has
    one eigensystem per category, the float64 lnL with every category reading part 0 is far off, so that a kernel
    reading the wrong part fails; and at least 10 % of the patterns have a tip observing state S-1 or S-2, the last
    float4 chunk of a partials row next to the padding at S = 62 and 63."""
    sh = SHAPES[name]
    pr = shape_problem(sh, 97, 8, 3, seed=11)
    mm = ShapeModels(pr, sh, seed=5)
    rng = np.random.default_rng(1)
    with mm.create(oracle_lib) as o, mm.create(oracle_lib) as scratch:
        o.set_arith(1)
        scratch.set_arith(1)
        mm.assert_models_differ(scratch, range(3))
        for ch in range(3):
            (lo,), (so,) = o.evaluate(mm.full(ch))
            assert so == abi.EVAL_OK
            lf = mm.f64(ch)
            assert abs(lo - lf) < RTOL * abs(lf), f"chain {ch}: {abs(lo - lf) / abs(lf):.2e}"
        for it in range(5):
            ch = it % 3
            old = pr.tree[ch].length.copy()
            sp = mm.update(ch, rng)
            (lo,), _ = o.evaluate(sp)
            lf = mm.f64(ch)
            assert abs(lo - lf) < RTOL * abs(lf), f"update {it}: {abs(lo - lf) / abs(lf):.2e}"
            if it == 2:
                pr.reject(ch, sp, old)
    if sh.parts > 1:
        for ch in range(3):
            m = mm.models[ch]
            wrong = f64_lnl(pr, ch, Q=np.broadcast_to(m.Q[0], m.Q.shape), freqs=m.freqs, rates=m.rates,
                            cat_weights=m.cat_weights, p_invar=m.p_invar, weights=mm.weights[m.row])[1]
            own = mm.f64(ch)
            assert abs(wrong - own) > 1e-3 * abs(own), f"chain {ch}: part 0 for every category changes lnL too little"
    full = np.uint64((1 << sh.S) - 1) if sh.S < 64 else np.uint64(~0 & 0xFFFFFFFFFFFFFFFF)
    last = np.uint64(3 << (sh.S - 2))
    observed = (pr.masks != full) & ((pr.masks & last) != 0)
    assert observed.any(axis=0).mean() >= 0.10
    if sh.kind == "covarion":
        assert len({(m.freqs[:sh.S0].sum()) for m in mm.models}) == len(mm.models)      # own switching rates per chain
