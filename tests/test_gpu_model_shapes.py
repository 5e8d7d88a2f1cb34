"""GPU: general-state evaluations at the shapes production models send down the CUDA-core route, against the CPU
oracle and the float64 reference.

The route is eval_gen_kernel with the stand-alone P(t) builders: tiprobs_kernel up to 32 states, tiprobs_mm_kernel
with cijk_factor_kernel above, and above 32 states the device eigensolver builds the slots (the seam's default
there).  The models come from tests/model_shapes.py:
  codon      60 (vertmt), 62 (invermt and the other 62-codon codes), 63 (ciliate: odd S, 64-float rows, solver N = 64)
             sense codons with one Q, or one Q per omega category in K = 3 or 4 cijk parts (NY98 / M3); 61 codons with
             four omega categories (the tensor-core kernel takes K <= 3 only)
  covarion   + gamma on 8 and 40 states, one Q per rate category (parts = K, host eigensystems through set_cijk), tip
             masks replicated into both hidden blocks, one slow-switching chain per shape
  protein    20 states with 5 and 20 gamma categories (the tensor-core kernel takes K <= 4 only)
Geometry of the generic kernel at these shapes (mb200_create_instance): at S = 63, K = 3 the P matrices of all
categories take 48 384 B, just under the 48 KB line for all categories per pass, and 32-pattern tiles need 97 920 B of
shared memory, just under 96 KB; they happen only when C >= 32 x SMs, so that case runs C = 32 x SMs + 1 (the last
tile holds one pattern) next to a small C (4-pattern tiles).  S = 63, K = 4 and S = 40, K = 8 take one category
per pass, S = 40, K = 4 all of them.

Each shape: 8 chains with their own models (slot 0 and weights row 0 decoys), one call of all full evaluations, two
calls of branch updates over all chains with every third update rejected, and one call of root-only evaluations
that reads what the rejections restored.  Every evaluation against the oracle (lnL and status; every partials
buffer and node and site scaler it wrote, at the generic kernel's tolerances), against the same evaluation sent
alone to a twin instance (bit for bit), and against the float64 reference after the full evaluations, after the
last updates and after the rejections.  The kernel counters show the route.  engine_checks.SHAPES_TOL says why the
partials and node scalers get wider bounds here than on the other generic tests."""
import numpy as np
import pytest
from scipy.linalg import expm

from model_shapes import (CODE_OF_STATES, P_EPS, P_TIMES, SHAPES, ShapeModels, cijk_block, codon_model, codon_q,
                          shape_problem, solver_cases)
from engine_checks import SHAPES_TOL, SYN_RTOL, check_with_oracle, eigen_instance, num_sms, rel
from mrbayes_b200 import abi

pytestmark = pytest.mark.gpu


# (shape, pattern count: "tp32" = 32 x SMs + 1, else C)
RUNS = [
    ("codon60", 130), ("codon60_m3", 130), ("codon62", 130), ("codon62_m3", 130), ("codon63", 130),
    ("codon63_m3", 130), ("codon63_m3", "tp32"), ("codon63_m3_host", 130), ("codon63_m4", 130),
    ("codon61_m4", 129), ("covarion8_g4", 300), ("covarion8_g20", 150), ("covarion40_g4", 200),
    ("covarion40_g8", 200), ("protein_g5", 257), ("protein_g20", 150),
]


@pytest.mark.parametrize("name,C", RUNS)
def test_generic_route_at_production_shape(engine_lib, oracle_lib, name, C):
    sh = SHAPES[name]
    if C == "tp32":
        C = 32 * num_sms() + 1
    seed = 9000 + sum(map(ord, name)) + C
    pr = shape_problem(sh, C, seed=seed)
    mm = ShapeModels(pr, sh, seed=seed)
    n = pr.n_chains
    rng = np.random.default_rng(seed)
    worst = {"f64": 0.0, "oracle": 0.0, "partials": 0.0, "partials_of_peak": 0.0}

    def against_f64(lnl):
        for ch in range(n):
            r = rel(lnl[ch], mm.f64(ch))
            worst["f64"] = max(worst["f64"], r)
            assert r < SYN_RTOL, f"float64 reference, chain {ch}: {r:.2e}"

    with mm.create(engine_lib) as e, mm.create(engine_lib) as twin, mm.create(oracle_lib) as o:
        o.set_arith(1)

        def call(specs):
            lnl, st = e.evaluate(specs)
            for i, sp in enumerate(specs):
                (la,), (sa,) = twin.evaluate(sp)
                assert sa == st[i] and la == lnl[i], f"evaluation {i}: alone {la!r}, batched {lnl[i]!r}"
            for k, x in zip(("oracle", "partials", "partials_of_peak"),
                            check_with_oracle(e, o, specs, lnl, st, SYN_RTOL, SHAPES_TOL)):
                worst[k] = max(worst[k], x)
            return lnl

        against_f64(call([mm.full(ch) for ch in range(n)]))
        updates = 0
        for g in range(2):
            specs, rejects = [], []
            for ch in range(n):
                old = pr.tree[ch].length.copy()
                specs.append(mm.update(ch, rng))
                updates += 1
                if updates % 3 == 0:
                    rejects.append((ch, specs[-1], old))
            lnl = call(specs)
            if g == 1:
                against_f64(lnl)
            for ch, sp, old in rejects:
                pr.reject(ch, sp, old)
        assert updates >= 10 and rejects
        against_f64(call([mm.root_only(ch) for ch in range(n)]))
        assert e.kernel_launches(abi.KERNEL_GENERIC) == 4
        assert e.kernel_launches(abi.KERNEL_TIPROBS) == 3          # the root-only call rebuilds no matrix
        assert e.kernel_launches(abi.KERNEL_TENSOR) == e.kernel_launches(abi.KERNEL_NUC4) == 0
    print(f"\n{name} C={C}: lnL vs float64 {worst['f64']:.2e}, vs oracle {worst['oracle']:.2e}, "
          f"partials vs oracle {worst['partials']:.2e} relative (entries above 1e-6 of the pattern's largest), "
          f"excess over 2e-6 relative {worst['partials_of_peak']:.2e} of the pattern's largest")


# ---- the device eigensolver at the new sizes -------------------------------------------------------------------------
def p_bound(want):
    """|P_device - expm| allowed per entry: 2 ulp of the float-rounded entry + P_EPS (model_shapes.py)"""
    return 2.0 * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + P_EPS


@pytest.mark.parametrize("name", list(solver_cases()))
def test_device_eigensystem_entry_by_entry(engine_lib, name):
    """mb200_set_rate_matrices on codon Q's (60, 62, 63 states; one and three parts) and covarion Q's (8 and 40
    states, four parts; the seam solves those on the host, but their spectra, nearly repeated with slow switching,
    are the solver's hardest).  P(t) at four lengths, entry by entry: within p_bound of expm (the existing
    test_gpu_eigen.py bound of 2e-7 absolute cannot see a 20 % error on the 1e-6 entries of a short codon branch),
    within twice that of the host-eigensystem path (set_cijk), and with parts > 1 far outside it for another part's
    matrix."""
    Qs, pi = solver_cases()[name]
    parts, S = Qs.shape[0], Qs.shape[1]
    K = parts if parts > 1 else 2
    rates = np.ones(K) if parts > 1 else np.array([0.5, 1.5])
    mats = np.zeros(len(P_TIMES), abi.MAT_DTYPE)
    for i, t in enumerate(P_TIMES):
        mats[i] = (i, 1, t)
    worst = 0.0
    with eigen_instance(engine_lib, S, K, parts) as dev, eigen_instance(engine_lib, S, K, parts) as host:
        dev.set_rate_matrices(1, Qs, pi)
        host.set_cijk(1, cijk_block(Qs, pi))
        dev.update_transition_matrices(mats, rates, pi)
        host.update_transition_matrices(mats, rates, pi)
        for i, t in enumerate(P_TIMES):
            Pd = np.asarray(dev.get_transition_matrix(i), np.float64).reshape(K, S, S)
            Ph = np.asarray(host.get_transition_matrix(i), np.float64).reshape(K, S, S)
            for k in range(K):
                want = expm(Qs[k if parts > 1 else 0] * (t * rates[k]))
                b = p_bound(want)
                d = np.abs(Pd[k] - want)
                worst = max(worst, float(d.max()))
                assert (d <= b).all(), f"t {t}, category {k}: {d.max():.2e}, {(d / b).max():.2f} x the bound"
                assert (np.abs(Pd[k] - Ph[k]) <= 2 * b).all(), f"t {t}, category {k}: device vs host eigensystem"
                if parts > 1:
                    other = expm(Qs[(k + 1) % parts] * (t * rates[k]))
                    assert (np.abs(other - Pd[k]) / b).max() > 1e3, f"t {t}: part {(k + 1) % parts} is as close"
    print(f"\n{name}: P(t) vs expm {worst:.2e}")


def test_warm_started_codon_chain(engine_lib):
    """40 links at 63 states, three omega categories: each proposal changes kappa, the omegas and pi a little and warm
    starts from the current slot's eigenvectors; accepted or not, the slots ping-pong.  Every link entry by entry
    against expm within p_bound."""
    code, S = CODE_OF_STATES[63], 63
    rng = np.random.default_rng(63)
    kappa, omegas = 2.5, np.array([0.05, 0.5, 3.0])
    _, pi = codon_model(code, rng, kappa, omegas, 1.0)
    mats = np.zeros(1, abi.MAT_DTYPE)
    cur, worst = 0, 0.0
    with eigen_instance(engine_lib, S, 3, 3) as dev:
        for link in range(40):
            kappa *= np.exp(0.2 * (rng.random() - 0.5))
            omegas = omegas * np.exp(0.2 * (rng.random(3) - 0.5))
            pi = pi * np.exp(0.1 * (rng.random(S) - 0.5))
            pi /= pi.sum()
            Qs = np.stack([codon_q(code, kappa, w, pi) for w in omegas])
            new = 1 - cur
            dev.set_rate_matrices(new, Qs, pi, like=cur)
            mats[0] = (0, new, 0.37)
            dev.update_transition_matrices(mats, np.ones(3), pi)
            P = np.asarray(dev.get_transition_matrix(0), np.float64).reshape(3, S, S)
            for k in range(3):
                want = expm(Qs[k] * 0.37)
                d = np.abs(P[k] - want)
                worst = max(worst, float(d.max()))
                assert (d <= p_bound(want)).all(), (link, k, float(d.max()))
            if rng.random() < 0.5:
                cur = new
    print(f"\nwarm-started chain: P(t) vs expm {worst:.2e}")
