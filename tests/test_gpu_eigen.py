"""Device eigensolver (mb200_set_rate_matrices, SURVEY 8 f3) against independent references.

What it replaces is the host half of UpDateCijk (GetEigens src/utils.c:11201 + CalcCijk src/utils.c:9734).  Checked here
through the C-ABI: P(t) built from the device's eigensystem vs (a) scipy's matrix exponential of Q t (no eigensystem
involved) and (b) the same engine fed the host's eigensystem the way the seam feeds it (mb200_set_cijk with V, V^-1 from
numpy.linalg.eig, i.e. a general non-symmetric solver like the reference's).  Tolerance: P(t) is stored as float; the
double-precision sums behind it agree to ~1e-13, so the stored values may differ in the last float place only."""
import numpy as np
import pytest
from scipy.linalg import expm

from engine_checks import eigen_instance, reversible_q
from mrbayes_b200 import abi

pytestmark = pytest.mark.gpu


def cijk_block(Q, pi):
    lam, V = np.linalg.eig(Q)
    assert np.abs(lam.imag).max() < 1e-9
    lam, V = lam.real, V.real
    if np.linalg.cond(V) > 1e8:                  # repeated eigenvalues: the general solver's basis may be degenerate
        d = np.sqrt(pi)
        lam, U = np.linalg.eigh(0.5 * ((d[:, None] * Q / d[None, :]) + (d[:, None] * Q / d[None, :]).T))
        V = U / d[:, None]
    Vi = np.linalg.inv(V)
    S = Q.shape[0]
    c = np.einsum("ik,kj->ijk", V, Vi)
    return np.concatenate([lam, np.zeros(S), c.ravel()])


CASES = [
    # S, K, parts, sparse, skew, equal
    (4, 4, 1, False, False, False),
    (4, 1, 1, False, True, True),        # F81-like: a threefold eigenvalue
    (16, 2, 1, True, False, False),      # doublet-sized
    (20, 4, 1, False, True, False),
    (61, 1, 1, True, True, False),       # codon M0-sized, odd S: padded pairing
    (61, 3, 3, True, False, False),      # one rate matrix per omega category
    (64, 1, 1, False, False, False),
]


@pytest.mark.parametrize("S,K,parts,sparse,skew,equal", CASES)
def test_device_eigensystem_gives_the_matrix_exponential(engine_lib, S, K, parts, sparse, skew, equal):
    rng = np.random.default_rng(1000 * S + K)
    base, pi = reversible_q(rng, S, sparse, skew, equal)
    Qs = np.stack([base * (0.4 + 0.8 * p) for p in range(parts)])        # same pi, different speeds (NY98-like)
    rates = np.ones(K) if parts > 1 else np.linspace(0.2, 2.5, K)
    lengths = [0.004, 0.11, 0.9, 3.7]
    mats = np.zeros(len(lengths), abi.MAT_DTYPE)
    with eigen_instance(engine_lib, S, K, parts) as dev, eigen_instance(engine_lib, S, K, parts) as host:
        dev.set_rate_matrices(1, Qs, pi)
        host.set_cijk(1, np.concatenate([cijk_block(q, pi) for q in Qs]))
        for i, t in enumerate(lengths):
            mats[i] = (i, 1, t)
        dev.update_transition_matrices(mats, rates, pi)
        host.update_transition_matrices(mats, rates, pi)
        for i, t in enumerate(lengths):
            Pd = np.asarray(dev.get_transition_matrix(i), np.float64).reshape(K, S, S)
            Ph = np.asarray(host.get_transition_matrix(i), np.float64).reshape(K, S, S)
            for k in range(K):
                want = expm(Qs[k if parts > 1 else 0] * (t * rates[k]))
                assert np.abs(Pd[k] - want).max() < 2e-7, (S, k, t, np.abs(Pd[k] - want).max())
                assert np.abs(Pd[k].sum(1) - 1.0).max() < 5e-6
                assert np.abs(Pd[k] - Ph[k]).max() < 2e-7, (S, k, t, np.abs(Pd[k] - Ph[k]).max())


def test_slots_can_be_rewritten_back_to_back(engine_lib):
    """The staging area of a slot is reused only after its previous copy has been consumed: the LAST matrices win."""
    rng = np.random.default_rng(7)
    S = 61
    with eigen_instance(engine_lib, S, 1, 1) as dev:
        last = None
        for rep in range(6):
            Q, pi = reversible_q(rng, S, sparse=True)
            dev.set_rate_matrices(rep % 2, Q, pi)
            last = (rep % 2, Q, pi) if rep >= 4 else last
            if rep == 4:
                first = (rep % 2, Q, pi)
        mats = np.zeros(2, abi.MAT_DTYPE)
        mats[0] = (0, first[0], 0.3); mats[1] = (1, last[0], 0.3)
        dev.update_transition_matrices(mats, np.ones(1), pi)
        for i, (_, Q, _) in enumerate((first, last)):
            P = np.asarray(dev.get_transition_matrix(i), np.float64).reshape(S, S)
            assert np.abs(P - expm(Q * 0.3)).max() < 2e-7


def test_rejects_what_it_cannot_diagonalise(engine_lib):
    Q, pi = reversible_q(np.random.default_rng(3), 4)
    bad = pi.copy(); bad[2] = 0.0
    with eigen_instance(engine_lib, 4, 1, 1) as dev:
        rc = engine_lib.fn("set_rate_matrices")(dev.handle, 0, -1, abi._ptr(np.ascontiguousarray(Q), abi.C.c_double), abi._ptr(bad, abi.C.c_double))
        assert rc != 0
        rc = engine_lib.fn("set_rate_matrices")(dev.handle, 9, -1, abi._ptr(np.ascontiguousarray(Q), abi.C.c_double), abi._ptr(pi, abi.C.c_double))
        assert rc != 0
        rc = engine_lib.fn("set_rate_matrices")(dev.handle, 0, 9, abi._ptr(np.ascontiguousarray(Q), abi.C.c_double), abi._ptr(pi, abi.C.c_double))
        assert rc != 0


@pytest.mark.parametrize("S,parts", [(4, 1), (20, 1), (61, 1), (61, 3)])
def test_warm_started_chain_of_proposals(engine_lib, S, parts):
    """What a run does: every proposal's matrices are a small change of the chain's current ones and start from their
    eigenvectors (like = the other slot); accepted or not, the slots ping-pong.  80 links, i.e. more than two of the
    engine's forced cold restarts; every link against the matrix exponential."""
    rng = np.random.default_rng(S + parts)
    K = parts if parts > 1 else 2
    rates = np.ones(K) if parts > 1 else np.array([0.5, 1.5])
    Q, pi = reversible_q(rng, S, sparse=(S > 20))
    R = Q / pi[None, :]; np.fill_diagonal(R, 0.0)          # exchangeabilities
    mats = np.zeros(1, abi.MAT_DTYPE)
    cur = 0
    with eigen_instance(engine_lib, S, K, parts) as dev:
        for link in range(80):
            # a multiplier move on a block of exchangeabilities and a Dirichlet-like nudge of the frequencies
            i, j = rng.integers(0, S, 2)
            if i != j and R[i, j] > 0:
                f = np.exp(0.4 * (rng.random() - 0.5)); R[i, j] *= f; R[j, i] *= f
            pi = pi * np.exp(0.1 * (rng.random(S) - 0.5)); pi /= pi.sum()
            Qn = R * pi[None, :]; np.fill_diagonal(Qn, 0.0); np.fill_diagonal(Qn, -Qn.sum(1)); Qn /= -(pi * np.diag(Qn)).sum()
            Qs = np.stack([Qn * (0.5 + 0.7 * p) for p in range(parts)])
            new = 1 - cur if rng.random() < 0.7 else cur ^ 1
            dev.set_rate_matrices(new, Qs, pi, like=cur)
            mats[0] = (0, new, 0.37)
            dev.update_transition_matrices(mats, rates, pi)
            P = np.asarray(dev.get_transition_matrix(0), np.float64).reshape(K, S, S)
            for k in range(K):
                want = expm(Qs[k if parts > 1 else 0] * (0.37 * rates[k]))
                assert np.abs(P[k] - want).max() < 2e-7, (link, k, np.abs(P[k] - want).max())
            if rng.random() < 0.5:
                cur = new                                    # accepted
