"""Model builders for the shapes production models send down the generic (CUDA-core) route: codon models under
the genetic codes with 60, 62 and 63 sense codons (one Q, or one Q per omega category on a shared pi, the NY98 / M3
shape), covarion + gamma (one Q per rate category on 2 S0 hidden states), and the replicated tip masks the seam
builds for covarion divisions.  No likelihood arithmetic lives here, only inputs, as in workloads.py.

ShapeModels is a chain_models.MixedModels whose eigensystems come from these builders: per-chain slots, the decoy
slot and row, device or host eigensystems and the float64 lnL by per-category expm all carry over.  Models with one
eigensystem per category send category_rates as the seam does for them: the constant correction factor (3 for codon
models, 1 otherwise), since the category's rate already sits in its Q."""
import numpy as np

from chain_models import MixedModels, cijk_of
from mrbayes_b200 import workloads

# The public NCBI translation tables, 64 codons in TCAG order (first base slowest), '*' a stop codon
CODES = {
    "universal":  "FFLLSSSSYY**CC*WLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG",    # table 1
    "vertmt":     "FFLLSSSSYY**CCWWLLLLPPPPHHQQRRRRIIMMTTTTNNKKSS**VVVVAAAADDEEGGGG",    # table 2
    "yeast":      "FFLLSSSSYY**CCWWTTTTPPPPHHQQRRRRIIMMTTTTNNKKSSRRVVVVAAAADDEEGGGG",    # table 3
    "mycoplasma": "FFLLSSSSYY**CCWWLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG",    # table 4
    "invermt":    "FFLLSSSSYY**CCWWLLLLPPPPHHQQRRRRIIMMTTTTNNKKSSSSVVVVAAAADDEEGGGG",    # table 5
    "ciliate":    "FFLLSSSSYYQQCC*WLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG",    # table 6
    "echinoderm": "FFLLSSSSYY**CCWWLLLLPPPPHHQQRRRRIIIMTTTTNNNKSSSSVVVVAAAADDEEGGGG",    # table 9
    "euplotid":   "FFLLSSSSYY**CCCWLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG",    # table 10
}
CODE_OF_STATES = {61: "universal", 60: "vertmt", 62: "invermt", 63: "ciliate"}
BASES = "TCAG"
TRANSITIONS = {frozenset("TC"), frozenset("AG")}


def sense_codons(code):
    """-> [(codon string, amino acid)] of the sense codons of `code`, in table order"""
    aa = CODES[code]
    cod = [a + b + c for a in BASES for b in BASES for c in BASES]
    return [(c, a) for c, a in zip(cod, aa) if a != "*"]


def position_freqs(rng, freq_skew):
    """[3, 4] nucleotide frequencies per codon position: at freq_skew = 1 each position takes 0.04, 0.16, 0.3 and 0.5
    in a random order, so the rarest codon has a frequency near 1e-4; freq_skew = 0 is uniform"""
    skewed = np.array([rng.permutation([0.04, 0.16, 0.3, 0.5]) for _ in range(3)])
    return (1.0 - freq_skew) * 0.25 + freq_skew * skewed


def codon_freqs(code, f3x4):
    """F3x4: the product of the per-position nucleotide frequencies, renormalised over the sense codons"""
    pi = np.array([np.prod([f3x4[p, BASES.index(c[p])] for p in range(3)]) for c, _ in sense_codons(code)])
    return pi / pi.sum()


def scaled(Q, pi):
    """Q with its diagonal set to minus the row sums, scaled to one expected substitution per unit time"""
    Q = Q.copy()
    np.fill_diagonal(Q, 0.0)
    np.fill_diagonal(Q, -Q.sum(1))
    return Q / -(pi * np.diag(Q)).sum()


def codon_q(code, kappa, omega, pi):
    """GY94-type codon rate matrix: q_ij = pi_j for codons one nucleotide apart, times kappa for a transition and
    omega for a nonsynonymous change; 0 for codons further apart"""
    sc = sense_codons(code)
    S = len(sc)
    Q = np.zeros((S, S))
    for i, (ci, ai) in enumerate(sc):
        for j, (cj, aj) in enumerate(sc):
            diff = [p for p in range(3) if ci[p] != cj[p]]
            if len(diff) != 1:
                continue
            p = diff[0]
            r = kappa if frozenset(ci[p] + cj[p]) in TRANSITIONS else 1.0
            Q[i, j] = r * (1.0 if ai == aj else omega) * pi[j]
    return scaled(Q, pi)


def codon_model(code, rng, kappa, omegas, freq_skew):
    """-> (Q [len(omegas), S, S], pi [S]): one rate matrix per omega value on a shared F3x4 pi"""
    pi = codon_freqs(code, position_freqs(rng, freq_skew))
    return np.stack([codon_q(code, kappa, w, pi) for w in omegas]), pi


def covarion_model(S0, K, rng, s01, s10, alpha):
    """-> (Q [K, 2 S0, 2 S0], pi [2 S0]).  States 0 .. S0-1 are the "on" copies of the observable states, S0 .. 2 S0-1
    the "off" copies.  Category k: the on block is a random reversible S0-state model times the k-th discrete-gamma
    rate, on -> off of the same state at rate s01, off -> on at s10, no substitutions in the off block.
    pi = pi0 (x) (s10, s01) / (s01 + s10)."""
    pi0, V, Vi, lam = workloads.reversible_model(S0, rng)
    Q0 = (V * lam) @ Vi
    rates = workloads.discrete_gamma_rates(alpha, K)
    pi = np.concatenate([pi0 * s10, pi0 * s01]) / (s01 + s10)
    Qs = []
    for r in rates:
        Q = np.zeros((2 * S0, 2 * S0))
        Q[:S0, :S0] = Q0 * r
        Q[np.arange(S0), S0 + np.arange(S0)] = s01
        Q[S0 + np.arange(S0), np.arange(S0)] = s10
        np.fill_diagonal(Q, 0.0)
        np.fill_diagonal(Q, -Q.sum(1))
        Qs.append(Q)
    return np.stack(Qs), pi


def covarion_masks(masks0, S0):
    """Each observation in both hidden blocks: bit i and bit i + S0, as the seam sets the tip states"""
    m = np.asarray(masks0, np.uint64) & np.uint64((1 << S0) - 1)
    return m | (m << np.uint64(S0))


def eig_of_reversible(Q, pi):
    """-> (V, V^-1, lambda) of a reversible Q through the symmetric form D Q D^-1, D = diag(sqrt(pi))"""
    d = np.sqrt(pi)
    B = (d[:, None] * Q) / d[None, :]
    lam, U = np.linalg.eigh(0.5 * (B + B.T))
    return np.ascontiguousarray(U / d[:, None]), np.ascontiguousarray(U.T * d[None, :]), lam


def cijk_block(Qs, pi):
    """the set_cijk block of a slot with one part per rate matrix in Qs [parts, S, S]"""
    return np.concatenate([cijk_of(*eig_of_reversible(Q, pi)) for Q in Qs])


def neighbours(code):
    """[S] lists: the sense codons one nucleotide away from each sense codon"""
    sc = [c for c, _ in sense_codons(code)]
    return [[j for j, b in enumerate(sc) if sum(x != y for x, y in zip(a, b)) == 1] for a in sc]


def shape_masks(shape, n_tips, C, rng, edge_fraction=0.15):
    """Tip masks over the shape's S0 observable states.  Each pattern has a base state that `edge_fraction` of the
    patterns take from the last two, S0-1 and S0-2; each tip observes it or, with probability 1/4, another state:
    any state, or for codon models a codon one nucleotide away.  (Random codons at every tip make patterns whose
    likelihood rests on P(t) entries near 1e-19, three changes on a short branch.  A P(t) summed from an eigensystem
    in double, as the reference, the oracle and the engine build it, is good to ~1e-14 absolute per entry, so on such
    data all three differ from the expm-based float64 reference by up to 5e-5 in lnL.  Real alignments do not look
    like that.)  2 % missing, partial ambiguity on tips 0-2 (the others keep the terminal-branch shortcut)."""
    S0 = shape.S0
    base = rng.integers(0, S0, size=C)
    edge = rng.random(C) < edge_fraction
    base[edge] = S0 - 1 - rng.integers(0, 2, size=int(edge.sum()))
    st = np.tile(base, (n_tips, 1))
    mut = rng.random((n_tips, C)) < 0.25
    if shape.kind == "codon":
        nb = neighbours(CODE_OF_STATES[shape.S])
        for t, c in zip(*np.nonzero(mut)):
            st[t, c] = rng.choice(nb[base[c]])
    else:
        st[mut] = rng.integers(0, S0, size=int(mut.sum()))
    masks = np.uint64(1) << st.astype(np.uint64)
    masks[rng.random((n_tips, C)) < 0.02] = np.uint64((1 << S0) - 1)
    for t in range(3):
        amb = rng.random(C) < 0.2
        extra = np.uint64(1) << rng.integers(0, S0, size=C).astype(np.uint64)
        masks[t] = np.where(amb, masks[t] | extra, masks[t])
    return masks


class Shape:
    """One production shape: kind "codon" (S sense codons, K omega categories, parts = K or 1), "covarion" (2 S0
    states, K gamma categories, parts = K) or "gamma" (a random reversible S-state model, K gamma categories, one
    eigensystem); device: the engine's eigensolver builds the slots"""

    def __init__(self, kind, S, K, parts, device):
        self.kind, self.S, self.K, self.parts, self.device = kind, S, K, parts, device

    @property
    def S0(self):
        return self.S // 2 if self.kind == "covarion" else self.S

    def __repr__(self):
        return f"{self.kind}-S{self.S}-K{self.K}-p{self.parts}-{'dev' if self.device else 'host'}"


# every shape the GPU tests run (their pattern counts are chosen there)
SHAPES = {
    "codon60": Shape("codon", 60, 1, 1, True),
    "codon60_m3": Shape("codon", 60, 3, 3, True),
    "codon62": Shape("codon", 62, 1, 1, True),
    "codon62_m3": Shape("codon", 62, 3, 3, True),
    "codon63": Shape("codon", 63, 1, 1, True),
    "codon63_m3": Shape("codon", 63, 3, 3, True),
    "codon63_m3_host": Shape("codon", 63, 3, 3, False),
    "codon63_m4": Shape("codon", 63, 4, 4, True),
    "codon61_m4": Shape("codon", 61, 4, 4, True),
    "covarion8_g4": Shape("covarion", 8, 4, 4, False),
    "covarion8_g20": Shape("covarion", 8, 20, 20, False),
    "covarion40_g4": Shape("covarion", 40, 4, 4, False),
    "covarion40_g8": Shape("covarion", 40, 8, 8, False),
    "protein_g5": Shape("gamma", 20, 5, 1, False),
    "protein_g20": Shape("gamma", 20, 20, 1, False),
}

SLOW_CHAIN = 1          # covarion: this chain switches slowly (s01, s10 ~ 0.01), nearly repeated eigenvalues


class ShapeModels(MixedModels):
    """MixedModels whose chains carry models of `shape`: codon (own kappa, omegas and F3x4 skew per chain),
    covarion (own switching rates and gamma shape; chain SLOW_CHAIN switches slowly) or gamma"""

    def __init__(self, pr, shape, seed, rows=4):
        self.shape = shape
        self._ch = -1
        super().__init__(pr, seed, rows=rows, parts=shape.parts, inline=False, device_eigen=shape.device,
                         ambiguous_tips=0)

    def _eig(self, rng, freqs=None):
        sh = self.shape
        if sh.kind == "gamma":
            return super()._eig(rng, freqs)
        if sh.kind == "codon":
            kappa = float(rng.uniform(1.5, 6.0))
            omegas = np.sort(rng.uniform(0.02, 0.3, sh.parts)) * np.geomspace(1.0, 12.0, sh.parts)
            Qs, pi = codon_model(CODE_OF_STATES[sh.S], rng, kappa, omegas, float(rng.uniform(0.8, 1.0)))
            if freqs is not None:
                pi = np.asarray(freqs, float)
                Qs = np.stack([codon_q(CODE_OF_STATES[sh.S], kappa, w, pi) for w in omegas])
        else:
            assert freqs is None, "a covarion model's frequencies follow from its switching rates"
            slow = self._ch == SLOW_CHAIN
            s01, s10 = (0.01, 0.013) if slow else tuple(rng.uniform(0.1, 1.5, 2))
            Qs, pi = covarion_model(sh.S0, sh.K, rng, s01, s10, float(rng.uniform(0.2, 2.0)))
        return pi, [eig_of_reversible(Q, pi) for Q in Qs]

    def _model(self, rng, slot, ch):
        self._ch = ch if slot else -1
        m = super()._model(rng, slot, ch)
        if self.shape.parts > 1:             # the category's rate is in its Q: category_rates = the correction factor
            m = m.replace(rates=np.full(self.shape.K, 3.0 if self.shape.kind == "codon" else 1.0))
        return m


P_TIMES = (0.004, 0.11, 0.9, 3.7)
# P(t) from an eigensystem against expm: |dP| <= 2 ulp_f32(P) + P_EPS per entry.  The float rounding of the stored
# matrix is the ulp term; P_EPS covers the double-precision sum behind it, which numpy's eigh-based P(t) gets within
# ~1.3e-14 of expm on solver_cases() (test_model_shapes.py), and leaves room for the device's Jacobi tolerance.
P_EPS = 1e-12


def solver_cases():
    """name -> (Q [parts, S, S], pi): what the device-eigensolver tests diagonalise -- codon Q's at 60, 62 and 63
    sense codons with one and three omega values, covarion Q's (four gamma categories) at 8 and 40 states, with
    moderate and with slow switching (nearly repeated eigenvalues)"""
    out = {}
    for S in (60, 62, 63):
        for omegas in ([0.3], [0.05, 0.5, 3.0]):
            out[f"codon{S}_p{len(omegas)}"] = codon_model(CODE_OF_STATES[S], np.random.default_rng(S), 2.5, omegas, 1.0)
    for S0 in (4, 20):
        out[f"covarion{2 * S0}"] = covarion_model(S0, 4, np.random.default_rng(S0), 0.4, 0.9, 0.5)
        out[f"covarion{2 * S0}_slow"] = covarion_model(S0, 4, np.random.default_rng(S0 + 1), 0.01, 0.013, 0.5)
    return out


def shape_problem(shape, C, n_tips=10, n_chains=8, seed=0):
    """workloads.Problem of `shape` with shape_masks (replicated into both hidden blocks for covarion)"""
    pr = workloads.make_problem(shape.S, shape.K, C, n_tips, n_chains, seed=seed)
    masks = shape_masks(shape, n_tips, C, np.random.default_rng(seed + 1))
    pr.masks = covarion_masks(masks, shape.S0) if shape.kind == "covarion" else masks
    return pr
