"""Per-chain models for chain-batched evaluations.

After the first model move of an MC^3 run every chain sits at its own point of the model space, and the
seam's chain-batched generation sends all chains in one call: each evaluation carries its own eigen slot
(or an inline 4-state eigensystem), state frequencies, rates, category weights, p_invar, flags and weights
row.  MixedModels gives every chain of a workloads.Problem (or StdProblem) such a model of its own and
rewrites the EvalSpecs the problem builds; workloads.py itself stays as bench.py uses it.

Eigen slot 0 and weights row 0 hold decoys that no evaluation uses, so a kernel that reads slot or row 0
instead of the evaluation's own gets a different likelihood.  Chain ch uses slot ch + 1.  Within one call,
category weights are equal in some evaluations and Dirichlet in others, p_invar is off in some, the 4-state
flags alternate, and (4 states) half the chains send their eigensystem inline."""
import copy

import numpy as np

from f64_reference import f64_lnl
from mrbayes_b200 import abi, workloads

ROWS = 4                 # weights rows: 0 is the decoy, chains use 1 .. ROWS - 1
FLAG_CYCLE = [0, abi.FLAG_NUC4_PINVAR_QUIRK, abi.FLAG_TIP_SHORTCUTS, abi.FLAG_NUC4_PINVAR_QUIRK | abi.FLAG_TIP_SHORTCUTS]


def cijk_of(V, Vinv, lam):
    """cijk block [lambda_re, lambda_im, c_ijk = V[i][k] Vinv[k][j]] of one eigensystem"""
    S = len(lam)
    return np.concatenate([lam, np.zeros(S), np.einsum("ik,kj->ijk", V, Vinv).ravel()])


class ChainModel:
    """One chain's model.  eig: [(V, Vinv, lambda)] per eigen part (None for Std); rates and cat_weights are
    what the evaluation sends, used as given."""

    def __init__(self, slot, eig, freqs, rates, cat_weights, p_invar, flags, row, inline):
        self.slot, self.eig, self.freqs, self.rates = slot, eig, np.asarray(freqs, float), np.asarray(rates, float)
        self.cat_weights, self.p_invar, self.flags, self.row, self.inline = np.asarray(cat_weights, float), p_invar, flags, row, inline

    @property
    def Q(self):
        return np.array([(V * lam) @ Vi for V, Vi, lam in self.eig])

    def block(self):
        return np.concatenate([cijk_of(*e) for e in self.eig])

    def replace(self, **kw):
        m = copy.copy(self)
        for k, v in kw.items():
            setattr(m, k, v)
        return m

    def with_p_invar(self, p):
        """the same rates, the category weights rescaled to 1 - p"""
        w = self.cat_weights / self.cat_weights.sum()
        return self.replace(p_invar=p, cat_weights=(1.0 - p) * w)


class MixedModels:
    def __init__(self, pr, seed, rows=ROWS, parts=1, inline=None, device_eigen=False, ambiguous_tips=3):
        """pr: a freshly made Problem / StdProblem; parts: eigen parts per slot (MB200_CONFIG_CIJK_PARTS);
        inline: half the chains carry their eigensystem inline (default: 4 states); device_eigen: the engine
        solves the slots itself (mb200_set_rate_matrices), the oracle gets the host eigensystem of the same Q."""
        self.pr, self.rows, self.parts, self.device_eigen = pr, rows, parts, device_eigen
        self.std = isinstance(pr, workloads.StdProblem)
        self.inline = (pr.S == 4) if inline is None else inline
        rng = np.random.default_rng(seed)
        C = pr.C
        if not self.std and ambiguous_tips:
            # partial ambiguity on a few tips only: the others keep the terminal-branch shortcut
            for t in range(ambiguous_tips):
                amb = rng.random(C) < 0.2
                extra = np.uint64(1) << rng.integers(0, pr.S, size=C).astype(np.uint64)
                pr.masks[t] = np.where(amb, pr.masks[t] | extra, pr.masks[t])
        # row r: the problem's weights times r, some patterns zeroed and some doubled (lnL roughly scales with
        # the row, which keeps the chains' likelihoods apart); the decoy row: other weights, larger again
        W = np.zeros((rows, C), np.float32)
        W[0] = rng.integers(2 * rows, 4 * rows, size=C)
        for r in range(1, rows):
            w = r * np.asarray(pr.weights, np.float32)
            u = rng.random(C)
            w[u < 0.15] = 0.0
            w[u > 0.8] *= 2.0
            W[r] = w
        if self.std:
            W[:, :pr.dummy] = 0.0
        self.weights = W
        self.decoy = self._model(rng, 0, 0)
        self.models = [self._model(rng, ch + 1, ch) for ch in range(pr.n_chains)]

    def _eig(self, rng, freqs=None):
        S = self.pr.S
        pi, V, Vi, lam = workloads.reversible_model(S, rng, freqs=freqs)
        eig = [(V, Vi, lam)]
        for p in range(1, self.parts):              # omega-category-like: same frequencies, other exchangeabilities
            _, V, Vi, lam = workloads.reversible_model(S, rng, freqs=pi)
            eig.append((V, Vi, lam * (0.4 + 0.8 * p)))
        return pi, eig

    def _model(self, rng, slot, ch):
        pr, K = self.pr, self.pr.K
        pinv = 0.0 if (ch % 3 == 0 or self.std) else float(rng.uniform(0.05, 0.3))
        # overall rate multipliers in [0.5, 2], one stratum per chain: models far apart in the rate
        mult = 0.5 * 4.0 ** ((ch + rng.uniform(0.25, 0.75)) / self.pr.n_chains if slot else rng.random())
        base = workloads.discrete_gamma_rates(float(rng.uniform(0.2, 2.0)), K) * mult
        w = np.full(K, 1.0 / K) if ch % 2 == 0 else rng.dirichlet(np.full(K, 2.0))
        if self.std:
            pi, eig = pr.freqs, None
        else:
            pi, eig = self._eig(rng)
        row = 1 + ch % (self.rows - 1) if slot else 0
        return ChainModel(slot, eig, pi, base / (1.0 - pinv), (1.0 - pinv) * w, pinv, FLAG_CYCLE[ch % 4], row,
                          bool(self.inline and slot and ch % 4 in (1, 2)))

    def new_eigensystem(self, ch, seed):
        """chain ch's model with another Q (same frequencies): what a rate-matrix move leaves"""
        _, eig = self._eig(np.random.default_rng(seed), self.models[ch].freqs)
        return self.models[ch].replace(eig=eig)

    # ---- instances ---------------------------------------------------------------------------
    def config(self, max_evaluations=None):
        c = self.pr.config(max_evaluations)
        c["eigen_count"] = self.pr.n_chains + 1
        c["weight_rows"] = self.rows
        if self.parts > 1:
            c["flags"] = c.get("flags", 0) | (self.parts << 8)
        return c

    def create(self, lib, max_evaluations=None, flags=0) -> abi.Instance:
        pr = self.pr
        cfg = self.config(max_evaluations)
        cfg["flags"] = cfg.get("flags", 0) | flags
        inst = abi.Instance(lib, **cfg)
        if self.std:
            inst.set_pattern_states(pr.state_counts, pr.matrix_offsets, pr.freq_offsets, pr.matrix_length,
                                    pr.dummy, pr.uncompressed)
        for t in range(pr.n_tips):
            inst.set_tip_states(t, pr.masks[t])
        for r in range(self.rows):
            inst.set_pattern_weights(r, self.weights[r])
        if not self.std:
            for m in [self.decoy] + self.models:
                self.load(inst, m.slot, m)
        return inst

    def load(self, inst, slot, m):
        """m's eigensystem into eigen slot `slot`"""
        if self.device_eigen and inst.lib.prefix == "mb200_":
            inst.set_rate_matrices(slot, m.Q, m.freqs)
        elif self.parts > 1:
            inst.set_cijk(slot, m.block())
        else:
            inst.set_eigen_decomposition(slot, *m.eig[0])

    def set_weights(self, insts, row, w):
        self.weights[row] = w
        for inst in insts:
            inst.set_pattern_weights(row, self.weights[row])

    # ---- evaluations ---------------------------------------------------------------------------
    def apply(self, sp, m=None) -> abi.EvalSpec:
        """sp with the model of its chain (or m): slot or inline eigensystem, and every per-evaluation value"""
        m = self.models[sp.chain] if m is None else m
        if len(sp.mats) and not self.std:
            sp.mats = sp.mats.copy()
            sp.mats["eigen"] = abi.EIGEN_INLINE if m.inline else m.slot
        sp.inline_eigen = m.block() if m.inline else None
        sp.rates, sp.cat_weights, sp.freqs = m.rates.copy(), m.cat_weights.copy(), m.freqs.copy()
        sp.p_invar, sp.has_p_invar = m.p_invar, int(m.p_invar > 0)
        sp.flags, sp.weights_row = m.flags, m.row
        return sp

    def full(self, ch):
        return self.apply(self.pr.full_evaluation(ch))

    def update(self, ch, rng):
        return self.apply(self.pr.random_branch_update(ch, rng))

    def root_only(self, ch):
        """root integration of the chain's current buffers: no matrix update, no operation"""
        st, tr = self.pr.chains[ch], self.pr.tree[ch]
        return self.apply(abi.EvalSpec(site_dst=abi.NONE, site_src=st.site, root=int(st.cl[tr.root_left]), chain=ch))

    def no_matrix_update(self, ch, rng):
        """the path from a tip to the root recomputed with every P(t) clean: operations, no matrix update"""
        tr = self.pr.tree[ch]
        tip = int(rng.integers(0, tr.n_tips - 1))
        tip = tip if tip != tr.root else tr.n_tips - 2
        return self.apply(self.pr._spec(ch, [], set(tr.path_to_root(tip)), False))

    def f64(self, ch, m=None):
        """float64 lnL of chain ch on its current tree under m (default its own model)"""
        m = self.models[ch] if m is None else m
        return f64_lnl(self.pr, ch, Q=m.Q, freqs=m.freqs, rates=m.rates, cat_weights=m.cat_weights,
                       p_invar=m.p_invar, weights=self.weights[m.row])[1]

    def detached_full(self, ch):
        """a full evaluation of chain ch that leaves the chain's index tables as they were"""
        snap = workloads.snapshot(self.pr)
        sp = self.pr.full_evaluation(ch)
        self.pr.chains[ch] = snap[0][ch]
        return sp

    def assert_models_differ(self, scratch, chains, rtol=1e-4):
        """Sensitivity: on a scratch oracle instance made by create(), chain ch's lnL under its own model
        differs by more than rtol (relative) from its lnL under every other chain's model and the decoy, so
        that an evaluation handed another evaluation's model, slot or row cannot pass within tolerance."""
        for ch in chains:
            sp = self.detached_full(ch)
            (own,), (st,) = scratch.evaluate(self.apply(copy.copy(sp), self.models[ch]))
            assert st == abi.EVAL_OK
            for other in [self.decoy] + self.models:
                if other is self.models[ch]:
                    continue
                (l,), _ = scratch.evaluate(self.apply(copy.copy(sp), other))
                assert abs(l - own) > rtol * abs(own), f"chain {ch}: slot {other.slot}'s model gives the same lnL"
