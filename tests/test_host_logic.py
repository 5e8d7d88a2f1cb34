"""CPU: host-side logic -- ABI surface, workload generator's index protocol, pattern
compression (integer, bit-exact), and loud failure without a GPU."""
import ctypes
import re

import numpy as np
import pytest

from conftest import ROOT
from mrbayes_b200 import abi, workloads


def declared_symbols():
    text = (ROOT / "include" / "mb200.h").read_text()
    return sorted(set(re.findall(r"\b(mb200_[a-z_0-9]+)\s*\(", text)))


def test_engine_library_exports_every_declared_symbol():
    lib = abi.engine_library()
    syms = declared_symbols()
    assert len(syms) >= 29
    for s in syms:
        assert hasattr(lib.lib, s), f"libmb200.so does not export {s}"
    assert lib.fn("abi_version")() == 1


def test_struct_sizes_match_the_header():
    assert ctypes.sizeof(abi.Operation) == 36
    assert ctypes.sizeof(abi.MatrixUpdate) == 16
    assert ctypes.sizeof(abi.InstanceConfig) == 48
    # int, ptr, int, ptr, 5 ints, double, int, 20+20+64 doubles (natural alignment)
    assert ctypes.sizeof(abi.Evaluation) == 8 + 8 + 8 + 8 + 24 + 8 + 8 + 8 * (20 + 20 + 64) + 8


def test_no_cpu_fallback_without_device():
    """Without an H100 the engine must refuse, not compute somewhere else."""
    lib = abi.engine_library()
    if lib.fn("device_count")() > 0:
        pytest.skip("a device is present; covered by the gpu tests")
    with pytest.raises(abi.AbiError) as e:
        abi.Instance(lib, tip_count=4, partials_count=10, state_count=4, pattern_count=8, category_count=1,
                     matrix_count=12, scaler_count=6, eigen_count=1)
    assert e.value.code == abi.ERROR_NO_DEVICE


def test_pattern_compression_first_occurrence(oracle_lib):
    rng = np.random.default_rng(3)
    n_taxa, n_sites = 7, 400
    base = rng.integers(0, 3, size=(n_taxa, 40)).astype(np.uint64)
    cols = rng.integers(0, 40, size=n_sites)
    mat = np.ascontiguousarray((np.uint64(1) << base[:, cols]))
    pos = np.zeros(n_sites, np.int32); first = np.zeros(n_sites, np.int32); w = np.zeros(n_sites, np.int32)
    P = ctypes.POINTER
    n = oracle_lib.fn("compress_patterns")(mat.ctypes.data_as(P(ctypes.c_uint64)), n_taxa, n_sites,
                                            pos.ctypes.data_as(P(ctypes.c_int)), first.ctypes.data_as(P(ctypes.c_int)),
                                            w.ctypes.data_as(P(ctypes.c_int)))
    # python restatement: first-occurrence order, integer counts
    seen = {}
    for s in range(n_sites):
        seen.setdefault(mat[:, s].tobytes(), len(seen))
    assert n == len(seen)
    assert w[:n].sum() == n_sites
    assert [seen[mat[:, s].tobytes()] for s in range(n_sites)] == list(pos)
    assert all(pos[first[p]] == p for p in range(n))
    assert list(first[:n]) == sorted(first[:n])


@pytest.mark.parametrize("S,K,C,tips", [(4, 4, 97, 9), (20, 2, 33, 6), (61, 1, 17, 5)])
def test_incremental_updates_equal_full_recomputation(oracle_lib, S, K, C, tips):
    """The index protocol of the workload generator (flip / copy / remove / reject) is the
    reference's: after a series of partial updates and rejections the incrementally maintained
    lnL equals a from-scratch evaluation of the same state."""
    pr = workloads.make_problem(S, K, C, tips, 2, seed=11, p_invar=0.15 if S == 4 else 0.0)
    rng = np.random.default_rng(2)
    with pr.create(oracle_lib) as inst:
        inst.evaluate([pr.full_evaluation(ch) for ch in range(2)])
        last = {}
        for it in range(12):
            ch = it % 2
            old = pr.tree[ch].length.copy()
            sp = pr.random_branch_update(ch, rng)
            lnl, st = inst.evaluate(sp)
            assert st[0] == abi.EVAL_OK
            if it % 4 == 3:
                pr.reject(ch, sp, old)
            else:
                last[ch] = lnl[0]
        pr2 = workloads.make_problem(S, K, C, tips, 2, seed=11, p_invar=0.15 if S == 4 else 0.0)
        for ch in range(2):
            pr2.tree[ch].length[:] = pr.tree[ch].length
        with pr2.create(oracle_lib) as inst2:
            fresh, _ = inst2.evaluate([pr2.full_evaluation(ch) for ch in range(2)])
        # incremental float site scalers vs fresh sums: rounding-level agreement only
        for ch in range(2):
            if ch in last:
                cur, _ = inst.evaluate(pr.full_evaluation(ch))
                assert cur[0] == pytest.approx(fresh[ch], rel=1e-12)


def test_discrete_gamma_rates_have_unit_mean():
    for alpha in (0.1, 0.5, 2.0):
        r = workloads.discrete_gamma_rates(alpha, 4)
        assert r.mean() == pytest.approx(1.0, abs=1e-9)
        assert np.all(np.diff(r) > 0)


def test_reversible_model_eigensystem():
    rng = np.random.default_rng(0)
    pi, V, Vinv, lam = workloads.reversible_model(20, rng)
    assert np.allclose(V @ Vinv, np.eye(20), atol=1e-10)
    Q = V @ np.diag(lam) @ Vinv
    assert np.allclose(Q.sum(1), 0, atol=1e-10)
    assert -(pi * np.diag(Q)).sum() == pytest.approx(1.0)
    assert np.allclose(pi[:, None] * Q, (pi[:, None] * Q).T, atol=1e-12)
