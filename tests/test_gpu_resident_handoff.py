"""The resident generation kernel hands data from one job to the next without a kernel boundary: a CTA of
generation g+1 may read what a different CTA wrote in generation g.  This cycle makes that happen on purpose
and compares it bit for bit with one launch per generation:

  - generation g updates one tip branch per chain, so the CTA of pattern tile 0 rebuilds that branch's P(t)
    and publishes it to the matrix buffer;
  - generation g+1 updates the sibling of that tip, so every tile reads the tip's P(t) as a clean branch
    from the matrix buffer, and lists the chains in reverse order, so evaluation row y reads the partials
    and scalers that row 7 - y wrote in generation g."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402

pytestmark = pytest.mark.gpu

GENERATIONS = 96


def _cycle(job):
    """-> [batch handle] of the alternating tip / sibling cycle on the job's primates instance"""
    inst, pr, nl = job.insts[0], job.parts[0], job.n_local
    rng = np.random.default_rng(20261015)
    batches = []
    for g in range(GENERATIONS // 2):
        tips, specs = [], []
        for ch in range(nl):
            tr = pr.tree[ch]
            tip = int(rng.integers(0, tr.n_tips))
            while tip == tr.root:
                tip = int(rng.integers(0, tr.n_tips))
            tips.append(tip)
            specs.append(pr.branch_update(ch, tip, float(tr.length[tip] * np.exp(0.5 * (rng.random() - 0.5)))))
        batches.append(inst.pack(specs))
        specs = []
        for ch in reversed(range(nl)):
            tr = pr.tree[ch]
            p = int(tr.anc[tips[ch]])
            sib = int(tr.right[p]) if int(tr.left[p]) == tips[ch] else int(tr.left[p])
            specs.append(pr.branch_update(ch, sib, float(tr.length[sib] * np.exp(0.5 * (rng.random() - 0.5)))))
        batches.append(inst.pack(specs))
    return batches


def _run(lib, mode):
    job = bench.Job("primates", 0, 1, lib, 0, 8)
    try:
        inst = job.insts[0]
        batches = _cycle(job)
        n0 = inst.launch_count()
        lnls = []
        for b in batches:
            if mode == "resident":
                lnl = np.zeros(8, np.float64)
                st = np.zeros(8, np.int32)
                assert lib.fn("replay_begin")(inst.handle, b) == 0
                assert lib.fn("replay_end")(inst.handle, lnl.ctypes.data_as(C.POINTER(C.c_double)),
                                            st.ctypes.data_as(C.POINTER(C.c_int))) == 0
            else:
                inst.replay(b)
                lnl, st = inst.replay_results(b, 8)
            assert not st.any()
            lnls.append(lnl)
        launches = inst.launch_count() - n0
        inst.synchronize()
        pr, nl = job.parts[0], job.n_local                # every interior buffer and scaler of every chain
        parts = [inst.get_partials(b) for b in range(pr.n_tips, pr.n_tips + 2 * nl * pr.n_int)]
        scalers = [inst.get_scalers(s) for s in range(2 * nl * (pr.n_int + 1))]
        return np.array(lnls), parts, scalers, launches
    finally:
        job.close()


def test_resident_handoff_between_ctas_equals_launch_path(engine_lib):
    lnl, parts, scal, launches = _run(engine_lib, "resident")
    want_lnl, want_parts, want_scal, want_launches = _run(engine_lib, "launch")
    assert want_launches == GENERATIONS
    assert launches <= GENERATIONS // 8                # the resident kernel served the cycle
    assert np.isfinite(lnl).all()
    assert np.array_equal(lnl, want_lnl)
    assert all(np.array_equal(a, b) for a, b in zip(parts, want_parts))
    assert all(np.array_equal(a, b) for a, b in zip(scal, want_scal))
