"""The resident generation kernel of mb200_replay_begin / _end: one kernel serves many generations
through a mailbox in mapped host memory, and must compute exactly what one launch per generation
computes.  Every comparison is bitwise."""
from __future__ import annotations

import sys
import time
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402
from engine_checks import written_buffers  # noqa: E402
from mrbayes_b200 import workloads  # noqa: E402

pytestmark = pytest.mark.gpu

CYCLE = 32


def _state(job):
    """Every partials buffer and scaler the cycle writes."""
    inst = job.insts[0]
    dests, scalers = written_buffers(job.steps[0])
    return [inst.get_partials(b) for b in dests], [inst.get_scalers(s) for s in scalers]


def _run(lib, mode, generations, pause_at=(), between=None):
    """Bench-shaped cycle (rejections included) on a fresh primates instance, the only one on the device.
    mode 'resident': replay_begin / _end; mode 'launch': mb200_replay + replay_results."""
    job = bench.Job("primates", 0, 1, lib, 0, CYCLE)
    try:
        inst = job.insts[0]
        batches = [inst.pack(job.steps[0][i]) for i in range(CYCLE)]
        n0 = inst.launch_count()
        lnls = []
        for g in range(generations):
            if g in pause_at:
                time.sleep(0.02)                       # far longer than the kernel's idle timeout
            if between is not None:
                between(g, inst)
            b = batches[g % CYCLE]
            if mode == "resident":
                inst.replay_begin(b)
                lnl, st = inst.replay_end()
            else:
                inst.replay(b)
                lnl, st = inst.replay_results(b, 8)
            assert not st.any()
            lnls.append(lnl)
        launches = inst.launch_count() - n0
        inst.synchronize()
        parts, scal = _state(job)
        return np.array(lnls), parts, scal, launches
    finally:
        job.close()


@pytest.fixture(scope="module")
def launched(engine_lib):
    return _run(engine_lib, "launch", 2 * CYCLE)


def test_resident_equals_launch_path(engine_lib, launched):
    lnl, parts, scal, launches = _run(engine_lib, "resident", 2 * CYCLE)
    assert np.array_equal(lnl, launched[0])
    assert all(np.array_equal(a, b) for a, b in zip(parts, launched[1]))
    assert all(np.array_equal(a, b) for a, b in zip(scal, launched[2]))
    # one kernel serves the generations (a host hiccup past the idle timeout may cost a relaunch)
    assert 1 <= launches <= CYCLE // 4


def test_resident_survives_pauses_longer_than_idle_timeout(engine_lib, launched):
    lnl, parts, scal, launches = _run(engine_lib, "resident", 2 * CYCLE, pause_at=(5, 6, 40))
    assert np.array_equal(lnl, launched[0])
    assert all(np.array_equal(a, b) for a, b in zip(parts, launched[1]))
    assert launches >= 4                              # the kernel exited during each pause and was relaunched


def test_other_calls_between_generations(engine_lib, launched):
    import torch

    def between(g, inst):
        if g % 7 == 3:
            inst.get_scalers(0)                       # stops the resident kernel first
        if g % 11 == 5:
            inst.synchronize()
            assert torch.cuda.ExternalStream(inst.stream()).query()     # nothing left running on the stream

    lnl, parts, scal, _ = _run(engine_lib, "resident", 2 * CYCLE, between=between)
    assert np.array_equal(lnl, launched[0])
    assert all(np.array_equal(a, b) for a, b in zip(parts, launched[1]))
    assert all(np.array_equal(a, b) for a, b in zip(scal, launched[2]))


def test_replay_between_begin_and_end(engine_lib, launched):
    """A synchronous mb200_replay (results to device memory) while a replay_begin is pending must not change
    how replay_end collects the pending results: the tile partials are still summed on the host."""
    job = bench.Job("primates", 0, 1, engine_lib, 0, CYCLE)
    try:
        inst = job.insts[0]
        batches = [inst.pack(job.steps[0][i]) for i in range(CYCLE)]
        lnls = []
        for g in range(CYCLE):
            b = batches[g]
            inst.replay_begin(b)
            if g % 4 == 1:
                inst.replay(b)                        # the same evaluation again: same inputs, same outputs
            lnl, st = inst.replay_end()
            assert not st.any()
            lnls.append(lnl)
    finally:
        job.close()
    assert np.array_equal(np.array(lnls), launched[0][:CYCLE])


def test_second_instance_falls_back_to_launches(engine_lib, launched):
    other = workloads.make_problem(4, 4, 64, 8, 1, seed=3)
    with other.create(engine_lib):
        lnl, parts, _, launches = _run(engine_lib, "resident", CYCLE)
    assert launches == CYCLE                          # one launch per generation
    assert np.array_equal(lnl, launched[0][:CYCLE])
