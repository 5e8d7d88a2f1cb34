"""GPU: the engine's resources across calls that replace or refuse them -- the variable-state tables and matrix
buffer set a second time, an allocation the device refuses, and a packed batch freed while an evaluation that
writes its results there is pending.  The instance must keep computing what a fresh instance computes."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402
from mrbayes_b200 import abi, workloads  # noqa: E402
from engine_checks import rel  # noqa: E402
from std_problems import make_std_division, model_block, random_block  # noqa: E402

pytestmark = pytest.mark.gpu

ERROR_OUT_OF_MEMORY = -2
ERROR_OUT_OF_RANGE = -3


def std_instance(lib, pr, matrix_length):
    """pr's division on an instance whose branch matrix blocks are matrix_length floats"""
    inst = abi.Instance(lib, **pr.config())
    inst.set_pattern_states(pr.state_counts, pr.matrix_offsets, pr.freq_offsets, matrix_length, pr.dummy,
                            pr.uncompressed)
    for t in range(pr.n_tips):
        inst.set_tip_states(t, pr.masks[t])
    inst.set_pattern_weights(0, pr.weights)
    return inst


def supplied_full_evaluation(pr, insts):
    """chain 0's full evaluation with every branch's block supplied by the caller: the model's matrices in the
    first pr.matrix_length floats of each instance's block, 0.5 in the rest"""
    sp = pr.full_evaluation(0)
    node_of = pr.node_of_matrix(0)
    for m in sp.mats["matrix"]:
        blk = model_block(pr, pr.tree[0].length[node_of[int(m)]], pr.chain_rates[0])
        for inst, length in insts:
            padded = np.full(length, 0.5, np.float32)
            padded[:len(blk)] = blk
            inst.set_transition_matrix(int(m), padded)
    sp.mats = sp.mats[:0].copy()
    return sp


def test_std_tables_set_again_with_longer_matrices(engine_lib, oracle_lib):
    """set_pattern_states, matrices through the pinned ring, set_pattern_states again with a longer matrix block,
    matrices of the new length: the lnL of an instance created with the longer blocks, bit for bit"""
    pr = make_std_division(60, 2, 8, 1, seed=41, states=(2, 3, 4))
    L, L2 = pr.matrix_length, 3 * pr.matrix_length + 5
    rng = np.random.default_rng(2)
    with std_instance(engine_lib, pr, L) as e, std_instance(engine_lib, pr, L2) as fresh, \
         pr.create(oracle_lib) as o:
        for m in range(6):
            e.set_transition_matrix(m, random_block(pr, rng))
        e.set_pattern_states(pr.state_counts, pr.matrix_offsets, pr.freq_offsets, L2, pr.dummy, pr.uncompressed)
        sp = supplied_full_evaluation(pr, [(e, L2), (fresh, L2), (o, L)])
        (le,), (se,) = e.evaluate(sp)
        (lf,), (sf,) = fresh.evaluate(sp)
        (lo,), (so,) = o.evaluate(sp)
        assert se == sf == so == abi.EVAL_OK
        assert le == lf, f"tables set again {le!r}, fresh instance {lf!r}"
        assert rel(le, lo) < 1e-9, f"engine {le!r}, oracle {lo!r}"
        assert np.array_equal(e.get_transition_matrix(int(sp.ops["matrix1"][0])),
                              fresh.get_transition_matrix(int(sp.ops["matrix1"][0])))


def test_refused_matrix_buffer_keeps_the_tables(engine_lib):
    """a matrix block so long that the matrix buffer exceeds any device: set_pattern_states fails, and the instance
    evaluates as before with its old tables and matrices"""
    pr = make_std_division(60, 2, 40, 1, seed=43, states=(2, 3, 4))
    huge = 2**31 - 1
    assert pr.config()["matrix_count"] * huge * 4 > 2**40
    with pr.create(engine_lib) as e:
        sp = pr.full_evaluation(0)
        (l0,), (s0,) = e.evaluate(sp)
        assert s0 == abi.EVAL_OK
        with pytest.raises(abi.AbiError) as err:
            e.set_pattern_states(pr.state_counts, pr.matrix_offsets, pr.freq_offsets, huge, pr.dummy, pr.uncompressed)
        assert err.value.code == ERROR_OUT_OF_MEMORY
        (l1,), (s1,) = e.evaluate(sp)
        assert s1 == abi.EVAL_OK and l1 == l0, f"before {l0!r}, after the refused call {l1!r}"


@pytest.mark.parametrize("route", ["resident", "launch"])
def test_free_batch_refused_while_pending(engine_lib, route):
    """replay_begin, then free_batch on that batch: refused with MB200_ERROR_OUT_OF_RANGE; replay_end still gives
    the lnL mb200_evaluate gives, and afterwards the batch can be freed.  route 'resident': the instance is alone on
    the device; 'launch': a second live instance keeps the replay on launches."""
    other = workloads.make_problem(4, 4, 64, 8, 1, seed=3).create(engine_lib) if route == "launch" else None
    job = bench.Job("primates", 0, 1, engine_lib, 0, 4)
    try:
        inst, specs = job.insts[0], job.steps[0][0]
        batch = inst.pack(specs)
        inst.replay_begin(batch)
        with pytest.raises(abi.AbiError) as err:
            inst.free_batch(batch)
        assert err.value.code == ERROR_OUT_OF_RANGE
        lnl, st = inst.replay_end()
        assert not st.any()
        want, st = inst.evaluate(specs)
        assert not st.any()
        assert np.array_equal(lnl, want)
        inst.free_batch(batch)
        with pytest.raises(abi.AbiError):
            inst.free_batch(batch)                      # gone
    finally:
        job.close()
        if other is not None:
            other.close()
