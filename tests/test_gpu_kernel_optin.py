"""GPU: two live instances whose shared kernel needs more dynamic shared memory in the one created first.  That limit
is one per process and device, so an instance created later must not lower it below what a live one launches with --
as two codon partitions under different omega models, or a codon partition next to a covarion protein partition, do
in one MrBayes process.  Each case keeps both instances open, creates the one that needs more first, then evaluates
each, first-created first, against the oracle."""
import pytest

from mrbayes_b200 import workloads
from engine_checks import check_with_oracle, lnl_tol, num_sms, parity_tol

pytestmark = pytest.mark.gpu

# (S, K, (a, b)) per instance, larger need first; the pattern count is a * SMs + b
CASES = {
    # eval_tcp_kernel<61>: two operand-ring stages at K = 1, one at K = 3
    "tcp_kernel_61": ((61, 1, (0, 130)), (61, 3, (0, 130))),
    # eval_gen_kernel<256>: 32 patterns per tile at C = 32 SMs + 1, 8 at C = 8 SMs + 1
    "gen_kernel_63": ((63, 3, (32, 1)), (63, 3, (8, 1))),
    # tiprobs_mm_kernel: two 61 x 64 double matrices, then two 40 x 40
    "tiprobs_mm_kernel": ((61, 1, (0, 130)), (40, 4, (0, 130))),
}


@pytest.mark.parametrize("case", list(CASES))
def test_later_instance_keeps_earlier_launches(engine_lib, oracle_lib, case):
    sms = num_sms()
    prs = [workloads.make_problem(S, K, a * sms + b, 5, 1, seed=300 + i)
           for i, (S, K, (a, b)) in enumerate(CASES[case])]
    with prs[0].create(engine_lib) as first, prs[1].create(engine_lib) as second:
        for pr, e in ((prs[0], first), (prs[1], second)):
            sp = pr.full_evaluation(0)
            lnl, st = e.evaluate(sp)
            with pr.create(oracle_lib) as o:
                o.set_arith(1)
                check_with_oracle(e, o, [sp], lnl, st, lnl_tol(pr.S), parity_tol(pr.S))
