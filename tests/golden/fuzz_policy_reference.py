#!/usr/bin/env python
"""Differential fuzz of oracle/policy_oracle.c against the reference's own loop code (build container only).

    python tests/golden/fuzz_policy_reference.py [n_cases] [first_seed]

Every case is policy_case(seed) of tests/test_policy_fuzz_cpu.py -- the generator of the GPU fuzz: 1 .. 64 GPUs
per node, up to 140 nodes, slot-bound nodes, leaks, jobs wider than the cluster, bursts of arrivals, whole-tick and
sub-tick durations, 1 .. 8 dlas queues with limits up to 2^31 + 6 * 10^9, gittins quanta -- at its full range of up to
600 jobs (the reference runs such a case in well under a second, so no cap is needed) and with the gittins table the
reference itself derives from the trace.  It executes the reference's smallest_first_sim_jobs / dlas_sim_jobs / gittins_sim_jobs VERBATIM through make_policy_golden.py's stub
harness and compares every completion and every checkpoint with the C restatement.  A reference run
that raises (its own list.remove / assertion failures on inputs outside its domain) is reported as
"reference raised" and skipped.  Needs /root/reference, so it is NOT part of the suite; its last run is
recorded in DESIGN.md section 5.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, HERE)

import make_policy_golden as mpg  # noqa: E402
from gpuschedule_b200 import capi, policies  # noqa: E402
import oracle  # noqa: E402
from test_policy_fuzz_cpu import policy_case  # noqa: E402
from test_policy_golden import check_against_expected  # noqa: E402


def run_case(seed):
    """policy_case(seed) of tests/test_policy_fuzz_cpu.py (the cases the GPU fuzz runs), its gittins table rebuilt
    from the trace: the reference derives that table from the trace itself (parse_job_dist)"""
    case = policy_case(seed)
    table = case.table
    try:
        comp, chk, gtab, unfinished = mpg.run_reference_policy(table, case.ckw, case.name, **case.pkw)
    except Exception as e:                                           # noqa: BLE001 - the reference's own failures
        return case, f"reference raised {type(e).__name__}: {e}"
    kw = dict(case.pkw)
    if case.name == "gittins":
        kw["gittins_table"] = policies.build_gittins_table(policies.gittins_samples(table), kw.get("gittins_delta", 3250.0))
    res = oracle.run_policy(capi.make_cluster(**case.ckw), capi.make_policy(case.name, **kw), table)
    check_against_expected(table, res, {"completions": comp, "checkpoints": chk, "unfinished": unfinished})
    return case, None


def main():
    n_cases = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    first = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    ok = raised = 0
    for seed in range(first, first + n_cases):
        try:
            case, msg = run_case(seed)
        except AssertionError:
            case = policy_case(seed)
            print(f"MISMATCH seed {seed}: {case.name} {case.ckw} {case.pkw} n={case.table.n}")
            raise
        if msg:
            raised += 1
            print(f"seed {seed} ({case.name} {case.ckw} {case.pkw}): {msg}")
        else:
            ok += 1
    print(f"{ok} cases identical, {raised} outside the reference's domain (it raised)")


if __name__ == "__main__":
    main()
