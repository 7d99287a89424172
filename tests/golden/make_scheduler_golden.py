"""Golden records of the reference's own TwoPhaseScheduler (common/scheduling/two_phase_scheduler.py, imported
unmodified by oracle/ref_sched.py) in every scenario of tests/test_scheduler_vs_reference.py.

    python tests/golden/make_scheduler_golden.py          (needs the reference source tree, see oracle/ref_import.py)
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_sched  # noqa: E402
from test_scheduler_vs_reference import SCENARIOS, TIMEOUT_SCENARIOS, run_scenario, scenario_id  # noqa: E402


def main():
    Ref = ref_sched.load()
    rec = {"source": "reference two_phase_scheduler.py, imported unmodified",
           "scenarios": {scenario_id(kw): run_scenario(Ref, **kw) for kw in SCENARIOS},
           "timeouts": {scenario_id(kw): run_scenario(Ref, **kw) for kw in TIMEOUT_SCENARIOS}}
    with open(os.path.join(HERE, "scheduler_reference.json"), "w") as f:
        json.dump(rec, f)


if __name__ == "__main__":
    main()
