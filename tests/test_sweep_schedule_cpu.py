"""
Static schedule of the fast PGS sweeps of the bench Kuka kernel (scripts/sweep_schedule.py, from `cuobjdump -sass` of the built library):
the copy of the loop that watches contacts must issue nearly as densely as the quiet copy.  It runs whenever any env of a warp has a
candidate contact, which in the bench workload is most physics steps, so a watch loop that ptxas schedules far worse than the quiet one
(1.89x the quiet loop's static cycles when every lane carried all four watched rows) is a regression of the headline rollout.
"""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("sweep_schedule", os.path.join(ROOT, "scripts", "sweep_schedule.py"))
sweep_schedule = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sweep_schedule)


def test_watch_sweep_issues_nearly_as_densely_as_the_quiet_sweep():
    if not os.path.exists(sweep_schedule.DEFAULT_LIB):
        pytest.skip("library not built")
    if sweep_schedule.find_cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    loops = {l["copy"]: l for l in sweep_schedule.schedule(sweep_schedule.DEFAULT_LIB)}
    assert set(loops) == {"quiet", "watch"}, loops
    quiet, watch = loops["quiet"], loops["watch"]
    assert quiet["ffma_sat"] == 12 and watch["ffma_sat"] == 12, loops
    assert watch["stall_cycles"] <= 1.3 * quiet["stall_cycles"], loops
