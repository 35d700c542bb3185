"""tools/sched_sim.py, variant `pull` (ENC_PULL of enc_kernels.cu): pulled A / Bs batches must complete every macroblock, fill
batches beyond the warp count, and keep the other lists' batches at one task per warp."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


@pytest.mark.parametrize("pull", [1, 2, 3])
def test_pull_variant_completes(pull):
    import sched_sim
    r = sched_sim.simulate(n_streams=24, warps=23, n_cta=4, variant="pull", pull=pull)      # asserts completion internally
    assert r["kernel_ms"] > 0 and 0 < r["warp_busy_frac"] <= 1.0
    assert r["fill"][sched_sim.B] <= 23 and r["fill"][sched_sim.C] <= 23
    if pull > 1:
        assert r["fill"][sched_sim.A] > 23


def test_pull_one_is_the_base_policy():
    import sched_sim
    a = sched_sim.simulate(n_streams=6, warps=23, n_cta=8)
    b = sched_sim.simulate(n_streams=6, warps=23, n_cta=8, variant="pull", pull=1)
    assert a["kernel_ms"] == b["kernel_ms"] and a["fill"] == b["fill"]
