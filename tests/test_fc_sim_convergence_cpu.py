"""The fused CartPole search's simulation loop runs without divergent-collective code (common.cuh, LaneGroup::converge).

Where ptxas cannot prove the warp converged at a shuffle, ballot or __syncwarp it puts a run-time divergence test (BRA.DIV)
in front of it and an out-of-line WARPSYNC.COLLECTIVE ... ENDCOLLECTIVE fallback behind it.  The persistent loop over games
has a lane-dependent trip count as far as ptxas can tell, so before LaneGroup::converge every collective of every
simulation carried one.  This disassembles the built library's headline instantiation, fc_search_kernel<16, false,
CartPoleShape, 1>, and attributes each instruction to the root, the simulation loop or the write-out by its source line in
fc_search.cu (scripts/sass_sim_lines.py): the simulation loop must have no ENDCOLLECTIVE and no BRA.DIV, and its
WARPSYNC, BSSY and BRA counts must stay at or below what the change reached."""
import os
import sys

import pytest

from muzero_general_b200 import build as b

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import sass_sim_lines  # noqa: E402

# the simulation loop of the headline instantiation (CUDA 12.9, sm_90a); before: ENDC 53, WSYNC 54, BDIV 14, BSSY 82, BRA 156
LIMITS = {"ENDC": 0, "BDIV": 0, "WSYNC": 1, "BSSY": 63, "BRA": 125}


@pytest.mark.skipif(sass_sim_lines._tool("nvdisasm") is None or sass_sim_lines._tool("cuobjdump") is None,
                    reason="nvdisasm / cuobjdump not found next to nvcc")
def test_simulation_loop_has_no_divergent_collectives():
    assert os.path.exists(b.LIB), "build the library first (python -m muzero_general_b200.build)"
    fn, n, per_region, _ = sass_sim_lines.count(b.LIB)
    sim = per_region["sim"]
    assert sim["inst"] > 500, (fn, dict(sim))          # the attribution found the loop
    over = {k: (sim[k], lim) for k, lim in LIMITS.items() if sim[k] > lim}
    assert not over, (fn, over)
