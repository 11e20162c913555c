"""The lane-group kernels take the full warp mask on every collective (common.cuh, LaneGroup).

A mask that depends on the lane makes nvcc wrap each collective region in a run-time convergence check - MATCH.ANY and
REDUX.OR of the mask, then a divergent-branch fallback - which sits on the per-simulation critical path of the fused
search.  With the full mask there is nothing to check.  This reads the built library's SASS and asserts that no
instantiation of the tree-search and FC kernels with groups narrower than a warp carries such a check."""
import os
import re
import shutil
import subprocess

import pytest

from muzero_general_b200 import build as b

KERNELS = ("fc_search_kernel", "tree_step_kernel", "tree_adopt_root_kernel", "fc_inference_kernel")
GUARDS = ("MATCH.ANY", "REDUX.OR")


def _cuobjdump():
    exe = os.path.join(os.path.dirname(b.NVCC), "cuobjdump")
    return exe if os.path.exists(exe) else shutil.which("cuobjdump")


def _guards_per_function(lib):
    sass = subprocess.run([_cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    counts, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            counts[fn] = 0
        elif fn and any(g in line for g in GUARDS):
            counts[fn] += 1
    return counts


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not found next to nvcc")
def test_narrow_group_kernels_have_no_convergence_guards():
    assert os.path.exists(b.LIB), "build the library first (python -m muzero_general_b200.build)"
    counts = _guards_per_function(b.LIB)
    narrow = {}
    for fn, n in counts.items():
        m = re.search(r"(" + "|".join(KERNELS) + r")ILi(\d+)E", fn)
        if m and int(m.group(2)) < 32:
            narrow[fn] = n
    # every group width the launchers instantiate: 4, 8 and 16 lanes (the headline CartPole search runs at 16)
    kinds = {(re.search("|".join(KERNELS), fn).group(0), re.search(r"ILi(\d+)E", fn).group(1)) for fn in narrow}
    assert {(k, g) for k in KERNELS for g in ("4", "8", "16")} <= kinds, sorted(kinds)
    guarded = {fn: n for fn, n in narrow.items() if n}
    assert not guarded, guarded
