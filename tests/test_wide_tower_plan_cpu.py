"""The wide 128-channel tower's planner (mz_debug_wide_tower_plan, host only) and the built kernel's resources, without a GPU:
which boards it accepts and why it refuses the others, the budget it plans (shared memory, threads x registers), the
launch count, the SASS of the kernel (no spills, registers inside the plan's assumption), and the routes of Gomoku-shaped
nets that do not opt in (the fused CUDA-core tower and conv3x3 plans are what they were)."""
import os
import re
import shutil
import subprocess

import pytest

from muzero_general_b200 import build as b
from muzero_general_b200.engine import debug_wide_tower_plan

SMEM_LIMIT = 227 * 1024
REGFILE = 65536


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("board", [(11, 11), (1, 1), (1, 11), (11, 1), (5, 5), (8, 11), (6, 7), (10, 10)])
@pytest.mark.parametrize("blocks,stem", [(6, True), (6, False), (0, True), (1, False), (10, True)])
def test_accepts_gomoku_and_the_case_table_boards(board, blocks, stem, sms):
    H, W = board
    for n in (1, 128, 4096):
        plan, why = debug_wide_tower_plan(n, 128, H, W, blocks, stem, sms)
        assert plan, why
        m = -(-H * (W + 1) // 64)
        assert plan["m_tiles"] == m and plan["threads"] == 128 * m
        assert plan["smem"] <= SMEM_LIMIT
        assert plan["threads"] * plan["reg_cap"] <= REGFILE
        assert plan["layers"] == int(stem) + 2 * blocks and plan["stages"] == 2
        assert plan["wave"] == plan["ctas_per_sm"] * sms and plan["ctas_per_sm"] >= 1
        assert plan["launches"] == 1                   # one CTA per board: any batch is one launch


def test_gomoku_budget():
    """11 x 11: 160 plane rows x 128 B x 4 planes + 2 x 32 KB ring + 132 x 136 fp32 residual rows + barriers."""
    plan, _ = debug_wide_tower_plan(128, 128, 11, 11, 6, True, 132)
    assert plan["smem"] == 4 * 160 * 128 + 2 * 32768 + 132 * 136 * 4 + 32 == 219296
    assert (plan["m_tiles"], plan["threads"], plan["ctas_per_sm"], plan["wave"]) == (3, 384, 1, 132)


@pytest.mark.parametrize("args,reason", [
    ((128, 64, 11, 11, 6, True), "128 channels"),
    ((128, 256, 6, 6, 6, True), "128 channels"),
    ((128, 128, 15, 15, 6, True), "three M-tiles"),
    ((128, 128, 16, 16, 6, True), "three M-tiles"),
    ((128, 128, 12, 12, 6, True), "shared memory"),
    ((128, 128, 11, 12, 6, False), "shared memory"),
    ((128, 128, 11, 11, 11, True), "layers"),
    ((128, 128, 11, 11, 0, False), "layers"),
])
def test_refusals_name_the_reason(args, reason):
    for sms in (132, 114):
        plan, why = debug_wide_tower_plan(*args, sms)
        assert plan is None and reason in why, why


def _cuobjdump():
    exe = os.path.join(os.path.dirname(b.NVCC), "cuobjdump")
    return exe if os.path.exists(exe) else shutil.which("cuobjdump")


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not found next to nvcc")
def test_kernel_resources_inside_the_plan():
    """Every instantiation of the wide kernel in the built library: no local memory (spills) and at most the registers
    the plan assumes, so 3 warpgroups x 128 threads fit the register file."""
    assert os.path.exists(b.LIB), "build the library first (python -m muzero_general_b200.build)"
    out = subprocess.run([_cuobjdump(), "-res-usage", b.LIB], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*conv_tower_wide_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert found, "conv_tower_wide_kernel not in the library"
    plan, _ = debug_wide_tower_plan(1, 128, 11, 11, 6, True, 132)
    for fn, reg, stack, local in found:
        assert int(local) == 0 and int(stack) == 0, fn
        assert int(reg) <= plan["reg_cap"], (fn, reg)


def test_unset_routes_are_unchanged():
    """Without MZ_TC_WIDE the Gomoku towers keep their routes: the fused CUDA-core tower refuses 128 channels on 11 x 11
    (so conv3x3_kernel runs one launch per conv) with the plans the conv3x3 planner gives."""
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import debug_small_tower_plan
    import ctypes as C
    for stem, cin, blocks in ((True, 129, 6), (False, 128, 6), (True, 3, 6)):
        plan, why = debug_small_tower_plan(128, cin, 128, 11, 11, blocks, stem, 132)
        assert plan is None and why
    lib = _lib.load_library()
    out = (C.c_int64 * 12)()
    for cin in (3, 128, 129):
        assert lib.mz_debug_conv3x3_plan(128, cin, 128, 11, 11, 1, out)
        # P = 1, stride 1, 4 items, 3 bands of 4 rows, one board per CTA, grid (128 boards, 2 cout tiles, 3 bands)
        assert list(out)[:6] == [1, 1, 4, 3, 4, 1] and list(out)[7:10] == [128, 2, 3] and out[11] == 64
