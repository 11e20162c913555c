"""The 256-channel tower's planner (mz_debug_wide256_tower_plan, host only) and the built kernel's resources, without a GPU:
which boards it accepts and why it refuses the others, the games/atari.py budget it plans (boards stacked per CTA pair,
M-tiles, threads, shared memory, boards per wave), the SASS of conv_tower_wide256_kernel next to the unchanged 128-channel
wide kernels, the CUDA-core launch plans Atari's towers keep without MZ_TC_WIDE=3, and the CPU oracle against the
reference's traced Atari searches (oracle/gen_golden_atari_search.py)."""
import ctypes as C
import os
import re
import subprocess

import numpy
import pytest

from muzero_general_b200 import _lib
from muzero_general_b200 import build as b
from muzero_general_b200.engine import debug_small_tower_plan, debug_wide256_tower_plan
from test_wide_tower_plan_cpu import _cuobjdump

SMEM_LIMIT = 227 * 1024
REGFILE = 65536


def _budget(boards, H, W):
    """Per CTA: 8 planes (x_h, x_l of 4 K-quarters) of 1 + S + boards (H + 1) S rows rounded to 8, the 2 x 32 KB ring, the
    fp32 residual of 128 channels (+ 8) over the (boards (H + 1) - 1) S interior rows, 4 mbarriers."""
    S = W + 1
    interior = (boards * (H + 1) - 1) * S
    rows = (1 + S + boards * (H + 1) * S + 7) & ~7
    return -(-interior // 64), 8 * rows * 128 + 2 * 32768 + interior * 136 * 4 + 32


def _fits(boards, H, W):
    m, smem = _budget(boards, H, W)
    return m <= 2 and smem <= 232448


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("board", [(1, 1), (1, 9), (9, 1), (1, 40), (40, 1), (6, 6), (3, 5), (4, 7), (2, 3), (9, 9)])
@pytest.mark.parametrize("blocks,stem", [(16, True), (16, False), (0, True), (1, False), (5, True)])
def test_accepts_boards_up_to_the_largest(board, blocks, stem, sms):
    H, W = board
    want = max(k for k in range(1, 9) if _fits(k, H, W))
    m, smem = _budget(want, H, W)
    for n in (1, 128, 4096):
        plan, why = debug_wide256_tower_plan(n, 256, H, W, blocks, stem, sms)
        assert plan, why
        assert plan["boards"] == want and plan["m_tiles"] == m and plan["threads"] == 128 * m
        assert plan["smem"] == smem <= SMEM_LIMIT
        assert plan["threads"] * plan["reg_cap"] <= REGFILE
        assert plan["layers"] == int(stem) + 2 * blocks and plan["stages"] == 2
        assert plan["ctas_per_sm"] == 1 and plan["wave"] == sms // 2 * want
        assert plan["launches"] == 1                   # one CTA pair per group of boards: any batch is one launch
    for k in range(1, want + 1):                       # every smaller stack may be forced
        plan, why = debug_wide256_tower_plan(128, 256, H, W, blocks, stem, sms, boards=k)
        assert plan and plan["boards"] == k and plan["smem"] == _budget(k, H, W)[1], why


def test_atari_budget():
    """games/atari.py's 6 x 6 hidden board, S = 7: two boards per CTA pair, 1 + 7 + 2 x 49 = 106 -> 112 plane rows x 128 B
    x 8 planes + 2 x 32 KB ring + 91 x 136 fp32 residual rows + barriers = 229,760 B; 2 M-tiles, 256 threads; 66 pairs x
    2 boards per wave on 132 SMs.  The 33-layer dynamics tower fits the cap."""
    plan, _ = debug_wide256_tower_plan(128, 256, 6, 6, 16, True, 132)
    assert plan["smem"] == 8 * 112 * 128 + 2 * 32768 + 91 * 136 * 4 + 32 == 229760
    assert (plan["boards"], plan["m_tiles"], plan["threads"], plan["wave"], plan["layers"]) == (2, 2, 256, 132, 33)
    assert _budget(3, 6, 6)[0] == 3                    # three boards need a third M-tile
    assert debug_wide256_tower_plan(128, 256, 6, 6, 16, True, 114)[0]["wave"] == 114


@pytest.mark.parametrize("args,reason", [
    ((128, 128, 6, 6, 16, True, 0), "256 channels"),
    ((128, 64, 6, 6, 2, True, 0), "256 channels"),
    ((128, 256, 6, 6, 17, True, 0), "layers"),
    ((128, 256, 6, 6, 0, False, 0), "layers"),
    ((128, 256, 10, 10, 16, True, 0), "shared memory"),
    ((128, 256, 9, 10, 16, True, 0), "shared memory"),
    ((128, 256, 1, 200, 1, True, 0), "two M-tiles"),
    ((128, 256, 6, 6, 16, True, 3), "forced boards per CTA exceed the 128 rows of two M-tiles"),
    ((128, 256, 1, 1, 1, True, 9), "1 to 8"),
])
def test_refusals_name_the_reason(args, reason):
    for sms in (132, 114):
        plan, why = debug_wide256_tower_plan(*args[:6], sms, args[6])
        assert plan is None and reason in why, why


def _resources():
    out = subprocess.run([_cuobjdump(), "-res-usage", b.LIB], capture_output=True, text=True, check=True).stdout
    return {fn: tuple(map(int, v)) for fn, *v in
            re.findall(r"Function (\S*conv_tower_wide\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not found next to nvcc")
def test_kernel_resources_inside_the_plan():
    """conv_tower_wide256_kernel: no local memory (spills) or stack, registers at most the plan's cap."""
    assert os.path.exists(b.LIB), "build the library first (python -m muzero_general_b200.build)"
    res = _resources()
    found = [(fn, r) for fn, r in res.items() if "conv_tower_wide256_kernel" in fn]
    assert found, "conv_tower_wide256_kernel not in the library"
    plan, _ = debug_wide256_tower_plan(1, 256, 6, 6, 16, True, 132)
    for fn, (reg, stack, local) in found:
        assert local == 0 and stack == 0, fn
        assert reg <= plan["reg_cap"], (fn, reg)


def test_atari_keeps_its_cuda_core_plans():
    """Without MZ_TC_WIDE=3 Atari's towers run one conv3x3_kernel per conv (the fused tower refuses 33 and 32 layers), with
    the plans they had: P = 6, one band, 2 boards per CTA, 64 (65 for the stem) input channels staged at a time, 4
    cout tiles."""
    for cin, stem in ((257, True), (256, False)):
        plan, why = debug_small_tower_plan(128, cin, 256, 6, 6, 16, stem, 132)
        assert plan is None and "layers" in why
    lib = _lib.load_library()
    out = (C.c_int64 * 12)()
    for cin, chunk, smem in ((256, 64, 180224), (257, 65, 183040)):
        for n, grid in ((2, 1), (128, 64)):
            assert lib.mz_debug_conv3x3_plan(n, cin, 256, 6, 6, 1, out)
            assert list(out) == [6, 1, 1, 1, 6, 2, chunk, grid, 4, 1, smem, 64]


# ---------------------------------------------------------------------------------------------- reference fixtures
def atari_search_cases():
    """mcts_atari_n50.json (oracle/gen_golden_atari_search.py): traced reference searches of games/atari.py's net, each
    observation stored as its seed."""
    from conftest import golden_json
    from oracle.gen_golden_atari_search import observation
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config
    spec = netspec_from_config(load_game_module("atari").MuZeroConfig())
    cases = golden_json("mcts_atari_n50.json")
    for c in cases:
        c["obs"] = observation(spec, c["obs_seed"])
    return cases


def test_python_oracle_reproduces_the_atari_searches():
    from oracle import mcts as om
    from oracle.net import OracleNet
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    cfg = load_game_module("atari").MuZeroConfig()
    assert (cfg.blocks, cfg.channels) == (16, 256)
    spec = netspec_from_config(cfg)
    net = OracleNet(spec, synthetic_weights(spec, 0))
    cases = atari_search_cases()
    assert len(cases) == 3 and all(c["num_simulations"] == 50 and c["add_noise"] for c in cases)
    for case in cases:
        params = om.SearchParams.from_config(cfg, case["num_simulations"])
        res = om.TreeSearch(params).run(om.ModelEvaluator(net, spec.support_size), case["obs"], case["legal"], case["to_play"],
                                        case["add_noise"], om.LegacyNumpyDraws(numpy.random.RandomState(case["seed"])))
        assert res.root_actions == case["root_actions"] and res.root_visits == case["root_visits"]
        assert res.root_value == case["root_value"] and res.max_tree_depth == case["max_tree_depth"]
        assert [s.path_actions for s in res.sims] == [s["actions"] for s in case["sims"]]
