"""The CTA-pair 128-channel tower's planner (mz_debug_wide_pair_tower_plan, host only), the built pair kernel's resources and
the reference fixtures of Gomoku's 6 x 128 net on 15 x 15 and 16 x 16 boards (oracle/gen_golden_gomoku_pair.py), without a
GPU: which boards the pair accepts and why it refuses the others, the per-CTA budget it plans, the SASS of
conv_tower_wide_pair_kernel, and the CPU oracle against the reference's outputs."""
import os
import re
import subprocess

import numpy
import pytest
import torch

from conftest import golden_json, golden_npz
from muzero_general_b200 import build as b
from muzero_general_b200.engine import debug_wide_pair_tower_plan, debug_wide_tower_plan
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
from test_wide_tower_plan_cpu import _cuobjdump

torch.set_num_threads(1)

SMEM_LIMIT = 227 * 1024
REGFILE = 65536
ONE_CTA_BOARDS = ((11, 11), (11, 1), (5, 5), (8, 11), (6, 7), (10, 10), (2, 3))


def _budget(H, W):
    """The one-CTA budget formula applied to one half: ceil(H / 2) board rows plus a halo row above and below."""
    h, S = -(-H // 2), W + 1
    rows = ((h + 2) * S + 1 + 7) & ~7
    return h, -(-h * S // 64), 4 * rows * 128 + 2 * 32768 + h * S * 136 * 4 + 32


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("board", [(12, 12), (13, 13), (14, 14), (15, 15), (16, 16), (12, 16), (16, 12), (2, 16)]
                         + list(ONE_CTA_BOARDS))
@pytest.mark.parametrize("blocks,stem", [(6, True), (6, False), (0, True), (1, False), (10, True)])
def test_accepts_large_boards_rectangles_and_the_one_cta_boards(board, blocks, stem, sms):
    H, W = board
    h, m, smem = _budget(H, W)
    for n in (1, 128, 4096):
        plan, why = debug_wide_pair_tower_plan(n, 128, H, W, blocks, stem, sms)
        assert plan, why
        assert plan["rows0"] == h and plan["m_tiles"] == m and plan["threads"] == 128 * m
        assert plan["smem"] == smem <= SMEM_LIMIT
        assert plan["threads"] * plan["reg_cap"] <= REGFILE
        assert plan["layers"] == int(stem) + 2 * blocks and plan["stages"] == 2
        assert plan["wave"] >= sms // 2 and plan["wave"] % (sms // 2) == 0
        assert plan["launches"] == 1                   # one CTA pair per board: any batch is one launch


@pytest.mark.parametrize("board", [(12, 12), (13, 13), (14, 14), (15, 15), (16, 16), (12, 16), (16, 12)])
def test_large_boards_are_what_one_cta_refuses(board):
    plan, why = debug_wide_tower_plan(128, 128, *board, 6, True, 132)
    assert plan is None and "board too large" in why


def test_gomoku15_and_16_budgets():
    """15 x 15: 8 + 7 rows, S = 16: 168 plane rows x 128 B x 4 planes + 2 x 32 KB ring + 8 x 16 x 136 fp32 residual rows +
    barriers, 2 M-tiles.  16 x 16: 8 + 8 rows, S = 17: 176 plane rows, 8 x 17 residual rows, 3 M-tiles.  One CTA per SM:
    half the SMs' worth of boards per wave."""
    p15, _ = debug_wide_pair_tower_plan(128, 128, 15, 15, 6, True, 132)
    assert p15["smem"] == 4 * 168 * 128 + 2 * 32768 + 8 * 16 * 136 * 4 + 32 == 221216
    assert (p15["rows0"], p15["m_tiles"], p15["threads"], p15["wave"]) == (8, 2, 256, 66)
    p16, _ = debug_wide_pair_tower_plan(128, 128, 16, 16, 6, True, 132)
    assert p16["smem"] == 4 * 176 * 128 + 2 * 32768 + 8 * 17 * 136 * 4 + 32 == 229664
    assert (p16["rows0"], p16["m_tiles"], p16["threads"], p16["wave"]) == (8, 3, 384, 66)


@pytest.mark.parametrize("args,reason", [
    ((128, 128, 17, 17, 6, True), "shared memory"),
    ((128, 128, 16, 24, 6, True), "three M-tiles per CTA"),
    ((128, 128, 1, 11, 6, True), "H >= 2"),
    ((128, 128, 1, 1, 1, False), "H >= 2"),
    ((128, 64, 15, 15, 6, True), "128 channels"),
    ((128, 256, 6, 6, 6, True), "128 channels"),
    ((128, 128, 15, 15, 11, True), "layers"),
    ((128, 128, 15, 15, 0, False), "layers"),
])
def test_refusals_name_the_reason(args, reason):
    for sms in (132, 114):
        plan, why = debug_wide_pair_tower_plan(*args, sms)
        assert plan is None and reason in why, why


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not found next to nvcc")
def test_pair_kernel_resources_inside_the_plan():
    """The pair kernel in the built library: no local memory (spills) or stack, at most the registers the plan assumes."""
    assert os.path.exists(b.LIB), "build the library first (python -m muzero_general_b200.build)"
    out = subprocess.run([_cuobjdump(), "-res-usage", b.LIB], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*conv_tower_wide_pair_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert found, "conv_tower_wide_pair_kernel not in the library"
    plan, _ = debug_wide_pair_tower_plan(1, 128, 16, 16, 6, True, 132)
    for fn, reg, stack, local in found:
        assert int(local) == 0 and int(stack) == 0, fn
        assert int(reg) <= plan["reg_cap"], (fn, reg)


# ---------------------------------------------------------------------------------------------- reference fixtures
def gomoku_config(side):
    cfg = load_game_module("gomoku").MuZeroConfig(board_size=side)
    assert (cfg.blocks, cfg.channels) == (6, 128)
    return cfg


@pytest.mark.parametrize("side", [15, 16])
def test_oracle_net_matches_reference_outputs(side):
    from oracle.net import OracleNet, support_to_scalar
    spec = netspec_from_config(gomoku_config(side))
    net = OracleNet(spec, synthetic_weights(spec, 0))
    g = golden_npz(f"net_gomoku{side}.npz")
    assert g["obs"].shape[1:] == (3, side, side)
    v0, r0, p0, h0 = net.initial_inference(g["obs"])
    v1, r1, p1, h1 = net.recurrent_inference(h0, g["action"])
    v2, r2, p2, h2 = net.recurrent_inference(h1, (g["action"] + 1) % spec.action_space)
    tol = dict(rtol=1e-5, atol=1e-6)     # same ATen calls; allows for a different CPU ISA
    for got, key in ((v0, "init_value"), (p0, "init_policy"), (h0, "init_hidden"),
                     (v1, "rec_value"), (r1, "rec_reward"), (p1, "rec_policy"), (h1, "rec_hidden"),
                     (v2, "rec2_value"), (r2, "rec2_reward"), (p2, "rec2_policy"), (h2, "rec2_hidden")):
        numpy.testing.assert_allclose(got.numpy(), g[key], err_msg=key, **tol)
    S = spec.support_size
    numpy.testing.assert_allclose(support_to_scalar(v1, S).numpy()[:, 0], g["rec_value_scalar"], **tol)
    numpy.testing.assert_allclose(support_to_scalar(r1, S).numpy()[:, 0], g["rec_reward_scalar"], **tol)


def c128_search_cases():
    """mcts_gomoku15_c128.json in the form of the other mcts_*.json files."""
    from oracle import packing
    cases = golden_json("mcts_gomoku15_c128.json")
    for c in cases:
        c["legal"] = packing.unpack_subset(c["legal"])
        c["root_actions"] = list(c["legal"])
        visits = [0] * c["root_visits"]["n"]
        for i, v in c["root_visits"]["nonzero"].items():
            visits[int(i)] = v
        c["root_visits"] = visits
        for key in ("obs", "root_priors_raw", "noise", "root_priors", "root_child_value_sums"):
            c[key] = packing.unpack_floats(c[key])
        for sim in c["sims"]:
            sim["priors"] = packing.unpack_floats(sim["priors"])
    return cases


def test_python_oracle_reproduces_the_128_channel_15x15_searches():
    from oracle import mcts as om
    from oracle.net import OracleNet
    cfg = gomoku_config(15)
    spec = netspec_from_config(cfg)
    net = OracleNet(spec, synthetic_weights(spec, 0))
    cases = c128_search_cases()
    assert len(cases) == 2 and all(c["num_simulations"] == 50 for c in cases)
    for case in cases:
        params = om.SearchParams.from_config(cfg, case["num_simulations"])
        obs = numpy.array(case["obs"]).reshape(case["obs_shape"])
        res = om.TreeSearch(params).run(om.ModelEvaluator(net, spec.support_size), obs, case["legal"], case["to_play"],
                                        case["add_noise"], om.LegacyNumpyDraws(numpy.random.RandomState(case["seed"])))
        assert res.root_actions == case["root_actions"] and res.root_visits == case["root_visits"]
        assert res.root_value == case["root_value"] and res.max_tree_depth == case["max_tree_depth"]
        assert [s.path_actions for s in res.sims] == [s["actions"] for s in case["sims"]]
