"""The Gridworld plug-in on the CPU: its config is the reference's, its rules give the hand-derived views, walls, rewards
and ends, the device's placement (oracle/gridworld.py) is pinned to its bit recipe and uniform over the 15 x 4 starts,
the oracle reproduces the reference's network and search fixtures, and MZ_ENV_GRIDWORLD is the same number everywhere."""
import os
import re

import numpy
import pytest
import torch

from conftest import ROOT, golden_json, golden_npz, weights_for
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from oracle import gridworld, philox
from oracle import mcts as om
from oracle.net import OracleNet, support_to_scalar

torch.set_num_threads(1)

gw = load_game_module("gridworld")
EMPTY, WALL, GOAL = [1, 0, 0], [2, 5, 0], [8, 1, 0]
AHEAD = {0: (1, 0), 1: (0, 1), 2: (-1, 0), 3: (0, -1)}


def _env(x, y, d):
    env = gw.GridworldVector(1, places=[lambda: (x, y, d)])
    env.reset()
    return env


def _view(x, y, d):
    return _env(x, y, d).observations()[0].tolist()


def _cell(x, y):
    if x <= 0 or x >= 5 or y <= 0 or y >= 5:
        return WALL
    return GOAL if (x, y) == (4, 4) else EMPTY


def test_config_equals_the_reference():
    """Every value of the reference's MuZeroConfig (config_gridworld.json) and its temperature schedule."""
    fx = golden_json("config_gridworld.json")
    cfg = gw.MuZeroConfig()
    for k, v in fx["values"].items():
        mine = getattr(cfg, k)
        assert (list(mine) if isinstance(mine, tuple) else mine) == v, k
    for steps, t in fx["temperature"]:
        assert cfg.visit_softmax_temperature_fn(steps) == t, steps
    assert fx["values"]["observation_shape"] == [7, 7, 3] and fx["values"]["max_moves"] == 15


def test_worked_anchor():
    """The agent at (1, 1) facing +x: three empty cells ahead, then the east wall; the goal at [6][3]; everything left
    of the agent (x' <= 2) wall; its own cell empty."""
    obs = _view(1, 1, 0)
    assert obs[3][5] == obs[3][4] == obs[3][3] == EMPTY
    assert obs[3][2] == WALL and obs[6][3] == GOAL and obs[3][6] == EMPTY
    assert all(obs[xv][yv] == WALL for xv in range(3) for yv in range(7))
    o = _env(1, 1, 0).observations()
    assert o.dtype == numpy.uint8 and o.shape == (1, 7, 7, 3)


@pytest.mark.parametrize("x,y,d,goal_at", [(4, 2, 0, (5, 6)), (2, 4, 1, (1, 6)), (1, 3, 2, None), (3, 1, 3, None)])
def test_each_direction_facing_a_wall(x, y, d, goal_at):
    """Facing the wall next to it in each direction: the whole column ahead (x' = 3, y' < 6) is wall, read from the
    room and from beyond it; the goal shows where the rotation puts it (beside the agent, or behind it and unseen)."""
    obs = _view(x, y, d)
    assert all(obs[3][yv] == WALL for yv in range(6)), d
    assert obs[3][6] == EMPTY
    goals = [(xv, yv) for xv in range(7) for yv in range(7) if obs[xv][yv] == GOAL]
    assert goals == ([goal_at] if goal_at else [])


def test_view_is_the_cell_ahead_and_to_the_right():
    """For every start (and the goal cell), the slice-and-rotate of the rules puts at view cell (x', y') the cell
    6 - y' ahead of the agent and x' - 3 to its right (right of dir d is dir d + 1): the closed form csrc/selfplay.cu
    evaluates."""
    for x in range(1, 5):
        for y in range(1, 5):
            for d in range(4):
                fx, fy = AHEAD[d]
                obs = _view(x, y, d)
                for xv in range(7):
                    for yv in range(7):
                        ahead, right = 6 - yv, xv - 3
                        want = EMPTY if (xv, yv) == (3, 6) else _cell(x + ahead * fx - right * fy, y + ahead * fy + right * fx)
                        assert obs[xv][yv] == want, (x, y, d, xv, yv)


def test_turns_and_a_step_into_a_wall():
    """Turning changes the direction only; a forward step into a wall changes nothing but step_count."""
    env = _env(4, 2, 0)
    before = env.observations().copy()
    obs, reward, done = env.step([2])
    assert (env.x[0], env.y[0], env.dir[0], env.step_count[0]) == (4, 2, 0, 1)
    assert numpy.array_equal(obs, before) and reward[0] == 0.0 and not done[0]
    env.step([0])
    assert (env.x[0], env.y[0], env.dir[0]) == (4, 2, 3)
    env.step([1]); env.step([1])
    assert (env.x[0], env.y[0], env.dir[0], env.step_count[0]) == (4, 2, 1, 4)
    env.step([2])
    assert (env.x[0], env.y[0]) == (4, 3)


@pytest.mark.parametrize("k", [1, 2, 15, 100, 143, 144])
def test_reaching_the_goal_at_step_k(k):
    """Entering the goal on step k pays 1 - 0.9 * (k / 144) in fp64 and ends the game; the agent stands on the goal,
    its own cell reading empty."""
    game = gw.Game()
    game.env = _env(4, 3, 1)
    for t in range(k - 1):
        _, reward, done = game.step(t % 2)          # left, right, ...: the direction is back after every pair
        assert reward == 0.0 and not done
    if k % 2 == 0:
        game.env.dir[0] = 1
    obs, reward, done = game.step(2)
    assert type(reward) is float and reward == 1 - 0.9 * (k / 144) and done
    assert (game.env.x[0], game.env.y[0]) == (4, 4) and obs[3][6].tolist() == EMPTY
    assert not any(obs[xv][yv].tolist() == GOAL for xv in range(7) for yv in range(7))


def test_the_144_step_cap_ends_the_game():
    env = _env(2, 2, 0)
    for t in range(143):
        _, reward, done = env.step([t % 2])
        assert not done[0] and reward[0] == 0.0
    _, reward, done = env.step([0])
    assert done[0] and reward[0] == 0.0 and env.step_count[0] == 144


def test_game_facade():
    """Game(seed): uint8 (7, 7, 3) observations, float rewards, the three actions and the reference's strings."""
    game = gw.Game(5)
    obs = game.reset()
    assert obs.dtype == numpy.uint8 and obs.shape == tuple(gw.MuZeroConfig().observation_shape)
    assert game.legal_actions() == [0, 1, 2] and game.to_play() == 0
    _, reward, done = game.step(0)
    assert type(reward) is float and type(done) is bool
    assert [game.action_to_string(a) for a in range(3)] == ["0. Turn left", "1. Turn right", "2. Move forward"]
    assert numpy.array_equal(gw.Game(5).reset(), gw.Game(5).reset())


def _chi_square(counts):
    expected = counts.sum() / counts.size
    return float(((counts - expected) ** 2 / expected).sum())


def test_placements_are_free_cells_and_uniform():
    """Over 60000 game ids the device placement (and over 6000 games the numpy default) never lands on a wall or the
    goal, reaches all 15 x 4 (cell, dir) starts, and passes a chi-square test of uniformity (59 degrees of freedom;
    99.9 % quantile 98.3)."""
    free = [(x, y) for y in range(1, 5) for x in range(1, 5) if (x, y) != (4, 4)]
    for draws in ([gridworld.placement(0x6A1D, g) for g in range(60000)],
                  [gw.numpy_placement(s)() for s in range(6000)]):
        counts = numpy.zeros((15, 4), numpy.int64)
        for x, y, d in draws:
            assert (x, y) in free and 0 <= d < 4
            counts[free.index((x, y)), d] += 1
        assert (counts > 0).all()
        assert _chi_square(counts) < 98.3


def test_numpy_placement_draw_order():
    """MiniGrid's place_agent on RandomState(seed): randint(0, 6) for x, then y, again on a taken cell, then
    randint(0, 4) for the direction; each game of a vector takes seed + g."""
    for seed in range(40):
        rs = numpy.random.RandomState(seed)
        while True:
            x, y = rs.randint(0, 6), rs.randint(0, 6)
            if 1 <= x <= 4 and 1 <= y <= 4 and (x, y) != (4, 4):
                break
        assert gw.numpy_placement(seed)() == (x, y, rs.randint(0, 4))
    env = gw.GridworldVector(3, seed=10)
    env.reset()
    assert [(env.x[g], env.y[g], env.dir[g]) for g in range(3)] == [gw.numpy_placement(10 + g)() for g in range(3)]


def test_placement_bit_recipe():
    """placement(seed, game): u_k = words 0 and 1 of Philox4x32-10 at counter (game_lo, k, 0, game_hi), key (seed_lo,
    seed_hi ^ 0x7169E007), as a 53-bit uniform; cell i = floor(15 u_0) at x = 1 + i % 4, y = 1 + i // 4, dir
    floor(4 u_1)."""
    rs = numpy.random.RandomState(4)
    for _ in range(300):
        seed, game = int(rs.randint(0, 2**62)), int(rs.randint(0, 2**45))
        u = []
        for k in range(2):
            w = philox.philox4x32_10((game & 0xFFFFFFFF, k, 0, game >> 32), (seed & 0xFFFFFFFF, (seed >> 32) ^ 0x7169E007))
            u.append(((w[0] >> 5) * 2**26 + (w[1] >> 6)) / 2.0**53)
        i = int(15 * u[0])
        assert gridworld.placement(seed, game) == (1 + i % 4, 1 + i // 4, int(4 * u[1]))
    assert gridworld.TAG_PLACE == 0x7169E007


def test_oracle_network_matches_the_reference():
    """The oracle network on the plug-in's config reproduces the reference network's outputs (net_gridworld.npz)."""
    cfg = gw.MuZeroConfig()
    spec = netspec_from_config(cfg)
    net = OracleNet(spec, weights_for("gridworld", spec))
    g = golden_npz("net_gridworld.npz")
    v0, r0, p0, h0 = net.initial_inference(g["obs"])
    v1, r1, p1, h1 = net.recurrent_inference(h0, g["action"])
    v2, r2, p2, h2 = net.recurrent_inference(h1, (g["action"] + 1) % spec.action_space)
    for got, key in ((v0, "init_value"), (p0, "init_policy"), (h0, "init_hidden"),
                     (v1, "rec_value"), (r1, "rec_reward"), (p1, "rec_policy"), (h1, "rec_hidden"),
                     (v2, "rec2_value"), (r2, "rec2_reward"), (p2, "rec2_policy"), (h2, "rec2_hidden")):
        numpy.testing.assert_allclose(got.numpy(), g[key], rtol=1e-5, atol=1e-6, err_msg=key)
    numpy.testing.assert_allclose(support_to_scalar(v1, spec.support_size).numpy()[:, 0], g["rec_value_scalar"],
                                  rtol=1e-5, atol=1e-6)


def test_oracle_search_reproduces_the_reference():
    """Same weights, same legacy numpy seed: the oracle search builds the reference's tree (mcts_gridworld.json) on
    observations of the plug-in's rules, fp64 equal."""
    cfg = gw.MuZeroConfig()
    spec = netspec_from_config(cfg)
    net = OracleNet(spec, weights_for("gridworld", spec))
    cases = golden_json("mcts_gridworld.json")
    assert len(cases) == 4
    for case in cases:
        params = om.SearchParams.from_config(cfg, case["num_simulations"])
        obs = numpy.array(case["obs"]).reshape(case["obs_shape"])
        draws = om.LegacyNumpyDraws(numpy.random.RandomState(case["seed"]))
        res = om.TreeSearch(params).run(om.ModelEvaluator(net, spec.support_size), obs, case["legal"],
                                        case["to_play"], case["add_noise"], draws)
        assert res.root_visits == case["root_visits"] and res.root_value == case["root_value"]
        assert res.root_priors == case["root_priors"] and res.max_tree_depth == case["max_tree_depth"]
        assert [s.path_actions for s in res.sims] == [s["actions"] for s in case["sims"]]
        assert [s.value for s in res.sims] == [s["value"] for s in case["sims"]]


def test_environment_code_matches_the_header():
    """#define MZ_ENV_GRIDWORLD of include/mzb200.h is _lib's constant, the loop's name table entry and the plug-in's
    DEVICE_ENV; it is none of the other codes."""
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import DeviceSelfPlayLoop
    header = open(os.path.join(ROOT, "include", "mzb200.h")).read()
    (code,) = [int(v) for v in re.findall(r"#define\s+MZ_ENV_GRIDWORLD\s+(\d+)", header)]
    assert code == _lib.MZ_ENV_GRIDWORLD == DeviceSelfPlayLoop.ENVS["gridworld"] == 7
    assert gw.Game.DEVICE_ENV == "gridworld"
    others = [v for k, v in DeviceSelfPlayLoop.ENVS.items() if k != "gridworld"] + [_lib.MZ_ENV_HOST]
    assert code not in others
