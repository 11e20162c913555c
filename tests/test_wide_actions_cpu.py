"""Action spaces beyond 128 and Gomoku boards beyond 11 x 11, without a GPU: the oracles against the reference's
15 x 15 / 16 x 16 fixtures (oracle/gen_golden_wide.py), the plug-in's board_size, and the limit's three statements."""
import os
import re

import numpy
import pytest

from conftest import ROOT, golden_json
from helpers import oracle_replay, random_teacher, teacher_from_cases
from muzero_general_b200 import _lib
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
from oracle import build_c
from oracle import packing
from oracle import mcts as om


def wide_config(A=None, board_size=11, **over):
    """games/gomoku.py's config on a small net; A: an action space that is no board (the search alone is under test)."""
    cfg = load_game_module("gomoku").MuZeroConfig(board_size=board_size)
    cfg.blocks, cfg.channels = 2, 16
    if A is not None:
        cfg.action_space = list(range(A))
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def wide_env_games(side):
    """env_gomoku15.json's games of one side, and its cut, with every step in the form of the other env_*.json files."""
    fx = golden_json("env_gomoku15.json")
    games = fx["sides"][str(side)]
    for steps in games:
        for s in steps:
            s["legal"], s["obs"] = packing.unpack_subset(s["legal"]), packing.unpack_board(s["obs"], side * side)
    return games, fx["cut"]


def wide_search_cases():
    """mcts_gomoku15.json in the form of the other mcts_*.json files."""
    cases = golden_json("mcts_gomoku15.json")
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


def test_packing_is_exact():
    values = [0.1, float(numpy.float32(0.1)), 0.0, 1e-300]
    assert packing.unpack_floats(packing.pack_floats(values)) == values and "f64" in packing.pack_floats(values)
    f32 = [float(numpy.float32(x)) for x in (0.1, 0.25, 3e-20)]
    assert packing.unpack_floats(packing.pack_floats(f32)) == f32 and "f32" in packing.pack_floats(f32)
    assert packing.unpack_subset(packing.pack_subset([0, 2, 5], 6)) == [0, 2, 5]
    obs = numpy.zeros((3, 5, 5)); obs[0, 1, 2] = 1; obs[1, 4, 4] = 1; obs[2] = -1
    assert packing.unpack_board(packing.pack_board(obs), 25) == obs.astype(numpy.int8).ravel().tolist()


def test_python_oracle_reproduces_the_225_action_searches_bit_for_bit():
    from oracle.net import OracleNet
    cfg = wide_config(board_size=15)
    spec = netspec_from_config(cfg)
    net = OracleNet(spec, synthetic_weights(spec, 0))
    cases = wide_search_cases()
    assert any(max(c["legal"]) == 224 for c in cases) and all(c["first_index"] is not None for c in cases)
    for case in cases:
        params = om.SearchParams.from_config(cfg, case["num_simulations"])
        obs = numpy.array(case["obs"]).reshape(case["obs_shape"])
        res = om.TreeSearch(params).run(om.ModelEvaluator(net, spec.support_size), obs, case["legal"], case["to_play"],
                                        case["add_noise"], om.LegacyNumpyDraws(numpy.random.RandomState(case["seed"])))
        assert res.root_actions == case["root_actions"] and res.root_visits == case["root_visits"]
        assert res.root_value == case["root_value"] and res.root_priors == case["root_priors"]
        assert res.max_tree_depth == case["max_tree_depth"]
        assert [s.path_actions for s in res.sims] == [s["actions"] for s in case["sims"]]
        assert [s.priors for s in res.sims] == [s["priors"] for s in case["sims"]]


def test_c_oracle_reproduces_the_225_action_searches():
    cfg = wide_config(board_size=15)
    for c in wide_search_cases():
        N = c["num_simulations"]
        t, legal, noise, first, to_play = teacher_from_cases([c], 225, N)
        r = build_c.tree_search(1, N, 225, 2, cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction,
                                legal, to_play, noise, first, cfg.seed, None, None, t)
        assert [int(r["visit_counts"][0, a]) for a in c["root_actions"]] == c["root_visits"]
        assert r["root_value"][0] == c["root_value"] and r["max_depth"][0] == c["max_tree_depth"]
        assert [[int(a) for a in r["actions"][0, s, :r["depth"][0, s]]] for s in range(N)] == [s["actions"] for s in c["sims"]]


@pytest.mark.parametrize("A", [225, 256])
def test_c_oracle_matches_python_oracle(A):
    cfg = wide_config(A)
    N, n, P = 40, 6, 2
    rs = numpy.random.RandomState(5 + A)
    legal = (rs.uniform(size=(n, A)) < 0.7).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    t = random_teacher(rs, n, N, A, reward_scale=0.0, legal=legal)
    if A == 256:
        t["priors"][:3] = numpy.float32(1.0 / A); t["value"][:3] = 0; t["reward"][:3] = 0
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    gid = (77 + numpy.arange(n)).astype(numpy.int64)
    mv = rs.randint(0, 9, n).astype(numpy.int32)
    r = build_c.tree_search(n, N, A, P, cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction,
                            legal, to_play, noise, None, cfg.seed, gid, mv, t)
    params = om.SearchParams.from_config(cfg, N)
    ties = 0
    for i in range(n):
        acts = [a for a in range(A) if legal[i, a]]
        res, draws = oracle_replay(params, acts, int(to_play[i]),
                                   (t["root_value"][i], t["root_reward"][i], [t["root_priors"][i, a] for a in acts]),
                                   [(t["value"][i, s], t["reward"][i, s], t["priors"][i, s]) for s in range(N)],
                                   [noise[i, a] for a in acts], None, seed=cfg.seed, game=int(gid[i]), move=int(mv[i]))
        assert [int(r["visit_counts"][i, a]) for a in acts] == res.root_visits
        assert r["root_value"][i] == res.root_value and r["ties"][i] == draws.later_ties
        assert [[int(a) for a in r["actions"][i, s, :r["depth"][i, s]]] for s in range(N)] == [s.path_actions for s in res.sims]
        ties += draws.later_ties
    assert A != 256 or ties > 0


@pytest.mark.parametrize("side", [15, 16])
def test_plugin_replays_the_reference_playouts(side):
    """Edge wins in the four directions end on their last move with reward 1; the random playout is still running when
    the fixture stops."""
    mod = load_game_module("gomoku")
    games, cut = wide_env_games(side)
    assert [g[-1]["done"] for g in games] == [True] * 4 + [False] and len(games[-1]) == cut
    for steps in games:
        g = mod.Game(0, board_size=side)
        obs = g.reset()
        assert obs.shape == (3, side, side) and g.legal_actions() == list(range(side * side)) and g.to_play() == 0
        for s in steps:
            obs, reward, done = g.step(s["action"])
            assert obs.astype(numpy.int8).ravel().tolist() == s["obs"] and reward == s["reward"] and done == s["done"]
            assert g.legal_actions() == s["legal"] and g.to_play() == s["to_play"]
    vec = mod.Game.sized(side).vector(3, 0)
    assert vec.observations().shape == (3, 3, side, side) and mod.Game.sized(side)(0).env.H == side


def test_default_board_is_the_existing_fixture():
    mod = load_game_module("gomoku")
    cfg = mod.MuZeroConfig()
    assert cfg.observation_shape == (3, 11, 11) and cfg.action_space == list(range(121)) and cfg.board_size == 11
    big = mod.MuZeroConfig(board_size=15)
    assert big.observation_shape == (3, 15, 15) and big.action_space == list(range(225))
    assert mod.Game(0).action_to_string(120) == "KK" and mod.Game(0, board_size=15).action_to_string(224) == "OO"
    for steps in golden_json("env_gomoku.json")["games"][:4]:
        g = mod.Game(0)
        g.reset()
        for s in steps:
            obs, reward, done = g.step(s["action"])
            assert obs.astype(numpy.int8).ravel().tolist() == s["obs"] and reward == s["reward"] and done == s["done"]


def test_limit_is_stated_once_everywhere():
    header = open(os.path.join(ROOT, "include", "mzb200.h")).read()
    assert int(re.search(r"#define MZ_MAX_ACTIONS (\d+)", header).group(1)) == _lib.MZ_MAX_ACTIONS == 256
    abi = open(os.path.join(ROOT, "muzero_general_b200", "csrc", "abi.cu")).read()
    assert "action_space must be in [1, 256]" in abi
    for doc in ("DESIGN.md", "INTEGRATION.md"):
        assert "MZ_MAX_ACTIONS = 256" in open(os.path.join(ROOT, doc)).read(), doc
