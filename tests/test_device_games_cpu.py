"""The Twenty-One and Simple Grid plug-ins, Gomoku's full-board rule and the card stream, on the CPU: the plug-ins
replay the reference environments step for step (tests/golden/env_*.json), their configs' networks and searches
reproduce the reference's fixtures through the oracle, the card draw is pinned to its bit recipe, and the new
environment codes are the header's."""
import os
import re

import numpy
import pytest
import torch

from conftest import ROOT, golden_json, golden_npz, weights_for
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from oracle import cards, philox
from oracle import mcts as om
from oracle.net import OracleNet, support_to_scalar

torch.set_num_threads(1)

NEW_GAMES = ["twentyone", "simple_grid"]


@pytest.mark.parametrize("name", NEW_GAMES)
def test_plugins_replay_the_reference_environments(name):
    """Game(g) replays the reference's Game(g) playout g: observations and their dtype, rewards and their type, done
    flags, legal actions and the side to move."""
    fx = golden_json(f"env_{name}.json")
    mod = load_game_module(name)
    ends = set()
    for g, steps in enumerate(fx["games"]):
        game = mod.Game(g)
        obs = game.reset()
        assert str(obs.dtype) == fx["obs_dtype"] == "float64"
        assert obs.shape == tuple(mod.MuZeroConfig().observation_shape)
        for s in steps:
            obs, reward, done = game.step(s["action"])
            assert str(obs.dtype) == fx["obs_dtype"]
            assert obs.astype(numpy.int8).ravel().tolist() == s["obs"], (g, s)
            assert type(reward) is int and reward == s["reward"] and done == s["done"]
            assert game.legal_actions() == s["legal"] == [0, 1] and game.to_play() == s["to_play"] == 0
        assert steps[-1]["done"]
        ends.add(steps[-1]["reward"])
    assert ends == ({-10, 10} if name == "twentyone" else {10})        # the playouts hold wins and losses


def test_twentyone_vector_takes_any_card_source():
    """The rules with a scripted card source: player 10 + 6, dealer 7; a hit on 9 busts, the dealer does not draw;
    a stand on 16 lets the dealer draw past 16 (7 + 5 + 4 + 3 = 19) and lose the player the hand."""
    tw = load_game_module("twentyone")
    deck = iter([10, 7, 9])
    env = tw.TwentyOneVector(1, cards=[lambda: next(deck)])
    env.reset()
    env.player[0] = 16
    obs, reward, done = env.step([0])
    assert done[0] and reward[0] == -10 and env.player[0] == 25 and env.dealer[0] == 7
    deck = iter([10, 7, 5, 4, 3])
    env = tw.TwentyOneVector(1, cards=[lambda: next(deck)])
    env.reset()
    env.player[0] = 16
    obs, reward, done = env.step([1])
    assert done[0] and reward[0] == -10 and env.dealer[0] == 19
    assert obs[0, 0].tolist() == [[16.0] * 3] * 3 and (obs[0, 2] == 0).all()


def _full_board_without_five():
    """Cells of 11 x 11 coloured (x + 2 y + k) mod 4 < 2 -> +1: runs of at most two in every direction.  Returns the
    forced actions, +1 and -1 alternating, that fill the board (the offset k gives +1 the 61 cells it moves on)."""
    for k in range(4):
        colour = numpy.array([[1 if (x + 2 * y + k) % 4 < 2 else -1 for x in range(11)] for y in range(11)]).ravel()
        if (colour == 1).sum() == 61:
            plus, minus = list(numpy.nonzero(colour == 1)[0]), list(numpy.nonzero(colour == -1)[0])
            return [int(plus[i // 2]) if i % 2 == 0 else int(minus[i // 2]) for i in range(121)]
    raise AssertionError("no colouring with 61 cells")


def test_gomoku_full_board_pays_the_mover():
    """A forced sequence that fills the board with no five in a row ends on move 121 with reward 1 (games/gomoku.py
    pays the mover whenever the game ends); no earlier move ends the game or pays."""
    game = load_game_module("gomoku").Game(0)
    game.reset()
    actions = _full_board_without_five()
    for t, a in enumerate(actions):
        assert a in game.legal_actions()
        _, reward, done = game.step(a)
        assert (reward, done) == ((1, True) if t == 120 else (0, False)), t


@pytest.mark.parametrize("name", NEW_GAMES)
def test_oracle_network_matches_the_reference(name):
    """The oracle network on the plug-in's config reproduces the reference network's outputs (net_*.npz)."""
    cfg = load_game_module(name).MuZeroConfig()
    spec = netspec_from_config(cfg)
    net = OracleNet(spec, weights_for(name, spec))
    g = golden_npz(f"net_{name}.npz")
    v0, r0, p0, h0 = net.initial_inference(g["obs"])
    v1, r1, p1, h1 = net.recurrent_inference(h0, g["action"])
    v2, r2, p2, h2 = net.recurrent_inference(h1, (g["action"] + 1) % spec.action_space)
    for got, key in ((v0, "init_value"), (p0, "init_policy"), (h0, "init_hidden"),
                     (v1, "rec_value"), (r1, "rec_reward"), (p1, "rec_policy"), (h1, "rec_hidden"),
                     (v2, "rec2_value"), (r2, "rec2_reward"), (p2, "rec2_policy"), (h2, "rec2_hidden")):
        numpy.testing.assert_allclose(got.numpy(), g[key], rtol=1e-5, atol=1e-6, err_msg=key)
    numpy.testing.assert_allclose(support_to_scalar(v1, spec.support_size).numpy()[:, 0], g["rec_value_scalar"],
                                  rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", NEW_GAMES)
def test_oracle_search_reproduces_the_reference(name):
    """Same weights, same legacy numpy seed: the oracle search builds the reference's tree (mcts_*.json), fp64 equal."""
    cfg = load_game_module(name).MuZeroConfig()
    spec = netspec_from_config(cfg)
    net = OracleNet(spec, weights_for(name, spec))
    for case in golden_json(f"mcts_{name}.json"):
        params = om.SearchParams.from_config(cfg, case["num_simulations"])
        obs = numpy.array(case["obs"]).reshape(case["obs_shape"])
        draws = om.LegacyNumpyDraws(numpy.random.RandomState(case["seed"]))
        res = om.TreeSearch(params).run(om.ModelEvaluator(net, spec.support_size), obs, case["legal"],
                                        case["to_play"], case["add_noise"], draws)
        assert res.root_visits == case["root_visits"] and res.root_value == case["root_value"]
        assert res.root_priors == case["root_priors"] and res.max_tree_depth == case["max_tree_depth"]
        assert [s.path_actions for s in res.sims] == [s["actions"] for s in case["sims"]]
        assert [s.value for s in res.sims] == [s["value"] for s in case["sims"]]


def test_card_draw_bit_recipe():
    """card(seed, game, k): words 0 and 1 of Philox4x32-10 at counter (game_lo, k, 0, game_hi), key (seed_lo,
    seed_hi ^ 0x7169E006), as a 53-bit uniform u; card 1 + floor(12 u), worth min(card, 10).  Over many draws every
    card 1..12 is equally likely."""
    rs = numpy.random.RandomState(3)
    for _ in range(300):
        seed, game, k = int(rs.randint(0, 2**62)), int(rs.randint(0, 2**45)), int(rs.randint(0, 40))
        w = philox.philox4x32_10((game & 0xFFFFFFFF, k, 0, game >> 32), (seed & 0xFFFFFFFF, (seed >> 32) ^ 0x7169E006))
        u = ((w[0] >> 5) * 2**26 + (w[1] >> 6)) / 2.0**53
        assert cards.card(seed, game, k) == min(1 + int(12.0 * u), 10)
    assert cards.TAG_CARD == 0x7169E006
    raw = numpy.array([1 + int(12.0 * philox.uniform53(7, g, k, 0, cards.TAG_CARD)) for g in range(400) for k in range(30)])
    counts = numpy.bincount(raw, minlength=13)[1:]
    assert counts.min() > 0.85 * len(raw) / 12 and counts.max() < 1.15 * len(raw) / 12


def test_environment_codes_match_the_header():
    """MZ_ENV_* of include/mzb200.h: the existing values unchanged, Gomoku 3, Twenty-One 4, Simple Grid 5; the Python
    binding and the loop's name table agree."""
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import DeviceSelfPlayLoop
    header = open(os.path.join(ROOT, "include", "mzb200.h")).read()
    codes = {k: int(v) for k, v in re.findall(r"(MZ_ENV_[A-Z_0-9]+)\s*=\s*(\d+)", header)}
    assert codes == {"MZ_ENV_CARTPOLE": 0, "MZ_ENV_TICTACTOE": 1, "MZ_ENV_CONNECT4": 2, "MZ_ENV_GOMOKU": 3,
                     "MZ_ENV_TWENTYONE": 4, "MZ_ENV_SIMPLE_GRID": 5}
    for k, v in codes.items():
        assert getattr(_lib, k) == v
    for name in ("cartpole", "tictactoe", "connect4", "gomoku", "twentyone", "simple_grid"):
        assert DeviceSelfPlayLoop.ENVS[name] == codes["MZ_ENV_" + name.upper()]
        assert load_game_module(name).Game.DEVICE_ENV == name
