"""Host side of Reanalyse's fresh search (config.reanalyse_search): every bundled plug-in's Game.legal_masks hook against
legal_actions() along the reference playouts and random playouts, the wiring of Reanalyse (game ids, the
store_visit_counts row rule, the missing-hook error, no search with the option off), PackedGameHistory keeping lists set
before it materialises, the reference's ReplayBuffer.make_target taking the fresh rows as policy targets, and the
resources of the new kernel in the built library."""
import copy
import os
import pickle
import re
import subprocess

import numpy
import pytest
import torch

from conftest import golden_json, weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import build as b
from muzero_general_b200 import reanalyse as ra
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from test_reanalyse_device_cpu import _cuobjdump, _packed_history

torch.set_num_threads(1)

PLUGINS = ["tictactoe", "connect4", "gomoku", "cartpole", "twentyone", "simple_grid", "gridworld", "breakout", "atari"]


@pytest.mark.parametrize("fixture", ["tictactoe", "connect4", "gomoku", "twentyone", "simple_grid"])
def test_legal_masks_equal_the_reference_playouts(fixture):
    """Game.legal_masks of every observation of the reference's playouts (tests/golden/env_*.json) == the legal
    actions the reference reported there."""
    fx = golden_json(f"env_{fixture}.json")
    mod = load_game_module(fixture)
    checked = 0
    for steps in fx["games"]:
        obs = numpy.array([s["obs"] for s in steps], numpy.float64)
        side = int(round((obs.shape[1] / 3) ** 0.5)) if fixture.startswith("gomoku") else None
        shape = (3, side, side) if side else tuple(mod.MuZeroConfig().observation_shape)
        masks = mod.Game.legal_masks(obs.reshape((len(steps),) + shape))
        assert masks.dtype == numpy.uint8
        for s, m in zip(steps, masks):
            if s["done"]:
                continue
            assert numpy.nonzero(m)[0].tolist() == s["legal"], (fixture, s)
            checked += 1
    assert checked > 0


@pytest.mark.parametrize("name", PLUGINS + ["gomoku7"])
def test_legal_masks_equal_legal_actions_along_random_playouts(name):
    """Along seeded random playouts of the plug-in's Game: legal_masks(observations) == legal_actions() at every state."""
    mod = load_game_module(name.rstrip("7"))
    Game = mod.Game.sized(7) if name == "gomoku7" else mod.Game
    rs = numpy.random.RandomState(0)
    states = 0
    for g in range(4 if name in ("breakout", "atari") else 40):
        game = Game(g)
        obs = game.reset()
        for _ in range(30 if name in ("breakout", "atari") else 200):
            legal = game.legal_actions()
            mask = Game.legal_masks(numpy.asarray(obs)[None])
            assert mask.dtype == numpy.uint8 and mask.shape[0] == 1
            assert numpy.nonzero(mask[0])[0].tolist() == sorted(legal), (name, g)
            states += 1
            obs, _, done = game.step(int(rs.choice(legal)))
            if done:
                break
    assert states >= 20


class SearchRecorder(FakeSearchEngine):
    """FakeSearchEngine (the oracle's values) that records reanalyse_search's arguments and answers position q, action
    a with (q + a) % 3 + 1 visits for legal actions and 0 for the others."""
    searches = []

    def reanalyse_search(self, frames, frame_offsets, actions, action_offsets, positions, legal_mask=None,
                         to_play=None, game_id=None, add_exploration_noise=True, stacked_observations=None):
        SearchRecorder.searches.append(dict(N=self.N, max_games=self.max_games, seed=self.seed, positions=positions,
                                            legal=legal_mask,
                                            to_play=to_play, game_id=game_id, noise=add_exploration_noise))
        q, a = numpy.meshgrid(numpy.arange(len(legal_mask)), numpy.arange(self.A), indexing="ij")
        visits = numpy.where(legal_mask != 0, (q + a) % 3 + 1, 0).astype(numpy.int32)
        return visits, numpy.arange(len(legal_mask), dtype=numpy.float64)


def _games(cfg, lengths, rs):
    out = []
    for T in lengths:
        gh = sp.GameHistory()
        gh.action_history = [0] + [int(a) for a in rs.randint(0, 9, T)]
        boards = numpy.zeros((T + 1, 9), numpy.int32)
        for t in range(T):                                  # stones fill cells in order: legal masks change per position
            boards[t + 1:, t] = 1 if t % 2 == 0 else -1
        gh.observation_history = [numpy.stack([(b == 1).reshape(3, 3), (b == -1).reshape(3, 3),
                                               numpy.full((3, 3), 1 - 2 * (t % 2))]).astype(numpy.int32)
                                  for t, b in enumerate(boards)]
        gh.to_play_history = [t % 2 for t in range(T + 1)]
        gh.child_visits = [[1 / 9] * 9 for _ in range(T)]
        gh.root_values = [0.0] * T
        gh.reward_history = [0] * (T + 1)
        out.append(gh)
    return out


def _actor(monkeypatch, search, Game="default", **kw):
    monkeypatch.setattr(ra, "SearchEngine", SearchRecorder)
    SearchRecorder.searches = []
    mod = load_game_module("tictactoe")
    cfg = mod.MuZeroConfig()
    cfg.num_simulations = 7
    if search:
        cfg.reanalyse_search = True
    w = weights_for("tictactoe", netspec_from_config(cfg))
    return ra.Reanalyse({"weights": w}, cfg, max_positions=5, Game=mod.Game if Game == "default" else Game, **kw), cfg


def test_wiring_ids_rows_and_the_search_handle(monkeypatch):
    """With reanalyse_search: one reanalyse_search per call on a handle of config.num_simulations and
    max_positions, game ids SEARCH_GAME_IDS + the buffer ids, noise on, legal masks from Game.legal_masks and
    to_play_history of every position (a PackedGameHistory's read from its block), and every position's child_visits
    the store_visit_counts row; the values are the option-off actor's."""
    actor, cfg = _actor(monkeypatch, True)
    rs = numpy.random.RandomState(0)
    packed = _packed_history(rs, (3, 3, 3), 9, 3)
    packed._packed[0]["obs"][:] = 0                         # an empty board: every action legal
    games = _games(cfg, (4, 1, 0, 6), rs) + [packed]
    ids = [5, 9, 2, 40, 7]
    plain = [copy.deepcopy(g) for g in games]
    actor.reanalyse_games(games, ids)
    assert len(SearchRecorder.searches) == 1
    call = SearchRecorder.searches[0]
    assert call["N"] == 7 and call["max_games"] == 5 and call["noise"] is True
    assert ra.Reanalyse.SEARCH_GAME_IDS == 1 << 41 > sp.SelfPlay.TEST_GAME_IDS
    # the Philox key is (seed low word, seed high word ^ tag): the search handle's high word is none of a self-play
    # worker's (config.seed + worker index)
    assert call["seed"] == ra.Reanalyse.search_seed(cfg.seed) == cfg.seed ^ (0x7169E0A5 << 32)
    assert all((call["seed"] >> 32) != ((cfg.seed + w) >> 32) for w in range(1024))
    assert call["game_id"].tolist() == [(1 << 41) + i for i in ids]
    assert call["positions"].tolist() == [4, 1, 0, 6, 3]
    want_legal = numpy.concatenate([load_game_module("tictactoe").Game.legal_masks(
        numpy.stack(gh.observation_history[:len(gh.root_values)])) for gh in plain if len(gh.root_values)])
    assert numpy.array_equal(call["legal"], want_legal)
    assert call["to_play"].tolist() == [p for gh in plain for p in gh.to_play_history[:len(gh.root_values)]]
    off = 0
    for gh in games:
        T = len(gh.root_values)
        assert len(gh.child_visits) == T
        for i, row in enumerate(gh.child_visits):
            legal = want_legal[off + i]
            visits = [(off + i + a) % 3 + 1 if legal[a] else 0 for a in range(9)]
            assert row == [visits[a] / sum(visits) if legal[a] else 0 for a in range(9)]
            assert all(type(x) is int for x, m in zip(row, legal) if not m)          # the reference's int 0
        off += T
    off_actor, _ = _actor(monkeypatch, False)
    off_actor.reanalyse_games(plain, ids)
    for a, b in zip(plain, games):
        assert numpy.array_equal(numpy.atleast_1d(a.reanalysed_predicted_root_values),
                                 numpy.atleast_1d(b.reanalysed_predicted_root_values))


def test_frames_are_packed_once_per_call(monkeypatch):
    """With stacked observations and the search on, reanalyse_games packs the games' frames once for both calls."""
    actor, cfg = _actor(monkeypatch, True)
    cfg.stacked_observations = 2
    packs, real = [], ra.pack_frames
    monkeypatch.setattr(ra, "pack_frames", lambda sources: (packs.append(len(sources)), real(sources))[1])
    seen = []
    actor.engine.reanalyse_values = lambda frames, *a, **k: (seen.append(frames), numpy.zeros(int(a[-1].sum()), numpy.float32))[1]
    games = _games(cfg, (3, 5), numpy.random.RandomState(5))
    actor.reanalyse_games(games, [0, 1])
    assert packs == [2] and len(SearchRecorder.searches) == 1 and len(seen) == 1


def test_no_search_with_the_option_off(monkeypatch):
    actor, cfg = _actor(monkeypatch, False, Game=None)
    assert actor.search_engine is None
    games = _games(cfg, (3, 2), numpy.random.RandomState(1))
    rows = copy.deepcopy([gh.child_visits for gh in games])
    actor.reanalyse_games(games)
    assert not SearchRecorder.searches and [gh.child_visits for gh in games] == rows


def test_loop_passes_the_buffer_ids(monkeypatch):
    actor, cfg = _actor(monkeypatch, True)
    games = _games(cfg, (3, 2, 4), numpy.random.RandomState(2))

    class Storage:
        d = dict(training_step=0, terminate=False, num_played_games=3, weights={})
        def get_info(self, k):
            if k == "training_step":
                self.d[k] += 1
            return self.d[k]
        def set_info(self, k, v=None):
            pass

    class Buffer:
        def sample_game(self, force_uniform=False):
            return 20 + 3 * (len(SearchRecorder.searches) % 3), games[len(SearchRecorder.searches) % 3], None
        def update_game_history(self, game_id, gh):
            pass

    actor.set_weights = lambda w: None
    actor.games_per_call = 1
    cfg.training_steps = 2
    actor.reanalyse(Buffer(), Storage())
    assert [c["game_id"].tolist() for c in SearchRecorder.searches] == [[(1 << 41) + 20]]


@pytest.mark.parametrize("Game", [None, object])
def test_the_option_without_the_hook_is_refused(monkeypatch, Game):
    with pytest.raises(ValueError, match=r"Game\.legal_masks"):
        _actor(monkeypatch, True, Game=Game)


def test_packed_history_keeps_lists_set_before_it_materialises():
    """child_visits set on a PackedGameHistory whose lists were never built survive the next list access and pickling;
    the other lists are built from the block as before."""
    rs = numpy.random.RandomState(3)
    gh = _packed_history(rs, (3, 3, 3), 9, 4)
    fresh = [[0.25 if a < 4 else 0 for a in range(9)] for _ in range(4)]
    gh.child_visits = fresh
    assert len(gh.observation_history) == 5 and gh.child_visits is fresh
    gh2 = _packed_history(numpy.random.RandomState(3), (3, 3, 3), 9, 4)
    gh2.child_visits = fresh
    back = pickle.loads(pickle.dumps(gh2))
    assert back.child_visits == fresh and len(back.root_values) == 4
    assert back.action_history == gh.action_history


@pytest.mark.skipif(not __import__("oracle.refload", fromlist=["x"]).reference_available(), reason="reference not present")
def test_reference_make_target_takes_the_fresh_rows(monkeypatch):
    """The reference's ReplayBuffer.make_target returns the reanalysed child_visits rows as the policy targets."""
    from oracle.refload import load_reference
    _, _, ref_rb, _ = load_reference()
    actor, cfg = _actor(monkeypatch, True)
    games = _games(cfg, (6,), numpy.random.RandomState(4))
    actor.reanalyse_games(games, [0])
    buf = ref_rb.ReplayBuffer({"num_played_games": 0, "num_played_steps": 0}, {}, cfg)
    _, _, policies, _ = buf.make_target(games[0], 1)
    assert policies[:5] == games[0].child_visits[1:6]
    assert policies[5] == [1 / 9] * 9


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not found next to nvcc")
def test_new_kernel_does_not_spill():
    assert os.path.exists(b.LIB), "build the library first (python -m muzero_general_b200.build)"
    out = subprocess.run([_cuobjdump(), "-res-usage", b.LIB], capture_output=True, text=True, check=True).stdout
    res = re.findall(r"Function (\S*reanalyse_search_inputs\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert res and all(int(st) == 0 and int(local) == 0 for _, _, st, local in res), res
