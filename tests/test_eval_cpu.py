"""Test-mode games (SelfPlay.play_test_games, mz_selfplay_begin_vs) on the CPU: packed blocks with opponent moves
materialise into the reference's test-mode GameHistory, the summary is the test worker's formulas, games are
selected by id rather than by finish order, and the binding declares the new entry points."""
import ctypes as C
import os
import re

import numpy
import pytest

from conftest import ROOT, weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import _lib
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config


def pack_block(gid, slot, first_to_play, root, visits, action, reward, to_play, obs):
    """One staged block in the layout of include/mzb200.h (what the packing warp writes)."""
    T, A = visits.shape
    O = obs.shape[1]
    body = b"".join([numpy.asarray(root, numpy.float64).tobytes(), numpy.asarray(visits, numpy.int32).tobytes(),
                     numpy.asarray(action, numpy.int32).tobytes(), numpy.asarray(reward, numpy.float32).tobytes(),
                     numpy.asarray(to_play, numpy.int32).tobytes(), numpy.zeros(T, numpy.float32).tobytes(),
                     numpy.asarray(obs, numpy.float32).tobytes()])
    size = (_lib.MZ_STAGED_HEADER_BYTES + len(body) + 7) & ~7
    head = numpy.array([gid], numpy.int64).tobytes() + numpy.array([slot, T, first_to_play, O, A, size], numpy.int32).tobytes()
    return (head + body).ljust(size, b"\0")


def packed_games(blocks, game="tictactoe"):
    vec = load_game_module(game).Game.VECTOR
    cfg = load_game_module(game).MuZeroConfig()
    buf, index, off = b"", [], 0
    for blk, slot, T in blocks:
        index.append((off, (slot << 32) | T))
        buf += blk
        off += len(blk)
    games = sp.PackedGames(cfg.observation_shape, vec.OBS_DTYPE, int)
    games.add(buf, numpy.array(index, numpy.uint64).reshape(-1, 2))
    return games


class _Root:
    """What store_search_statistics reads from a search root: children's visit counts and value()."""

    def __init__(self, visits, legal, value):
        self.children = {a: sp.Node(0) for a in numpy.nonzero(legal)[0].tolist()}
        for a, ch in self.children.items():
            ch.visit_count = int(visits[a])
        self._value = value

    def value(self):
        return self._value


def _play(game, muzero_player, rs, gid):
    """One test-mode game on the host environment in the reference's order (self_play.py:110-183), MuZero's moves
    from made-up search results, the opponent's from the host expert -> (reference GameHistory, packed block)."""
    mod = load_game_module(game)
    cfg = mod.MuZeroConfig()
    env = mod.Game(0)
    A = len(cfg.action_space)
    gh = sp.GameHistory()
    obs = env.reset()
    gh.action_history.append(0)
    gh.observation_history.append(obs)
    gh.reward_history.append(0)
    gh.to_play_history.append(env.to_play())
    rec = dict(root=[], visits=[], action=[], reward=[], to_play=[], obs=[numpy.asarray(obs, numpy.float32).ravel()])
    done = False
    while not done and len(gh.action_history) <= cfg.max_moves:
        legal = numpy.zeros(A, numpy.uint8)
        legal[env.legal_actions()] = 1
        if muzero_player == env.to_play():
            visits = rs.randint(0, 6, A) * legal
            visits[numpy.nonzero(legal)[0][0]] += 1
            value = 0.0 if len(rec["root"]) in (2, 3) else float(rs.uniform(-1, 1))  # MuZero's second move: `if value` drops it
            root = _Root(visits, legal, value)
            action = int(numpy.argmax(numpy.where(legal > 0, visits, -1)))
            rec["root"].append(value)
            rec["visits"].append(visits)
        else:
            numpy.random.seed(int(rs.randint(1 << 30)))
            action, root = int(env.expert_agent()), None
            rec["root"].append(float("nan"))
            rec["visits"].append(numpy.zeros(A, numpy.int32))
        obs, reward, done = env.step(action)
        gh.store_search_statistics(root, cfg.action_space)
        gh.action_history.append(action)
        gh.observation_history.append(obs)
        gh.reward_history.append(reward)
        gh.to_play_history.append(env.to_play())
        rec["action"].append(action)
        rec["reward"].append(reward)
        rec["to_play"].append(env.to_play())
        rec["obs"].append(numpy.asarray(obs, numpy.float32).ravel())
    T = len(rec["action"])
    blk = pack_block(gid, gid % 7, gh.to_play_history[0], rec["root"], numpy.array(rec["visits"]), rec["action"],
                     rec["reward"], rec["to_play"], numpy.array(rec["obs"]))
    return gh, (blk, gid % 7, T)


def _worker_report(gh, muzero_player):
    """The test worker's per-game report, as written in self_play.py:67-90."""
    return {
        "episode_length": len(gh.action_history) - 1,
        "total_reward": sum(gh.reward_history),
        "mean_value": numpy.mean([value for value in gh.root_values if value]),
        "muzero_reward": sum(reward for i, reward in enumerate(gh.reward_history)
                             if gh.to_play_history[i - 1] == muzero_player),
        "opponent_reward": sum(reward for i, reward in enumerate(gh.reward_history)
                               if gh.to_play_history[i - 1] != muzero_player),
    }


@pytest.mark.parametrize("game", ["tictactoe", "connect4"])
@pytest.mark.parametrize("muzero_player", [0, 1])
def test_opponent_moves_materialise_in_the_reference_test_mode_shape(game, muzero_player):
    """A packed block whose opponent moves carry NaN root values and zero visits becomes the GameHistory
    play_game(0, ..., "expert", muzero_player) builds: None in root_values at the opponent's moves, child_visits rows
    for MuZero's moves only and in order, the same to_play, action, reward and observation histories."""
    rs = numpy.random.RandomState(7 + muzero_player)
    host, blocks = [], []
    for gid in range(12):
        gh, blk = _play(game, muzero_player, rs, gid)
        host.append(gh)
        blocks.append(blk)
    games = packed_games(blocks, game)
    assert len(games) == len(host)
    nones = 0
    for gh, got in zip(host, games):
        assert got.root_values[0] is None if muzero_player == 1 else got.root_values[0] is not None
        assert [v is None for v in got.root_values] == [v is None for v in gh.root_values]
        assert [v for v in got.root_values if v is not None] == [v for v in gh.root_values if v is not None]
        assert got.child_visits == gh.child_visits
        assert len(got.child_visits) == sum(v is not None for v in gh.root_values)
        assert got.to_play_history == gh.to_play_history
        assert [int(a) for a in got.action_history] == [int(a) for a in gh.action_history]
        assert got.reward_history == gh.reward_history
        assert all(numpy.array_equal(a, b) for a, b in zip(got.observation_history, gh.observation_history))
        nones += sum(v is None for v in gh.root_values)
    assert nones > 0


@pytest.mark.parametrize("muzero_player", [0, 1])
def test_summary_is_the_test_worker_report(muzero_player):
    """summarise_test_games over packed blocks equals the means over games of the test worker's formulas applied to
    the host GameHistory objects of the same games, and its win / draw / loss counts are MuZero's."""
    rs = numpy.random.RandomState(3)
    host, blocks = [], []
    for gid in range(40):
        gh, blk = _play("tictactoe", muzero_player, rs, gid)
        host.append(gh)
        blocks.append(blk)
    got = sp.summarise_test_games(packed_games(blocks), muzero_player, 2)
    reports = [_worker_report(gh, muzero_player) for gh in host]
    for key in ("episode_length", "total_reward", "mean_value", "muzero_reward", "opponent_reward"):
        assert got[key] == numpy.mean([r[key] for r in reports]), key
    wins = sum(r["muzero_reward"] > r["opponent_reward"] for r in reports)
    losses = sum(r["muzero_reward"] < r["opponent_reward"] for r in reports)
    assert (got["games"], got["wins"], got["losses"], got["draws"]) == (40, wins, losses, 40 - wins - losses)
    assert losses > 0 and got["draws"] + wins > 0


def test_self_play_blocks_materialise_unchanged():
    """A self-play block (no NaN) keeps one child_visits row and one float root value per move."""
    rs = numpy.random.RandomState(0)
    T, A = 5, 9
    visits = rs.randint(1, 5, (T, A)).astype(numpy.int32)
    root = rs.uniform(-1, 1, T)
    blk = pack_block(3, 0, 0, root, visits, rs.randint(0, A, T), numpy.zeros(T), numpy.arange(T) % 2,
                     rs.randint(0, 2, (T + 1, 27)))
    gh = packed_games([(blk, 0, T)])[0]
    assert gh.root_values == root.tolist()
    assert gh.child_visits == (visits / visits.sum(1, keepdims=True)).tolist()


# ------------------------------------------------------------------------------------------ selection by id
class _FakeLoop:
    """DeviceSelfPlayLoop stand-in: slot g plays ids first + g + k * stride; a game's length depends on its id so that
    the games of slot 0 are long and every other slot's are short (they finish first and recycle their slots)."""
    made = []

    def __init__(self, engine, env, max_moves, first_game_id=0, game_id_stride=0, opponent="self", muzero_player=0,
                 td_steps=0, **kw):
        self.B = engine.max_games
        self.first, self.stride = first_game_id, game_id_stride or self.B
        self.ids = first_game_id + numpy.arange(self.B)
        self.moves_played = numpy.zeros(self.B, numpy.int64)
        self.kw = dict(opponent=opponent, muzero_player=muzero_player, td_steps=td_steps, env=env)
        self.with_priorities = False
        self.stats = _lib.MzSelfPlayStats()
        self.staged = []
        _FakeLoop.made.append(self)

    def length(self, gid):
        return 9 if (gid - self.first) % self.stride == 0 else 5 + gid % 2

    def enqueue(self, n, temperature):
        for _ in range(n):
            self.moves_played += 1
            for g in range(self.B):
                T = int(self.moves_played[g])
                if T == self.length(int(self.ids[g])):
                    z = numpy.zeros(T)
                    self.staged.append((pack_block(int(self.ids[g]), g, 0, z, numpy.ones((T, 9), numpy.int32), z, z, z,
                                                   numpy.zeros((T + 1, 27))), g, T))
                    self.ids[g] += self.stride
                    self.moves_played[g] = 0
        self.stats.staged_bytes = sum(len(b) for b, _, _ in self.staged)
        self.stats.staging_capacity = 1 << 20

    def wait(self):
        return self.stats

    def drain_pointers(self):
        buf = b"".join(b for b, _, _ in self.staged)
        offs = numpy.cumsum([0] + [len(b) for b, _, _ in self.staged])[:-1]
        index = numpy.array([(o, (g << 32) | T) for o, (_, g, T) in zip(offs, self.staged)], numpy.uint64).reshape(-1, 2)
        self.staged = []
        return buf, index

    @staticmethod
    def copy_staged(pointers):
        return pointers

    def peek(self):
        return {"game_id": self.ids.copy()}


@pytest.fixture()
def fake_device(monkeypatch):
    monkeypatch.setattr(sp, "SearchEngine", FakeSearchEngine)
    monkeypatch.setattr(sp, "DeviceSelfPlayLoop", _FakeLoop)
    _FakeLoop.made = []


def _eval_worker(name="tictactoe", B=4, **over):
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = B, "philox", 2
    for k, v in over.items():
        setattr(cfg, k, v)
    return sp.SelfPlay({"weights": weights_for(name, netspec_from_config(cfg))}, mod.Game, cfg, 0), cfg


def test_play_test_games_selects_by_id_not_by_finish_order(fake_device):
    """n_games = 10 on 4 slots: the returned ids are the 10 smallest this call plays (three rounds, the third one
    partial), although slots 1-3 finish many more short games before slot 0 finishes its long ones; games begun past
    the quota are discarded.  The loop gets the config's opponent and muzero_player and no priorities; a second call
    uses ids past every id the first one began."""
    worker, cfg = _eval_worker(PER=True)
    games, summary = worker.play_test_games(10)
    loop = _FakeLoop.made[-1]
    assert loop.kw == dict(opponent="expert", muzero_player=cfg.muzero_player, td_steps=0, env="tictactoe")
    first = sp.SelfPlay.TEST_GAME_IDS
    assert loop.first == first
    want = {first + k * 4 + g for k in range(3) for g in range(4)}
    want = set(sorted(want)[:10])
    got = [g.game_id for g in games]
    assert len(got) == 10 and set(got) == want
    # finish order would have picked short games of slots 1-3 only, past the quota of the later rounds
    assert max(loop.ids) > max(want) + 4
    assert summary["games"] == 10 and summary["episode_length"] == numpy.mean([len(g) for g in games])
    games2, _ = worker.play_test_games(3, opponent="random", muzero_player=1)
    loop2 = _FakeLoop.made[-1]
    assert loop2.kw["opponent"] == "random" and loop2.kw["muzero_player"] == 1
    assert loop2.first > int(loop.ids.max()) and (loop2.first - first) % 4 == 0
    assert {g.game_id for g in games2} == {loop2.first + g for g in range(3)}


def test_play_test_games_one_player_plays_self(fake_device):
    worker, cfg = _eval_worker("cartpole", B=3)
    games, summary = worker.play_test_games(3)
    assert _FakeLoop.made[-1].kw["opponent"] == "self"
    assert "muzero_reward" not in summary and summary["games"] == 3


def test_play_test_games_refusals(fake_device):
    """No device environment: NotImplementedError naming play_game.  A running self-play loop on the worker: refused
    rather than dropped."""
    worker, _ = _eval_worker(rng_mode="numpy")
    with pytest.raises(NotImplementedError, match="play_game"):
        worker.play_test_games(4)
    worker, _ = _eval_worker()
    worker.play_moves(1, 1.0)
    with pytest.raises(RuntimeError, match="reset_stream"):
        worker.play_test_games(4)
    worker.reset_stream()
    assert len(worker.play_test_games(4)[0]) == 4


# ------------------------------------------------------------------------------------------ binding
def test_binding_declares_the_opponent_entry_points():
    header = open(os.path.join(ROOT, "include", "mzb200.h")).read()
    enum = dict((k, int(v)) for k, v in re.findall(r"(MZ_OPPONENT_[A-Z]+) = (\d+)", header))
    assert enum == {"MZ_OPPONENT_SELF": 0, "MZ_OPPONENT_EXPERT": 1, "MZ_OPPONENT_RANDOM": 2}
    for k, v in enum.items():
        assert getattr(_lib, k) == v
    symbols = {name: (res, args) for name, res, args in _lib.SYMBOLS}
    assert symbols["mz_selfplay_begin_vs"] == (C.c_int, [C.c_void_p, C.POINTER(_lib.MzSelfPlayDesc), C.c_int32, C.c_int32])
    assert len(symbols["mz_debug_opponent_action"][1]) == 9
