"""Test-mode games of host-stepped games (mz_selfplay_begin_host_vs / _host_opponent_turn / _host_opponent_act,
engine.HostEnvSelfPlayLoop with an opponent, SelfPlay.play_test_games on loop_path "device-host-env"): they equal the
device environments' test games field by field, plug-ins without a vector game play legal, reproducible games against
their own expert_agent, host-kept observations give the same games, and the refusals of the ABI."""
import ctypes as C

import numpy
import pytest

from conftest import weights_for
from muzero_general_b200 import _lib
from muzero_general_b200 import self_play as sp
from muzero_general_b200.engine import HostEnvSelfPlayLoop, SearchEngine, parse_staged_game
from muzero_general_b200.games import load_game_module
from muzero_general_b200.games.abstract_game import AbstractGame
from muzero_general_b200.netspec import netspec_from_config
from test_host_env_loop_gpu import _block_bytes, _cfg, _worker

pytestmark = pytest.mark.gpu

MZ_EINVAL, MZ_EUNSUPPORTED, MZ_ESTATE = -1, -3, -4        # include/mzb200.h


def _games(packed):
    """game id -> parsed block of every game of ``packed`` (the kept blocks of each drain)."""
    return {g["game_id"]: g for g in (parse_staged_game(buf, int(off)) for buf, index in packed._chunks
                                      for off in index[:, 0])}


def _same_games(a, b):
    assert sorted(a) == sorted(b)
    for gid in a:
        x, y = a[gid], b[gid]
        assert (x["length"], x["first_to_play"]) == (y["length"], y["first_to_play"]), gid
        assert x["root_value"].tobytes() == y["root_value"].tobytes(), gid
        for key in ("visits", "action", "reward", "to_play", "priority", "obs"):
            assert x[key].tobytes() == y[key].tobytes(), (gid, key)


def _same_summary(a, b, rel=0.0):
    assert set(a) == set(b)
    for k in a:
        assert abs(a[k] - b[k]) <= rel * abs(a[k]) or (a[k] != a[k] and b[k] != b[k]), k


def _opponent_moves_staged_alike(games, muzero_player):
    """Every move whose side to move was not MuZero's has a NaN root value and zero visit counts, MuZero's none."""
    n = 0
    for g in games.values():
        mover = numpy.concatenate(([g["first_to_play"]], g["to_play"][:-1]))
        opp = mover != muzero_player
        assert numpy.isnan(g["root_value"][opp]).all() and not g["visits"][opp].any()
        assert not numpy.isnan(g["root_value"][~opp]).any() and (g["visits"][~opp].sum(axis=1) > 0).all()
        n += int(opp.sum())
    return n


# name, B, config overrides, opponent, muzero_player, temperature, park (a staging area of three maximum-length games)
PARITY_CASES = [
    ("tictactoe", 16, {}, "random", 0, 0.0, False),
    ("tictactoe", 16, {}, "random", 1, 1.0, False),
    ("tictactoe", 16, {}, "expert", 0, 1.0, False),
    ("tictactoe", 16, {}, "expert", 1, 0.0, True),
    ("connect4", 12, dict(stacked_observations=2, max_moves=16), "expert", 0, 1.0, False),
    ("connect4", 12, dict(stacked_observations=2, max_moves=16), "random", 1, 0.0, False),
    ("connect4", 12, dict(max_moves=16), "expert", 1, 1.0, True),
    ("connect4", 12, dict(max_moves=16), "random", 0, 0.0, True),
    ("simple_grid", 16, {}, "self", 0, 1.0, False),
]


@pytest.mark.parametrize("name,B,over,opponent,muzero_player,T,park", PARITY_CASES)
def test_host_test_games_equal_the_device_environments(name, B, over, opponent, muzero_player, T, park, monkeypatch):
    """play_test_games(n) of the same worker config with the device environment and with the game's host vector (the
    expert from BoardVector.expert_actions), same seed, first_game_id and stride, twice in a row: the same ids, and
    every game identical - first_to_play, root values bit for bit (NaN included), visits, actions, rewards, to_play,
    observations - with equal summaries.  With a small staging area both loops park games; the games of the first
    call are still the same."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    _, _, cfg = _cfg(name, B, 4, **over)
    if park:
        A, O = len(cfg.action_space), int(numpy.prod(cfg.observation_shape))
        over = dict(over, selfplay_staging_bytes=3 * _block_bytes(cfg.max_moves, A, O))
    got = {}
    n = 2 * B + 5
    for host in (False, True):
        w, _ = _worker(name, B, 4, seed=11, host=host, first_game_id=3, game_id_stride=B + 2, **over)
        got[host] = [w.play_test_games(n, opponent, muzero_player, temperature=T) for _ in range(2)]
        got[host] = [(_games(packed), summary) for packed, summary in got[host]]
        w.close()
    # a call's ids start past every game the previous call began, which with parking depends on the loop: compare the
    # first call there; its means add the games drain by drain, so parking may change their last bits
    for (dev, s_dev), (hst, s_hst) in zip(got[False], got[True][:1] if park else got[True]):
        assert len(dev) == n
        _same_games(dev, hst)
        _same_summary(s_dev, s_hst, rel=1e-12 if park else 0.0)
        if opponent != "self":
            assert _opponent_moves_staged_alike(hst, muzero_player) > 0
    assert min(got[True][1][0]) > max(got[True][0][0])            # fresh ids per call


class ObjectTicTacToe(AbstractGame):
    """A two-player plug-in without a vector game (the driver takes the _ObjectVector path): TicTacToe through its
    Game object, whose expert_agent is the reference's threat scan with a numpy.random fallback."""

    def __init__(self, seed=None):
        self.g = load_game_module("tictactoe").Game(seed)

    def step(self, action):
        return self.g.step(action)

    def to_play(self):
        return self.g.to_play()

    def legal_actions(self):
        return self.g.legal_actions()

    def reset(self):
        return self.g.reset()

    def render(self):
        pass

    def expert_agent(self):
        return self.g.expert_agent()


def test_object_plugin_plays_legal_reproducible_games(monkeypatch):
    """The object plug-in against its expert_agent, both sides opening: every move is legal when replayed on a fresh
    game, the opponent's moves are staged with NaN and zero visits, and two workers with the same seed (numpy's
    global stream included) play the same games."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    assert not hasattr(ObjectTicTacToe, "vector")
    runs = []
    for _ in range(2):
        mod = load_game_module("tictactoe")
        cfg = mod.MuZeroConfig()
        cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations, cfg.host_env_device_loop = 8, "philox", 4, True
        w = sp.SelfPlay({"weights": weights_for("tictactoe", netspec_from_config(cfg))}, ObjectTicTacToe, cfg, seed=4)
        assert w.loop_path == "device-host-env"
        out = []
        for mp in (0, 1):
            packed, summary = w.play_test_games(13, "expert", mp)
            games = _games(packed)
            assert len(games) == 13 and summary["games"] == 13
            assert _opponent_moves_staged_alike(games, mp) > 0
            for g in games.values():
                ref = ObjectTicTacToe()
                ref.reset()
                for t, a in enumerate(g["action"]):
                    assert int(a) in ref.legal_actions(), (g["game_id"], t)
                    ref.step(int(a))
            out.append(games)
        runs.append(out)
        w.close()
    for a, b in zip(*runs):
        _same_games(a, b)


def _force(monkeypatch, obs_history):
    def make(*args, obs_history=None, _mode=obs_history, **kw):
        return HostEnvSelfPlayLoop(*args, obs_history=_mode, **kw)
    monkeypatch.setattr(sp, "HostEnvSelfPlayLoop", make)


@pytest.mark.parametrize("name,B,over,opponent,muzero_player", [
    ("connect4", 12, dict(stacked_observations=2, max_moves=16), "expert", 1),
    ("breakout", 6, dict(stacked_observations=2, max_moves=12), "self", 0),
])
def test_window_test_games_equal_device_history(name, B, over, opponent, muzero_player, monkeypatch):
    """The same test games with the observations kept on the device and on the host (mz_selfplay_begin_host_vs with
    window 0 and 1): identical records, host-kept observation_history equal to the staged observations byte for byte
    (the opponent's steps included), equal summaries."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    got = {}
    for mode in ("device", "host"):
        _force(monkeypatch, mode)
        w, _ = _worker(name, B, 4, seed=5, host=True, **over)
        packed, summary = w.play_test_games(B + 3, opponent, muzero_player, temperature=1.0)
        assert all((g["obs"].shape[1] == 0) == (mode == "host") for g in _games(packed).values())
        got[mode] = ({gh.game_id: (gh._packed[0], gh) for gh in packed}, summary)
        w.close()
    (dev, s_dev), (hst, s_hst) = got["device"], got["host"]
    _same_summary(s_dev, s_hst)
    assert sorted(dev) == sorted(hst) and len(dev) == B + 3
    for gid in dev:
        a, b = dev[gid][0], hst[gid][0]                   # b["obs"]: the host-kept rows (the block carries none)
        for key in ("root_value", "visits", "action", "reward", "to_play", "obs"):
            assert a[key].tobytes() == b[key].tobytes(), (gid, key)
        obs = numpy.stack([numpy.asarray(o) for o in hst[gid][1].observation_history])
        assert obs.reshape(len(obs), -1).astype(numpy.float32).tobytes() == a["obs"].tobytes(), gid


# ------------------------------------------------------------------------------------------ refusals
def _engine(name, B=4, **over):
    _, _, cfg = _cfg(name, B, 2, **over)
    eng = SearchEngine(cfg, max_games=B, num_simulations=2)
    eng.load_weights(weights_for(name, netspec_from_config(cfg)))
    return cfg, eng


def _code(fn, *args):
    with pytest.raises(_lib.MzError) as e:
        fn(*args)
    return e.value.code


def test_opponent_calls_out_of_order_are_refused():
    """TicTacToe against the expert, MuZero opening: host_act before the turn, opponent_act before the turn, a second
    turn after one that found nothing, host_act while the opponent's moves are due: MZ_ESTATE.  NULL actions on an
    EXPERT loop and an illegal action: MZ_EINVAL, after which the right moves are accepted.  On a loop without an
    opponent the opponent calls answer MZ_ESTATE."""
    _, eng = _engine("tictactoe")
    env = load_game_module("tictactoe").Game.vector(4)
    obs = env.reset()
    loop = HostEnvSelfPlayLoop(eng, (3, 3, 3), 9, obs, env.legal_mask(), env.to_play(), opponent="expert")
    assert _code(loop.act, 1.0) == MZ_ESTATE
    assert _code(loop.opponent_act, numpy.zeros(4)) == MZ_ESTATE
    assert loop.opponent_turn() is None                        # MuZero (to_play 0) opens every game
    assert _code(loop.opponent_turn) == MZ_ESTATE
    assert _code(loop.opponent_act, numpy.zeros(4)) == MZ_ESTATE
    a = loop.act(1.0).copy()
    assert (a >= 0).all()
    obs, reward, done = env.step(a)
    loop.observe(obs, reward, done, env.legal_mask(), env.to_play())
    assert _code(loop.act, 1.0) == MZ_ESTATE
    defaults = loop.opponent_turn().copy()
    assert (defaults >= 0).all() and env.legal_mask()[numpy.arange(4), defaults].all()
    assert _code(loop.act, 1.0) == MZ_ESTATE
    assert _code(loop.opponent_turn) == MZ_ESTATE
    assert _code(loop.opponent_act, None) == MZ_EINVAL
    assert _code(loop.opponent_act, a) == MZ_EINVAL             # the cells MuZero just took
    steps = loop.stats.env_steps
    expert = env.expert_actions(defaults, defaults >= 0)
    played = loop.opponent_act(expert).copy()
    assert played.tolist() == expert.tolist()
    obs, reward, done = env.step(played)
    loop.observe(obs, reward, done, env.legal_mask(), env.to_play())
    assert loop.stats.env_steps == steps + 4
    assert loop.opponent_turn() is None
    assert (loop.act(1.0) >= 0).all()
    eng.close()

    _, eng = _engine("tictactoe")
    obs = env.reset()
    loop = HostEnvSelfPlayLoop(eng, (3, 3, 3), 9, obs, env.legal_mask(), env.to_play())
    assert _code(loop.opponent_turn) == MZ_ESTATE
    assert _code(loop.opponent_act, None) == MZ_ESTATE
    eng.close()


def test_random_opponent_opens_with_the_default():
    """muzero_player 1: the RANDOM opponent opens every game with the turn's default (NULL actions)."""
    _, eng = _engine("tictactoe")
    env = load_game_module("tictactoe").Game.vector(4)
    obs = env.reset()
    loop = HostEnvSelfPlayLoop(eng, (3, 3, 3), 9, obs, env.legal_mask(), env.to_play(), opponent="random",
                               muzero_player=1)
    defaults = loop.opponent_turn().copy()
    assert (defaults >= 0).all()
    assert loop.opponent_act().tolist() == defaults.tolist()
    eng.close()


def _begin_vs(eng, cfg, opponent, muzero_player, window=0, td_steps=0):
    B, A = eng.max_games, len(cfg.action_space)
    shape = tuple(cfg.observation_shape)
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves, d.td_steps = _lib.MZ_ENV_HOST, cfg.max_moves, td_steps
    pw = (C.c_double * (td_steps + 1))(*([1.0] * (td_steps + 1)))
    d.per_alpha, d.discount_pow = 1.0, C.cast(pw, C.c_void_p)
    e = _lib.MzHostEnvDesc(*shape)
    obs = numpy.zeros((B, int(numpy.prod(shape))), numpy.float32)
    legal, tp = numpy.ones((B, A), numpy.uint8), numpy.zeros(B, numpy.int32)
    rc = eng.lib.mz_selfplay_begin_host_vs(eng._h, C.byref(d), C.byref(e), opponent, muzero_player, window,
                                           obs.ctypes.data, legal.ctypes.data, tp.ctypes.data)
    return rc, eng.lib.mz_last_error(eng._h).decode()


def test_begin_host_vs_refusals():
    """MZ_EINVAL: td_steps > 0 with an opponent, muzero_player 2, window 2, an opponent on a one-player handle;
    MZ_EUNSUPPORTED: an unknown opponent.  SELF with muzero_player 0 begins as mz_selfplay_begin_host does, and
    mz_selfplay_begin_vs still refuses MZ_ENV_HOST with an opponent."""
    cfg, eng = _engine("tictactoe")
    rc, msg = _begin_vs(eng, cfg, _lib.MZ_OPPONENT_RANDOM, 0, td_steps=5)
    assert rc == MZ_EINVAL and "td_steps must be 0" in msg, msg
    rc, msg = _begin_vs(eng, cfg, _lib.MZ_OPPONENT_EXPERT, 2)
    assert rc == MZ_EINVAL and "muzero_player must be 0 or 1" in msg, msg
    rc, msg = _begin_vs(eng, cfg, _lib.MZ_OPPONENT_EXPERT, 0, window=2)
    assert rc == MZ_EINVAL and "window" in msg, msg
    rc, msg = _begin_vs(eng, cfg, 3, 0)
    assert rc == MZ_EUNSUPPORTED and "unknown opponent 3" in msg, msg
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves = _lib.MZ_ENV_HOST, 9
    assert eng.lib.mz_selfplay_begin_vs(eng._h, C.byref(d), _lib.MZ_OPPONENT_RANDOM, 0) == MZ_EINVAL
    assert _begin_vs(eng, cfg, _lib.MZ_OPPONENT_SELF, 0, window=1)[0] == 0
    assert _begin_vs(eng, cfg, _lib.MZ_OPPONENT_EXPERT, 1)[0] == 0
    eng.close()
    cfg, eng = _engine("simple_grid")
    rc, msg = _begin_vs(eng, cfg, _lib.MZ_OPPONENT_RANDOM, 0)
    assert rc == MZ_EINVAL and "one player" in msg, msg
    eng.close()
