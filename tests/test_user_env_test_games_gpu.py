"""Test-mode games of user environments (mz_selfplay_begin_user_vs, engine.UserEnvSelfPlayLoop with an opponent,
SelfPlay.play_test_games on loop_path "device-user-env"): TicTacToe and Connect4 restated as sources with their expert
(tests/user_env_expert_sources.py) play the built-in device environments' test games field by field; the two-player
contract cases play the host-stepped route's test games under the same rules and expert written in Python; and the
refusals of the ABI."""
import ctypes as C

import numpy
import pytest

from conftest import weights_for
from muzero_general_b200 import _lib
from muzero_general_b200 import self_play as sp
from muzero_general_b200.engine import SearchEngine, UserEnvSelfPlayLoop, parse_staged_game
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
from user_env_contract_games import CASES, SEED, make_config
from user_env_expert_sources import SOURCES, make_expert_game
from user_env_sources import SOURCES as PLAIN_SOURCES

pytestmark = pytest.mark.gpu

MZ_EINVAL, MZ_EUNSUPPORTED = -1, -3        # include/mzb200.h


def _games(packed):
    """game id -> parsed block of every game of ``packed``."""
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
        assert abs(a[k] - b[k]) <= rel * abs(a[k]) or (a[k] != a[k] and b[k] != b[k]), (k, a[k], b[k])


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


def _block_bytes(T, A, O):
    """Bytes of one staged game of T moves (include/mzb200.h, "Staged games")."""
    return (_lib.MZ_STAGED_HEADER_BYTES + 8 * T + 4 * T * A + 16 * T + 4 * (T + 1) * O + 7) // 8 * 8


def _cfg(name, B, N, **over):
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = B, "philox", N
    for k, v in over.items():
        setattr(cfg, k, v)
    return mod, cfg


def _worker(name, B, user, source=None, **over):
    mod, cfg = _cfg(SOURCES[name][2], B, 4, **over)
    Game = mod.Game
    if user:
        Game = type("UserGame", (mod.Game,), dict(DEVICE_ENV=None, DEVICE_SOURCE=source or SOURCES[name][0],
                                                  DEVICE_STATE_BYTES=SOURCES[name][1]))
    w = sp.SelfPlay({"weights": weights_for(name, netspec_from_config(cfg))}, Game, cfg, seed=11, first_game_id=3,
                    game_id_stride=B + 2)
    assert w.loop_path == ("device-user-env" if user else "device")
    return w, cfg


# name, B, config overrides, opponent, muzero_player, temperature, park (a staging area of three maximum-length games)
PARITY_CASES = [
    ("tictactoe", 16, {}, "random", 0, 0.0, False),
    ("tictactoe", 16, {}, "random", 1, 1.0, False),
    ("tictactoe", 16, {}, "expert", 0, 1.0, False),
    ("tictactoe", 16, {}, "expert", 1, 0.0, False),
    ("tictactoe", 16, dict(stacked_observations=2), "expert", 1, 1.0, False),
    ("tictactoe", 16, {}, "expert", 1, 0.0, True),
    ("connect4", 12, dict(stacked_observations=2, max_moves=16), "expert", 0, 1.0, False),
    ("connect4", 12, dict(max_moves=16), "random", 1, 0.0, False),
    ("connect4", 12, dict(max_moves=16), "expert", 1, 1.0, False),
    ("connect4", 12, dict(max_moves=16), "random", 0, 0.0, True),
]


@pytest.mark.parametrize("name,B,over,opponent,muzero_player,T,park", PARITY_CASES)
def test_user_test_games_equal_the_device_environments(name, B, over, opponent, muzero_player, T, park, monkeypatch):
    """play_test_games(2B + 5) of the same worker config with the built-in device environment and with its restatement as
    a user source with the expert in CUDA, same seed, weights, first_game_id and stride, twice in a row: the same ids,
    every game identical - first_to_play, root values bit for bit (NaN included), visits, actions, rewards, to_play,
    observations - and equal summaries.  With a staging area of three games both loops park games; the games of the
    first call are still the same (a call's ids start past every game the previous call began, which with parking
    depends on the loop, and its means add the games drain by drain)."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    _, cfg = _cfg(name, B, 4, **over)
    if park:
        A, O = len(cfg.action_space), int(numpy.prod(cfg.observation_shape))
        over = dict(over, selfplay_staging_bytes=3 * _block_bytes(cfg.max_moves, A, O))
    got = {}
    n = 2 * B + 5
    for user in (False, True):
        w, _ = _worker(name, B, user, **over)
        calls = [w.play_test_games(n, opponent, muzero_player, temperature=T) for _ in range(2)]
        got[user] = [(_games(packed), summary) for packed, summary in calls]
        w.close()
    for (dev, s_dev), (usr, s_usr) in zip(got[False], got[True][:1] if park else got[True]):
        assert len(dev) == n
        _same_games(dev, usr)
        _same_summary(s_dev, s_usr, rel=1e-12 if park else 0.0)
        assert _opponent_moves_staged_alike(usr, muzero_player) > 0
    assert min(got[True][1][0]) > max(got[True][0][0])            # fresh ids per call


CONTRACT_CASES = [("turns33", "expert", 0), ("wide128", "random", 1), ("wide129", "expert", 1),
                  ("wide225", "expert", 0), ("wide256", "random", 0), ("row4097", "expert", 1)]


@pytest.mark.parametrize("name,opponent,muzero_player", CONTRACT_CASES)
def test_contract_test_games_equal_the_host_stepped_route(name, opponent, muzero_player, monkeypatch):
    """The two-player contract cases - the same player again on 30 % of moves, up to 256 actions, up to 4096 state
    bytes, terminal rows without a legal action, max_moves cuts - with CONTRACT_EXPERT in CUDA ("device-user-env") and
    in Python ("device-host-env"): play_test_games returns the same games, every opponent move staged with NaN and zero
    visits, and summaries equal up to the order the games were added in: the user route's two opponent passes per move
    reach a third consecutive opponent move one search later than the host's opponent phase does."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    case = CASES[name]
    assert case.P == 2
    n = case.B + 5
    got = {}
    for user in (True, False):
        cfg = make_config(case, host_env_device_loop=not user)
        spec = netspec_from_config(cfg)
        stride = case.B + 5
        Game = make_expert_game(case, sp.SelfPlay.TEST_GAME_IDS, stride, user=user)
        w = sp.SelfPlay({"weights": synthetic_weights(spec, 0)}, Game, cfg, seed=SEED, first_game_id=0,
                        game_id_stride=stride)
        assert w.loop_path == ("device-user-env" if user else "device-host-env")
        packed, summary = w.play_test_games(n, opponent, muzero_player, temperature=1.0)
        got[user] = (_games(packed), summary)
        w.close()
    (usr, s_usr), (hst, s_hst) = got[True], got[False]
    assert len(usr) == n
    _same_games(usr, hst)
    _same_summary(s_usr, s_hst, rel=1e-12)
    assert _opponent_moves_staged_alike(usr, muzero_player) > 0
    # consecutive moves of one side and games the opponent opens were both played
    movers = [numpy.concatenate(([g["first_to_play"]], g["to_play"][:-1])) for g in usr.values()]
    assert any((m[1:] == m[:-1]).any() for m in movers)
    assert any(m[0] != muzero_player for m in movers)


# ------------------------------------------------------------------------------------------ refusals
def _engine(name, B=4):
    _, cfg = _cfg(name, B, 2)
    eng = SearchEngine(cfg, max_games=B, num_simulations=2)
    eng.load_weights(weights_for(name, netspec_from_config(cfg)))
    return cfg, eng


def _begin_user_vs(eng, cfg, source, state_bytes, opponent, muzero_player, td_steps=0):
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves, d.td_steps = _lib.MZ_ENV_USER, cfg.max_moves, td_steps
    pw = (C.c_double * (td_steps + 1))(*([1.0] * (td_steps + 1)))
    d.per_alpha, d.discount_pow = 1.0, C.cast(pw, C.c_void_p)
    e = _lib.MzUserEnvDesc(source.encode(), state_bytes, *cfg.observation_shape)
    rc = eng.lib.mz_selfplay_begin_user_vs(eng._h, C.byref(d), C.byref(e), opponent, muzero_player)
    return rc, eng.lib.mz_last_error(eng._h).decode()


def test_begin_user_vs_refusals():
    """MZ_EINVAL: td_steps > 0 with an opponent, muzero_player 2, an opponent on a one-player handle, desc->env other
    than MZ_ENV_USER; MZ_EUNSUPPORTED: an unknown opponent, EXPERT on a source without mz_env_expert (naming the macro
    and the function).  A refused begin leaves the running loop as it was; SELF with muzero_player 0 begins as
    mz_selfplay_begin_user does."""
    cfg, eng = _engine("tictactoe")
    src, sb = SOURCES["tictactoe"][:2]
    assert _begin_user_vs(eng, cfg, src, sb, _lib.MZ_OPPONENT_RANDOM, 1)[0] == 0
    before = eng.lib.mz_debug_user_env_compiles(eng._h)
    rc, msg = _begin_user_vs(eng, cfg, src, sb, _lib.MZ_OPPONENT_RANDOM, 0, td_steps=5)
    assert rc == MZ_EINVAL and "td_steps must be 0" in msg, msg
    rc, msg = _begin_user_vs(eng, cfg, src, sb, _lib.MZ_OPPONENT_EXPERT, 2)
    assert rc == MZ_EINVAL and "muzero_player must be 0 or 1" in msg, msg
    rc, msg = _begin_user_vs(eng, cfg, src, sb, 3, 0)
    assert rc == MZ_EUNSUPPORTED and "unknown opponent 3" in msg, msg
    rc, msg = _begin_user_vs(eng, cfg, PLAIN_SOURCES["tictactoe"][0], sb, _lib.MZ_OPPONENT_EXPERT, 0)
    assert rc == MZ_EUNSUPPORTED and "MZ_ENV_EXPERT" in msg and "mz_env_expert" in msg, msg
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves = _lib.MZ_ENV_HOST, 9
    e = _lib.MzUserEnvDesc(src.encode(), sb, *cfg.observation_shape)
    assert eng.lib.mz_selfplay_begin_user_vs(eng._h, C.byref(d), C.byref(e), _lib.MZ_OPPONENT_RANDOM, 0) == MZ_EINVAL
    # the loop begun first still plays: every refusal came before it was dropped
    stats = _lib.MzSelfPlayStats()
    assert eng.lib.mz_selfplay_user_moves(eng._h, 3, 1.0, None, C.byref(stats)) == 0 and stats.env_steps > 0
    assert eng.lib.mz_debug_user_env_compiles(eng._h) == before + 1          # the plain source, compiled once
    assert _begin_user_vs(eng, cfg, PLAIN_SOURCES["tictactoe"][0], sb, _lib.MZ_OPPONENT_SELF, 0)[0] == 0
    eng.close()
    _, cfg = _cfg("simple_grid", 4, 2)
    eng = SearchEngine(cfg, max_games=4, num_simulations=2)
    eng.load_weights(weights_for("simple_grid", netspec_from_config(cfg)))
    rc, msg = _begin_user_vs(eng, cfg, PLAIN_SOURCES["simple_grid"][0], 8, _lib.MZ_OPPONENT_RANDOM, 0)
    assert rc == MZ_EINVAL and "one player" in msg, msg
    eng.close()


def test_an_illegal_expert_move_fails_the_call(monkeypatch):
    """An expert that answers an occupied cell at move 3: the call fails with MZ_EINVAL naming mz_env_expert, the loop
    must be begun again (a later call fails too), and after reset_stream() the same worker's self-play equals a fresh
    worker's."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    bad = SOURCES["tictactoe"][0].replace("    int a = default_action;\n",
                                          "    int a = default_action;\n    if (ctx.move == 3) return b->cell[0] ? 0 : 9;\n")
    assert bad != SOURCES["tictactoe"][0]
    w, _ = _worker("tictactoe", 8, True, source=bad)
    with pytest.raises(_lib.MzError) as e:
        w.play_test_games(8, "expert", 0)
    assert e.value.code == MZ_EINVAL and "mz_env_expert" in str(e.value), str(e.value)
    loop = UserEnvSelfPlayLoop(w.model.engine, bad, 10, (3, 3, 3), 9, opponent="expert")
    for n_moves in (6, 1):                                   # the loop stays failed until it is begun again
        with pytest.raises(_lib.MzError) as e:
            loop.moves(n_moves, 1.0)
        assert e.value.code == MZ_EINVAL
    w.reset_stream()
    mine = _games(w.play_moves(12, 1.0))
    w.close()
    fresh, _ = _worker("tictactoe", 8, True, source=bad)
    theirs = _games(fresh.play_moves(12, 1.0))
    fresh.close()
    assert len(mine) >= 8
    _same_games(mine, theirs)
