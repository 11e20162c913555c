"""The device loop for host-stepped games (MZ_ENV_HOST: mz_selfplay_begin_host / _host_act / _host_observe /
_host_restart, engine.HostEnvSelfPlayLoop, self_play.DeviceHostEnvSelfPlay): the games it plays equal the device-resident
loop's field by field where both can play them, the records of image games reproduce their searches, and the
refusals of the ABI."""
import ctypes as C

import numpy
import pytest

from conftest import weights_for
from muzero_general_b200 import _lib
from muzero_general_b200.engine import parse_staged_games
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config

pytestmark = pytest.mark.gpu

MZ_EINVAL, MZ_ESTATE, MZ_ENOMEM = -1, -4, -5        # include/mzb200.h


def _cfg(name, B, N, **over):
    mod = load_game_module(name)
    Game = mod.Game
    if name == "gomoku":                            # a 7 x 7 board and a small net: the loop is under test, not the towers
        cfg = mod.MuZeroConfig(board_size=7)
        cfg.blocks, cfg.channels = 1, 16
        Game = mod.Game.sized(7)
    else:
        cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = B, "philox", N
    for k, v in over.items():
        setattr(cfg, k, v)
    return mod, Game, cfg


def _worker(name, B, N, seed, host, first_game_id=0, game_id_stride=None, **over):
    from muzero_general_b200 import self_play as sp
    mod, Game, cfg = _cfg(name, B, N, **over)
    if host:
        cfg.device_envs, cfg.host_env_device_loop = False, True
    w = sp.SelfPlay({"weights": weights_for(name, netspec_from_config(cfg))}, Game, cfg, seed=seed,
                    first_game_id=first_game_id, game_id_stride=game_id_stride)
    assert w.loop_path == ("device-host-env" if host else "device")
    return w, cfg


def _block_bytes(T, A, O):
    """Bytes of one staged game of T moves (include/mzb200.h, "Staged games")."""
    return (_lib.MZ_STAGED_HEADER_BYTES + 8 * T + 4 * T * A + 16 * T + 4 * (T + 1) * O + 7) // 8 * 8


def _games(packed):
    return {g["game_id"]: g for buf, index in packed._chunks for g in parse_staged_games(buf, index)}


# name, B, config overrides, the temperature of each call, park (a staging area of three maximum-length games)
PARITY_CASES = [
    ("tictactoe", 32, dict(temperature_threshold=4), (1.0, 0.5, 0.0, 1.0), False),
    ("tictactoe", 32, {}, (1.0,) * 4, True),
    ("connect4", 24, dict(stacked_observations=2, max_moves=12), (1.0, 0.5, 0.0, 0.5), False),
    ("connect4", 24, dict(stacked_observations=2, max_moves=12), (0.5,) * 4, True),
    ("gomoku", 16, dict(max_moves=10), (1.0, 0.5, 0.0, 1.0), False),
    ("gomoku", 16, dict(max_moves=10, stacked_observations=1), (0.0,) * 4, True),
    ("simple_grid", 32, dict(temperature_threshold=2), (1.0, 0.5, 0.0, 1.0), False),
    ("simple_grid", 32, {}, (0.0,) * 4, True),
]


@pytest.mark.parametrize("name,B,over,temps,park", PARITY_CASES)
def test_host_stepped_games_equal_the_device_loop(name, B, over, temps, park, monkeypatch):
    """The same worker config played by the device environment and by the game's host vector through the new path,
    with the same seed, first_game_id and game_id_stride: every game both finished is identical - id, first_to_play,
    root values bit for bit (NaN included), visit counts, actions, rewards, to_play, PER priorities, observations.
    Without parking both loops finish the same games; with a staging area of three games, games park in both (they
    restart at different moves, so every call there has one temperature)."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    mod, _, cfg = _cfg(name, B, 4, **over)
    if park:
        A, O = len(cfg.action_space), int(numpy.prod(cfg.observation_shape))
        over = dict(over, selfplay_staging_bytes=3 * _block_bytes(cfg.max_moves, A, O))
    got, parked = {}, {}
    moves = cfg.max_moves // 2 + 1
    for host in (False, True):
        w, cfg = _worker(name, B, 4, seed=7, host=host, game_id_stride=B + 3, first_game_id=5, **over)
        games = {}
        for T in temps:
            games.update(_games(w.play_moves(moves, T)))
        assert w.played_games == len(games) and 0 < w.env_steps <= B * moves * len(temps)
        parked[host] = w._device_loop.parked_events
        got[host] = games
        w.close()
    dev, hst = got[False], got[True]
    common = sorted(set(dev) & set(hst))
    if not park:
        assert set(dev) == set(hst) and parked == {False: 0, True: 0} and len(common) >= B
    else:                                          # parked games restart later, differently in the two loops
        assert parked[False] > 0 and parked[True] > 0 and len(common) >= B // 2
    for gid in common:
        a, b = dev[gid], hst[gid]
        assert (a["length"], a["first_to_play"]) == (b["length"], b["first_to_play"]), gid
        assert a["root_value"].tobytes() == b["root_value"].tobytes(), gid
        for key in ("visits", "action", "reward", "to_play", "priority", "obs"):
            assert a[key].tobytes() == b[key].tobytes(), (gid, key)
        assert b["priority"].any() or (b["root_value"] == 0).all()


@pytest.mark.parametrize("s", [0, 2])
def test_breakout_records_reproduce_their_searches(s, monkeypatch):
    """Breakout's synthetic 3 x 96 x 96 frames through the new path: for every recorded move, the stacked observation
    rebuilt from the packed game with GameHistory.get_stacked_observations, searched by engine.search with the game's id
    and move index, gives the recorded visit counts and root value bit for bit."""
    from muzero_general_b200.engine import SearchEngine
    monkeypatch.setenv("MZ_TC_MODE", "off")
    B, N = 4, 4
    w, cfg = _worker("breakout", B, N, seed=3, host=True, max_moves=6, stacked_observations=s)
    games = list(w.play_moves(8, 1.0))
    w.close()
    assert len(games) >= B and all(len(g) == 6 for g in games)
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=3)
    eng.load_weights(weights_for("breakout", spec))
    A = spec.action_space
    rows = [(gh, t) for gh in games for t in range(len(gh))]
    for k in range(0, len(rows), B):
        chunk = rows[k:k + B]
        chunk += [chunk[-1]] * (B - len(chunk))
        obs = numpy.stack([numpy.asarray(gh.get_stacked_observations(t, s, A), numpy.float32).ravel() for gh, t in chunk])
        assert obs.shape[1] == spec.obs_elems
        out = eng.search(obs=obs, legal_mask=numpy.ones((B, A), numpy.uint8), to_play=numpy.zeros(B, numpy.int32),
                         add_exploration_noise=True, game_id=numpy.array([gh.game_id for gh, _ in chunk], numpy.int64),
                         move_index=numpy.array([t for _, t in chunk], numpy.int32))
        for i, (gh, t) in enumerate(chunk):
            rec = gh._packed[0]
            assert out.visit_counts[i].tolist() == rec["visits"][t].tolist(), (gh.game_id, t)
            assert out.root_value[i] == rec["root_value"][t], (gh.game_id, t)
    eng.close()


def _engine(name, B=4, **over):
    from muzero_general_b200.engine import SearchEngine
    _, _, cfg = _cfg(name, B, 2, **over)
    eng = SearchEngine(cfg, max_games=B, num_simulations=2)
    eng.load_weights(weights_for(name, netspec_from_config(cfg)))
    return cfg, eng


def _rows(B, O, A, legal=1, to_play=0):
    return (numpy.zeros((B, O), numpy.float32), numpy.full((B, A), legal, numpy.uint8), numpy.full(B, to_play, numpy.int32))


def _begin(eng, shape, max_moves, obs, legal, to_play, env=_lib.MZ_ENV_HOST):
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves = env, max_moves
    e = _lib.MzHostEnvDesc(*shape)
    rc = eng.lib.mz_selfplay_begin_host(eng._h, C.byref(d), C.byref(e), obs.ctypes.data, legal.ctypes.data,
                                        to_play.ctypes.data)
    return rc, eng.lib.mz_last_error(eng._h).decode()


def test_begin_host_refusals():
    """MZ_EINVAL for an observation that does not give the handle's input, a row without a legal action, a to_play
    outside the players, desc->env other than MZ_ENV_HOST, an opponent other than "self" (mz_selfplay_begin_vs) and
    MZ_ENV_HOST through mz_selfplay_begin; MZ_ENOMEM naming the bytes per slot for records that do not fit."""
    cfg, eng = _engine("tictactoe")
    B, A, O = 4, 9, 27
    obs, legal, tp = _rows(B, O, A)
    rc, msg = _begin(eng, (3, 3, 4), 9, numpy.zeros((B, 36), numpy.float32), legal, tp)
    assert rc == MZ_EINVAL and "obs_c" in msg and "27 input values" in msg, msg
    bad = legal.copy()
    bad[2] = 0
    rc, msg = _begin(eng, (3, 3, 3), 9, obs, bad, tp)
    assert rc == MZ_EINVAL and "row 2 has no legal action" in msg, msg
    rc, msg = _begin(eng, (3, 3, 3), 9, obs, legal, numpy.array([0, 1, 2, 0], numpy.int32))
    assert rc == MZ_EINVAL and "row 2 has to_play 2" in msg, msg
    rc, msg = _begin(eng, (3, 3, 3), 9, obs, legal, tp, env=_lib.MZ_ENV_TICTACTOE)
    assert rc == MZ_EINVAL and "MZ_ENV_HOST" in msg, msg
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves = _lib.MZ_ENV_HOST, 9
    for opponent in (_lib.MZ_OPPONENT_EXPERT, _lib.MZ_OPPONENT_RANDOM):
        assert eng.lib.mz_selfplay_begin_vs(eng._h, C.byref(d), opponent, 0) == MZ_EINVAL
        assert "against themselves only" in eng.lib.mz_last_error(eng._h).decode()
    assert eng.lib.mz_selfplay_begin(eng._h, C.byref(d)) == MZ_EINVAL
    assert "mz_selfplay_begin_host" in eng.lib.mz_last_error(eng._h).decode()
    assert _begin(eng, (3, 3, 3), 9, obs, legal, tp)[0] == 0
    eng.close()
    # games/atari.py's max_moves with 96 x 96 frames: [B][27001][3 * 96 * 96] floats do not fit
    cfg, eng = _engine("breakout", B=64)
    obs, legal, tp = _rows(64, 3 * 96 * 96, 4)
    rc, msg = _begin(eng, (3, 96, 96), 27000, obs, legal, tp)
    assert rc == MZ_ENOMEM and "bytes per slot" in msg and "27001 observations of 27648 floats" in msg, msg
    eng.close()


def test_calls_out_of_order_are_refused():
    """MZ_ESTATE: observe without an act, a second act before the observe, restart with an observe pending, restart of a
    slot with no packed game, act while finished slots wait for their restart, mz_selfplay_moves on a host-stepped
    loop; the protocol then goes on normally."""
    from muzero_general_b200.engine import HostEnvSelfPlayLoop
    cfg, eng = _engine("simple_grid", B=4)
    env = load_game_module("simple_grid").Game.vector(4)
    obs = env.reset()
    loop = HostEnvSelfPlayLoop(eng, (1, 1, 9), 2, obs, env.legal_mask(), env.to_play())

    def code(fn, *args):
        with pytest.raises(_lib.MzError) as e:
            fn(*args)
        return e.value.code

    row = (obs, numpy.zeros(4), numpy.zeros(4, bool), env.legal_mask(), env.to_play())
    assert code(loop.observe, *row) == MZ_ESTATE
    assert code(loop.moves, 1, 1.0) == MZ_ESTATE
    a = loop.act(1.0).copy()
    assert (a >= 0).all()
    assert code(loop.act, 1.0) == MZ_ESTATE
    assert code(loop.restart, numpy.ones(4, bool), obs, env.legal_mask(), env.to_play()) == MZ_ESTATE
    obs, reward, done = env.step(a)
    assert not loop.observe(obs, reward, done, env.legal_mask(), env.to_play()).any()     # max_moves = 2: none yet
    assert code(loop.restart, numpy.ones(4, bool), obs, env.legal_mask(), env.to_play()) == MZ_ESTATE
    obs, reward, done = env.step(loop.act(1.0))
    finished = loop.observe(obs, reward, done, env.legal_mask(), env.to_play())
    assert finished.all() and loop.stats.games_finished == 4
    assert code(loop.act, 1.0) == MZ_ESTATE
    obs = env.reset(finished)
    loop.restart(finished[:2].tolist() + [False, False], obs, env.legal_mask(), env.to_play())
    assert code(loop.act, 1.0) == MZ_ESTATE                    # slots 2, 3 still wait
    loop.restart([False, False, True, True], obs, env.legal_mask(), env.to_play())
    assert (loop.act(1.0) >= 0).all()
    pk = loop.peek()
    assert pk["game_id"].tolist() == [4, 5, 6, 7] and (pk["move_index"] == 0).all()
    games = parse_staged_games(*loop.drain())
    assert sorted(g["game_id"] for g in games) == [0, 1, 2, 3] and all(g["length"] == 2 for g in games)
    assert parse_staged_games(*loop.drain()) == []             # a second drain before the next move: nothing
    eng.close()
