"""User environments (MZ_ENV_USER: mz_selfplay_begin_user / _user_moves, engine.UserEnvSelfPlayLoop, the
"device-user-env" route of SelfPlay.play_moves): four built-in device environments restated as CUDA sources
(tests/user_env_sources.py) play the built-in environments' games bit for bit, the compiled module is cached per handle,
and the ABI's refusals."""
import ctypes as C

import numpy
import pytest

from conftest import weights_for
from muzero_general_b200 import _lib
from muzero_general_b200.engine import SearchEngine, UserEnvSelfPlayLoop, parse_staged_games
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
from user_env_sources import SOURCES

pytestmark = pytest.mark.gpu

MZ_EINVAL, MZ_ESTATE = -1, -4        # include/mzb200.h


def _cfg(name, B, N, **over):
    mod = load_game_module(SOURCES[name][2])
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = B, "philox", N
    for k, v in over.items():
        setattr(cfg, k, v)
    return mod, cfg


def _worker(name, B, N, seed, user, **over):
    from muzero_general_b200 import self_play as sp
    mod, cfg = _cfg(name, B, N, **over)
    Game = mod.Game
    if user:
        source, state_bytes, _ = SOURCES[name]
        Game = type("UserGame", (mod.Game,), dict(DEVICE_ENV=None, DEVICE_SOURCE=source, DEVICE_STATE_BYTES=state_bytes))
    w = sp.SelfPlay({"weights": weights_for(name, netspec_from_config(cfg))}, Game, cfg, seed=seed, first_game_id=5,
                    game_id_stride=B + 3)
    assert w.loop_path == ("device-user-env" if user else "device")
    return w, cfg


def _block_bytes(T, A, O):
    """Bytes of one staged game of T moves (include/mzb200.h, "Staged games")."""
    return (_lib.MZ_STAGED_HEADER_BYTES + 8 * T + 4 * T * A + 16 * T + 4 * (T + 1) * O + 7) // 8 * 8


def _games(packed):
    return {g["game_id"]: g for buf, index in packed._chunks for g in parse_staged_games(buf, index)}


# name, B, config overrides, the temperature of each call, park (a staging area of three maximum-length games)
PARITY_CASES = [
    ("simple_grid", 32, dict(temperature_threshold=2), (1.0, 0.0, 1.0), False),
    ("simple_grid", 32, {}, (0.0,) * 3, True),
    ("cartpole", 64, dict(max_moves=60), (1.0, 0.0, 1.0), False),
    ("cartpole", 48, dict(max_moves=40, stacked_observations=2), (1.0,) * 3, True),
    ("gridworld", 32, dict(stacked_observations=2), (1.0, 0.0, 1.0), False),
    ("tictactoe", 32, dict(stacked_observations=2), (1.0, 0.0, 1.0), False),
    ("tictactoe", 32, {}, (1.0,) * 3, True),
]


@pytest.mark.parametrize("name,B,over,temps,park", PARITY_CASES)
def test_user_sources_play_the_built_in_games(name, B, over, temps, park, monkeypatch):
    """The same worker config played by the built-in device environment and by its restatement as a user source, with
    the same seed, weights, first_game_id and game_id_stride, over several calls: every game both finished is identical -
    id, first_to_play, root values bit for bit, visit counts, actions, rewards, to_play, PER priorities, observations.
    Without parking both loops finish the same games and play the same moves, with a weight refresh between calls; with
    a staging area of three games, games park in both (they restart at different moves and so in different calls: every
    call there has one temperature and the same weights)."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    _, cfg = _cfg(name, B, 4, **over)
    if park:
        A, O = len(cfg.action_space), int(numpy.prod(cfg.observation_shape))
        over = dict(over, selfplay_staging_bytes=3 * _block_bytes(cfg.max_moves, A, O))
    spec = netspec_from_config(cfg)
    refreshed = [weights_for(name, spec), synthetic_weights(spec, 1)]
    got, parked, steps = {}, {}, {}
    moves = max(3, min(cfg.max_moves // 2 + 1, 24))
    for user in (False, True):
        w, cfg = _worker(name, B, 4, seed=7, user=user, **over)
        games = {}
        for i, T in enumerate(temps):
            w.model.set_weights(refreshed[0 if park else i % 2])
            games.update(_games(w.play_moves(moves, T)))
        assert w.played_games == len(games) and 0 < w.env_steps <= B * moves * len(temps)
        parked[user], steps[user], got[user] = w._device_loop.parked_events, w.env_steps, games
        w.close()
    dev, usr = got[False], got[True]
    common = sorted(set(dev) & set(usr))
    if not park:
        assert set(dev) == set(usr) and parked == {False: 0, True: 0} and len(common) >= B // 2
        assert steps[False] == steps[True]
    else:                                          # parked games restart later, differently in the two loops
        assert parked[False] > 0 and parked[True] > 0 and len(common) >= B // 4
    for gid in common:
        a, b = dev[gid], usr[gid]
        assert (a["length"], a["first_to_play"]) == (b["length"], b["first_to_play"]), gid
        assert a["root_value"].tobytes() == b["root_value"].tobytes(), gid
        for key in ("visits", "action", "reward", "to_play", "priority", "obs"):
            assert a[key].tobytes() == b[key].tobytes(), (gid, key)
    if cfg.PER:
        assert any(usr[g]["priority"].any() for g in common)
    if name == "tictactoe":                        # both players moved, and legal masks changed under the search
        assert any(set(usr[g]["to_play"].tolist()) == {0, 1} and usr[g]["length"] >= 5 for g in common)


def _engine(name, B=8):
    _, cfg = _cfg(name, B, 2)
    eng = SearchEngine(cfg, max_games=B, num_simulations=2)
    eng.load_weights(weights_for(name, netspec_from_config(cfg)))
    return cfg, eng


def _loop(eng, cfg, source, state_bytes=8, max_moves=6):
    return UserEnvSelfPlayLoop(eng, source, state_bytes, cfg.observation_shape, max_moves)


def test_the_compiled_module_is_cached_per_handle():
    """Beginning the loop again on the same handle with the same source compiles nothing; another source compiles once;
    the cached module plays."""
    cfg, eng = _engine("simple_grid")
    src = SOURCES["simple_grid"][0]
    loop = _loop(eng, cfg, src)
    assert loop.compiles == 1
    loop.moves(4, 1.0)
    loop = _loop(eng, cfg, src)
    assert loop.compiles == 1
    st = loop.moves(6, 1.0)
    assert st.games_finished == 8 and st.env_steps >= 8 * 4
    loop = _loop(eng, cfg, src + "\n// another source\n")
    assert loop.compiles == 2
    loop = _loop(eng, cfg, src)
    assert loop.compiles == 2
    eng.close()


def test_user_loop_refusals():
    """MZ_EINVAL: state_bytes beyond the limit, desc->env other than MZ_ENV_USER, a source that does not compile (the
    log in the message), a reset that leaves a slot with to_play outside the players; MZ_ESTATE: mz_selfplay_moves on a
    user loop and mz_selfplay_user_moves on a device loop."""
    cfg, eng = _engine("simple_grid")
    src = SOURCES["simple_grid"][0]

    def begin(source, state_bytes=8, env=_lib.MZ_ENV_USER):
        d = _lib.MzSelfPlayDesc()
        d.env, d.max_moves = env, 6
        e = _lib.MzUserEnvDesc(source.encode(), state_bytes, *cfg.observation_shape)
        return eng.lib.mz_selfplay_begin_user(eng._h, C.byref(d), C.byref(e)), eng.lib.mz_last_error(eng._h).decode()

    rc, msg = begin(src, _lib.MZ_USER_ENV_MAX_STATE_BYTES + 1)
    assert rc == MZ_EINVAL and "state_bytes" in msg
    rc, msg = begin(src, env=_lib.MZ_ENV_HOST)
    assert rc == MZ_EINVAL and "MZ_ENV_USER" in msg
    rc, msg = begin(src.replace("++s->col;", "++s->col"))
    assert rc == MZ_EINVAL and "error" in msg
    rc, msg = begin(src.replace("s->col = 0;", "s->col = 0; *row.to_play = 3;"))
    assert rc == MZ_EINVAL and "to_play" in msg
    assert begin(src)[0] == 0
    stats = _lib.MzSelfPlayStats()
    assert eng.lib.mz_selfplay_moves(eng._h, 1, 1.0, None, C.byref(stats)) == MZ_ESTATE
    assert eng.lib.mz_selfplay_user_moves(eng._h, 1, 1.0, None, C.byref(stats)) == 0
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves = _lib.MZ_ENV_SIMPLE_GRID, 6
    assert eng.lib.mz_selfplay_begin(eng._h, C.byref(d)) == 0
    assert eng.lib.mz_selfplay_user_moves(eng._h, 1, 1.0, None, C.byref(stats)) == MZ_ESTATE
    eng.close()
