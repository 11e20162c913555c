"""Host-stepped games with the observations kept on the host (mz_selfplay_begin_host_window,
engine.HostEnvSelfPlayLoop(obs_history="host")): the games equal those of the device-history loop field by field, their
records reproduce their searches from the host-kept observations, and games/atari.py as shipped - refused by the
device-history begin - plays on the window with device memory that does not grow with its observations."""
import numpy
import pytest

from conftest import weights_for
from muzero_general_b200 import _lib
from muzero_general_b200 import self_play as sp
from muzero_general_b200.engine import HostEnvSelfPlayLoop, parse_staged_games
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from test_host_env_loop_gpu import PARITY_CASES, _block_bytes, _cfg, _worker

pytestmark = pytest.mark.gpu

WIDE256_ROUTE = "256-channel towers on the tensor cores, output channels split across CTA pairs"   # mz_numerics


def _force(monkeypatch, obs_history):
    """Make self_play's driver begin its loops with ``obs_history``."""
    def make(*args, obs_history=None, _mode=obs_history, **kw):
        return HostEnvSelfPlayLoop(*args, obs_history=_mode, **kw)
    monkeypatch.setattr(sp, "HostEnvSelfPlayLoop", make)


def _games(packed):
    """game id -> (parsed block, PackedGameHistory) of every game of ``packed``."""
    return {gh.game_id: (gh._packed[0], gh) for gh in packed}


# Breakout's synthetic 3 x 96 x 96 frames, without a stack, with a window that wraps within a game (s = 2, 3 rows for
# 12 moves) and with games/atari.py's s = 32
BREAKOUT_CASES = [
    ("breakout", 8, dict(max_moves=12, stacked_observations=s), (1.0, 0.5, 0.0, 1.0), False) for s in (0, 2, 32)
] + [("breakout", 8, dict(max_moves=12, stacked_observations=2), (1.0,) * 4, True)]


@pytest.mark.parametrize("name,B,over,temps,park", PARITY_CASES + BREAKOUT_CASES)
def test_window_games_equal_the_device_history(name, B, over, temps, park, monkeypatch):
    """The same worker played with obs_history="device" and "host" (same seed, first_game_id, game_id_stride): every game
    both finish is identical - length, first_to_play, root values bit for bit (NaN included), visit counts, actions,
    rewards, to_play, PER priorities - and the host-kept observation_history equals the device-history loop's staged
    observations byte for byte, dtype included.  The window's blocks carry no observations.  With parking, each loop's
    staging area holds three of its own maximum-length blocks."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    mod, _, cfg = _cfg(name, B, 4, **over)
    A, O = len(cfg.action_space), int(numpy.prod(cfg.observation_shape))
    got, parked = {}, {}
    moves = cfg.max_moves // 2 + 1
    for mode in ("device", "host"):
        _force(monkeypatch, mode)
        extra = dict(selfplay_staging_bytes=3 * _block_bytes(cfg.max_moves, A, O if mode == "device" else 0)) if park else {}
        w, wcfg = _worker(name, B, 4, seed=7, host=True, game_id_stride=B + 3, first_game_id=5, **over, **extra)
        games = {}
        for T in temps:
            packed = w.play_moves(moves, T)
            assert w._device_loop.loop.obs_history == mode
            if mode == "host":
                assert all(g["obs"].shape == (g["length"] + 1, 0) for buf, ix in packed._chunks
                           for g in parse_staged_games(buf, ix))
                assert not w._device_loop.loop._finished_rows
            games.update(_games(packed))
        assert w.played_games == len(games)
        parked[mode] = w._device_loop.parked_events
        got[mode] = games
        w.close()
    dev, hst = got["device"], got["host"]
    common = sorted(set(dev) & set(hst))
    if park and name == "breakout":
        # the synthetic frames come from one random stream for the whole batch, so a game begun after a park depends on
        # which slots won the staging space, which the device does not order: compare the games every slot began with
        common = [gid for gid in common if gid < 5 + B]
    if not park:
        assert set(dev) == set(hst) and parked == {"device": 0, "host": 0} and len(common) >= B
    else:
        assert parked["device"] > 0 and parked["host"] > 0 and len(common) >= B // 2
    shape = tuple(cfg.observation_shape)
    for gid in common:
        (a, ga), (b, gb) = dev[gid], hst[gid]
        T = a["length"]
        assert (T, a["first_to_play"]) == (b["length"], b["first_to_play"]), gid
        assert a["root_value"].tobytes() == b["root_value"].tobytes(), gid
        for key in ("visits", "action", "reward", "to_play", "priority"):
            assert a[key].tobytes() == b[key].tobytes(), (gid, key)
        staged = a["obs"].reshape((T + 1,) + shape).astype(ga._packed[2])
        kept = numpy.stack(gb.observation_history)
        assert kept.dtype == staged.dtype and kept.tobytes() == staged.tobytes(), gid
        assert numpy.stack(ga.observation_history).tobytes() == kept.tobytes(), gid


@pytest.mark.parametrize("s", [2, 32])
def test_window_records_reproduce_their_searches(s, monkeypatch):
    """Breakout through the window: for every recorded move, the stacked observation rebuilt with
    GameHistory.get_stacked_observations from the host-kept observation_history, searched by engine.search with the
    game's id and move index, gives the recorded visit counts and root value bit for bit."""
    from muzero_general_b200.engine import SearchEngine
    monkeypatch.setenv("MZ_TC_MODE", "off")
    _force(monkeypatch, "host")
    B, N = 4, 4
    w, cfg = _worker("breakout", B, N, seed=3, host=True, max_moves=6, stacked_observations=s)
    games = list(w.play_moves(8, 1.0))
    assert w._device_loop.loop.obs_history == "host"
    w.close()
    assert len(games) >= B and all(len(g) == 6 and len(g.observation_history) == 7 for g in games)
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


@pytest.mark.parametrize("wide", [None, "3"])
def test_atari_as_shipped_plays_on_the_window(wide, monkeypatch):
    """games/atari.py as shipped (max_moves = 27000, stacked_observations = 32, the 16 x 256 net), 64 slots, N = 2, on
    the CUDA-core towers and on MZ_TC_WIDE=3: the device-history begin answers MZ_ENOMEM; the window's device
    allocation for 27000 moves exceeds the one for 64 moves by the per-move records alone, T x (8 + 4A + 12) bytes per
    slot; and SelfPlay.play_moves falls back to the window and finishes every slot's 64-move synthetic episode with its
    65 observations kept on the host."""
    import torch
    for k in ("MZ_TC_MODE", "MZ_NO_TC", "MZ_TC_WIDE"):
        monkeypatch.delenv(k, raising=False)
    if wide:
        monkeypatch.setenv("MZ_TC_WIDE", wide)
    mod = load_game_module("atari")
    cfg = mod.MuZeroConfig()
    assert (cfg.max_moves, cfg.stacked_observations, cfg.blocks, cfg.channels) == (27000, 32, 16, 256)
    B, N, A = 64, 2, len(cfg.action_space)
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations, cfg.host_env_device_loop = B, "philox", N, True
    w = sp.SelfPlay({"weights": weights_for("atari", netspec_from_config(cfg))}, mod.Game, cfg, seed=1)
    assert w.loop_path == "device-host-env"
    eng = w.model.engine
    assert (WIDE256_ROUTE in eng.numerics) == bool(wide), eng.numerics
    env = mod.Game.vector(B, 0)
    rows = (env.reset(), env.legal_mask(), numpy.zeros(B, numpy.int32))
    shape = tuple(cfg.observation_shape)
    with pytest.raises(_lib.MzError) as e:
        HostEnvSelfPlayLoop(eng, shape, cfg.max_moves, *rows, stacked_observations=32)
    assert e.value.code == _lib.MZ_ENOMEM and "27001 observations of 27648 floats" in str(e.value), str(e.value)

    def window(max_moves):
        HostEnvSelfPlayLoop(eng, shape, max_moves, *rows, stacked_observations=32, obs_history="host")
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    window(64)                                     # each begin frees the loop before it
    free_short = window(64)
    free_long = window(27000)
    records = (27000 - 64) * (8 + 4 * A + 12) * B
    granularity = 5 * (2 << 20)                    # five record buffers grow, each rounded to the allocator's 2 MiB
    assert abs((free_short - free_long) - records) <= granularity, (free_short - free_long, records)

    games = w.play_moves(64, 1.0)
    loop = w._device_loop.loop
    assert loop.obs_history == "host" and not loop._finished_rows
    assert len(games) == B and sorted(g.game_id for g in games) == list(range(B))
    for gh in games[:4]:
        assert len(gh) == 64 and len(gh.observation_history) == 65
        assert gh.observation_history[0].shape == shape and gh.observation_history[0].dtype == numpy.float32
        assert numpy.isfinite(gh.root_values).all()
    assert (WIDE256_ROUTE in eng.numerics) == bool(wide), eng.numerics
    w.close()
