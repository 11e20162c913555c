"""The search re-run at every stored position (mz_reanalyse_search, csrc/reanalyse.cu): visit counts and root values
against the host route (host stacks through engine.search with the same chunk boundaries, legal masks, to_play, game ids
and move indices) bit for bit on every route, order invariance, games/atari.py on the CUDA-core towers and on
MZ_TC_WIDE=3, the device self-play loop's own searches reproduced, bounded memory on a long game, the refusals,
Reanalyse.reanalyse_games end to end, and the search handle's noise being none of self-play's."""
import copy
import ctypes as C
import pickle
import tracemalloc

import numpy
import pytest

from conftest import weights_for
from muzero_general_b200 import _lib
from muzero_general_b200 import reanalyse as ra
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config

pytestmark = pytest.mark.gpu

MZ_EINVAL, MZ_ESTATE = -1, -4                    # include/mzb200.h


def _cfg(name, s, N, **over):
    cfg = load_game_module("gomoku").MuZeroConfig(board_size=7) if name == "gomoku7" else load_game_module(name).MuZeroConfig()
    cfg.stacked_observations, cfg.num_simulations = s, N
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def _engine(cfg, name, B, N=None):
    from muzero_general_b200.engine import SearchEngine
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=N)
    eng.load_weights(weights_for(name.rstrip("7"), spec))
    return eng


def _games(rs, cfg, lengths):
    """Seeded histories: T moves, T + 1 float32 frames, the action history with its leading 0, a random side to move
    per position; with random legal masks (at least one legal action per position) in game order."""
    A, P = len(cfg.action_space), len(cfg.players)
    games, legal = [], []
    for T in lengths:
        gh = sp.GameHistory()
        gh.action_history = [0] + [int(a) for a in rs.randint(0, A, T)]
        gh.observation_history = [rs.random_sample(tuple(cfg.observation_shape)).astype(numpy.float32) for _ in range(T + 1)]
        gh.to_play_history = [int(p) for p in rs.randint(0, P, T + 1)]
        gh.root_values = [0.0] * T
        m = rs.random_sample((T, A)) < 0.6
        m[numpy.arange(T), rs.randint(0, A, T)] = True
        legal.append(m.astype(numpy.uint8))
        games.append(gh)
    return games, numpy.concatenate(legal) if legal else numpy.zeros((0, A), numpy.uint8)


def _to_play(games):
    return numpy.array([gh.to_play_history[i] for gh in games for i in range(len(gh.root_values))], numpy.int32)


def _host_route(eng, games, s, legal, to_play, gids, B, noise=True):
    """engine.search on host-built get_stacked_observations(i, s, A), chunks of B positions in game order."""
    stacks, idx, gid = [], [], []
    for g, gh in enumerate(games):
        for i in range(len(gh.root_values)):
            stacks.append(numpy.asarray(gh.get_stacked_observations(i, s, eng.A), numpy.float32).reshape(-1))
            idx.append(i)
            gid.append(gids[g])
    visits, root = [numpy.zeros((0, eng.A), numpy.int32)], [numpy.zeros(0)]
    for lo in range(0, len(stacks), B):
        hi = min(len(stacks), lo + B)
        out = eng.search(obs=numpy.stack(stacks[lo:hi]), legal_mask=legal[lo:hi], to_play=to_play[lo:hi],
                         add_exploration_noise=noise, game_id=numpy.array(gid[lo:hi], numpy.int64),
                         move_index=numpy.array(idx[lo:hi], numpy.int32))
        visits.append(out.visit_counts)
        root.append(out.root_value)
    return numpy.concatenate(visits), numpy.concatenate(root)


def _packed(games):
    p = ra.pack_frames([ra._frame_source(gh) for gh in games])
    return p["frames"], p["frame_offsets"], p["actions"], p["action_offsets"], p["positions"]


def _device(args, legal, to_play):
    import torch
    frames, fo, actions, ao, pos = args
    return (torch.from_numpy(frames).cuda(), fo, torch.from_numpy(actions).cuda(), ao, pos,
            torch.from_numpy(legal).cuda(), torch.from_numpy(to_play).cuda())


# (game, s): every route of the search - the fused small search, step-wise towers, the fused FC kernel, wide actions
CASES = [("tictactoe", 0), ("tictactoe", 2), ("connect4", 0), ("connect4", 8), ("gomoku7", 0), ("cartpole", 0),
         ("twentyone", 0), ("simple_grid", 3), ("gridworld", 0), ("breakout", 2)]
LENGTHS = (0, 9, 1, 20, 0, 3)                    # games of 0 and 1 positions, and longer than a chunk of 7


@pytest.mark.parametrize("B", [1, 7, 64])
@pytest.mark.parametrize("name,s", CASES, ids=[f"{n}-s{s}" for n, s in CASES])
def test_equals_the_host_route(name, s, B):
    """Host and CUDA frames: visit counts and root values == engine.search on host stacks, bit for bit."""
    cfg = _cfg(name, s, 6)
    eng = _engine(cfg, name, B)
    rs = numpy.random.RandomState(B + s)
    games, legal = _games(rs, cfg, LENGTHS)
    to_play = _to_play(games)
    gids = rs.randint(0, 1 << 40, len(games)).astype(numpy.int64)
    args = _packed(games)
    got_v, got_r = eng.reanalyse_search(*args, legal, to_play, gids)
    dev_v, dev_r = eng.reanalyse_search(*_device(args, legal, to_play), gids)
    want_v, want_r = _host_route(eng, games, s, legal, to_play, gids, B)
    eng.close()
    assert got_v.dtype == numpy.int32 and got_r.dtype == numpy.float64 and got_v.shape == (sum(LENGTHS), len(cfg.action_space))
    assert (want_v.sum(1) == cfg.num_simulations).all()
    assert numpy.array_equal(got_v, want_v) and numpy.array_equal(got_r.view(numpy.int64), want_r.view(numpy.int64))
    assert numpy.array_equal(dev_v.cpu().numpy(), want_v)
    assert numpy.array_equal(dev_r.cpu().numpy().view(numpy.int64), want_r.view(numpy.int64))


@pytest.mark.parametrize("name,s", [("tictactoe", 2), ("connect4", 8)])
def test_order_and_chunking_do_not_change_a_position(name, s):
    """Permuting the games and changing max_positions changes no position's result."""
    cfg = _cfg(name, s, 8)
    rs = numpy.random.RandomState(3)
    games, legal = _games(rs, cfg, (5, 12, 1, 30, 7))
    to_play = _to_play(games)
    gids = numpy.arange(len(games), dtype=numpy.int64) * 977
    T = [len(gh.root_values) for gh in games]
    first = numpy.concatenate([[0], numpy.cumsum(T)])
    results = []
    for B, perm in ((64, [0, 1, 2, 3, 4]), (5, [3, 0, 4, 2, 1]), (11, [4, 3, 2, 1, 0])):
        eng = _engine(cfg, name, B)
        sel = numpy.concatenate([numpy.arange(first[g], first[g + 1]) for g in perm])
        v, r = eng.reanalyse_search(*_packed([games[g] for g in perm]), legal[sel], to_play[sel], gids[perm])
        eng.close()
        back_v, back_r = numpy.empty_like(v), numpy.empty_like(r)
        back_v[sel], back_r[sel] = v, r
        results.append((back_v, back_r))
    for v, r in results[1:]:
        assert numpy.array_equal(v, results[0][0]) and numpy.array_equal(r, results[0][1])


@pytest.mark.parametrize("wide", ["0", "3"])
def test_atari_equals_the_host_route(wide, monkeypatch):
    """games/atari.py (16 x 256, s = 32), short games, N = 3, on the CUDA-core towers and on MZ_TC_WIDE=3, host and
    device frames: bit for bit the host route."""
    for k in ("MZ_TC_MODE", "MZ_NO_TC", "MZ_TC_WIDE"):
        monkeypatch.delenv(k, raising=False)
    if wide != "0":
        monkeypatch.setenv("MZ_TC_WIDE", wide)
    cfg = _cfg("atari", 32, 3)
    B = 16
    eng = _engine(cfg, "atari", B)
    rs = numpy.random.RandomState(5)
    games, legal = _games(rs, cfg, (20, 4))
    to_play = _to_play(games)
    gids = numpy.array([11, 12], numpy.int64)
    args = _packed(games)
    got_v, got_r = eng.reanalyse_search(*args, legal, to_play, gids)
    dev_v, dev_r = eng.reanalyse_search(*_device(args, legal, to_play), gids)
    want_v, want_r = _host_route(eng, games, 32, legal, to_play, gids, B)
    eng.close()
    assert numpy.isfinite(want_r).all()
    assert numpy.array_equal(got_v, want_v) and numpy.array_equal(got_r, want_r)
    assert numpy.array_equal(dev_v.cpu().numpy(), want_v) and numpy.array_equal(dev_r.cpu().numpy(), want_r)


@pytest.mark.parametrize("name", ["tictactoe", "connect4"])
def test_reproduces_the_device_self_play_searches(name):
    """Games played on the device loop, reanalysed with the same weights and seed, their own self-play game ids, legal
    masks from Game.legal_masks and noise on: the visit counts and root values the loop recorded, bit for bit."""
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 16, "philox", 12
    spec = netspec_from_config(cfg)
    w = weights_for(name, spec)
    seed = 3
    worker = sp.SelfPlay({"weights": w}, mod.Game, cfg, seed=seed)
    assert worker.loop_path == "device"
    games = []
    for _ in range(8):
        games += list(worker.play_moves(8, 1.0))
    worker.close()
    assert len(games) >= 8
    from muzero_general_b200.engine import SearchEngine
    eng = SearchEngine(cfg, max_games=32, seed=seed)
    eng.load_weights(w)
    sources = [ra._frame_source(gh) for gh in games]
    p = ra.pack_frames(sources)
    legal = numpy.concatenate([mod.Game.legal_masks(rows[:T].reshape((T,) + tuple(cfg.observation_shape)))
                               for rows, _, T in sources])
    to_play = numpy.concatenate([ra._to_play(gh, T) for gh, (_, _, T) in zip(games, sources)])
    visits, root = eng.reanalyse_search(p["frames"], p["frame_offsets"], p["actions"], p["action_offsets"],
                                        p["positions"], legal, to_play, [gh.game_id for gh in games])
    eng.close()
    block = [gh._packed[0] for gh in games]
    assert numpy.array_equal(visits, numpy.concatenate([g["visits"] for g in block]))
    assert numpy.array_equal(root, numpy.concatenate([g["root_value"] for g in block]))


def test_long_game_bounded_memory():
    """A games/atari.py-shaped game of 3000 moves (s = 32, 3 x 96 x 96 frames, a small net, N = 2): the device memory
    the call takes stays within mz_reanalyse_search's documented bound, the host builds no per-position stacks
    (tracemalloc peak: the frames plus one chunk's bookkeeping), and the first and last chunks equal the host route."""
    import torch
    T, B, s, A = 3000, 256, 32, 4
    cfg = _cfg("atari", s, 2, blocks=1, channels=16, reduced_channels_reward=2, reduced_channels_value=2,
               reduced_channels_policy=2, resnet_fc_reward_layers=[8], resnet_fc_value_layers=[8],
               resnet_fc_policy_layers=[8], reanalyse_search=True)
    spec = netspec_from_config(cfg)
    re = ra.Reanalyse({"weights": weights_for("atari", spec)}, cfg, max_positions=B, Game=load_game_module("atari").Game)
    eng = re.search_engine
    rs = numpy.random.RandomState(3)
    gh = _games(rs, cfg, (T,))[0][0]
    gh.to_play_history = [0] * (T + 1)
    for _ in range(2):                                     # the search's kernels are loaded and its graph captured
        eng.search(obs=numpy.zeros((B, spec.obs_elems), numpy.float32), legal_mask=numpy.ones((B, A), numpy.uint8),
                   add_exploration_noise=True)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    O = 3 * 96 * 96
    frames_bytes = (T + 1) * O * 4
    tracemalloc.start()
    visits, root, legal = re.fresh_search([gh], [0])[0]
    _, peak = tracemalloc.get_traced_memory()
    tracemalloc.stop()
    free2 = torch.cuda.mem_get_info()[0]
    bound = 2 * ((B + s) * (O + 1) * 4 + B * (32 + A) + 8 * 256)
    assert free1 - free2 <= bound + 16 * 1024 * 1024, (free1 - free2, bound)      # + module and graph memory
    assert peak <= frames_bytes + 16 * 1024 * 1024, (peak, frames_bytes)
    assert visits.shape == (T, A) and (visits.sum(1) == 2).all() and numpy.isfinite(root).all()
    assert (legal == 1).all()
    last = (T - 1) // B * B
    for lo in (0, last):
        hi = min(T, lo + B)
        stacks = numpy.stack([numpy.asarray(gh.get_stacked_observations(i, s, A), numpy.float32).reshape(-1)
                              for i in range(lo, hi)])
        out = eng.search(obs=stacks, legal_mask=legal[lo:hi], to_play=numpy.zeros(hi - lo, numpy.int32),
                         add_exploration_noise=True, game_id=numpy.full(hi - lo, re.SEARCH_GAME_IDS, numpy.int64),
                         move_index=numpy.arange(lo, hi, dtype=numpy.int32))
        assert numpy.array_equal(visits[lo:hi], out.visit_counts) and numpy.array_equal(root[lo:hi], out.root_value), lo
    re.close()


def _call(eng, games, legal, to_play, s=None, visits=True):
    keep = []
    io, total, _ = eng._reanalyse_io(*_packed(games), s, keep)
    sio = _lib.MzReanalyseSearchIO()
    sio.games = C.addressof(io)
    sio.legal_mask = legal.ctypes.data
    sio.to_play = to_play.ctypes.data
    sio.add_exploration_noise = 1
    v = numpy.full((max(total, 1), eng.A), 7, numpy.int32)
    r = numpy.full(max(total, 1), 7.0)
    sio.visit_counts = v.ctypes.data if visits else None
    sio.root_value = r.ctypes.data
    rc = eng.lib.mz_reanalyse_search(eng._h, C.byref(sio))
    return rc, eng.lib.mz_last_error(eng._h).decode(), v, r


def test_refusals_name_the_problem_and_write_nothing():
    """MZ_EINVAL with a message, the outputs untouched, for: the caller's s not the handle's, an action out of range,
    a position without a legal action, a to_play outside [0, num_players), no visit_counts; MZ_ESTATE for an
    inference-only handle."""
    cfg = _cfg("tictactoe", 0, 4)
    eng = _engine(cfg, "tictactoe", 8)
    games, legal = _games(numpy.random.RandomState(1), cfg, (4, 6))
    to_play = _to_play(games)
    rc, msg, v, r = _call(eng, games, legal, to_play)
    assert rc == 0 and (v.sum(1) == 4).all(), msg

    def expect(words, code=MZ_EINVAL, e=eng, g=games, lg=legal, tp=to_play, **kw):
        rc, msg, v, r = _call(e, g, lg, tp, **kw)
        assert rc == code and all(w in msg for w in words), msg
        assert (v == 7).all() and (r == 7.0).all()

    expect(["stacked_observations = 3", "implies s = 0"], s=3)
    bad = copy.deepcopy(games)
    bad[1].action_history[2] = 9
    expect(["action 9", "outside [0, 9)"], g=bad)
    lg = legal.copy()
    lg[6] = 0
    expect(["position 2 of game 1", "no legal action"], lg=lg)
    tp = to_play.copy()
    tp[3] = 2
    expect(["position 3 of game 0", "to_play 2", "outside [0, 2)"], tp=tp)
    expect(["visit_counts is required"], visits=False)
    eng.close()
    eng0 = _engine(cfg, "tictactoe", 8, N=0)
    expect(["num_simulations = 0"], code=MZ_ESTATE, e=eng0)
    eng0.close()


def test_reanalyse_games_end_to_end():
    """Reanalyse.reanalyse_games on games the device loop played (s = 2): child_visits are the store_visit_counts rows
    of the host route's searches under the ids SEARCH_GAME_IDS + buffer id, they survive pickling the
    PackedGameHistory, reanalysed_predicted_root_values are bit-identical with the option on and off, and with it off
    no search is made."""
    mod = load_game_module("tictactoe")
    cfg = mod.MuZeroConfig()
    cfg.stacked_observations, cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 2, 16, "philox", 10
    spec = netspec_from_config(cfg)
    w = weights_for("tictactoe", spec)
    worker = sp.SelfPlay({"weights": w}, mod.Game, cfg, seed=0)
    games = []
    for _ in range(4):
        games += list(worker.play_moves(6, 1.0))
    worker.close()
    assert len(games) >= 4 and all(isinstance(g, sp.PackedGameHistory) for g in games)
    ids = [100 + 3 * k for k in range(len(games))]
    B = 16
    off = ra.Reanalyse({"weights": w}, cfg, max_positions=B)
    assert off.search_engine is None
    plain = off.reanalyse_games([copy.deepcopy(g) for g in games], ids)
    off.close()
    cfg_on = copy.deepcopy(cfg)
    cfg_on.reanalyse_search = True
    on = ra.Reanalyse({"weights": w}, cfg_on, max_positions=B, Game=mod.Game)
    done = on.reanalyse_games(games, ids)
    for a, b in zip(plain, done):
        assert numpy.array_equal(numpy.atleast_1d(a.reanalysed_predicted_root_values).view(numpy.int32),
                                 numpy.atleast_1d(b.reanalysed_predicted_root_values).view(numpy.int32))
    legal = numpy.concatenate([mod.Game.legal_masks(numpy.stack(gh.observation_history[:len(gh.root_values)]))
                               for gh in copy.deepcopy(done)])
    to_play = _to_play(copy.deepcopy(done))
    want_v, _ = _host_route(on.search_engine, copy.deepcopy(done), 2, legal, to_play,
                            [on.SEARCH_GAME_IDS + i for i in ids], B)
    want = ra.policy_rows(want_v, legal, cfg.action_space)
    got = [row for gh in done for row in gh.child_visits]
    assert got == want
    again = [pickle.loads(pickle.dumps(gh)) for gh in done]
    assert [row for gh in again for row in gh.child_visits] == want
    assert all(type(gh) is sp.GameHistory for gh in again)
    on.close()


def test_search_noise_is_not_a_self_play_draw():
    """The same positions searched as self-play would (self-play seeds config.seed + worker index, game id k, move i)
    and as Reanalyse does (its search handle, game id SEARCH_GAME_IDS + k): the root Dirichlet noise differs at every
    position, and so, in aggregate, do the visit counts."""
    from muzero_general_b200.engine import SearchEngine
    cfg = _cfg("tictactoe", 0, 25, reanalyse_search=True)
    spec = netspec_from_config(cfg)
    w = weights_for("tictactoe", spec)
    re = ra.Reanalyse({"weights": w}, cfg, max_positions=32, Game=load_game_module("tictactoe").Game)
    rs = numpy.random.RandomState(8)
    n, A = 32, spec.action_space
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    legal = numpy.ones((n, A), numpy.uint8)
    k = numpy.arange(n, dtype=numpy.int64) % 4
    move = (numpy.arange(n) // 4).astype(numpy.int32)

    def search(eng, ids):
        out = eng.search(obs=obs, legal_mask=legal, to_play=numpy.zeros(n, numpy.int32), add_exploration_noise=True,
                         game_id=ids, move_index=move, trace=True)
        return out.trace["noise"], out.visit_counts

    mine_noise, mine_visits = search(re.search_engine, re.SEARCH_GAME_IDS + k)
    assert numpy.isfinite(mine_noise).all() and (mine_noise > 0).any(axis=1).all()
    for worker in range(3):
        eng = SearchEngine(cfg, max_games=n, seed=cfg.seed + worker)
        eng.load_weights(w)
        noise, visits = search(eng, k)
        eng.close()
        assert (noise != mine_noise).any(axis=1).all(), worker
        assert not numpy.array_equal(visits, mine_visits), worker
    re.close()
