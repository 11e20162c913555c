"""Reanalyse with stacked observations on the device (mz_reanalyse_values, csrc/reanalyse.cu): the stacked inputs each
chunk builds against GameHistory.get_stacked_observations byte for byte, the values against the host route (host
stacks through mz_initial_inference with the same chunk boundaries) bit for bit and against the fp64 oracle, bounded
device and host memory on a long games/atari.py-shaped game, the refusals, and Reanalyse.reanalyse end to end on games
the device self-play loop played."""
import copy
import ctypes as C
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

MZ_EINVAL = -1                                  # include/mzb200.h


def _cfg(name, s, **over):
    cfg = load_game_module(name).MuZeroConfig()
    cfg.stacked_observations = s
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def _engine(cfg, name, B):
    from muzero_general_b200.engine import SearchEngine
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=0)
    w = weights_for(name, spec)
    eng.load_weights(w)
    return eng, spec, w


def _games(rs, cfg, lengths, dtype, extra_frames=0):
    """Seeded histories of T moves each (T + 1 observations in `dtype`, the action history with its leading 0)."""
    A = len(cfg.action_space)
    out = []
    for T in lengths:
        gh = sp.GameHistory()
        gh.action_history = [0] + [int(a) for a in rs.randint(0, A, T)]
        shape = tuple(cfg.observation_shape)
        if numpy.dtype(dtype).kind == "i":
            gh.observation_history = [rs.randint(-1, 3, shape).astype(dtype) for _ in range(T + 1 + extra_frames)]
        else:
            gh.observation_history = [rs.random_sample(shape).astype(dtype) for _ in range(T + 1 + extra_frames)]
        gh.root_values = [0.0] * T
        out.append(gh)
    return out


def _host_stacks(games, s, A):
    return [numpy.asarray(gh.get_stacked_observations(i, s, A), dtype=numpy.float32).reshape(-1)
            for gh in games for i in range(len(gh.root_values))]


def _packed(games):
    return ra.pack_frames([ra._frame_source(gh) for gh in games])


def _args(p):
    return p["frames"], p["frame_offsets"], p["actions"], p["action_offsets"], p["positions"]


# (game, s, max_games, game lengths, frame dtype): positions i < s, one-position games, chunk boundaries inside a game
# and chunks spanning many games in every case
STACK_CASES = [
    ("tictactoe", 3, 4, (1, 2, 5, 9, 9, 3, 1), numpy.int32),
    ("tictactoe", 12, 7, (1, 5, 9, 2, 9, 1, 1, 4), numpy.float64),
    ("connect4", 8, 16, (1, 7, 20, 42, 13, 3), numpy.float32),
    ("cartpole", 4, 16, (1, 3, 30, 57, 2), numpy.float64),
    ("simple_grid", 8, 5, (1, 4, 12, 6, 1, 2), numpy.int32),
    ("breakout", 2, 4, (1, 2, 9, 3), numpy.float32),
    ("atari", 32, 16, (1, 5, 40, 3), numpy.float32),
]


@pytest.mark.parametrize("name,s,B,lengths,dtype", STACK_CASES, ids=[f"{c[0]}-s{c[1]}" for c in STACK_CASES])
def test_stacked_inputs_byte_for_byte(name, s, B, lengths, dtype):
    """Every chunk's stacked inputs (mz_debug_reanalyse_stack) == numpy.asarray(gh.get_stacked_observations(i, s, A),
    float32), bit for bit, for float32, float64 and int32 observations."""
    cfg = _cfg(name, s)
    eng, spec, _ = _engine(cfg, name, B)
    games = _games(numpy.random.RandomState(7), cfg, lengths, dtype)
    want = _host_stacks(games, s, spec.action_space)
    p = _packed(games)
    chunks = -(-sum(lengths) // B)
    got = numpy.concatenate([eng.debug_reanalyse_stack(c, *_args(p)) for c in range(chunks)])
    eng.close()
    assert got.shape == (len(want), spec.obs_elems)
    for q, w in enumerate(want):
        assert numpy.array_equal(got[q].view(numpy.uint32), w.view(numpy.uint32)), (name, q)


def _host_route(eng, stacks, B):
    """The host route: host stacks through mz_initial_inference, chunks of max_games positions."""
    out = [eng.initial_inference(numpy.stack(stacks[lo:lo + B]))["value"] for lo in range(0, len(stacks), B)]
    return numpy.concatenate(out)


VALUE_CASES = [c for c in STACK_CASES if c[0] != "atari"]


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("name,s,B,lengths,dtype", VALUE_CASES, ids=[f"{c[0]}-s{c[1]}" for c in VALUE_CASES])
def test_values_equal_the_host_route_and_the_oracle(name, s, B, lengths, dtype, mem):
    """reanalyse_values == the host route bit for bit (the same network calls on the same inputs: every route is
    deterministic for a given batch), and the fp64 oracle at test_batched_reanalyse_on_device's tolerances."""
    import torch
    from oracle.net import OracleNet, support_to_scalar
    cfg = _cfg(name, s)
    eng, spec, w = _engine(cfg, name, B)
    games = _games(numpy.random.RandomState(11), cfg, lengths, dtype)
    stacks = _host_stacks(games, s, spec.action_space)
    p = _packed(games)
    if mem == "device":
        frames, fo, actions, ao, pos = _args(p)
        got = eng.reanalyse_values(torch.from_numpy(frames).cuda(), fo, torch.from_numpy(actions).cuda(), ao, pos)
        got = got.cpu().numpy()
    else:
        got = eng.reanalyse_values(*_args(p))
    want = _host_route(eng, stacks, B)
    eng.close()
    assert got.dtype == numpy.float32 and numpy.array_equal(got, want), numpy.abs(got - want).max()
    net = OracleNet(spec, w)
    x = numpy.stack(stacks).reshape((len(stacks), spec.in_channels) + tuple(spec.obs_shape[1:]))
    ref = support_to_scalar(net.initial_inference(x)[0], cfg.support_size).numpy()[:, 0]
    numpy.testing.assert_allclose(got, ref, rtol=2e-4, atol=5e-4)


@pytest.mark.parametrize("wide", ["0", "3"])
def test_atari_values_equal_the_host_route(wide, monkeypatch):
    """games/atari.py (16 x 256, s = 32) with 80-move games, on the CUDA-core towers and on MZ_TC_WIDE=3, with host and
    device frames: bit for bit the host route."""
    import torch
    for k in ("MZ_TC_MODE", "MZ_NO_TC", "MZ_TC_WIDE"):
        monkeypatch.delenv(k, raising=False)
    if wide != "0":
        monkeypatch.setenv("MZ_TC_WIDE", wide)
    cfg = _cfg("atari", 32)
    B = 64
    eng, spec, _ = _engine(cfg, "atari", B)
    games = _games(numpy.random.RandomState(5), cfg, (80, 80), numpy.float32)
    p = _packed(games)
    got_host = eng.reanalyse_values(*_args(p))
    frames, fo, actions, ao, pos = _args(p)
    got_dev = eng.reanalyse_values(torch.from_numpy(frames).cuda(), fo, torch.from_numpy(actions).cuda(), ao, pos).cpu().numpy()
    want = _host_route(eng, _host_stacks(games, 32, spec.action_space), B)
    eng.close()
    assert numpy.isfinite(want).all()
    assert numpy.array_equal(got_host, want) and numpy.array_equal(got_dev, want)


def test_long_game_bounded_memory():
    """A games/atari.py-shaped game of 3000 moves (s = 32, 3 x 96 x 96 frames; a small net, the stack is under test):
    the device memory the call takes stays within the staging bound of mz_reanalyse_values, the host builds no
    per-position stacks (tracemalloc peak: the frames plus one chunk's bookkeeping), and sampled positions - the first
    s + 1, both sides of every chunk boundary, the last - equal host stacks; the values are the host route's."""
    import torch
    T, B, s = 3000, 256, 32
    cfg = _cfg("atari", s, blocks=1, channels=16, reduced_channels_reward=2, reduced_channels_value=2,
               reduced_channels_policy=2, resnet_fc_reward_layers=[8], resnet_fc_value_layers=[8],
               resnet_fc_policy_layers=[8])
    spec = netspec_from_config(cfg)
    re = ra.Reanalyse({"weights": weights_for("atari", spec)}, cfg, max_positions=B)
    eng = re.engine
    gh = _games(numpy.random.RandomState(3), cfg, (T,), numpy.float32)[0]
    eng.initial_inference(numpy.zeros((2, spec.obs_elems), numpy.float32))      # the network's kernels are loaded
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    O = 3 * 96 * 96
    frames_bytes = (T + 1) * O * 4
    tracemalloc.start()
    values = re.fresh_root_values([gh])[0]
    _, peak = tracemalloc.get_traced_memory()
    tracemalloc.stop()
    free2 = torch.cuda.mem_get_info()[0]
    staging = 2 * ((B + s) * (O + 1) * 4 + B * 20)
    assert free1 - free2 <= staging + 16 * 1024 * 1024, (free1 - free2, staging)     # + the stack kernel's module
    assert peak <= frames_bytes + 16 * 1024 * 1024, (peak, frames_bytes)
    assert values.shape == (T,) and values.dtype == numpy.float32 and numpy.isfinite(values).all()
    sample = sorted(set(range(s + 1)) | {c * B + d for c in range(1, -(-T // B)) for d in (-1, 0)} | {T - 1})
    p = _packed([gh])
    for c in sorted({i // B for i in sample}):
        got = eng.debug_reanalyse_stack(c, *_args(p))
        for i in sample:
            if i // B == c:
                want = numpy.asarray(gh.get_stacked_observations(i, s, 4), numpy.float32).reshape(-1)
                assert numpy.array_equal(got[i - c * B], want), i
    # the host route on the first and the last chunk: bit for bit
    last = (T - 1) // B * B
    for lo in (0, last):
        stacks = [numpy.asarray(gh.get_stacked_observations(i, s, 4), numpy.float32).reshape(-1)
                  for i in range(lo, min(T, lo + B))]
        assert numpy.array_equal(values[lo:lo + len(stacks)], _host_route(eng, stacks, B)), lo
    re.close()


def _call(eng, p, s=None, values=None):
    io, keep = None, []
    io, total, _ = eng._reanalyse_io(p["frames"], p["frame_offsets"], p["actions"], p["action_offsets"], p["positions"],
                                     s, keep)
    out = numpy.full(max(total, 1), 7.0, numpy.float32) if values is None else values
    io.values = out.ctypes.data
    rc = eng.lib.mz_reanalyse_values(eng._h, C.byref(io))
    return rc, eng.lib.mz_last_error(eng._h).decode(), out


def test_refusals_name_the_problem_and_write_nothing():
    """MZ_EINVAL with a message, and the values untouched, for: the caller's s not the handle's, frames of an O that
    does not fit, decreasing offsets, T_g > frames_g, an action history shorter than T_g, an action out of range."""
    cfg = _cfg("tictactoe", 3)
    eng, spec, _ = _engine(cfg, "tictactoe", 8)
    games = _games(numpy.random.RandomState(1), cfg, (4, 6), numpy.float32)
    good = _packed(games)
    rc, msg, out = _call(eng, good)
    assert rc == 0 and numpy.isfinite(out).all()

    def expect(p, words, s=None):
        rc, msg, out = _call(eng, p, s)
        assert rc == MZ_EINVAL and all(w in msg for w in words), msg
        assert (out == 7.0).all()

    expect(good, ["stacked_observations = 8", "implies s = 3"], s=8)
    bad = copy.deepcopy(good)
    bad["frames"] = numpy.zeros((len(bad["frames"]), 26), numpy.float32)
    expect(bad, ["O = 26", "obs_elems"])
    bad = copy.deepcopy(good)
    bad["frame_offsets"] = numpy.array([0, 5, 4], numpy.int64)
    expect(bad, ["non-decreasing"])
    bad = copy.deepcopy(good)
    bad["positions"] = numpy.array([6, 6], numpy.int64)              # game 0 has 5 frames
    expect(bad, ["game 0", "positions must be in [0, frames]"])
    bad = copy.deepcopy(good)
    bad["action_offsets"] = numpy.array([0, 3, 10], numpy.int64)     # game 0: 3 actions for 4 positions
    expect(bad, ["game 0", "action history of 3"])
    bad = copy.deepcopy(good)
    bad["actions"][7] = 9
    expect(bad, ["action 9", "outside [0, 9)"])
    eng.close()
    # a handle built for a different s refuses these frames
    eng8, _, _ = _engine(_cfg("tictactoe", 8), "tictactoe", 8)
    rc, msg, out = _call(eng8, good, s=3)
    assert rc == MZ_EINVAL and "implies s = 8" in msg and (out == 7.0).all(), msg
    eng8.close()


def test_reanalyse_end_to_end_on_device_games():
    """Games played with s = 2 on the device self-play loop (PackedGameHistory), through Reanalyse.reanalyse against a
    buffer and storage stand-in, then handed on with save_games: the reanalysed values are the host route's and the
    priorities use them."""
    mod = load_game_module("tictactoe")
    cfg = mod.MuZeroConfig()
    cfg.stacked_observations, cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 2, 16, "philox", 6
    cfg.training_steps, cfg.PER, cfg.td_steps = 3, True, 2          # bootstrap values inside the games: they are read
    spec = netspec_from_config(cfg)
    w = weights_for("tictactoe", spec)
    worker = sp.SelfPlay({"weights": w}, mod.Game, cfg, seed=0)
    assert worker.loop_path == "device"
    games = []
    for _ in range(6):
        games += list(worker.play_moves(4, 1.0))
    worker.close()
    assert len(games) >= 6 and all(isinstance(g, sp.PackedGameHistory) for g in games)

    class Storage:
        def __init__(self):
            self.d = dict(weights=w, training_step=0, terminate=False, num_played_games=len(games), num_reanalysed_games=0)
        def get_info(self, k):
            if k == "training_step":
                self.d[k] += 1
            return self.d[k]
        def set_info(self, k, v=None):
            self.d.update(k if isinstance(k, dict) else {k: v})

    class Buffer:
        def __init__(self):
            self.buffer, self.updated, self.saved = dict(enumerate(games)), set(), []
        def sample_game(self, force_uniform=False):
            i = int(numpy.random.randint(len(self.buffer)))
            return i, self.buffer[i], None
        def update_game_history(self, game_id, gh):
            self.updated.add(game_id); self.buffer[game_id] = gh
        def save_game(self, gh, storage=None):
            self.saved.append(gh)

    B = 32
    actor = ra.Reanalyse({"weights": w, "num_reanalysed_games": 0}, cfg, max_positions=B, games_per_call=len(games))
    st, buf = Storage(), Buffer()
    actor.reanalyse(buf, st)
    assert buf.updated and st.d["num_reanalysed_games"] == actor.num_reanalysed_games > 0
    done = [buf.buffer[i] for i in sorted(buf.updated)]
    for gh in done:
        assert "observation_history" not in gh.__dict__          # reanalysed without building the lists
    want = _host_route(actor.engine, _host_stacks(done, 2, spec.action_space), B)
    got = numpy.concatenate([numpy.atleast_1d(gh.reanalysed_predicted_root_values) for gh in done])
    assert numpy.array_equal(got, want)
    for gh in done:
        gh.priorities = None
    ra.save_games(buf, done, cfg)
    for gh in buf.saved:
        plain = copy.deepcopy(gh)
        plain.reanalysed_predicted_root_values, plain.priorities = None, None
        pri, top = ra.initial_priorities(gh, cfg)
        assert numpy.array_equal(gh.priorities, pri) and gh.game_priority == top
        assert not numpy.array_equal(pri, ra.initial_priorities(plain, cfg)[0])
    actor.close()
