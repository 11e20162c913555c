"""Host side of Reanalyse with stacked observations (muzero_general_b200/reanalyse.py): what Reanalyse.fresh_root_values
hands to SearchEngine.reanalyse_values for GameHistory and PackedGameHistory inputs (offsets, float32 frames, int32
action histories, positions; no per-position stack), the s = 0 route's chunked gathering, and the resources of the
self-play kernels whose stack rule mz_reanalyse_values shares (csrc/stack.cuh)."""
import os
import re
import shutil
import subprocess

import numpy
import pytest
import torch

from conftest import weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import build as b
from muzero_general_b200 import reanalyse as ra
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config

torch.set_num_threads(1)


class RecordingEngine:
    """Stand-in for SearchEngine that records reanalyse_values' arguments and answers each position with a value
    that encodes (game, position): 1000 g + i."""

    def __init__(self, config, max_games=1, device=0, num_simulations=None, **_):
        self.config, self.max_games, self.calls = config, max_games, []

    def load_weights(self, w):
        pass

    def close(self):
        pass

    def reanalyse_values(self, frames, frame_offsets, actions, action_offsets, positions, stacked_observations=None):
        self.calls.append(dict(frames=frames, frame_offsets=frame_offsets, actions=actions, action_offsets=action_offsets,
                               positions=positions))
        return numpy.concatenate([1000.0 * g + numpy.arange(T) for g, T in enumerate(positions)]).astype(numpy.float32)


def _history(rs, shape, A, T, dtype):
    gh = sp.GameHistory()
    gh.action_history = [0] + [int(a) for a in rs.randint(0, A, T)]
    if numpy.dtype(dtype).kind == "i":
        gh.observation_history = [rs.randint(-1, 3, shape).astype(dtype) for _ in range(T + 1)]
    else:
        gh.observation_history = [rs.random_sample(shape).astype(dtype) for _ in range(T + 1)]
    gh.root_values = [0.5] * T
    return gh


def _packed_history(rs, shape, A, T):
    """A PackedGameHistory over a hand-made block (the fields mz_selfplay_drain stages)."""
    O = int(numpy.prod(shape))
    block = dict(game_id=3, slot=0, length=T, first_to_play=0, root_value=rs.standard_normal(T),
                 visits=rs.randint(1, 5, (T, A)).astype(numpy.int32), action=rs.randint(0, A, T).astype(numpy.int32),
                 reward=numpy.zeros(T, numpy.float32), to_play=numpy.zeros(T, numpy.int32),
                 priority=numpy.zeros(T, numpy.float32), obs=rs.random_sample((T + 1, O)).astype(numpy.float32))
    return sp.PackedGameHistory(block, shape, numpy.float64, float)


def _actor(monkeypatch, name, s, max_positions=7):
    monkeypatch.setattr(ra, "SearchEngine", RecordingEngine)
    cfg = load_game_module(name).MuZeroConfig()
    cfg.stacked_observations = s
    return ra.Reanalyse({"weights": {}}, cfg, max_positions=max_positions), cfg


def test_packing_of_game_histories_and_packed_games(monkeypatch):
    """One call per fresh_root_values: frames [sum (T + 1)][O] float32 (float32, float64 and int32 observations, each
    rounded once like the host's .float()), action histories int32 with their leading 0, int64 offsets and positions;
    a PackedGameHistory gives its block's sections and its lists stay unbuilt; the values come back per game in the
    reference's shapes."""
    actor, cfg = _actor(monkeypatch, "tictactoe", 3)
    rs = numpy.random.RandomState(0)
    shape, A = tuple(cfg.observation_shape), len(cfg.action_space)
    games = [_history(rs, shape, A, 4, numpy.float64), _history(rs, shape, A, 1, numpy.int32),
             _packed_history(rs, shape, A, 6), _history(rs, shape, A, 0, numpy.float32),
             _history(rs, shape, A, 3, numpy.float32)]
    out = actor.fresh_root_values(games)
    assert len(actor.engine.calls) == 1
    call = actor.engine.calls[0]
    assert call["frames"].dtype == numpy.float32 and call["actions"].dtype == numpy.int32
    assert call["frame_offsets"].dtype == call["action_offsets"].dtype == call["positions"].dtype == numpy.int64
    assert call["frame_offsets"].tolist() == [0, 5, 7, 14, 15, 19]
    assert call["action_offsets"].tolist() == [0, 5, 7, 14, 15, 19]
    assert call["positions"].tolist() == [4, 1, 6, 0, 3]
    assert "observation_history" not in games[2].__dict__                       # the packed lists were not built
    for g, gh in enumerate(games):
        lo, hi = call["frame_offsets"][g], call["frame_offsets"][g + 1]
        want = numpy.stack([numpy.asarray(o, numpy.float32).reshape(-1) for o in gh.observation_history])
        assert numpy.array_equal(call["frames"][lo:hi], want), g
        lo, hi = call["action_offsets"][g], call["action_offsets"][g + 1]
        assert call["actions"][lo:hi].tolist() == [int(a) for a in gh.action_history], g
    assert [v.shape for v in out] == [(4,), (), (6,), (0,), (3,)]
    assert all(v.dtype == numpy.float32 for v in out)
    assert out[2].tolist() == [2000.0 + i for i in range(6)] and float(out[1]) == 1000.0


def test_games_without_positions_make_no_call(monkeypatch):
    actor, cfg = _actor(monkeypatch, "tictactoe", 2)
    rs = numpy.random.RandomState(1)
    out = actor.fresh_root_values([_history(rs, tuple(cfg.observation_shape), 9, 0, numpy.float32)])
    assert not actor.engine.calls and out[0].shape == (0,)


def _today(actor, games):
    """fresh_root_values as it was before chunked gathering: every position stacked up front, then chunks."""
    cfg = actor.config
    A = len(cfg.action_space)
    obs = [numpy.asarray(gh.get_stacked_observations(i, cfg.stacked_observations, A), dtype=numpy.float32)
           for gh in games for i in range(len(gh.root_values))]
    obs = numpy.stack(obs).reshape(len(obs), -1)
    values = numpy.empty(len(obs), numpy.float32)
    for lo in range(0, len(obs), actor.max_positions):
        values[lo:lo + actor.max_positions] = actor.engine.initial_inference(obs[lo:lo + actor.max_positions])["value"]
    return values


@pytest.mark.parametrize("name", ["tictactoe", "cartpole"])
def test_unstacked_route_gathers_chunk_by_chunk(name, monkeypatch):
    """s = 0: initial_inference per max_positions positions, each chunk gathered when it is due, and the values of the
    route that stacked every position first; a PackedGameHistory is read from its block."""
    monkeypatch.setattr(ra, "SearchEngine", FakeSearchEngine)
    cfg = load_game_module(name).MuZeroConfig()
    assert cfg.stacked_observations == 0
    spec = netspec_from_config(cfg)
    actor = ra.Reanalyse({"weights": weights_for(name, spec)}, cfg, max_positions=5)
    rs = numpy.random.RandomState(2)
    shape, A = tuple(cfg.observation_shape), len(cfg.action_space)
    games = [_history(rs, shape, A, T, dt) for T, dt in ((3, numpy.float64), (1, numpy.int32), (9, numpy.float32))]
    games.append(_packed_history(rs, shape, A, 4))
    sizes = []
    real = actor.engine.initial_inference
    actor.engine.initial_inference = lambda obs: (sizes.append(len(obs)), real(obs))[1]
    got = actor.fresh_root_values(games)
    assert sizes == [5, 5, 5, 2]
    actor.engine.initial_inference = real
    want = _today(actor, games)
    assert numpy.array_equal(numpy.concatenate([numpy.atleast_1d(v) for v in got]), want)
    assert got[1].shape == () and got[0].shape == (3,)


def _cuobjdump():
    nvcc = os.path.realpath(b.NVCC) if os.path.exists(b.NVCC) else shutil.which("nvcc")
    if not nvcc:
        return None
    path = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    return path if os.path.exists(path) else None


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not found next to nvcc")
def test_selfplay_kernels_keep_their_resources():
    """stack_fill and reanalyse_stack_kernel share the stack rule (stack_tail_element); the self-play kernels keep their
    resources: selfplay_step_kernel<128> 54 registers and a 1072-byte stack frame (<256>: 54, 2096), no spills."""
    assert os.path.exists(b.LIB), "build the library first (python -m muzero_general_b200.build)"
    out = subprocess.run([_cuobjdump(), "-res-usage", b.LIB], capture_output=True, text=True, check=True).stdout
    res = {fn: tuple(map(int, v)) for fn, *v in
           re.findall(r"Function (\S*(?:selfplay_step|reanalyse_stack)\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    step = {fn: v for fn, v in res.items() if "selfplay_step_kernel" in fn}
    assert sorted(step.values()) == [(54, 1072, 0), (54, 2096, 0)], step
    stack = [v for fn, v in res.items() if "reanalyse_stack_kernel" in fn]
    assert stack and all(local == 0 and st == 0 for _, st, local in stack), stack
