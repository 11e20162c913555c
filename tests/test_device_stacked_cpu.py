"""Stacked observations on the device self-play loop, host side: a config with stacked_observations > 0 takes the device
loop and hands its stacked_observations to DeviceSelfPlayLoop, and the descriptor field that carries it sits where the
header puts it."""
import ctypes as C

import pytest

from conftest import weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import _lib
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from test_eval_cpu import _FakeLoop


class _StackLoop(_FakeLoop):
    def __init__(self, *args, stacked_observations=0, **kw):
        super().__init__(*args, **kw)
        self.stacked = stacked_observations


@pytest.fixture()
def fake_device(monkeypatch):
    monkeypatch.setattr(sp, "SearchEngine", FakeSearchEngine)
    monkeypatch.setattr(sp, "DeviceSelfPlayLoop", _StackLoop)
    _FakeLoop.made = []


def _worker(name, **over):
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 4, "philox", 2
    for k, v in over.items():
        setattr(cfg, k, v)
    return sp.SelfPlay({"weights": weights_for(name, netspec_from_config(cfg))}, mod.Game, cfg, 0)


@pytest.mark.parametrize("name", ["cartpole", "tictactoe", "connect4", "gomoku", "twentyone", "simple_grid"])
def test_stacked_config_takes_the_device_loop(name, fake_device):
    assert _worker(name, stacked_observations=2).loop_path == "device"
    assert _worker(name, stacked_observations=2, device_envs=False).loop_path == "host"
    assert _worker(name, stacked_observations=2, rng_mode="numpy").loop_path == "host"


@pytest.mark.parametrize("s", [0, 2, 8])
def test_stacked_observations_reach_the_device_loop(s, fake_device):
    """Self-play and test games both build their loop with the config's stacked_observations."""
    worker = _worker("tictactoe", stacked_observations=s)
    worker.play_moves(1, 1.0)
    assert _FakeLoop.made[-1].stacked == s and _FakeLoop.made[-1].kw["opponent"] == "self"
    worker.reset_stream()
    games, _ = worker.play_test_games(4)
    assert len(games) == 4
    assert _FakeLoop.made[-1].stacked == s and _FakeLoop.made[-1].kw["opponent"] == "expert"


def test_descriptor_field_keeps_the_layout():
    """stacked_observations takes the int32 after td_steps; per_alpha and the size stay where they were."""
    d = _lib.MzSelfPlayDesc
    names = [f[0] for f in d._fields_]
    assert "reserved" not in names and names.index("stacked_observations") == names.index("td_steps") + 1
    assert (d.stacked_observations.offset, d.stacked_observations.size) == (36, 4)
    assert d.td_steps.offset == 32 and d.per_alpha.offset == 40 and C.sizeof(d) == 64
