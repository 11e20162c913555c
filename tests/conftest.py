import json
import os
import sys

import numpy
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def golden_json(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def golden_npz(name):
    return dict(numpy.load(os.path.join(GOLDEN, name)))


@pytest.fixture(scope="session")
def game_configs():
    from muzero_general_b200.games import load_game_module
    return {n: load_game_module(n).MuZeroConfig() for n in ("cartpole", "tictactoe", "connect4", "breakout", "atari", "gomoku")}


def weights_for(name, spec):
    """Weights matching the golden fixtures: synthetic seed 0, or the shipped CartPole checkpoint."""
    from muzero_general_b200.netspec import stress_weights, synthetic_weights
    if name == "cartpole_pretrained":
        return golden_npz("weights_cartpole_pretrained.npz")
    if "_stress_" in name:                      # e.g. connect4_stress_large (oracle/gen_golden.py::main_round2)
        return stress_weights(spec, 0, name.rsplit("_", 1)[1])
    return synthetic_weights(spec, 0)
