"""Bulk callers either side of the self-play path (muzero_general_b200/reanalyse.py) on the CPU: PER priorities against
those of the unmodified reference ReplayBuffer, batched Reanalyse against the oracle network."""
import copy

import numpy
import pytest
import torch

from conftest import golden_npz, weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import reanalyse as ra
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config

torch.set_num_threads(1)


def _random_history(rs, cfg, T, players):
    gh = sp.GameHistory()
    A = len(cfg.action_space)
    gh.action_history = [0] + [int(a) for a in rs.randint(0, A, T)]
    gh.observation_history = [rs.random_sample(cfg.observation_shape).astype(numpy.float32) for _ in range(T + 1)]
    gh.reward_history = [0] + [float(r) for r in rs.choice([0.0, 1.0, -1.0, 0.5], T)]
    gh.to_play_history = [int(i % players) for i in range(T + 1)] if players > 1 else [0] * (T + 1)
    cv = rs.random_sample((T, A)); gh.child_visits = (cv / cv.sum(1, keepdims=True)).tolist()
    gh.root_values = [float(v) for v in rs.standard_normal(T)]
    return gh


PRIORITY_CASES = [("tictactoe", 20, 1, 0.5, False), ("cartpole", 50, 0.997, 0.5, False), ("cartpole", 7, 0.9, 1.0, True),
                  ("connect4", 3, 1, 0.7, True)]
PRIORITY_LENGTHS = (1, 2, 9, 42, 130)


def priority_histories(name, td, reanalysed, cfg):
    """(fixture key, GameHistory) of the seeded histories the priority fixtures were computed on."""
    rs = numpy.random.RandomState(4)
    for T in PRIORITY_LENGTHS:
        gh = _random_history(rs, cfg, T, len(cfg.players))
        if reanalysed:
            gh.reanalysed_predicted_root_values = rs.standard_normal(T).astype(numpy.float32)
        yield f"{name}_td{td}_T{T}", gh


class _Recorder:
    def __init__(self):
        self.buffer = []

    def save_game(self, game_history, shared_storage=None):
        self.buffer.append(game_history)


@pytest.mark.parametrize("name,td,discount,alpha,reanalysed", PRIORITY_CASES)
def test_bulk_priorities_equal_the_reference_save_game(name, td, discount, alpha, reanalysed):
    """initial_priorities == what the unmodified ReplayBuffer.save_game computed (tests/golden/per_priorities.npz, from
    oracle/gen_golden.py --priorities), bit for bit (float32 priorities, game priority), for one- and two-player games,
    with and without reanalysed values, short and long td horizons; save_games hands them to the buffer as they are."""
    cfg = load_game_module(name).MuZeroConfig()
    cfg.td_steps, cfg.discount, cfg.PER_alpha, cfg.PER = td, discount, alpha, True
    gold = golden_npz("per_priorities.npz")
    for key, gh in priority_histories(name, td, reanalysed, cfg):
        mine, top = ra.initial_priorities(copy.deepcopy(gh), cfg)
        assert mine.dtype == gold[key].dtype == numpy.float32
        assert numpy.array_equal(mine, gold[key]), key
        assert top == gold[key + "_top"]
        buf = _Recorder()
        ra.save_games(buf, [copy.deepcopy(gh)], cfg)
        assert numpy.array_equal(buf.buffer[0].priorities, gold[key]) and buf.buffer[0].game_priority == top


def test_batched_reanalyse_matches_per_game_inference(monkeypatch):
    """One batched call over many games == the reference's per-game computation (replay_buffer.py:345-366) done with
    the oracle network; the actor loop updates the buffer and the counter."""
    from oracle.net import OracleNet, support_to_scalar
    monkeypatch.setattr(ra, "SearchEngine", FakeSearchEngine)
    mod = load_game_module("tictactoe")
    cfg = mod.MuZeroConfig()
    cfg.training_steps = 3
    spec = netspec_from_config(cfg)
    w = weights_for("tictactoe", spec)
    rs = numpy.random.RandomState(2)
    games = [_random_history(rs, cfg, T, 2) for T in (1, 5, 9, 3)]
    for g in games:
        g.observation_history = [rs.randint(0, 2, cfg.observation_shape).astype(numpy.int32) for _ in g.observation_history]
    actor = ra.Reanalyse({"weights": w, "num_reanalysed_games": 0}, cfg, max_positions=7)      # forces several chunks
    actor.reanalyse_games(games)
    net = OracleNet(spec, w)
    for g in games:
        T = len(g.root_values)
        obs = numpy.array([g.get_stacked_observations(i, cfg.stacked_observations, 9) for i in range(T)], dtype=numpy.float32)
        want = torch.squeeze(support_to_scalar(net.initial_inference(obs)[0], cfg.support_size)).numpy()
        assert g.reanalysed_predicted_root_values.shape == want.shape and g.reanalysed_predicted_root_values.dtype == numpy.float32
        numpy.testing.assert_allclose(g.reanalysed_predicted_root_values, want, rtol=1e-6, atol=1e-7)
    assert actor.num_reanalysed_games == 4

    class Storage:
        def __init__(self):
            self.d = dict(weights=w, training_step=0, terminate=False, num_played_games=4, num_reanalysed_games=0)
        def get_info(self, k):
            if k == "training_step":
                self.d[k] += 1
            return self.d[k]
        def set_info(self, k, v=None):
            self.d.update(k if isinstance(k, dict) else {k: v})

    class Buffer:
        def __init__(self):
            self.buffer = {i: copy.deepcopy(g) for i, g in enumerate(games)}
            self.updated = set()
        def sample_game(self, force_uniform=False):
            i = int(rs.randint(len(self.buffer)))
            return i, self.buffer[i], None
        def update_game_history(self, game_id, gh):
            self.updated.add(game_id); self.buffer[game_id] = gh

    st, buf = Storage(), Buffer()
    actor.games_per_call = 3
    actor.reanalyse(buf, st)
    assert buf.updated and st.d["num_reanalysed_games"] == actor.num_reanalysed_games > 4
