"""Host side of the device loop for host-stepped games (self_play.DeviceHostEnvSelfPlay) on the CPU: which worker takes
the path, and the order of its calls - act, step of the playing slots only, observe, reset of the packed games,
restart - against a stand-in for engine.HostEnvSelfPlayLoop that parks a game the way the library does."""
import types

import numpy
import pytest

from conftest import weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import self_play as sp
from muzero_general_b200.games import load_game_module
from muzero_general_b200.games.abstract_game import AbstractGame
from muzero_general_b200.netspec import netspec_from_config

LOG = []


class LogGame(AbstractGame):
    """Simple Grid's shapes; the game built with seed g ends after 2 + g % 2 moves and logs its steps and resets."""

    def __init__(self, seed=None):
        self.slot, self.t = int(seed), 0

    def _obs(self):
        o = numpy.zeros((1, 1, 9))
        o[0, 0, self.t] = 1
        return o

    def step(self, action):
        LOG.append(("step", self.slot, int(action)))
        self.t += 1
        return self._obs(), 1, self.t >= 2 + self.slot % 2

    def legal_actions(self):
        return [0, 1]

    def reset(self):
        LOG.append(("reset", self.slot))
        self.t = 0
        return self._obs()

    def render(self):
        pass


class FakeHostLoop:
    """The call protocol of HostEnvSelfPlayLoop with the library's slot states: a slot's first finished game parks
    (action -1 for the next two moves) when the slot is in PARK, then observe reports it finished."""
    PARK = {1}

    def __init__(self, engine, obs_shape, max_moves, obs, legal_mask, to_play, **kw):
        self.B = len(to_play)
        self.with_priorities = False
        self.stats = types.SimpleNamespace(parked_slots=0, staged_bytes=0, staging_capacity=1, env_steps=0)
        self.parked, self.awaiting, self.due = {}, set(), False
        self.park = set(self.PARK)
        LOG.append(("begin", numpy.stack(obs).argmax(-1).ravel().tolist()))

    def act(self, temperature, **inject):
        assert not self.due and not self.awaiting
        self.acted = numpy.array([-1 if g in self.parked else g % 2 for g in range(self.B)], numpy.int32)
        self.due = True
        LOG.append(("act", self.acted.tolist()))
        return self.acted

    def observe(self, obs, reward, done, legal_mask, to_play):
        assert self.due
        self.due = False
        finished = numpy.zeros(self.B, bool)
        for g in range(self.B):
            if self.acted[g] < 0:
                self.parked[g] -= 1
                if self.parked[g] == 0:
                    del self.parked[g]
                    finished[g] = True
            elif done[g]:
                if g in self.park:
                    self.park.discard(g)
                    self.parked[g] = 2
                else:
                    finished[g] = True
        self.awaiting |= set(numpy.nonzero(finished)[0].tolist())
        self.stats.parked_slots = len(self.parked)
        LOG.append(("observe", numpy.nonzero(finished)[0].tolist()))
        return finished

    def restart(self, which, obs, legal_mask, to_play):
        which = set(numpy.nonzero(which)[0].tolist())
        assert which and which == self.awaiting
        self.awaiting.clear()
        LOG.append(("restart", sorted(which), [int(numpy.asarray(obs[g]).argmax()) for g in sorted(which)]))

    def drain(self):
        LOG.append(("drain",))
        return b"", numpy.zeros((0, 2), numpy.uint64)


def _worker(Game, name="simple_grid", **over):
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games = 4
    for k, v in over.items():
        setattr(cfg, k, v)
    spec = netspec_from_config(cfg)
    return sp.SelfPlay({"weights": weights_for(name, spec)}, Game or mod.Game, cfg, seed=0)


@pytest.fixture()
def fakes(monkeypatch):
    monkeypatch.setattr(sp, "SearchEngine", FakeSearchEngine)
    monkeypatch.setattr(sp, "HostEnvSelfPlayLoop", FakeHostLoop)
    LOG.clear()


@pytest.mark.parametrize("name,game,over,path", [
    ("simple_grid", LogGame, dict(rng_mode="philox"), "host"),                                   # off by default
    ("simple_grid", LogGame, dict(rng_mode="philox", host_env_device_loop=True), "device-host-env"),
    ("simple_grid", LogGame, dict(rng_mode="numpy", host_env_device_loop=True), "host"),         # numpy draws: host loop
    ("tictactoe", None, dict(rng_mode="philox", host_env_device_loop=True), "device"),           # device env in use
    ("tictactoe", None, dict(rng_mode="philox", host_env_device_loop=True, device_envs=False), "device-host-env"),
    ("tictactoe", None, dict(rng_mode="philox", device_envs=False), "host"),
])
def test_loop_path(fakes, name, game, over, path):
    assert _worker(game, name, **over).loop_path == path


def test_driver_steps_only_playing_slots_and_restarts_packed_games(fakes):
    """Four slots, games of 2 or 3 moves; slot 1's first game parks for two moves.  Every move is act -> the steps of
    the slots with an action, in slot order -> observe -> the resets of the slots it reports -> restart of exactly those
    slots with their reset observations; a parked slot is neither stepped nor reset until observe reports it."""
    w = _worker(LogGame, rng_mode="philox", host_env_device_loop=True)
    assert w.loop_path == "device-host-env"
    w.play_moves(8, 1.0)
    assert LOG[:5] == [("reset", 0), ("reset", 1), ("reset", 2), ("reset", 3), ("begin", [0, 0, 0, 0])]
    moves, cur = [], None
    for e in LOG[5:]:
        if e[0] == "act":
            cur = [e]
            moves.append(cur)
        else:
            cur.append(e)
    assert len(moves) == 8 and LOG[-1] == ("drain",)
    parked_moves = 0
    for m in moves:
        acted = m[0][1]
        kinds = [e[0] for e in m]
        k_obs = kinds.index("observe")
        assert m[1:k_obs] == [("step", g, a) for g, a in enumerate(acted) if a >= 0]
        finished = m[k_obs][1]
        rest = [e for e in m[k_obs + 1:] if e[0] != "drain"]
        if finished:
            assert rest[:-1] == [("reset", g) for g in finished]
            assert rest[-1] == ("restart", finished, [0] * len(finished))
        else:
            assert rest == []
        parked_moves += acted[1] < 0
    assert parked_moves == 2
    # slot 1 finished its first game at move 3 (parked), was reported at move 5, restarted; slot 0 every 2 moves
    assert [i for i, m in enumerate(moves) if 1 in m[[e[0] for e in m].index("observe")][1]] == [4, 7]
    assert [i for i, m in enumerate(moves) if 0 in m[[e[0] for e in m].index("observe")][1]] == [1, 3, 5, 7]


def test_vector_games_step_whole_with_a_filler_action(fakes):
    """A VectorGame steps all its games: a parked slot takes action 0 and its rows are ignored."""
    calls = []

    class Vec:
        def __init__(self, Game, num_games, seed, A):
            self.inner = sp._ObjectVector(Game, num_games, seed, A)
            self.num_games = num_games

        def step(self, actions):
            calls.append(numpy.asarray(actions).tolist())
            return self.inner.step(actions)

        def __getattr__(self, name):
            return getattr(self.inner, name)

    class VecGame(LogGame):
        @classmethod
        def vector(cls, num_games, seed=None):
            return Vec(cls, num_games, seed, 2)

    w = _worker(VecGame, rng_mode="philox", host_env_device_loop=True)
    w.play_moves(6, 1.0)
    acts = [e[1] for e in LOG if e[0] == "act"]
    assert len(calls) == 6
    for a, c in zip(acts, calls):
        assert c == [x if x >= 0 else 0 for x in a]
    assert any(x < 0 for a in acts for x in a)
