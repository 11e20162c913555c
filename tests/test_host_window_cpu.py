"""Host-kept observations of host-stepped games (engine.HostEnvSelfPlayLoop with obs_history="host",
mz_selfplay_begin_host_window) on the CPU: the rows each game keeps, their hand-over with the drained blocks, the
fall-back from the device-history begin on MZ_ENOMEM, pickling, and the declarations of the new entry point.  The
library is a stand-in with its slot states (parking included) that stages blocks without observations."""
import ctypes as C
import os
import pickle
import re

import numpy
import pytest

from conftest import ROOT, weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import _lib
from muzero_general_b200 import self_play as sp
from muzero_general_b200.engine import HostEnvSelfPlayLoop
from muzero_general_b200.games import load_game_module
from muzero_general_b200.games.abstract_game import AbstractGame
from muzero_general_b200.netspec import netspec_from_config


def _view(addr, ctype, n):
    return numpy.ctypeslib.as_array(C.cast(addr, C.POINTER(ctype)), (n,))


class FakeWindowLib:
    """The host-stepped calls of the library for B slots of A actions: a slot's first finished game parks when the slot
    is in ``park`` (action -1 for two moves, then reported finished), and drains return blocks with obs_elems = 0."""

    def __init__(self, B, A, park=(), device_rc=0):
        self.B, self.A, self.park, self.device_rc = B, A, set(park), device_rc
        self.begun = []

    def mz_last_error(self, h):
        return b"fake"

    def _begin(self, kind, d_ref):
        d = d_ref._obj
        self.begun.append(kind)
        self.stride = d.game_id_stride if d.game_id_stride > 0 else self.B
        self.ids = [d.first_game_id + g for g in range(self.B)]
        self.t = [0] * self.B
        self.parked = {}
        self.staged = []
        return 0

    def mz_selfplay_begin_host(self, h, d_ref, e_ref, obs, legal, to_play):
        if self.device_rc:
            self.begun.append("device refused")
            return self.device_rc
        return self._begin("device", d_ref)

    def mz_selfplay_begin_host_window(self, h, d_ref, e_ref, obs, legal, to_play):
        return self._begin("window", d_ref)

    def mz_selfplay_host_act(self, h, temperature, inj, actions):
        self.acted = numpy.array([-1 if g in self.parked else g % self.A for g in range(self.B)], numpy.int32)
        _view(actions, C.c_int32, self.B)[:] = self.acted
        return 0

    def mz_selfplay_host_observe(self, h, obs, reward, done, legal, to_play, finished, stats_ref):
        done = _view(done, C.c_uint8, self.B)
        out = _view(finished, C.c_uint8, self.B)
        out[:] = 0
        for g in range(self.B):
            if self.acted[g] < 0:
                self.parked[g] -= 1
                if self.parked[g]:
                    continue
                del self.parked[g]
            else:
                self.t[g] += 1
                if not done[g]:
                    continue
                if g in self.park:
                    self.park.discard(g)
                    self.parked[g] = 2
                    continue
            self.staged.append((self.ids[g], g, self.t[g]))
            out[g] = 1
        st = stats_ref._obj
        st.parked_slots, st.staged_bytes, st.staging_capacity = len(self.parked), 0, 1
        return 0

    def mz_selfplay_host_restart(self, h, which, obs, legal, to_play):
        for g in numpy.nonzero(_view(which, C.c_uint8, self.B))[0]:
            self.ids[g] += self.stride
            self.t[g] = 0
        return 0

    def mz_selfplay_drain(self, h, data_ref, bytes_ref, n_ref, index_ref):
        A, blocks, index, off = self.A, [], [], 0
        for gid, slot, T in self.staged:
            n = (_lib.MZ_STAGED_HEADER_BYTES + 8 * T + 4 * T * A + 16 * T + 7) // 8 * 8
            b = bytearray(n)
            b[0:8] = numpy.int64(gid).tobytes()
            b[8:32] = numpy.array([slot, T, 0, 0, A, n], numpy.int32).tobytes()
            blocks.append(bytes(b))
            index.append((off, (slot << 32) | T))
            off += n
        self.staged = []
        self._buf = C.create_string_buffer(b"".join(blocks) or b"\0")
        self._index = numpy.array(index or [(0, 0)], numpy.uint64)
        data_ref._obj.value = C.addressof(self._buf)
        index_ref._obj.value = self._index.ctypes.data
        bytes_ref._obj.value, n_ref._obj.value = off, len(index)
        return 0


class FakeEngine(FakeSearchEngine):
    """The oracle engine with a stand-in library (``lib``), checked like SearchEngine._check."""
    PARK, DEVICE_RC = (), 0

    def __init__(self, config, max_games=1, **kw):
        super().__init__(config, max_games=max_games, **kw)
        self.lib, self._h = FakeWindowLib(max_games, self.A, self.PARK, self.DEVICE_RC), None

    def _check(self, rc):
        if rc != 0:
            raise _lib.MzError(rc, self.lib.mz_last_error(self._h).decode())


class RowGame(AbstractGame):
    """Simple Grid's shapes; the game built with seed g ends after 2 + g % 2 moves.  Observation: [slot, move, game of
    the slot, 0...], so every row names the game and move it belongs to."""

    def __init__(self, seed=None):
        self.slot, self.t, self.k = int(seed), 0, -1

    def _obs(self):
        o = numpy.zeros((1, 1, 9))
        o[0, 0, :3] = self.slot, self.t, self.k
        return o

    def step(self, action):
        self.t += 1
        return self._obs(), 1, self.t >= 2 + self.slot % 2

    def legal_actions(self):
        return [0, 1]

    def reset(self):
        self.t, self.k = 0, self.k + 1
        return self._obs()

    def render(self):
        pass


def _worker(monkeypatch, park=(), device_rc=0, B=4, stride=None):
    monkeypatch.setattr(FakeEngine, "PARK", tuple(park))
    monkeypatch.setattr(FakeEngine, "DEVICE_RC", device_rc)
    monkeypatch.setattr(sp, "SearchEngine", FakeEngine)
    cfg = load_game_module("simple_grid").MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.host_env_device_loop = B, "philox", True
    w = sp.SelfPlay({"weights": weights_for("simple_grid", netspec_from_config(cfg))}, RowGame, cfg, seed=0,
                    first_game_id=10, game_id_stride=stride)
    assert w.loop_path == "device-host-env"
    return w


def _check_rows(games, B, stride):
    """Every game's observations are its own rows, one per position: slot, move 0..T, the slot's k-th game."""
    assert len(games)
    for gh in games:
        slot, k = (gh.game_id - 10) % stride, (gh.game_id - 10) // stride
        T = len(gh)
        obs = numpy.stack(gh.observation_history)
        assert obs.shape == (T + 1, 1, 1, 9) and obs.dtype == numpy.float32, gh.game_id
        assert obs[:, 0, 0, 0].tolist() == [slot] * (T + 1), gh.game_id
        assert obs[:, 0, 0, 1].tolist() == list(range(T + 1)), gh.game_id
        assert obs[:, 0, 0, 2].tolist() == [k] * (T + 1), gh.game_id
        assert T == 2 + slot % 2


def test_enomem_on_the_device_history_selects_the_window(monkeypatch):
    """The driver begins with the device keeping the observations, as before; on MZ_ENOMEM it begins again with the
    window and keeps each game's rows on the host.  Any other refusal is raised."""
    w = _worker(monkeypatch, device_rc=_lib.MZ_ENOMEM)
    games = w.play_moves(6, 1.0)
    assert w._device_loop.loop.obs_history == "host"
    assert w.model.engine.lib.begun == ["device refused", "window"]
    _check_rows(games, 4, 4)
    assert sorted(g.game_id for g in games) == [10, 11, 12, 13, 14, 15, 16, 17, 18, 20]
    w = _worker(monkeypatch)
    w.play_moves(1, 1.0)
    assert w._device_loop.loop.obs_history == "device" and w.model.engine.lib.begun == ["device"]
    with pytest.raises(_lib.MzError):
        _worker(monkeypatch, device_rc=-1).play_moves(1, 1.0)


def test_parked_and_idle_slots_add_no_rows(monkeypatch):
    """Slot 1's first game parks for two moves: its environment is not stepped and the rows passed for it then are not
    its game's; the game arrives with exactly its T + 1 rows, and so do the games after it."""
    w = _worker(monkeypatch, park={1}, device_rc=_lib.MZ_ENOMEM, stride=7)
    games = w.play_moves(9, 1.0)
    assert w._device_loop.parked_events > 0
    assert 11 in [g.game_id for g in games] and 18 in [g.game_id for g in games]
    _check_rows(games, 4, 7)
    assert not w._device_loop.loop._finished_rows        # handed over with their blocks


def test_a_drain_after_the_restart_gets_the_finished_games_rows(monkeypatch):
    """observe reports a game finished, its slot restarts (a new game id), and only then does the drain return the
    block: the rows that go with it are the finished game's, not the next game's."""
    monkeypatch.setattr(sp, "SearchEngine", FakeEngine)
    cfg = load_game_module("simple_grid").MuZeroConfig()
    eng = FakeEngine(cfg, max_games=2)
    games = [RowGame(g) for g in range(2)]
    obs = [g.reset() for g in games]
    legal, tp = numpy.ones((2, 2), numpy.uint8), numpy.zeros(2, numpy.int32)
    loop = HostEnvSelfPlayLoop(eng, (1, 1, 9), 27000, obs, legal, tp, first_game_id=3, game_id_stride=5,
                               obs_history="host")
    for move in range(3):
        a = loop.act(1.0)
        steps = [games[g].step(a[g]) for g in range(2)]
        finished = loop.observe([s[0] for s in steps], [s[1] for s in steps], [s[2] for s in steps], legal, tp)
        if finished.any():
            for g in numpy.nonzero(finished)[0]:
                obs[g] = games[g].reset()
            loop.restart(finished, obs, legal, tp)
    assert loop._game_id == [8, 9]                      # both slots restarted before the drain
    buf, index, rows = loop.drain()
    packed = sp.PackedGames((1, 1, 9), numpy.float32, float)
    packed.add(buf, index, rows)
    assert sorted(rows) == [3, 4] and not loop._finished_rows
    got = {g.game_id: numpy.stack(g.observation_history)[:, 0, 0, :3].tolist() for g in packed}
    assert got == {3: [[0, t, 0] for t in range(3)], 4: [[1, t, 0] for t in range(4)]}
    # the games in flight kept their own first rows
    assert [len(r) for r in loop._rows_of] == [2, 1]
    assert [r[0][:3].tolist() for r in loop._rows_of] == [[0, 0, 1], [1, 0, 1]]


def test_pickle_gives_a_game_history_with_every_observation(monkeypatch):
    w = _worker(monkeypatch, device_rc=_lib.MZ_ENOMEM)
    games = w.play_moves(4, 1.0)
    gh = games[0]
    assert isinstance(gh, sp.PackedGameHistory) and gh._packed[0]["bytes"] > 0
    back = pickle.loads(pickle.dumps(gh))
    assert type(back) is sp.GameHistory
    assert len(back.observation_history) == len(gh) + 1 == len(back.action_history)
    assert numpy.array_equal(numpy.stack(back.observation_history), numpy.stack(gh.observation_history))


def test_obs_history_must_be_device_or_host(monkeypatch):
    cfg = load_game_module("simple_grid").MuZeroConfig()
    eng = FakeEngine(cfg, max_games=2)
    with pytest.raises(ValueError):
        HostEnvSelfPlayLoop(eng, (1, 1, 9), 4, numpy.zeros((2, 9)), numpy.ones((2, 2)), numpy.zeros(2), obs_history="gpu")


def test_the_window_entry_is_declared_alike():
    """include/mzb200.h, _lib.SYMBOLS and the INTEGRATION.md stub declare mz_selfplay_begin_host_window with the
    arguments of mz_selfplay_begin_host."""
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mzb200.h")).read(), flags=re.S)
    proto = {name: " ".join(args.split()) for name, args in
             re.findall(r"int (mz_selfplay_begin_host(?:_window)?)\((.*?)\);", header, flags=re.S)}
    assert proto["mz_selfplay_begin_host_window"] == proto["mz_selfplay_begin_host"] == (
        "MzHandle* h, const MzSelfPlayDesc* desc, const MzHostEnvDesc* env, const float* obs, const uint8_t* legal, "
        "const int32_t* to_play")
    sym = {name: (res, args) for name, res, args in _lib.SYMBOLS}
    assert sym["mz_selfplay_begin_host_window"] == sym["mz_selfplay_begin_host"]
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    stub = re.search(r"lib\.mz_selfplay_begin_host_window\((.*?)\) == 0", doc, flags=re.S)
    assert stub and " ".join(stub.group(1).split()) == (
        "h, C.byref(desc), C.byref(env), obs0.ctypes.data, legal0.ctypes.data, to_play0.ctypes.data")
