"""Host side of test-mode games of host-stepped games (self_play.DeviceHostEnvSelfPlay with an opponent,
SelfPlay.play_test_games on loop_path "device-host-env") on the CPU, against a stand-in for engine.HostEnvSelfPlayLoop
with the library's call order: the opponent phase after begin, observe and restart, the slots each phase steps, the
game ids of successive calls, the refusals raised in Python, and BoardVector.expert_actions against expert_agent."""
import types

import numpy
import pytest

from conftest import weights_for
from fake_engine import FakeSearchEngine
from muzero_general_b200 import _lib
from muzero_general_b200 import self_play as sp
from muzero_general_b200.engine import HostEnvSelfPlayLoop
from muzero_general_b200.games import load_game_module
from muzero_general_b200.games._boards import BoardVector
from muzero_general_b200.netspec import netspec_from_config

LOG = []


class FakeOpponentLoop:
    """HostEnvSelfPlayLoop's calls with the library's order checks: MuZero plays legal action (slot % legal moves), the
    turn's default is the first legal action, finished games are staged as blocks without observations."""

    def __init__(self, engine, obs_shape, max_moves, obs, legal_mask, to_play, first_game_id=0, game_id_stride=0,
                 opponent="self", muzero_player=0, **kw):
        self.B, self.max_moves = len(to_play), max_moves
        self.opponent, self.mp = opponent, muzero_player
        self.stride = game_id_stride or self.B
        self.ids = numpy.arange(self.B, dtype=numpy.int64) + first_game_id
        self.t = numpy.zeros(self.B, int)
        self.legal, self.to_play = numpy.array(legal_mask), numpy.array(to_play)
        self.with_priorities = False
        self.stats = types.SimpleNamespace(parked_slots=0, staged_bytes=0, staging_capacity=1, env_steps=0)
        self.phase = int(opponent != "self")
        self.observe_due, self.awaiting, self.staged = False, set(), []
        LOG.append(("begin", opponent, muzero_player))

    def opponent_turn(self):
        assert self.phase == 1 and not self.observe_due and not self.awaiting
        due = self.to_play != self.mp
        self.defaults = numpy.where(due, self.legal.argmax(axis=1), -1).astype(numpy.int32)
        self.phase = 2 if due.any() else 0
        LOG.append(("turn", numpy.nonzero(due)[0].tolist()))
        return self.defaults if due.any() else None

    def opponent_act(self, actions=None):
        assert self.phase == 2
        assert (actions is None) == (self.opponent == "random")
        due = self.defaults >= 0
        self.acted = numpy.where(due, self.defaults if actions is None else actions, -1).astype(numpy.int32)
        assert self.legal[due, self.acted[due]].all()
        self.phase, self.observe_due = 0, True
        LOG.append(("opponent_act", self.acted.tolist()))
        return self.acted

    def act(self, temperature, **inject):
        assert self.phase == 0 and not self.observe_due and not self.awaiting
        assert (self.to_play == self.mp).all() or self.opponent == "self"
        self.acted = numpy.array([numpy.nonzero(self.legal[g])[0][g % self.legal[g].sum()] for g in range(self.B)],
                                 numpy.int32)
        self.observe_due = True
        LOG.append(("act", self.acted.tolist()))
        return self.acted

    def observe(self, obs, reward, done, legal_mask, to_play):
        assert self.observe_due
        moved = self.acted >= 0
        self.t[moved] += 1
        finished = moved & (numpy.asarray(done, bool) | (self.t >= self.max_moves))
        self.legal[moved], self.to_play[moved] = numpy.asarray(legal_mask)[moved], numpy.asarray(to_play)[moved]
        for g in numpy.nonzero(finished)[0]:
            self.staged.append((int(self.ids[g]), int(g), int(self.t[g])))
        self.awaiting = set(numpy.nonzero(finished)[0].tolist())
        self.observe_due, self.phase = False, int(self.opponent != "self")
        LOG.append(("observe", numpy.nonzero(finished)[0].tolist()))
        return finished

    def restart(self, which, obs, legal_mask, to_play):
        which = numpy.asarray(which, bool)
        assert set(numpy.nonzero(which)[0].tolist()) == self.awaiting
        self.ids[which] += self.stride
        self.t[which] = 0
        self.legal[which], self.to_play[which] = numpy.asarray(legal_mask)[which], numpy.asarray(to_play)[which]
        self.awaiting, self.phase = set(), int(self.opponent != "self")
        LOG.append(("restart", numpy.nonzero(which)[0].tolist()))

    def drain(self):
        A, blocks, index, off = self.legal.shape[1], [], [], 0
        for gid, slot, T in self.staged:
            n = (_lib.MZ_STAGED_HEADER_BYTES + 8 * T + 4 * T * A + 16 * T + 7) // 8 * 8
            b = bytearray(n)
            b[0:8] = numpy.int64(gid).tobytes()
            b[8:32] = numpy.array([slot, T, 0, 0, A, n], numpy.int32).tobytes()
            blocks.append(bytes(b))
            index.append((off, (slot << 32) | T))
            off += n
        self.staged = []
        return b"".join(blocks), numpy.array(index, numpy.uint64).reshape(-1, 2)

    def peek(self):
        return {"game_id": self.ids.copy()}


STEPS = []


def _ids(games):
    """The game ids of ``PackedGames`` read from the blocks (the stand-in's blocks carry no observations)."""
    return sorted(int(numpy.frombuffer(buf, numpy.int64, 1, int(off))[0]) for buf, ix in games._chunks for off in ix[:, 0])


@pytest.fixture()
def fakes(monkeypatch):
    monkeypatch.setattr(sp, "SearchEngine", FakeSearchEngine)
    monkeypatch.setattr(sp, "HostEnvSelfPlayLoop", FakeOpponentLoop)
    step = BoardVector.step

    def logged(self, actions, which=None):
        before = self.board.copy()
        STEPS.append((numpy.asarray(actions).tolist(), None if which is None else numpy.nonzero(which)[0].tolist()))
        LOG.append(("step",))
        out = step(self, actions, which)
        if which is not None:                         # the slots left out keep their boards
            assert (self.board[~numpy.asarray(which, bool)] == before[~numpy.asarray(which, bool)]).all()
        return out

    monkeypatch.setattr(BoardVector, "step", logged)
    LOG.clear()
    STEPS.clear()


def _worker(name="tictactoe", B=4, Game=None, **over):
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.host_env_device_loop, cfg.device_envs = B, "philox", True, False
    for k, v in over.items():
        setattr(cfg, k, v)
    w = sp.SelfPlay({"weights": weights_for(name, netspec_from_config(cfg))}, Game or mod.Game, cfg, seed=0)
    assert w.loop_path == ("host" if cfg.rng_mode == "numpy" else "device-host-env")
    return w


@pytest.mark.parametrize("opponent,muzero_player", [("expert", 0), ("expert", 1), ("random", 1)])
def test_opponent_phase_order_and_stepped_slots(fakes, opponent, muzero_player):
    """Every begin, observe and restart is followed by a turn before MuZero's next act; a turn that finds due slots is
    followed by opponent_act, a step of exactly those slots (the others' boards unchanged) and an observe; the expert's
    moves are BoardVector.expert_actions of the turn's defaults, the random opponent's are the defaults (None)."""
    w = _worker()
    games, summary = w.play_test_games(9, opponent, muzero_player)
    assert len(games) == 9 and summary["games"] == 9
    kinds = [e[0] for e in LOG]
    assert kinds[0] == "begin" and LOG[0][1:] == (opponent, muzero_player) and kinds[1] == "turn"
    for i, k in enumerate(kinds):
        if k in ("begin", "observe", "restart") and i + 1 < len(kinds) and kinds[i + 1] != "restart":
            assert kinds[i + 1] == "turn", (i, kinds[i - 2:i + 3])
        if k == "opponent_act":
            assert kinds[i - 1] == "turn" and kinds[i + 1:i + 3] == ["step", "observe"]
    movers = [e[0] for e in LOG if e[0] in ("act", "opponent_act")]
    opp_steps = [st for st, m in zip(STEPS, movers) if m == "opponent_act"]
    assert len(STEPS) == len(movers) and any(which is not None for _, which in opp_steps)
    for (_, which), played in zip(opp_steps, [e[1] for e in LOG if e[0] == "opponent_act"]):
        assert (list(range(4)) if which is None else which) == [g for g, a in enumerate(played) if a >= 0]
    if opponent == "expert":
        first = [e for e in LOG if e[0] == "opponent_act"][0][1]
        env = load_game_module("tictactoe").Game.vector(4)
        env.reset()
        if muzero_player == 0:                         # MuZero's opening moves: legal action g % 9 of an empty board
            env.step(numpy.arange(4) % 9)
        dflt = numpy.where(env.to_play() != muzero_player, env.legal_mask().argmax(axis=1), -1)
        assert first == env.expert_actions(dflt, dflt >= 0).tolist()


def test_game_ids_across_calls(fakes):
    """The n smallest ids of the call (slot g plays first + g + k * stride), and a next call past every id begun."""
    w = _worker()
    first = sp.SelfPlay.TEST_GAME_IDS
    games, _ = w.play_test_games(6, "random", 0)
    assert _ids(games) == list(range(first, first + 6))
    again, _ = w.play_test_games(3, "random", 0)
    assert min(_ids(again)) >= first + 8 and (min(_ids(again)) - first) % 4 == 0


def test_refusals(fakes):
    """rng_mode="numpy": NotImplementedError naming play_game; a self-play loop in flight: RuntimeError; "human":
    NotImplementedError; "expert" on a vector game without expert_actions: NotImplementedError."""
    w = _worker(rng_mode="numpy")
    assert w.loop_path == "host"
    with pytest.raises(NotImplementedError, match="play_game"):
        w.play_test_games(2)
    w = _worker()
    w.play_moves(1, 1.0)
    with pytest.raises(RuntimeError, match="reset_stream"):
        w.play_test_games(2)
    w.reset_stream()
    assert len(w.play_test_games(2, "random", 0)[0]) == 2
    with pytest.raises(NotImplementedError, match="human"):
        HostEnvSelfPlayLoop(None, (3, 3, 3), 9, numpy.zeros((4, 27)), numpy.ones((4, 9)), numpy.zeros(4), opponent="human")

    class NoExpert(load_game_module("tictactoe").Game):
        @classmethod
        def vector(cls, num_games, seed=None):                 # a vector game without expert_actions
            v = cls.VECTOR(num_games, seed)
            return types.SimpleNamespace(num_games=num_games, reset=v.reset, step=v.step, legal_mask=v.legal_mask,
                                         to_play=v.to_play)

    w = _worker(Game=NoExpert)
    with pytest.raises(NotImplementedError, match="expert_actions"):
        w.play_test_games(2, "expert", 0)


@pytest.mark.parametrize("name", ["tictactoe", "connect4"])
def test_expert_actions_equal_expert_agent(name):
    """On positions of random playouts, BoardVector.expert_actions with the default expert_agent draws from numpy's
    global stream gives expert_agent's move, for every game of the batch at once."""
    mod = load_game_module(name)
    rs = numpy.random.RandomState(3)
    n = 24
    vec = mod.Game.vector(n)
    vec.reset()
    singles = [mod.Game() for _ in range(n)]
    for g in range(n):
        for _ in range(int(rs.randint(0, 7))):
            legal = singles[g].legal_actions()
            _, _, done = singles[g].step(int(rs.choice(legal)))
            if done or len(singles[g].legal_actions()) == 0:
                singles[g].reset()
        vec.board[g], vec.player[g] = singles[g].env.board[0], singles[g].env.player[0]
    defaults, expected = numpy.empty(n, numpy.int32), numpy.empty(n, numpy.int32)
    for g in range(n):
        numpy.random.seed(100 + g)
        defaults[g] = numpy.random.choice(singles[g].legal_actions())
        numpy.random.seed(100 + g)
        expected[g] = singles[g].expert_agent()
    which = numpy.arange(n) % 5 != 4
    got = vec.expert_actions(defaults, which)
    assert got[which].tolist() == expected[which].tolist() and (got[~which] == -1).all()
    assert (got[which] != defaults[which]).any()                   # some positions have a threat
