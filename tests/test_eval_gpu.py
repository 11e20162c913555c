"""Test-mode games on the device (mz_selfplay_begin_vs, mz_debug_opponent_action, SelfPlay.play_test_games) against
host oracles: the device opponent against the host expert (games/_boards.py::_threat_scan, pinned to the reference by
tests/golden/expert.json), the production loop against a host composition of search + sampling + opponent, and the
evaluation API against the test worker's formulas.  Everything goes through the C ABI."""
import ctypes as C

import numpy
import pytest

from conftest import golden_json, weights_for
from muzero_general_b200 import _lib
from muzero_general_b200.games import load_game_module
from muzero_general_b200.games._boards import _threat_scan
from muzero_general_b200.netspec import netspec_from_config
from oracle import mcts as om
from oracle import philox

pytestmark = pytest.mark.gpu

TAG_OPPONENT = 0x7169E005          # csrc/selfplay.cu kTagOpponent


def _default(legal, u):
    """numpy.random.choice(legal_actions) for the uniform u: the legal action with index floor(u * n)."""
    return legal[min(int(u * len(legal)), len(legal) - 1)]


def _host_opponent(Game, board, player, opponent, default):
    if opponent == "random":
        return default
    return _threat_scan(board, int(player), Game._expert_windows(None, board), default)


# ------------------------------------------------------------------------------------------ the opponent alone
@pytest.mark.parametrize("name", ["tictactoe", "connect4"])
def test_device_expert_replays_the_reference_fixture(name):
    """Every position of tests/golden/expert.json, with the fixture's numpy default re-drawn on the host from its seed:
    the device expert returns the reference's action."""
    from muzero_general_b200.engine import debug_opponent_action
    mod = load_game_module(name)
    boards, players, defaults, want = [], [], [], []
    for c in golden_json("expert.json")[name]:
        g = mod.Game(0)
        g.reset()
        for a in c["moves"]:
            g.step(a)
        numpy.random.seed(c["seed"])
        defaults.append(int(numpy.random.choice(g.legal_actions())))
        boards.append(g.env.board[0].copy())
        players.append(int(g.env.player[0]))
        want.append(c["action"])
    got = debug_opponent_action(name, boards, players, defaults=defaults)
    assert got.tolist() == want
    assert sum(d != w for d, w in zip(defaults, want)) > 20        # the scan changed the default often


def _playout_positions(name, n_games, rs):
    """(boards [n, H*W], players [n]) of every position of random playouts, both sides to move.  Half the playouts go
    on past a completed line until the board is full, so near-full boards and full columns are common."""
    vec = load_game_module(name).Game.VECTOR(n_games)
    vec.reset()
    boards, players = [], []
    alive = numpy.ones(n_games, bool)
    past_lines = numpy.arange(n_games) % 2 == 0
    while alive.any():
        legal = vec.legal_mask()
        alive &= legal.any(1)
        if not alive.any():
            break
        boards.append(vec.board[alive].copy())
        players.append(vec.player[alive].copy())
        r = rs.random_sample(legal.shape) * legal
        _, _, done = vec.step(numpy.argmax(r, 1))
        alive &= ~done | past_lines
    return numpy.concatenate(boards), numpy.concatenate(players)


@pytest.mark.parametrize("name,n_games", [("tictactoe", 7000), ("connect4", 1800)])
def test_device_opponent_equals_host_on_random_positions(name, n_games):
    """At least 50k positions per game from random playouts, with random uniforms: "expert" equals the host
    _threat_scan with default legal[floor(u * n)], "random" equals that default.  The positions include wins and
    blocks for both sides, full columns and boards with at most three empty cells."""
    from muzero_general_b200.engine import debug_opponent_action
    mod = load_game_module(name)
    vec = mod.Game.VECTOR
    rs = numpy.random.RandomState(17)
    boards, players = _playout_positions(name, n_games, rs)
    n = len(boards)
    assert n >= 50000, n
    u = rs.random_sample(n)
    u[:200] = numpy.nextafter(1.0, 0.0)
    expert = debug_opponent_action(name, boards, players, uniforms=u, opponent="expert")
    rand = debug_opponent_action(name, boards, players, uniforms=u, opponent="random")
    changed = full_cols = near_full = 0
    for i in range(n):
        b = boards[i].reshape(vec.H, vec.W)
        legal = [int(a) for a in numpy.nonzero(b[vec.H - 1] == 0 if vec.GRAVITY else b.ravel() == 0)[0]]
        d = _default(legal, u[i])
        assert rand[i] == d, i
        want = _host_opponent(mod.Game, b, players[i], "expert", d)
        assert expert[i] == want, (i, b.tolist(), int(players[i]), d)
        changed += want != d
        full_cols += vec.GRAVITY and len(legal) < vec.W
        near_full += (b == 0).sum() <= 3
    assert changed > n // 20 and near_full > 1000
    if vec.GRAVITY:
        assert full_cols > 5000


# ------------------------------------------------------------------------------------------ the production loop
def _make(name, B, N, seed, opponent, muzero_player, max_moves=None, staging=0):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    if max_moves:
        cfg.max_moves = max_moves
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    eng.load_weights(weights_for(name, spec))
    loop = DeviceSelfPlayLoop(eng, name, cfg.max_moves, reward_scale=mod.Game.VECTOR.REWARD_SCALE, staging_bytes=staging,
                              opponent=opponent, muzero_player=muzero_player)
    return mod, cfg, eng, loop


def _drain(loop):
    from muzero_general_b200.engine import parse_staged_games
    return parse_staged_games(*loop.drain())


def _check_record(mod, cfg, rec, expected, seed, opponent, muzero_player):
    """Replays one delivered game on the host environment: MuZero's moves carry the host search's visits, root value
    and action, the opponent's moves NaN, zero visits and the host opponent's action; rewards, observations, to_play
    and the end of the game replay.  Returns the number of opponent moves where the expert's scan changed the
    default."""
    env = mod.Game(0)
    env.reset()
    T, gid = rec["length"], rec["game_id"]
    assert rec["first_to_play"] == 0
    changed = 0
    for t in range(T):
        mover = env.to_play()
        if mover == muzero_player:
            visits, root, action = expected[(gid, t)]
            assert rec["visits"][t].tolist() == visits.tolist(), (gid, t)
            assert rec["root_value"][t] == root, (gid, t)
            assert rec["action"][t] == action, (gid, t)
        else:
            assert numpy.isnan(rec["root_value"][t]) and not rec["visits"][t].any(), (gid, t)
            d = _default(env.legal_actions(), philox.uniform53(seed, gid, t, 0, TAG_OPPONENT))
            board = env.env.board[0].reshape(env.env.H, env.env.W)
            want = _host_opponent(mod.Game, board, env.env.player[0], opponent, d)
            assert rec["action"][t] == want, (gid, t)
            changed += want != d
        obs, reward, done = env.step(int(rec["action"][t]))
        assert numpy.array_equal(numpy.asarray(obs, numpy.float32).ravel(), rec["obs"][t + 1]), (gid, t)
        assert float(reward) == float(rec["reward"][t]) and rec["to_play"][t] == env.to_play(), (gid, t)
        assert done == (t + 1 == T) or (not done and t + 1 == T == cfg.max_moves), (gid, t)
    return changed


CASES = [(name, opponent, mp, T) for name in ("tictactoe", "connect4") for opponent in ("expert", "random")
         for mp in (0, 1) for T in (0.0, 1.0)]


@pytest.mark.parametrize("name,opponent,muzero_player,T", CASES)
def test_production_loop_equals_host_composition(name, opponent, muzero_player, T, monkeypatch):
    """Run A plays one MuZero move per call.  Before each call every slot is at MuZero's turn; the host composes
    [search of the peeked state] + [uniform53(seed, game, move, 0, TAG_ACTION)] + [numpy's choice rule] for it.  Each
    delivered game replays on the host: MuZero's moves equal that composition bit for bit, the opponent's moves are NaN,
    zero visits and the host opponent's action for uniform53(seed, game, move, 0, 0x7169E005).  Connect4 is cut at
    max_moves = 12 - muzero_player, so the opponent may play the last move a game allows.  env_steps counts both sides'
    moves.  Run B plays the same seeded loop through enqueue / wait in chunks of 1, 3 and 8 moves with a staging area
    that parks games, until it has finished every game run A finished: each is identical."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    B, N, seed = 32, 6, 0x5EED_0000_0042 + muzero_player
    max_moves = 12 - muzero_player if name == "connect4" else None
    calls = 16 if name == "connect4" else 12
    mod, cfg, eng_a, loop_a = _make(name, B, N, seed, opponent, muzero_player, max_moves)
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    ref.load_weights(weights_for(name, netspec_from_config(cfg)))
    expected, recs_a = {}, {}
    for _ in range(calls):
        pk = loop_a.peek()
        assert (pk["to_play"] == muzero_player).all()               # no search is spent on an opponent's turn
        out = ref.search(obs=pk["obs"], legal_mask=pk["legal_mask"], to_play=pk["to_play"], add_exploration_noise=True,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        for g in range(B):
            gid, mv = int(pk["game_id"][g]), int(pk["move_index"][g])
            u = philox.uniform53(seed, gid, mv, 0, philox.TAG_ACTION)
            idx = [int(a) for a in numpy.nonzero(pk["legal_mask"][g])[0]]
            a = om.select_action(idx, out.visit_counts[g][idx], T, om.InjectedDraws(uniform=float(u)))
            expected[(gid, mv)] = (out.visit_counts[g].copy(), out.root_value[g], a)
        st = loop_a.moves(1, T)
        for rec in _drain(loop_a):
            recs_a[rec["game_id"]] = rec
    pk = loop_a.peek()
    assert st.env_steps == sum(r["length"] for r in recs_a.values()) + int(pk["move_index"].sum())
    eng_a.close(); ref.close()
    assert len(recs_a) >= B
    changed = sum(_check_record(mod, cfg, rec, expected, seed, opponent, muzero_player) for rec in recs_a.values())
    if opponent == "expert":
        assert changed > 0
    if name == "connect4":
        assert sum(r["length"] == max_moves for r in recs_a.values()) > 0

    L, A = cfg.max_moves, len(cfg.action_space)
    longest = 32 + 8 * L + 4 * L * A + 16 * L + 4 * (L + 1) * eng_a.obs_elems + 8      # a maximum-length block
    _, _, eng_b, loop_b = _make(name, B, N, seed, opponent, muzero_player, max_moves, staging=3 * longest)
    recs_b, parked, i = {}, 0, 0
    while not set(recs_a) <= set(recs_b) and i < 400:
        loop_b.enqueue([1, 3, 8][i % 3], T)
        parked = max(parked, loop_b.wait().parked_slots)
        for rec in _drain(loop_b):
            assert rec["game_id"] not in recs_b
            recs_b[rec["game_id"]] = rec
        i += 1
    eng_b.close()
    assert parked > 0 and set(recs_a) <= set(recs_b)
    for gid in sorted(recs_a):
        for key in ("length", "slot", "first_to_play", "action", "visits", "root_value", "reward", "to_play", "obs"):
            assert numpy.asarray(recs_a[gid][key]).tobytes() == numpy.asarray(recs_b[gid][key]).tobytes(), (gid, key)


@pytest.mark.parametrize("name,td_steps", [("tictactoe", 0), ("connect4", 0), ("cartpole", 0), ("tictactoe", 3)])
def test_begin_vs_self_is_begin(name, td_steps, monkeypatch):
    """mz_selfplay_begin_vs(..., MZ_OPPONENT_SELF, 0) and mz_selfplay_begin stage byte-identical games."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    if name == "cartpole":
        cfg.max_moves = 20
    spec = netspec_from_config(cfg)
    raw = []
    for variant in ("begin", "begin_vs"):
        eng = SearchEngine(cfg, max_games=24, num_simulations=5, seed=99)
        eng.load_weights(weights_for(name, spec))
        d = _lib.MzSelfPlayDesc()
        d.env, d.max_moves = DeviceSelfPlayLoop.ENVS[name], cfg.max_moves
        d.reward_scale = getattr(getattr(mod.Game, "VECTOR", None), "REWARD_SCALE", 1)
        pw = (C.c_double * (td_steps + 1))(*[cfg.discount ** k for k in range(td_steps + 1)])
        if td_steps:
            d.td_steps, d.per_alpha, d.discount_pow = td_steps, 1.0, C.cast(pw, C.c_void_p)
        if variant == "begin":
            eng._check(eng.lib.mz_selfplay_begin(eng._h, C.byref(d)))
        else:
            eng._check(eng.lib.mz_selfplay_begin_vs(eng._h, C.byref(d), _lib.MZ_OPPONENT_SELF, 0))
        loop = object.__new__(DeviceSelfPlayLoop)
        loop.engine, loop.stats = eng, _lib.MzSelfPlayStats()
        out = []
        for k in (1, 4, 8, 8, 16):
            st = loop.moves(k, 1.0)
            buf, index = loop.drain()
            # blocks are staged in the order their warps reserved space: compare them by game id, byte for byte up to
            # the padding (which nothing writes)
            blocks = {}
            for off in index[:, 0].astype(numpy.int64):
                _, T, _, O, A, _ = numpy.frombuffer(buf, numpy.int32, 6, off + 8).tolist()
                used = _lib.MZ_STAGED_HEADER_BYTES + T * 8 + T * A * 4 + T * 16 + (T + 1) * O * 4
                blocks[int(numpy.frombuffer(buf, numpy.int64, 1, off)[0])] = buf[off:off + used]
            out.append((blocks, st.env_steps))
        eng.close()
        raw.append(out)
    for (blocks_a, steps_a), (blocks_b, steps_b) in zip(*raw):
        assert blocks_a == blocks_b and steps_a == steps_b
    assert sum(len(b) for b, _ in raw[0]) > 24


# ------------------------------------------------------------------------------------------ evaluation API
def _worker_report(gh, muzero_player):
    """self_play.py:67-90, as the reference's test worker writes it."""
    return {
        "episode_length": len(gh.action_history) - 1,
        "total_reward": sum(gh.reward_history),
        "mean_value": numpy.mean([value for value in gh.root_values if value]),
        "muzero_reward": sum(reward for i, reward in enumerate(gh.reward_history)
                             if gh.to_play_history[i - 1] == muzero_player),
        "opponent_reward": sum(reward for i, reward in enumerate(gh.reward_history)
                               if gh.to_play_history[i - 1] != muzero_player),
    }


@pytest.mark.parametrize("muzero_player", [0, 1])
def test_play_test_games_returns_reference_shaped_games(muzero_player, monkeypatch):
    """Connect4 against the expert, 37 games on 16 slots: the returned ids are exactly the 37 smallest of the call,
    the histories have the shape of host play_game histories (None root values at the opponent's moves, child_visits
    rows for MuZero's moves only), the summary equals the test worker's formulas recomputed from the histories, a
    second call plays new ids, and a fresh worker with the same seed plays the same games."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.self_play import SelfPlay

    def worker():
        mod = load_game_module("connect4")
        cfg = mod.MuZeroConfig()
        cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations, cfg.muzero_player = 16, "philox", 8, muzero_player
        return SelfPlay({"weights": weights_for("connect4", netspec_from_config(cfg))}, mod.Game, cfg, 5), cfg

    w, cfg = worker()
    games, summary = w.play_test_games(37)
    first = SelfPlay.TEST_GAME_IDS
    assert sorted(g.game_id for g in games) == list(range(first, first + 37))
    reports = []
    for gh in games:
        T = len(gh.action_history) - 1
        assert T == len(gh) == len(gh.root_values) == len(gh.reward_history) - 1 == len(gh.to_play_history) - 1
        assert len(gh.observation_history) == T + 1 and gh.observation_history[0].shape == (3, 6, 7)
        mine = [gh.to_play_history[t] == muzero_player for t in range(T)]
        assert [v is not None for v in gh.root_values] == mine
        assert len(gh.child_visits) == sum(mine) and all(abs(sum(c) - 1) < 1e-12 for c in gh.child_visits)
        reports.append(_worker_report(gh, muzero_player))
    for key in ("episode_length", "total_reward", "mean_value", "muzero_reward", "opponent_reward"):
        assert summary[key] == numpy.mean([r[key] for r in reports]), key
    assert summary["games"] == 37 and summary["wins"] + summary["draws"] + summary["losses"] == 37
    again, _ = w.play_test_games(5)
    assert min(g.game_id for g in again) >= first + 48
    w.close()
    w2, _ = worker()
    games2, summary2 = w2.play_test_games(37)
    w2.close()
    key = lambda gs: sorted((g.game_id, tuple(int(a) for a in g.action_history)) for g in gs)
    assert key(games2) == key(games) and summary2 == summary


# ------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("name,kw,reason", [
    ("cartpole", dict(opponent="expert"), "CartPole has one player"),
    ("tictactoe", dict(opponent="expert", muzero_player=2), "muzero_player must be 0 or 1"),
    ("connect4", dict(opponent="random", td_steps=5), "td_steps must be 0"),
])
def test_begin_vs_refusals(name, kw, reason):
    """Each refusal fails at begin with MZ_EINVAL and its reason."""
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    eng = SearchEngine(cfg, max_games=4, num_simulations=2)
    with pytest.raises(_lib.MzError, match=reason) as e:
        DeviceSelfPlayLoop(eng, name, cfg.max_moves, **kw)
    assert e.value.code == -1
    eng.close()


def test_begin_vs_refuses_an_unknown_opponent():
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    cfg = load_game_module("tictactoe").MuZeroConfig()
    eng = SearchEngine(cfg, max_games=4, num_simulations=2)
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves = _lib.MZ_ENV_TICTACTOE, cfg.max_moves
    assert eng.lib.mz_selfplay_begin_vs(eng._h, C.byref(d), 3, 0) == _lib.MZ_EUNSUPPORTED
    assert "unknown opponent 3" in eng.lib.mz_last_error(eng._h).decode()
    with pytest.raises(NotImplementedError, match="human"):
        DeviceSelfPlayLoop(eng, "tictactoe", cfg.max_moves, opponent="human")
    eng.close()
