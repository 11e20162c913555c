"""Gomoku, Twenty-One and Simple Grid in the device self-play loop (csrc/selfplay.cu) against the reference's recorded
trajectories, the plug-ins' rules, host compositions of search + sampling + opponent, and the reference's network and
search fixtures.  Everything goes through the C ABI."""
import ctypes as C
import pickle

import numpy
import pytest

from conftest import golden_json, golden_npz, weights_for
from muzero_general_b200 import _lib
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from oracle import cards, philox
from oracle import mcts as om

pytestmark = pytest.mark.gpu

TAG_OPPONENT = 0x7169E005          # csrc/selfplay.cu kTagOpponent
SMALL_GOMOKU = dict(blocks=1, channels=16)      # loop tests: the rules are under test, not the 128-channel towers


def _cfg(name, **over):
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    for k, v in ({**SMALL_GOMOKU, **over} if name == "gomoku" else over).items():
        setattr(cfg, k, v)
    return mod, cfg


def _loop(name, B, N, seed=0, first_game_id=0, opponent="self", muzero_player=0, **over):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    mod, cfg = _cfg(name, **over)
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    eng.load_weights(weights_for(name, spec))
    loop = DeviceSelfPlayLoop(eng, name, cfg.max_moves, temperature_threshold=cfg.temperature_threshold,
                              reward_scale=mod.Game.VECTOR.REWARD_SCALE, first_game_id=first_game_id,
                              opponent=opponent, muzero_player=muzero_player)
    return mod, cfg, spec, eng, loop


def _drain(loop):
    from muzero_general_b200.engine import parse_staged_games
    return parse_staged_games(*loop.drain())


def _philox_cards(seed, gid):
    k = iter(range(1 << 20))
    return lambda: cards.card(seed, gid, next(k))


# ------------------------------------------------------------------------------------------ rules
@pytest.mark.parametrize("name", ["gomoku", "simple_grid"])
def test_environments_replay_the_reference_trajectories(name):
    """Slot g is driven through the reference's recorded game g (tests/golden/env_*.json) with forced actions: the
    device observations, legal masks, side to move, rewards and terminations are the reference's, bit for bit."""
    games = golden_json(f"env_{name}.json")["games"]
    B = len(games)
    # the playouts run to the end of the game; Simple Grid's moves off the edge can outlast its max_moves of 6
    mod, cfg, spec, eng, loop = _loop(name, B, 2, max_moves=200)
    first = numpy.asarray(mod.Game(0).reset(), numpy.float32).ravel()
    finished = {}
    pk = loop.peek()
    assert (pk["move_index"] == 0).all() and (pk["to_play"] == 0).all()
    for t in range(max(len(g) for g in games)):
        forced = numpy.array([games[g][t]["action"] if t < len(games[g]) else int(numpy.nonzero(pk["legal_mask"][g])[0][0])
                              for g in range(B)], numpy.int32)
        loop.moves(1, 1.0, forced_action=forced)
        pk = loop.peek()
        for g in range(B):
            if t < len(games[g]):
                s = games[g][t]
                if not s["done"]:
                    assert pk["obs"][g].astype(numpy.int8).tolist() == s["obs"], (name, g, t)
                    assert numpy.nonzero(pk["legal_mask"][g])[0].tolist() == s["legal"]
                    assert int(pk["to_play"][g]) == s["to_play"] and int(pk["move_index"][g]) == t + 1
                else:
                    assert int(pk["move_index"][g]) == 0 and int(pk["game_id"][g]) == g + B
        for rec in _drain(loop):
            if rec["game_id"] < B:
                finished[rec["game_id"]] = rec
    eng.close()
    assert sorted(finished) == list(range(B))
    for g, rec in finished.items():
        steps = games[g]
        assert rec["length"] == len(steps) and rec["first_to_play"] == 0 and rec["obs"][0].tolist() == first.tolist()
        assert rec["action"].tolist() == [s["action"] for s in steps]
        assert rec["reward"].tolist() == [float(s["reward"]) for s in steps]
        assert rec["to_play"].tolist() == [s["to_play"] for s in steps]
        assert rec["obs"][1:].astype(numpy.int8).tolist() == [s["obs"] for s in steps]


def test_gomoku_full_board_without_five_pays_the_last_mover():
    """A forced sequence filling all 121 cells with no five in a row: the game ends on move 121, which alone is paid."""
    from test_device_games_cpu import _full_board_without_five
    actions = _full_board_without_five()
    mod, cfg, spec, eng, loop = _loop("gomoku", 1, 2)
    recs = []
    for a in actions:
        loop.moves(1, 1.0, forced_action=numpy.array([a], numpy.int32))
        recs += _drain(loop)
    eng.close()
    assert len(recs) == 1 and recs[0]["length"] == 121 and recs[0]["action"].tolist() == actions
    assert recs[0]["reward"].tolist() == [0.0] * 120 + [1.0]


def test_twentyone_device_games_replay_through_the_plugin_rules():
    """Every game the device plays is replayed by games/twentyone.py's rules with cards from oracle.cards.card for its
    (seed, game id): identical observations, rewards and end."""
    tw = load_game_module("twentyone")
    seed, B = 0x2101, 64
    mod, cfg, spec, eng, loop = _loop("twentyone", B, 6, seed=seed)
    recs = []
    for _ in range(12):
        loop.moves(1, 1.0)
        recs += _drain(loop)
    eng.close()
    assert len(recs) > B
    rewards, hits = set(), 0
    for rec in recs:
        env = tw.TwentyOneVector(1, cards=[_philox_cards(seed, rec["game_id"])])
        obs = env.reset()
        assert numpy.array_equal(obs[0].astype(numpy.float32).ravel(), rec["obs"][0]), rec["game_id"]
        T = rec["length"]
        for t in range(T):
            obs, reward, done = env.step([int(rec["action"][t])])
            assert numpy.array_equal(obs[0].astype(numpy.float32).ravel(), rec["obs"][t + 1]), (rec["game_id"], t)
            assert float(reward[0]) == rec["reward"][t] and bool(done[0]) == (t + 1 == T), (rec["game_id"], t)
            hits += rec["action"][t] == 0
        rewards.add(float(rec["reward"][-1]))
    assert {-10.0, 10.0} <= rewards and hits > 0


# ------------------------------------------------------------------------------------------ the loop
@pytest.mark.parametrize("name,B,N,moves,over", [("gomoku", 16, 8, 10, {}), ("twentyone", 48, 10, 10, {}),
                                                  ("simple_grid", 48, 10, 10, {})])
def test_device_loop_equals_host_composition_with_injected_draws(name, B, N, moves, over, monkeypatch):
    """One move at a time with the host's draws injected (root noise, action uniforms): the action the device plays and
    the record it keeps equal [mz_search on the peeked observation] + [select_action with numpy's choice rule]."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    mod, cfg, spec, eng, loop = _loop(name, B, N, seed=5, **over)
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=5)
    ref.load_weights(weights_for(name, spec))
    A = spec.action_space
    rs = numpy.random.RandomState(17)
    expected, delivered = {}, []
    for t in range(moves):
        pk = loop.peek()
        legal = pk["legal_mask"]
        gam = rs.standard_gamma(cfg.root_dirichlet_alpha, size=(B, A)) * (legal > 0)
        noise = gam / gam.sum(1, keepdims=True)
        u = rs.random_sample(B)
        out = ref.search(obs=pk["obs"], legal_mask=legal, to_play=pk["to_play"], add_exploration_noise=True, noise=noise,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        want = numpy.array([om.select_action([int(a) for a in numpy.nonzero(legal[g])[0]],
                                             out.visit_counts[g][legal[g] > 0], 1.0, om.InjectedDraws(uniform=u[g]))
                            for g in range(B)])
        for g in range(B):
            expected.setdefault(int(pk["game_id"][g]), []).append((out.visit_counts[g].copy(), out.root_value[g], int(want[g])))
        loop.moves(1, 1.0, uniform=u, noise=noise)
        after = loop.peek()
        restarted = after["move_index"] == 0
        assert (after["last_action"][~restarted] == want[~restarted]).all()
        delivered += _drain(loop)
    eng.close(); ref.close()
    if name == "gomoku":
        assert not delivered                       # ten moves end no Gomoku game: the slots' state carried the moves
    for rec in delivered:
        exp = expected[rec["game_id"]]
        assert rec["length"] == len(exp)
        for t, (visits, root_value, action) in enumerate(exp):
            assert rec["visits"][t].tolist() == visits.tolist() and rec["root_value"][t] == root_value
            assert rec["action"][t] == action
    if name != "gomoku":
        assert len(delivered) >= B


@pytest.mark.parametrize("name,max_moves", [("gomoku", 9), ("twentyone", 21), ("simple_grid", 6)])
def test_histories_are_batch_and_rank_invariant(name, max_moves):
    """Global games 16..31 have the same histories as slots 16..31 of a 32-game batch and as slots 0..15 of a 16-game
    batch whose first id is 16: every draw, Twenty-One's cards included, is keyed by (seed, global game id, move)."""
    def games(B, first):
        mod, cfg, spec, eng, loop = _loop(name, B, 6, seed=3, first_game_id=first, max_moves=max_moves)
        out = {}
        for _ in range(max_moves + 2):
            loop.moves(1, 1.0)
            for rec in _drain(loop):
                out[rec["game_id"]] = rec
        eng.close()
        return out
    a, b = games(32, 0), games(16, 16)
    common = [g for g in range(16, 32) if g in a and g in b]
    assert len(common) == 16
    for g in common:
        for key in ("action", "visits", "root_value", "reward", "obs"):
            assert numpy.array_equal(a[g][key], b[g][key]), (g, key)


@pytest.mark.parametrize("name", ["gomoku", "twentyone", "simple_grid"])
def test_selfplay_api_on_the_device_loop(name, monkeypatch):
    """SelfPlay.play_moves with rng_mode="philox" takes the device loop: PackedGameHistory objects with the reference's
    attribute set, float64 observations and int rewards; they pickle as plain GameHistory; the device PER priorities
    equal reanalyse.initial_priorities (pinned to the reference's ReplayBuffer.save_game in the CPU suite).  Test games
    come back in the same shape."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200 import self_play as sp
    mod, cfg = _cfg(name, max_moves=14) if name == "gomoku" else _cfg(name)
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 24, "philox", 6
    worker = sp.SelfPlay({"weights": weights_for(name, netspec_from_config(cfg))}, mod.Game, cfg, seed=0)
    assert worker.loop_path == "device"
    games = []
    for _ in range(6):
        games += list(worker.play_moves(4, 1.0))
    assert games and worker.env_steps == 24 * 24 and worker.played_games == len(games)
    for gh in games[:16]:
        T = len(gh.action_history) - 1
        assert isinstance(gh, sp.GameHistory) and T == len(gh) >= 1
        assert len(gh.child_visits) == T == len(gh.root_values) and len(gh.observation_history) == T + 1
        assert gh.observation_history[0].shape == tuple(cfg.observation_shape)
        assert gh.observation_history[0].dtype == numpy.float64 and all(type(r) is int for r in gh.reward_history)
        assert all(abs(sum(c) - 1) < 1e-12 for c in gh.child_visits)
        plain = pickle.loads(pickle.dumps(gh))
        assert type(plain) is sp.GameHistory and plain.child_visits == gh.child_visits
        assert plain.reward_history == gh.reward_history
        want, _ = ra.initial_priorities(gh, cfg)
        numpy.testing.assert_allclose(gh.priorities, want, rtol=2e-7, atol=0)
    worker.reset_stream()
    tests, summary = worker.play_test_games(10)
    assert len(tests) == 10 == summary["games"]
    for gh in tests:
        assert type(pickle.loads(pickle.dumps(gh))) is sp.GameHistory
        if name == "gomoku":                     # the config's opponent, "random": no root value at its moves
            assert [v is not None for v in gh.root_values] == [tp == 0 for tp in gh.to_play_history[:-1]]
        else:
            assert all(v is not None for v in gh.root_values)
    worker.close()


def test_shipped_gomoku_net_on_the_device_loop(monkeypatch):
    """The shipped 6 x 128-channel Gomoku towers play the device loop at small B and N: every move legal, visit counts
    over legal cells only."""
    from muzero_general_b200 import self_play as sp
    cfg = load_game_module("gomoku").MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 2, "philox", 4
    worker = sp.SelfPlay({"weights": weights_for("gomoku", netspec_from_config(cfg))}, load_game_module("gomoku").Game,
                         cfg, seed=0)
    assert worker.loop_path == "device"
    worker.play_moves(3, 1.0)
    pk = worker._device_loop.loop.peek()
    worker.close()
    assert (pk["move_index"] == 3).all() and (pk["legal_mask"].sum(1) == 118).all()
    obs = pk["obs"].reshape(2, 3, 121)
    assert (obs[:, 0].sum(1) == 2).all() and (obs[:, 1].sum(1) == 1).all() and (obs[:, 2] == -1).all()


# ------------------------------------------------------------------------------------------ Gomoku test games
@pytest.mark.parametrize("muzero_player,T", [(0, 0.0), (0, 1.0), (1, 0.0), (1, 1.0)])
def test_gomoku_test_games_against_random_equal_host_composition(muzero_player, T, monkeypatch):
    """Gomoku against "random", cut at 12 - muzero_player moves (max_moves): MuZero's moves equal [search of the peeked state] +
    [uniform53(seed, game, move, 0, TAG_ACTION)] + [numpy's choice rule], the opponent's moves are NaN, zero visits and
    legal[floor(u * n_legal)] for uniform53(seed, game, move, 0, 0x7169E005); rewards, observations and ends replay."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    B, N, seed, L = 16, 6, 0x5EED_0000_0077 + muzero_player, 12 - muzero_player
    mod, cfg, spec, eng, loop = _loop("gomoku", B, N, seed=seed, opponent="random", muzero_player=muzero_player,
                                      max_moves=L)
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    ref.load_weights(weights_for("gomoku", spec))
    expected, recs = {}, {}
    for _ in range(8):
        pk = loop.peek()
        assert (pk["to_play"] == muzero_player).all()
        out = ref.search(obs=pk["obs"], legal_mask=pk["legal_mask"], to_play=pk["to_play"], add_exploration_noise=True,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        for g in range(B):
            gid, mv = int(pk["game_id"][g]), int(pk["move_index"][g])
            u = philox.uniform53(seed, gid, mv, 0, philox.TAG_ACTION)
            idx = [int(a) for a in numpy.nonzero(pk["legal_mask"][g])[0]]
            expected[(gid, mv)] = (out.visit_counts[g].copy(), out.root_value[g],
                                   om.select_action(idx, out.visit_counts[g][idx], T, om.InjectedDraws(uniform=float(u))))
        loop.moves(1, T)
        for rec in _drain(loop):
            recs[rec["game_id"]] = rec
    eng.close(); ref.close()
    assert len(recs) >= B
    for gid, rec in recs.items():
        env = mod.Game(0)
        env.reset()
        T = rec["length"]
        assert T <= L and rec["first_to_play"] == 0
        for t in range(T):
            if env.to_play() == muzero_player:
                visits, root, action = expected[(gid, t)]
                assert rec["visits"][t].tolist() == visits.tolist() and rec["root_value"][t] == root, (gid, t)
                assert rec["action"][t] == action, (gid, t)
            else:
                assert numpy.isnan(rec["root_value"][t]) and not rec["visits"][t].any(), (gid, t)
                legal = env.legal_actions()
                u = philox.uniform53(seed, gid, t, 0, TAG_OPPONENT)
                assert rec["action"][t] == legal[min(int(u * len(legal)), len(legal) - 1)], (gid, t)
            obs, reward, done = env.step(int(rec["action"][t]))
            assert numpy.array_equal(numpy.asarray(obs, numpy.float32).ravel(), rec["obs"][t + 1]), (gid, t)
            assert float(reward) == float(rec["reward"][t]) and rec["to_play"][t] == env.to_play(), (gid, t)
            assert done == (t + 1 == T < L) or (not done and t + 1 == T == L), (gid, t)


def test_gomoku_expert_is_refused():
    """The reference's Gomoku has no expert_agent: MZ_EUNSUPPORTED from mz_selfplay_begin_vs and from
    mz_debug_opponent_action, NotImplementedError from the Python loop."""
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine, debug_opponent_action
    mod, cfg = _cfg("gomoku")
    eng = SearchEngine(cfg, max_games=4, num_simulations=2)
    d = _lib.MzSelfPlayDesc()
    d.env, d.max_moves, d.reward_scale = _lib.MZ_ENV_GOMOKU, cfg.max_moves, 1
    assert eng.lib.mz_selfplay_begin_vs(eng._h, C.byref(d), _lib.MZ_OPPONENT_EXPERT, 0) == _lib.MZ_EUNSUPPORTED
    assert "no expert" in eng.lib.mz_last_error(eng._h).decode()
    with pytest.raises(NotImplementedError, match="no expert"):
        DeviceSelfPlayLoop(eng, "gomoku", cfg.max_moves, opponent="expert")
    for name in ("twentyone", "simple_grid"):
        _, c = _cfg(name)
        e2 = SearchEngine(c, max_games=4, num_simulations=2)
        with pytest.raises(_lib.MzError, match="one player") as err:
            DeviceSelfPlayLoop(e2, name, c.max_moves, opponent="random")
        assert err.value.code == -1
        e2.close()
    eng.close()
    with pytest.raises(_lib.MzError, match="no expert") as err:
        debug_opponent_action("gomoku", numpy.zeros((1, 121)), [1], uniforms=[0.5], opponent="expert")
    assert err.value.code == _lib.MZ_EUNSUPPORTED


def test_gomoku_random_opponent_on_random_positions():
    """debug_opponent_action("gomoku", ..., opponent="random") equals legal[floor(u * n_legal)] on 20000 random
    positions from empty to one free cell, with uniforms next to 0 and 1 included."""
    from muzero_general_b200.engine import debug_opponent_action
    rs = numpy.random.RandomState(29)
    n = 20000
    boards = numpy.zeros((n, 121), numpy.int8)
    for i in range(n):
        k = rs.randint(0, 121)
        cells = rs.permutation(121)[:k]
        boards[i, cells] = rs.choice([-1, 1], size=k)
    players = rs.choice([-1, 1], size=n)
    u = rs.random_sample(n)
    u[:100] = numpy.nextafter(1.0, 0.0)
    u[100:200] = 0.0
    got = debug_opponent_action("gomoku", boards, players, uniforms=u, opponent="random")
    for i in range(n):
        legal = numpy.nonzero(boards[i] == 0)[0]
        assert got[i] == legal[min(int(u[i] * len(legal)), len(legal) - 1)], i


# ------------------------------------------------------------------------------------------ networks and searches
@pytest.mark.parametrize("name", ["twentyone", "simple_grid"])
def test_network_matches_the_reference(name):
    """The reference network's outputs (net_*.npz) within DESIGN.md 3.6's fp32 tolerances: logits rtol 2e-4 /
    atol 2e-5, hidden states rtol 2e-4 / atol 5e-5, scalars 5e-4."""
    from muzero_general_b200.engine import SearchEngine
    _, cfg = _cfg(name)
    spec = netspec_from_config(cfg)
    g = golden_npz(f"net_{name}.npz")
    n = len(g["obs"])
    eng = SearchEngine(cfg, max_games=n, num_simulations=4)
    eng.load_weights(weights_for(name, spec))
    logits, hidden, scalar = dict(rtol=2e-4, atol=2e-5), dict(rtol=2e-4, atol=5e-5), dict(rtol=2e-4, atol=5e-4)
    r0 = eng.initial_inference(g["obs"])
    numpy.testing.assert_allclose(r0["hidden"], g["init_hidden"].reshape(n, -1), **hidden)
    numpy.testing.assert_allclose(r0["value_logits"], g["init_value"], **logits)
    numpy.testing.assert_allclose(r0["policy_logits"], g["init_policy"], **logits)
    numpy.testing.assert_allclose(r0["value"], g["init_value_scalar"], **scalar)
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(n, -1), g["action"])
    numpy.testing.assert_allclose(r1["hidden"], g["rec_hidden"].reshape(n, -1), **hidden)
    for key, ref_key in (("value_logits", "rec_value"), ("reward_logits", "rec_reward"), ("policy_logits", "rec_policy")):
        numpy.testing.assert_allclose(r1[key], g[ref_key], **logits)
    numpy.testing.assert_allclose(r1["value"], g["rec_value_scalar"], **scalar)
    numpy.testing.assert_allclose(r1["reward"], g["rec_reward_scalar"], **scalar)
    r2 = eng.recurrent_inference(g["rec_hidden"].reshape(n, -1), (g["action"] + 1) % spec.action_space)
    numpy.testing.assert_allclose(r2["hidden"], g["rec2_hidden"].reshape(n, -1), **hidden)
    numpy.testing.assert_allclose(r2["policy_logits"], g["rec2_policy"], **logits)
    eng.close()


@pytest.mark.parametrize("name", ["twentyone", "simple_grid"])
def test_search_reproduces_the_reference_visit_counts(name):
    """Own networks + the reference's noise and first pick (mcts_*.json): the reference's visit counts exactly."""
    from muzero_general_b200.engine import SearchEngine
    _, cfg = _cfg(name)
    spec = netspec_from_config(cfg)
    A = spec.action_space
    for c in golden_json(f"mcts_{name}.json"):
        eng = SearchEngine(cfg, max_games=1, num_simulations=c["num_simulations"])
        eng.load_weights(weights_for(name, spec))
        obs = numpy.array(c["obs"], numpy.float32).reshape(1, -1)
        noise = numpy.zeros((1, A)); noise[0, c["legal"]] = c["noise"]
        out = eng.search(obs=obs, legal_mask=numpy.ones((1, A), numpy.uint8), to_play=numpy.zeros(1, numpy.int32),
                         add_exploration_noise=True, noise=noise, first_index=numpy.array([c["first_index"]], numpy.int32))
        eng.close()
        assert [int(out.visit_counts[0, a]) for a in c["root_actions"]] == c["root_visits"]
        assert abs(out.root_value[0] - c["root_value"]) <= 2e-4 * max(1.0, abs(c["root_value"]))
