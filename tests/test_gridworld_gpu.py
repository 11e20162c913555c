"""Gridworld in the device self-play loop (csrc/selfplay.cu, MZ_ENV_GRIDWORLD) against the plug-in's rules with the
device's placement (oracle/gridworld.py), host compositions of search + sampling (+ the stack), the SelfPlay API, the
host-stepped loop on GridworldVector, and the reference's network and search fixtures.  Everything goes through the
C ABI."""
import itertools
import pickle

import numpy
import pytest

from conftest import golden_json, golden_npz, weights_for
from muzero_general_b200 import _lib
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from oracle import gridworld
from oracle import mcts as om

pytestmark = pytest.mark.gpu

gw = load_game_module("gridworld")


def _cfg(**over):
    cfg = gw.MuZeroConfig()
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def _loop(B, N, seed=0, first_game_id=0, opponent="self", **over):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    cfg = _cfg(**over)
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    eng.load_weights(weights_for("gridworld", spec))
    loop = DeviceSelfPlayLoop(eng, "gridworld", cfg.max_moves, temperature_threshold=cfg.temperature_threshold,
                              first_game_id=first_game_id, opponent=opponent,
                              stacked_observations=cfg.stacked_observations)
    return cfg, spec, eng, loop


def _drain(loop):
    from muzero_general_b200.engine import parse_staged_games
    return parse_staged_games(*loop.drain())


def _replay(rec, seed, max_moves):
    """Replays a staged game through the plug-in's rules from the device's placement: observations, fp32 rewards and
    the end must be the record's.  Returns the rewards."""
    gid, T = rec["game_id"], rec["length"]
    env = gw.GridworldVector(1, places=[lambda: gridworld.placement(seed, gid)])
    obs = env.reset()
    assert numpy.array_equal(obs[0].astype(numpy.float32).ravel(), rec["obs"][0]), gid
    rewards = []
    for t in range(T):
        obs, reward, done = env.step([int(rec["action"][t])])
        assert numpy.array_equal(obs[0].astype(numpy.float32).ravel(), rec["obs"][t + 1]), (gid, t)
        assert numpy.float32(reward[0]) == rec["reward"][t], (gid, t)
        assert not done[0] or t + 1 == T, (gid, t)
        rewards.append(float(reward[0]))
    assert done[0] or T == max_moves, gid
    return rewards, int(env.step_count[0])


# ------------------------------------------------------------------------------------------ rules
@pytest.mark.parametrize("max_moves", [15, 150])
def test_device_games_replay_through_the_plugin_rules(max_moves):
    """Every game the device plays is replayed by games/gridworld.py's rules with the placement of oracle.gridworld for
    its (seed, game id): identical observations (all four directions, walls beyond the room), fp32 rewards, ends and
    lengths.  At max_moves = 150 slot 0 only turns, so its game ends at the 144-step cap with reward 0."""
    seed, B = 0x6D1D, 128
    cfg, spec, eng, loop = _loop(B, 4, seed=seed, max_moves=max_moves)
    forced = numpy.full(B, -1, numpy.int32)
    forced[0] = 0
    recs = []
    for _ in range(max_moves + 2):
        loop.moves(1, 1.0, forced_action=forced if max_moves == 150 else None)
        recs += _drain(loop)
    eng.close()
    assert len(recs) >= B
    goals, dirs = 0, set()
    for rec in recs:
        rewards, steps = _replay(rec, seed, max_moves)
        goals += rewards[-1] > 0
        dirs.add(gridworld.placement(seed, rec["game_id"])[2])
        if rec["game_id"] == 0 and max_moves == 150:
            assert rec["length"] == 144 == steps and rewards == [0.0] * 144
    assert goals > 0 and dirs == {0, 1, 2, 3}


# ------------------------------------------------------------------------------------------ the loop
@pytest.mark.parametrize("T", [1.0, 0.0])
def test_device_loop_equals_host_composition_with_injected_draws(T, monkeypatch):
    """One move at a time with the host's draws injected (root noise, action uniforms): the action the device plays and
    the record it keeps equal [mz_search on the peeked observation] + [select_action with numpy's choice rule]."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    B, N, moves = 48, 10, 20
    cfg, spec, eng, loop = _loop(B, N, seed=5)
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=5)
    ref.load_weights(weights_for("gridworld", spec))
    A = spec.action_space
    rs = numpy.random.RandomState(17)
    expected, delivered = {}, []
    for _ in range(moves):
        pk = loop.peek()
        legal = pk["legal_mask"]
        assert (legal == 1).all() and (pk["to_play"] == 0).all()
        gam = rs.standard_gamma(cfg.root_dirichlet_alpha, size=(B, A)) * (legal > 0)
        noise = gam / gam.sum(1, keepdims=True)
        u = rs.random_sample(B)
        out = ref.search(obs=pk["obs"], legal_mask=legal, to_play=pk["to_play"], add_exploration_noise=True, noise=noise,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        want = numpy.array([om.select_action(list(range(A)), out.visit_counts[g], T, om.InjectedDraws(uniform=u[g]))
                            for g in range(B)])
        for g in range(B):
            expected.setdefault(int(pk["game_id"][g]), []).append((out.visit_counts[g].copy(), out.root_value[g], int(want[g])))
        loop.moves(1, T, uniform=u, noise=noise)
        after = loop.peek()
        restarted = after["move_index"] == 0
        assert (after["last_action"][~restarted] == want[~restarted]).all()
        delivered += _drain(loop)
    eng.close(); ref.close()
    assert len(delivered) >= B
    for rec in delivered:
        exp = expected[rec["game_id"]]
        assert rec["length"] == len(exp)
        for t, (visits, root_value, action) in enumerate(exp):
            assert rec["visits"][t].tolist() == visits.tolist() and rec["root_value"][t] == root_value
            assert rec["action"][t] == action


def test_histories_are_batch_and_rank_invariant():
    """Global games 16..31 have the same histories as slots 16..31 of a 32-game batch and as slots 0..15 of a 16-game
    batch whose first id is 16: every draw, the placement included, is keyed by (seed, global game id, draw)."""
    def games(B, first):
        cfg, spec, eng, loop = _loop(B, 6, seed=3, first_game_id=first)
        out = {}
        for _ in range(cfg.max_moves + 2):
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


def test_stacked_observations_equal_a_host_composition(monkeypatch):
    """stacked_observations = 2: every search input equals get_stacked_observations of the drained game (7 planes of
    7 x 3 per observation and a 7 x 3 action plane), and every action equals [mz_search on that input] + [sampling]
    with the host's draws injected."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    s, B, N = 2, 32, 6
    cfg, spec, eng, loop = _loop(B, N, seed=9, stacked_observations=s)
    assert eng.obs_elems == (7 * (s + 1) + s) * 7 * 3
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=9)
    ref.load_weights(weights_for("gridworld", spec))
    A = spec.action_space
    rs = numpy.random.RandomState(23)
    peeked, expected, recs = {}, {}, []
    for _ in range(2 * cfg.max_moves + 2):
        pk = loop.peek()
        gam = rs.standard_gamma(cfg.root_dirichlet_alpha, size=(B, A))
        noise = gam / gam.sum(1, keepdims=True)
        u = rs.random_sample(B)
        out = ref.search(obs=pk["obs"], legal_mask=pk["legal_mask"], to_play=pk["to_play"], add_exploration_noise=True,
                         noise=noise, game_id=pk["game_id"], move_index=pk["move_index"])
        for g in range(B):
            key = (int(pk["game_id"][g]), int(pk["move_index"][g]))
            peeked[key] = pk["obs"][g].copy()
            expected[key] = (out.visit_counts[g].copy(), om.select_action(list(range(A)), out.visit_counts[g], 1.0,
                                                                          om.InjectedDraws(uniform=u[g])))
        loop.moves(1, 1.0, uniform=u, noise=noise)
        recs += _drain(loop)
    eng.close(); ref.close()
    assert len(recs) >= B
    shape = tuple(cfg.observation_shape)
    for rec in recs:
        obs = [numpy.asarray(o, numpy.float64).reshape(shape) for o in rec["obs"]]
        actions = [0] + [int(a) for a in rec["action"]]
        for t in range(rec["length"]):
            key = (rec["game_id"], t)
            want = om.stacked_observation(obs, actions, t, s, A).astype(numpy.float32).ravel()
            assert peeked[key].tobytes() == want.tobytes(), key
            visits, action = expected[key]
            assert rec["visits"][t].tolist() == visits.tolist() and rec["action"][t] == action, key


def test_selfplay_api_on_the_device_loop(monkeypatch):
    """SelfPlay.play_moves with rng_mode="philox" takes the device loop: PackedGameHistory objects with uint8 (7, 7, 3)
    observations and float rewards that pickle as plain GameHistory; with PER = True and td_steps = 20 the device
    priorities equal reanalyse.initial_priorities.  Test games against "self" come back in the same shape."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200 import self_play as sp
    cfg = _cfg(PER=True, td_steps=20)
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 24, "philox", 6
    worker = sp.SelfPlay({"weights": weights_for("gridworld", netspec_from_config(cfg))}, gw.Game, cfg, seed=0)
    assert worker.loop_path == "device"
    games = []
    for _ in range(6):
        games += list(worker.play_moves(4, 1.0))
    assert games and worker.env_steps == 24 * 24 and worker.played_games == len(games)
    assert any(gh.reward_history[-1] > 0 for gh in games)
    for gh in games[:16]:
        T = len(gh.action_history) - 1
        assert isinstance(gh, sp.GameHistory) and T == len(gh) >= 1
        assert len(gh.child_visits) == T == len(gh.root_values) and len(gh.observation_history) == T + 1
        assert gh.observation_history[0].shape == (7, 7, 3) and gh.observation_history[0].dtype == numpy.uint8
        assert all(type(r) is float for r in gh.reward_history[1:])
        plain = pickle.loads(pickle.dumps(gh))
        assert type(plain) is sp.GameHistory and plain.reward_history == gh.reward_history
        want, _ = ra.initial_priorities(gh, cfg)
        numpy.testing.assert_allclose(gh.priorities, want, rtol=2e-7, atol=0)
    worker.reset_stream()
    tests, summary = worker.play_test_games(10)
    assert len(tests) == 10 == summary["games"]
    for gh in tests:
        assert type(pickle.loads(pickle.dumps(gh))) is sp.GameHistory and all(v is not None for v in gh.root_values)
    worker.close()


def test_an_opponent_is_refused():
    """Gridworld has one player: mz_selfplay_begin_vs refuses "random" and "expert" with MZ_EINVAL."""
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    cfg = _cfg()
    eng = SearchEngine(cfg, max_games=4, num_simulations=2)
    for opponent in ("random", "expert"):
        with pytest.raises(_lib.MzError, match="Gridworld has one player") as err:
            DeviceSelfPlayLoop(eng, "gridworld", cfg.max_moves, opponent=opponent)
        assert err.value.code == -1
    eng.close()


# ------------------------------------------------------------------------------------------ the host-stepped loop
def test_host_stepped_loop_plays_gridworld_vector_games(monkeypatch):
    """With device_envs = False and host_env_device_loop = True the host steps GridworldVector.  Given the device's
    placement for each slot's game ids, its games equal the device loop's field by field."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200 import self_play as sp
    B, seed = 32, 0x51
    weights = weights_for("gridworld", netspec_from_config(_cfg()))

    def play(device_envs):
        cfg = _cfg(PER=True)
        cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = B, "philox", 6
        cfg.device_envs, cfg.host_env_device_loop = device_envs, not device_envs
        worker = sp.SelfPlay({"weights": weights}, gw.Game, cfg, seed=seed)
        assert worker.loop_path == ("device" if device_envs else "device-host-env")
        games = {}
        for _ in range(8):
            for gh in worker.play_moves(4, 1.0):
                games[gh.game_id] = gh
        worker.close()
        return games

    def vector(num_games, _seed=None):
        places = []
        for g in range(num_games):
            ids = itertools.count(g, num_games)
            places.append(lambda ids=ids: gridworld.placement(seed, next(ids)))
        return gw.GridworldVector(num_games, places=places)

    device = play(True)
    monkeypatch.setattr(gw.Game, "vector", staticmethod(vector))
    host = play(False)
    common = sorted(set(device) & set(host))
    assert len(common) >= B
    for gid in common:
        a, b = device[gid], host[gid]
        assert a.action_history == b.action_history and a.reward_history == b.reward_history, gid
        assert a.root_values == b.root_values and a.child_visits == b.child_visits, gid
        assert all(numpy.array_equal(x, y) and y.dtype == numpy.uint8
                   for x, y in zip(a.observation_history, b.observation_history)), gid
        assert numpy.array_equal(a.priorities, b.priorities), gid


# ------------------------------------------------------------------------------------------ network and search
def test_network_matches_the_reference():
    """The reference network's outputs (net_gridworld.npz) within DESIGN.md 3.6's fp32 tolerances: logits rtol 2e-4 /
    atol 2e-5, hidden states rtol 2e-4 / atol 5e-5, scalars 5e-4."""
    from muzero_general_b200.engine import SearchEngine
    cfg = _cfg()
    spec = netspec_from_config(cfg)
    g = golden_npz("net_gridworld.npz")
    n = len(g["obs"])
    eng = SearchEngine(cfg, max_games=n, num_simulations=4)
    eng.load_weights(weights_for("gridworld", spec))
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


def test_search_reproduces_the_reference_visit_counts():
    """Own network + the reference's noise and first pick (mcts_gridworld.json): the reference's visit counts exactly."""
    from muzero_general_b200.engine import SearchEngine
    cfg = _cfg()
    spec = netspec_from_config(cfg)
    A = spec.action_space
    for c in golden_json("mcts_gridworld.json"):
        eng = SearchEngine(cfg, max_games=1, num_simulations=c["num_simulations"])
        eng.load_weights(weights_for("gridworld", spec))
        obs = numpy.array(c["obs"], numpy.float32).reshape(1, -1)
        noise = numpy.zeros((1, A)); noise[0, c["legal"]] = c["noise"]
        out = eng.search(obs=obs, legal_mask=numpy.ones((1, A), numpy.uint8), to_play=numpy.zeros(1, numpy.int32),
                         add_exploration_noise=True, noise=noise, first_index=numpy.array([c["first_index"]], numpy.int32))
        eng.close()
        assert [int(out.visit_counts[0, a]) for a in c["root_actions"]] == c["root_visits"]
        assert abs(out.root_value[0] - c["root_value"]) <= 2e-4 * max(1.0, abs(c["root_value"]))
