"""Action spaces of 129 to 256 actions (tree_wide.cu's eight-children-per-lane instantiation) and Gomoku on 15 x 15 and
16 x 16 in the device self-play loop: the tree against the C oracle bit for bit, the environment against the
reference's playouts, the loop against host compositions.  Everything goes through the C ABI."""
import ctypes as C
import pickle

import numpy
import pytest

from helpers import oracle_replay, paths_from_trace, random_teacher
from muzero_general_b200 import _lib
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
from oracle import mcts as om
from oracle import philox
from test_wide_actions_cpu import wide_config, wide_env_games, wide_search_cases

pytestmark = pytest.mark.gpu


def _engine(cfg, n, N, **kw):
    from muzero_general_b200.engine import SearchEngine
    return SearchEngine(cfg, max_games=n, num_simulations=N, **kw)


def _edge_masks(legal, A):
    """Rows 0..2: legal actions only above id 128, only in mask word 4 (ids 128..159), and the single id A - 1."""
    legal[0, :128] = 0; legal[0, A - 1] = 1
    legal[1] = 0; legal[1, 128:min(A, 160)] = 1
    legal[2] = 0; legal[2, A - 1] = 1
    return legal


# ------------------------------------------------------------------------------------------ the tree
@pytest.mark.parametrize("A", [121, 128, 129, 160, 225, 255, 256])
def test_teacher_forced_search_equals_the_c_oracle(A):
    """Host noise and first-simulation picks, partial legal masks, both players: visit counts, root values, value
    ranges, tie counts, depths and every selected path, bit for bit.  121 and 128 run the four-children instantiation."""
    from oracle import build_c
    cfg = wide_config(A)
    n, N, P, D = 24, 60, 2, 60
    rs = numpy.random.RandomState(1000 + A)
    legal = (rs.uniform(size=(n, A)) < 0.8).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    if A > 128:
        legal = _edge_masks(legal, A)
    t = random_teacher(rs, n, N, A, reward_scale=0.0, legal=legal)
    t["priors"][3:6] = numpy.float32(1.0 / 256); t["value"][3:6] = 0; t["reward"][3:6] = 0      # exact ties at every level
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n) * legal
    noise /= noise.sum(1, keepdims=True)
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    first = numpy.where(rs.uniform(size=n) < 0.5, rs.randint(0, A, n), -1).astype(numpy.int32)
    gid = rs.randint(0, 1 << 40, n).astype(numpy.int64)
    mv = rs.randint(0, 250, n).astype(numpy.int32)
    ref = build_c.tree_search(n, N, A, P, cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction,
                              legal, to_play, noise, first, cfg.seed, gid, mv, t, D=D)
    eng = _engine(cfg, n, N)
    out = eng.search(legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise, first_index=first,
                     game_id=gid, move_index=mv, teacher=t, trace=True, trace_depth=D, n_games=n)
    eng.close()
    assert (out.visit_counts == ref["visit_counts"]).all() and (out.visit_counts.sum(1) == N).all()
    assert (out.visit_counts[legal == 0] == 0).all()
    assert (out.root_value == ref["root_value"]).all()
    assert (out.max_tree_depth == ref["max_depth"]).all()
    assert (out.tie_count == ref["ties"]).all() and ref["ties"][3:6].sum() > 0
    assert (out.value_range == ref["range"]).all()
    assert (out.trace["depth"] == ref["depth"]).all()
    mask = numpy.arange(D)[None, None, :] < ref["depth"][:, :, None]
    assert (numpy.where(mask, out.trace["actions"], 0) == numpy.where(mask, ref["actions"], 0)).all()
    if A > 128:
        assert out.visit_counts[2, A - 1] == N and out.trace["actions"][2, :, 0].tolist() == [A - 1] * N


@pytest.mark.parametrize("A,alpha", [(129, 0.25), (225, 0.3), (256, 0.3)])
def test_device_drawn_noise_equals_restated_gamma(A, alpha):
    """Action k = lane + 32 j draws with counter k for j up to 7: the restated draws of oracle/philox.py, 1e-12 relative."""
    from test_selfplay_sampling_gpu import _check_noise, _noise_case
    cfg = wide_config(A, root_dirichlet_alpha=alpha)
    n, N = 96, 4
    legal, t, to_play, gid, mv = _noise_case(cfg, n, N, numpy.random.RandomState(A))
    legal = _edge_masks(legal, A)
    eng = _engine(cfg, n, N, seed=77)
    out = eng.search(legal_mask=legal, to_play=to_play, add_exploration_noise=True, game_id=gid, move_index=mv,
                     teacher=t, trace=True, n_games=n)
    eng.close()
    assert _check_noise(out.trace["noise"], legal, 77, gid, mv, alpha) > n // 2


def test_student_forced_search_and_continued_tree_on_225_actions(monkeypatch):
    """The device's own network outputs on the 15 x 15 synthetic net, replayed through the oracle tree, give the same
    search (trace actions up to 224 pass through the uint8 field); the exported tree, imported again, exports equal and
    continues as the root of a new search."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    cfg = wide_config(board_size=15)
    spec = netspec_from_config(cfg)
    cases = wide_search_cases()[1:]
    n, N, A = len(cases), cases[0]["num_simulations"], 225
    obs = numpy.array([c["obs"] for c in cases], numpy.float32).reshape(n, 3, 15, 15)
    legal = numpy.zeros((n, A), numpy.uint8)
    for i, c in enumerate(cases):
        legal[i, c["legal"]] = 1
    rs = numpy.random.RandomState(7)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n) * legal
    noise /= noise.sum(1, keepdims=True)
    first = rs.randint(0, 200, n).astype(numpy.int32)
    to_play = numpy.array([c["to_play"] for c in cases], numpy.int32)
    eng = _engine(cfg, n, N)
    eng.load_weights(synthetic_weights(spec, 0))
    out = eng.search(obs=obs, legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise, first_index=first,
                     trace=True, keep_tree=True, stepwise=True)
    params = om.SearchParams.from_config(cfg, N)
    tr = out.trace
    for i in range(n):
        acts = [int(a) for a in numpy.nonzero(legal[i])[0]]
        res, _ = oracle_replay(params, acts, int(to_play[i]),
                               (out.root_predicted_value[i], tr["root_reward"][i], [tr["root_priors_raw"][i, a] for a in acts]),
                               [(tr["value"][i, s], tr["reward"][i, s], tr["priors"][i, s]) for s in range(N)],
                               [noise[i, a] for a in acts], int(first[i]), seed=cfg.seed, game=i)
        assert [int(out.visit_counts[i, a]) for a in acts] == res.root_visits and out.root_value[i] == res.root_value
        assert paths_from_trace(tr, i, N) == [s.path_actions for s in res.sims]
        assert max(max(p) for p in paths_from_trace(tr, i, N) if p) > 128
    tree = eng.export_tree(0, with_hidden=True)
    eng.close()
    assert tree["n_expansions"] == N + 1 and tree["root_visit"] == N
    assert tree["child_visit"][:A].tolist() == out.visit_counts[0].tolist()
    one = _engine(cfg, 1, N, extra_expansions=N + 1)          # override_root_with: a single-game handle with room
    one.load_weights(synthetic_weights(spec, 0))
    one.import_tree(0, tree)
    again = one.export_tree(0, with_hidden=True)
    used = (N + 1) * A
    for k in ("child_visit", "child_value_sum", "child_reward", "child_prior", "child_expansion"):
        assert numpy.array_equal(numpy.asarray(tree[k])[:used], numpy.asarray(again[k])[:used]), k
    assert numpy.array_equal(tree["hidden"][:N + 1], again["hidden"][:N + 1])
    cont = one.search(add_exploration_noise=True, keep_tree=True, continue_tree=True, n_games=1, to_play=to_play[:1])
    assert cont.visit_counts[0].sum() > N and (cont.visit_counts[0] >= out.visit_counts[0]).all()
    one.close()


def test_fc_net_with_200_actions_against_the_oracle_network():
    """A fully connected net with 200 actions runs the step-wise route: policy logits of the initial and recurrent
    inference against the oracle network within the fp32 tolerances of the other FC routes, and a search that visits
    legal actions only."""
    import torch
    from oracle.net import OracleNet
    cfg = load_game_module("cartpole").MuZeroConfig()
    cfg.action_space = list(range(200))
    spec = netspec_from_config(cfg)
    w = synthetic_weights(spec, 0)
    n, N = 16, 12
    rs = numpy.random.RandomState(2)
    obs = rs.uniform(-0.05, 0.05, size=(n, 1, 1, 4)).astype(numpy.float32)
    eng = _engine(cfg, n, N)
    eng.load_weights(w)
    net = OracleNet(spec, w)
    r0 = eng.initial_inference(obs)
    v, r, pol, h = net.initial_inference(obs)
    assert r0["policy_logits"].shape == (n, 200)
    numpy.testing.assert_allclose(r0["policy_logits"], pol.numpy(), rtol=2e-5, atol=2e-6)
    act = rs.randint(128, 200, size=(n, 1)).astype(numpy.int64)
    r1 = eng.recurrent_inference(h.numpy(), act)
    v1, rw1, pol1, h1 = net.recurrent_inference(h, torch.from_numpy(act))
    numpy.testing.assert_allclose(r1["policy_logits"], pol1.numpy(), rtol=1e-4, atol=1e-5)
    numpy.testing.assert_allclose(r1["hidden"], h1.numpy(), rtol=1e-4, atol=1e-5)
    legal = numpy.zeros((n, 200), numpy.uint8)
    legal[:, 130:200:3] = 1
    out = eng.search(obs=obs, legal_mask=legal, add_exploration_noise=True)
    eng.close()
    assert (out.visit_counts.sum(1) == N).all() and (out.visit_counts[legal == 0] == 0).all()


# ------------------------------------------------------------------------------------------ Gomoku on the device
def _loop(side, B, N, seed=0, opponent="self", muzero_player=0, stack=0, **over):
    from muzero_general_b200.engine import DeviceSelfPlayLoop
    mod = load_game_module("gomoku")
    cfg = wide_config(board_size=side, blocks=1, stacked_observations=stack, **over)
    spec = netspec_from_config(cfg)
    eng = _engine(cfg, B, N, seed=seed)
    eng.load_weights(synthetic_weights(spec, 0))
    loop = DeviceSelfPlayLoop(eng, "gomoku", cfg.max_moves, temperature_threshold=cfg.temperature_threshold, reward_scale=1,
                              opponent=opponent, muzero_player=muzero_player, stacked_observations=stack)
    return mod, cfg, spec, eng, loop


def _drain(loop):
    from muzero_general_b200.engine import parse_staged_games
    return parse_staged_games(*loop.drain())


@pytest.mark.parametrize("side", [15, 16])
def test_device_gomoku_replays_the_reference_playouts(side):
    """Slot g is forced through the reference's game g: peeked observation, legal mask and side to move after every
    move; the four edge lines end their games with reward 1, the random playout is ended by max_moves alone."""
    games, cut = wide_env_games(side)
    B = len(games)
    mod, cfg, spec, eng, loop = _loop(side, B, 2, max_moves=cut)
    finished = {}
    pk = loop.peek()
    assert pk["obs"].shape == (B, 3 * side * side) and (pk["legal_mask"].sum(1) == side * side).all()
    for t in range(cut):
        forced = numpy.array([games[g][t]["action"] if t < len(games[g]) else int(numpy.nonzero(pk["legal_mask"][g])[0][0])
                              for g in range(B)], numpy.int32)
        loop.moves(1, 1.0, forced_action=forced)
        pk = loop.peek()
        for g in range(B):
            if t < len(games[g]) and not games[g][t]["done"] and t + 1 < cut:
                s = games[g][t]
                assert pk["obs"][g].astype(numpy.int8).tolist() == s["obs"], (g, t)
                assert numpy.nonzero(pk["legal_mask"][g])[0].tolist() == s["legal"]
                assert int(pk["to_play"][g]) == s["to_play"] and int(pk["move_index"][g]) == t + 1
        for rec in _drain(loop):
            finished.setdefault(rec["game_id"], rec)
    eng.close()
    for g in range(B):
        rec, steps = finished[g], games[g]
        assert rec["length"] == len(steps) and rec["action"].tolist() == [s["action"] for s in steps]
        assert rec["reward"].tolist() == [float(s["reward"]) for s in steps]
        assert rec["to_play"].tolist() == [s["to_play"] for s in steps]
        assert rec["obs"][1:].astype(numpy.int8).tolist() == [s["obs"] for s in steps]
    assert [finished[g]["reward"][-1] for g in range(B)] == [1.0] * 4 + [0.0] and finished[B - 1]["length"] == cut


@pytest.mark.parametrize("side,T,stack", [(15, 1.0, 0), (15, 0.0, 2), (16, 1.0, 2), (16, 0.0, 0)])
def test_device_loop_equals_host_composition(side, T, stack, monkeypatch):
    """One move at a time: the action the device plays equals [search of the peeked input] + [the device's uniform] +
    [numpy's choice rule], and the plug-in's step of that action gives the next peeked observation."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    B, N, seed, A = 8, 6, 0x5EED_0015, side * side
    mod, cfg, spec, eng, loop = _loop(side, B, N, seed=seed, stack=stack)
    ref = _engine(cfg, B, N, seed=seed)
    ref.load_weights(synthetic_weights(spec, 0))
    envs = mod.Game.vector(B, 0, side)
    envs.reset()
    for t in range(7):
        pk = loop.peek()
        assert numpy.array_equal(pk["obs"][:, :3 * A], envs.observations().reshape(B, -1).astype(numpy.float32))
        assert numpy.array_equal(pk["legal_mask"], envs.legal_mask())
        out = ref.search(obs=pk["obs"], legal_mask=pk["legal_mask"], to_play=pk["to_play"], add_exploration_noise=True,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        want = []
        for g in range(B):
            u = philox.uniform53(seed, int(pk["game_id"][g]), int(pk["move_index"][g]), 0, philox.TAG_ACTION)
            idx = [int(a) for a in numpy.nonzero(pk["legal_mask"][g])[0]]
            want.append(om.select_action(idx, out.visit_counts[g][idx], T, om.InjectedDraws(uniform=float(u))))
        loop.moves(1, T)
        assert loop.peek()["last_action"].tolist() == want, t
        envs.step(want)
        if stack:
            # GameHistory.get_stacked_observations: after the current observation, the previous one and its action plane
            tail = loop.peek()["obs"][:, 3 * A:7 * A].reshape(B, 4, A)
            assert numpy.array_equal(tail[:, :3].reshape(B, -1), pk["obs"][:, :3 * A])
            assert numpy.array_equal(tail[:, 3, 0], (numpy.array(want, numpy.float64) / A).astype(numpy.float32))
    eng.close(); ref.close()


@pytest.mark.parametrize("muzero_player", [0, 1])
def test_selfplay_api_at_board_size_15(muzero_player, monkeypatch):
    """MuZeroConfig(board_size=15) with rng_mode="philox" takes the device loop and plays whole games; histories
    pickle as plain GameHistory; the device priorities at td_steps 3 equal reanalyse.initial_priorities; test games
    against "random" come back for either side."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200 import self_play as sp
    mod = load_game_module("gomoku")
    cfg = wide_config(board_size=15, blocks=1, max_moves=14, td_steps=3, muzero_player=muzero_player)
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 12, "philox", 6
    worker = sp.SelfPlay({"weights": synthetic_weights(netspec_from_config(cfg), 0)}, mod.Game.sized(15), cfg, seed=0)
    assert worker.loop_path == "device"
    games = []
    for _ in range(4):
        games += list(worker.play_moves(4, 1.0))
    assert len(games) >= 12
    for gh in games[:12]:
        T = len(gh.action_history) - 1
        assert T == 14 and gh.observation_history[0].shape == (3, 15, 15) and len(gh.child_visits[0]) == 225
        assert max(gh.action_history) > 128 or T == 0
        plain = pickle.loads(pickle.dumps(gh))
        assert type(plain) is sp.GameHistory and plain.child_visits == gh.child_visits
        want, _ = ra.initial_priorities(gh, cfg)
        numpy.testing.assert_allclose(gh.priorities, want, rtol=2e-7, atol=0)
    worker.reset_stream()
    tests, summary = worker.play_test_games(6)
    assert len(tests) == 6 == summary["games"]
    for gh in tests:
        assert [v is not None for v in gh.root_values] == [tp == muzero_player for tp in gh.to_play_history[:-1]]
    worker.close()


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_are_host_side_checks():
    """257 actions at mz_create; a Gomoku action space that is no square, or whose side is outside 5..16, at
    mz_selfplay_begin - each a return code and a message that names the value."""
    with pytest.raises(NotImplementedError, match=r"\[1, 256\]"):          # MZ_EUNSUPPORTED, as the engine raises it
        _engine(wide_config(257), 2, 2)
    for A in (120, 16, 200):
        eng = _engine(wide_config(A, blocks=1), 2, 2)
        d = _lib.MzSelfPlayDesc()
        d.env, d.max_moves, d.reward_scale = _lib.MZ_ENV_GOMOKU, 20, 1
        assert eng.lib.mz_selfplay_begin(eng._h, C.byref(d)) == -1          # MZ_EINVAL
        assert f"has {A} actions" in eng.lib.mz_last_error(eng._h).decode()
        eng.close()
    eng = _engine(wide_config(225), 2, 4, extra_expansions=5)
    t = random_teacher(numpy.random.RandomState(0), 2, 4, 225)
    with pytest.raises(_lib.MzError, match="extra_expansions = 0"):
        eng.search(teacher=t, trace=True, n_games=2)
    eng.close()
