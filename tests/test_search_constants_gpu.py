"""Every tree-search route at search constants no shipped game uses (the sets K1..K4 of
oracle/gen_golden_search_constants.py: discounts 0.9, 0.5, 0.997 and 0, pb_c_base 5 to 1e6, pb_c_init 0.5 to 3, root
exploration fractions 0 to 1), in both player modes, against the C oracle bit for bit, and in closed loop against the
reference's own searches at those constants.

Teacher-forced batches carry rewards of both signs (root rewards too), games whose value range stays flat at a nonzero
value (lo == hi, where MinMaxStats.normalize returns its argument), a game whose path grows one level per simulation
(past every lane-group width G, into the backup's unpacked loop) and quantised games with exact ties; each case asserts
that this coverage was real on the device.

One-line faults of the tree, each built into the library and run against this file on an H100:

* M1 - the two-player node value of the backup without its discount, ``r + (-q)`` for ``r + discount * -q``
  (tree.cuh::tree_backup): the packed reciprocal branch (M1a), the packed IEEE branch (M1b), the unpacked loop (M1c).
* M2 - the root noise mixed at 0.25 instead of the config's fraction: tree.cuh::tree_init_root (M2a, the fused
  searches), tree_kernels.cu's root kernel (M2b, the step-wise pipeline), tree_wide.cu (M2c).
* M3 - the host's exploration tables at the default pb_c constants (engine.py's pb_c_table / ucb_table).  abi.cu's own
  tables are only built when a caller passes none, which engine.py never does, so that copy has no route from Python.
* M4 - value_range_normalize returning 0 for a flat range (hi <= lo) instead of the value.
* M5 - the two-player reward's sign flipped in the backup's unpacked value recurrence.

Which tests fail under each fault (H100 80GB HBM3 at 700 W).  The counts are of the 198 cases other than
test_continued_tree_matches_reference[K3]; that case was run against M1b and M2b only:

* M1a: 54 - test_teacher_forced_equals_c_oracle (48: the fused routes at P = 2, where the fused kernel takes the
  reciprocal branch), test_student_forced_cartpole_shape (4), test_teacher_forced_reference_traces (2).
* M1b: 48 - test_teacher_forced_equals_c_oracle (24: the step-wise kernels at P = 2), the wide tree (16), the closed loop
  (5), the reference traces (2), the continued tree at K1 (1; the K3 case passes).
* M1c: 89 - test_teacher_forced_equals_c_oracle (72), the wide tree (16), the reference traces (1): the game that grows
  one level per simulation takes every route into the unpacked loop.
* M2a: 82 - test_teacher_forced_equals_c_oracle (72), test_student_forced_cartpole_shape (4), the closed loop (5), the
  reference traces (1).
* M2b: test_continued_tree_matches_reference[K3] only.  tree_kernels.cu's noise mixing runs in tree_adopt_root_kernel,
  at the root of a search continued from an imported tree, so only a continued search at a fraction other than 0.25
  (the literal itself, K1's fraction) can see it.
* M2c: 16 - test_teacher_forced_wide_equals_c_oracle at every set whose fraction is not 0.25 (K2, K3).
* M3: 143 - every route at the sets with other pb_c constants: the teacher-forced tests (108 + 24), the closed loop (6),
  test_student_forced_cartpole_shape (4), the reference traces (1).
* M4: 176 - every teacher-forced case (144 + 32): each holds games whose range stays flat at a nonzero value.
* M5: 90 - test_teacher_forced_equals_c_oracle (72), the wide tree (16), the closed loop (1), the reference traces (1).
"""
import numpy
import pytest

from helpers import oracle_replay, paths_from_trace, teacher_from_cases
from muzero_general_b200.netspec import netspec_from_config
from oracle import build_c
from oracle import mcts as om
from oracle.gen_golden_search_constants import CONSTANTS, OVERRIDE_KEYS, load_fixture, reward_signed_weights
from test_search_constants_cpu import KEYS, N_FLAT, constants_config, flat_point, signed_case

pytestmark = pytest.mark.gpu


def _engine(cfg, n, N, **kw):
    from muzero_general_b200.engine import SearchEngine
    return SearchEngine(cfg, max_games=n, num_simulations=N, **kw)


def _lane_group(A):
    """Lanes per game of the step-wise tree kernels (tree_kernels.cu::launch_tree_step; 32 above 32 actions)."""
    G = 4
    while G < A:
        G <<= 1
    return min(G, 32)


def _assert_equals_c_oracle(out, ref, N, D):
    assert (out.visit_counts == ref["visit_counts"]).all()
    assert (out.root_value == ref["root_value"]).all()
    assert (out.max_tree_depth == ref["max_depth"]).all()
    assert (out.tie_count == ref["ties"]).all()
    assert (out.value_range == ref["range"]).all()
    assert (out.trace["depth"] == ref["depth"]).all()
    mask = numpy.arange(D)[None, None, :] < ref["depth"][:, :, None]
    assert (numpy.where(mask, out.trace["actions"], 0) == numpy.where(mask, ref["actions"], 0)).all()


def _teacher_forced(cfg, key, P, A, G, route, monkeypatch, n=12, N=40):
    t, legal, noise, to_play, gid, mv = signed_case(A, P, key, n, N, seed=31 * A + 5 * P + KEYS.index(key))
    first = numpy.full(n, -1, numpy.int32)
    first[1::2] = numpy.arange(1, n, 2) % A
    D = N + 1
    ref = build_c.tree_search(n, N, A, P, cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction,
                              legal, to_play, noise, first, cfg.seed, gid, mv, t, D=D)
    eng = _engine(cfg, n, N)
    n0 = eng.launch_count
    out = eng.search(legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise, first_index=first,
                     game_id=gid, move_index=mv, teacher=t, trace=True, trace_depth=D, stepwise=route == "stepwise",
                     n_games=n)
    launches = eng.launch_count - n0
    fc = eng.last_fc_launch if route != "stepwise" else None
    eng.close()
    if route != "stepwise":
        assert launches == 1 and fc["group"] == G            # the fused FC kernel ran, at this lane-group width
    _assert_equals_c_oracle(out, ref, N, D)
    # coverage: a path at least G deep, rewards of both signs on the paths, a flat nonzero range, exact ties
    assert out.max_tree_depth[0] >= G
    assert t["reward"].min() < 0 < t["reward"].max() and t["root_reward"].min() < 0 < t["root_reward"].max()
    _, v = flat_point(cfg.discount, P)
    assert (out.value_range[:N_FLAT] == v).all()
    assert out.tie_count.sum() > 0


@pytest.mark.parametrize("route", ["fused", "fused_one_level", "stepwise"])
@pytest.mark.parametrize("A", [2, 3, 7, 9, 16, 32])
@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("key", KEYS)
def test_teacher_forced_equals_c_oracle(key, P, A, route, monkeypatch, game_configs):
    """The fused FC kernel (default multi-level selection and one level per round) and the step-wise tree kernels."""
    cfg = constants_config(game_configs["cartpole"], key, A, P)
    G = 32 if A > 16 else 16
    monkeypatch.setenv("MZ_FC_GROUP", str(G))
    if route == "fused_one_level":
        monkeypatch.setenv("MZ_FC_SELECT_LEVELS", "1")
    else:
        monkeypatch.delenv("MZ_FC_SELECT_LEVELS", raising=False)
    _teacher_forced(cfg, key, P, A, _lane_group(A) if route == "stepwise" else G, route, monkeypatch)


@pytest.mark.parametrize("A", [64, 121, 129, 225])
@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("key", KEYS)
def test_teacher_forced_wide_equals_c_oracle(key, P, A, monkeypatch, game_configs):
    """tree_wide.cu: four children per lane up to 128 actions, eight above."""
    cfg = constants_config(game_configs["cartpole"], key, A, P)
    _teacher_forced(cfg, key, P, A, 32, "stepwise", monkeypatch, n=8, N=40)


@pytest.mark.parametrize("G", [16, 32])
@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("key", ["K1", "K2"])
def test_student_forced_cartpole_shape(key, P, G, monkeypatch, game_configs):
    """The unrolled CartPole-shaped network in the fused kernel, with P = 1 fixed and with run-time P: the device's own
    outputs, replayed through the oracle tree, give the same search."""
    cfg = constants_config(game_configs["cartpole"], key, P=P)
    spec = netspec_from_config(cfg)
    monkeypatch.setenv("MZ_FC_GROUP", str(G))
    monkeypatch.delenv("MZ_FC_SELECT_LEVELS", raising=False)
    monkeypatch.delenv("MZ_FC_GENERIC", raising=False)
    n, N, A = 48, 50, 2
    rs = numpy.random.RandomState(11 + G + P)
    obs = rs.uniform(-0.05, 0.05, size=(n, 1, 1, 4)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    first = rs.randint(0, A, n).astype(numpy.int32)
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    eng = _engine(cfg, n, N)
    eng.load_weights(reward_signed_weights("cartpole", spec))
    n0 = eng.launch_count
    out = eng.search(obs=obs, to_play=to_play, add_exploration_noise=True, noise=noise, first_index=first, trace=True,
                     trace_depth=N + 1)
    assert eng.launch_count - n0 == 1 and eng.last_fc_launch["group"] == G
    eng.close()
    params = om.SearchParams.from_config(cfg, N)
    tr = out.trace
    assert tr["reward"].min() < 0 < tr["reward"].max()
    for i in range(n):
        res, _ = oracle_replay(
            params, [0, 1], int(to_play[i]), (out.root_predicted_value[i], tr["root_reward"][i], list(tr["root_priors_raw"][i])),
            [(tr["value"][i, s], tr["reward"][i, s], tr["priors"][i, s]) for s in range(N)],
            list(noise[i]), int(first[i]), seed=cfg.seed, game=i)
        assert [int(v) for v in out.visit_counts[i]] == res.root_visits, i
        assert out.root_value[i] == res.root_value
        assert (out.value_range[i, 0], out.value_range[i, 1]) == (res.range_lo, res.range_hi)
        assert paths_from_trace(tr, i, N) == [s.path_actions for s in res.sims]


CLOSED_LOOP = [(k, g) for k in KEYS for g in CONSTANTS[k][4]]


@pytest.mark.parametrize("key,game", CLOSED_LOOP)
def test_closed_loop_matches_reference_counts(key, game, monkeypatch, game_configs):
    """Whole searches on the device's own networks (the reference's noise and first pick) give the reference's visit
    counts exactly and its depth; the root value within fp32 network tolerance."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    cfg = constants_config(game_configs[game], key)
    spec = netspec_from_config(cfg)
    w = reward_signed_weights(game, spec)
    for c in load_fixture()[key][game]:
        eng = _engine(cfg, 1, c["num_simulations"])
        eng.load_weights(w)
        obs = numpy.array(c["obs"], numpy.float32).reshape(1, *c["obs_shape"])
        legal = numpy.zeros((1, len(cfg.action_space)), numpy.uint8)
        legal[0, c["legal"]] = 1
        noise = numpy.zeros((1, len(cfg.action_space)))
        noise[0, c["legal"]] = c["noise"]
        out = eng.search(obs=obs, legal_mask=legal, to_play=numpy.array([c["to_play"]], numpy.int32),
                         add_exploration_noise=True, noise=noise, first_index=numpy.array([c["first_index"]], numpy.int32))
        eng.close()
        assert [int(out.visit_counts[0, a]) for a in c["root_actions"]] == c["root_visits"]
        assert out.max_tree_depth[0] == c["max_tree_depth"]
        assert abs(out.root_value[0] - c["root_value"]) <= 1e-4 * max(1.0, abs(c["root_value"]))


@pytest.mark.parametrize("key", ["K1", "K2"])
def test_teacher_forced_reference_traces(key, game_configs):
    """The reference's own per-simulation outputs at these constants, both routes, every traced field."""
    for game in CONSTANTS[key][4]:
        cfg = constants_config(game_configs[game], key)
        A = len(cfg.action_space)
        for stepwise in (False, True):
            for c in load_fixture()[key][game]:
                N = c["num_simulations"]
                t, legal, noise, first, to_play = teacher_from_cases([c], A, N)
                eng = _engine(cfg, 1, N)
                out = eng.search(legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise,
                                 first_index=first, teacher=t, trace=True, trace_depth=N + 1, stepwise=stepwise, n_games=1)
                eng.close()
                assert [int(out.visit_counts[0, a]) for a in c["root_actions"]] == c["root_visits"]
                assert out.root_value[0] == c["root_value"] and out.max_tree_depth[0] == c["max_tree_depth"]
                assert [out.root_priors[0, a] for a in c["root_actions"]] == c["root_priors"]
                assert paths_from_trace(out.trace, 0, N) == [s["actions"] for s in c["sims"]]


@pytest.mark.parametrize("key", ["K1", "K2"])
def test_fused_small_search_equals_stepwise_pipeline(key, monkeypatch, game_configs):
    """TicTacToe's small residual net at these constants: the one-launch search (small_search.cu) against the step-wise
    pipeline, bit for bit, two-player rewards of both signs included."""
    cfg = constants_config(game_configs["tictactoe"], key)
    spec = netspec_from_config(cfg)
    A, n, N = spec.action_space, 96, 30
    rs = numpy.random.RandomState(3)
    obs = rs.randint(0, 2, size=(n, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    legal = (rs.uniform(size=(n, A)) < 0.7).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    to_play = rs.randint(0, 2, n).astype(numpy.int32)
    results = []
    for on in ("0", "1"):
        monkeypatch.setenv("MZ_SMALL_SEARCH", on)
        eng = _engine(cfg, n, N)
        eng.load_weights(reward_signed_weights("tictactoe", spec))
        n0 = eng.launch_count
        runs = [eng.search(obs=obs, legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise,
                           keep_tree=True) for _ in range(3)]
        per_search = (eng.launch_count - n0) // 3
        trees = [eng.export_tree(i) for i in range(0, n, 8)]
        results.append((runs[-1], per_search, trees))
        eng.close()
    (a, la, ta), (b, lb, tb) = results
    assert la - lb == 5 * N - 1, (la, lb)             # one search launch instead of five per simulation
    assert numpy.array_equal(a.visit_counts, b.visit_counts)
    assert numpy.array_equal(a.root_value, b.root_value)
    assert numpy.array_equal(a.value_range, b.value_range)
    assert numpy.array_equal(a.max_tree_depth, b.max_tree_depth)
    assert numpy.array_equal(a.tie_count, b.tie_count)
    for x, y in zip(ta, tb):
        for k in ("child_visit", "child_value_sum", "child_reward"):
            assert numpy.array_equal(x[k], y[k]), k
    rewards = numpy.concatenate([x["child_reward"] for x in ta])
    assert rewards.min() < 0 < rewards.max()


@pytest.mark.parametrize("key", OVERRIDE_KEYS)
def test_continued_tree_matches_reference(key, monkeypatch):
    """override_root_with (self_play.py:275-277): the most visited child of a finished TicTacToe search becomes the root
    of a second one.  mz_import_tree restates each imported child's node value with the discount and the two-player sign,
    and the adopted root mixes fresh noise at the config's fraction (all noise at K3); the continued search reproduces the
    reference's visit counts exactly."""
    from muzero_general_b200 import self_play as sp
    from muzero_general_b200.games import load_game_module
    monkeypatch.setenv("MZ_TC_MODE", "off")
    fx = load_fixture()["override"][key]
    first, case = fx["first"], fx["cases"][0]
    mod = load_game_module("tictactoe")
    cfg = constants_config(mod.MuZeroConfig(), key)
    cfg.num_simulations = first["num_simulations"]
    worker = sp.SelfPlay({"weights": reward_signed_weights("tictactoe", netspec_from_config(cfg))}, mod.Game, cfg, 0)
    obs = numpy.array(first["obs"]).reshape(first["obs_shape"])
    numpy.random.seed(0)
    root, _ = sp.MCTS(cfg).run(worker.model, obs, first["legal"], first["to_play"], True)
    assert [root.children[a].visit_count for a in first["root_actions"]] == first["root_visits"]
    action = int(sp.SelfPlay.select_action(root, 0))
    assert action == case["action"]
    node = root.children[action]
    assert node.visit_count == case["pre_visits"]
    root2, info2 = sp.MCTS(cfg).run(worker.model, None, cfg.action_space, case["to_play"], True, node)
    worker.model.engine.close()
    assert list(root2.children.keys()) == case["root_actions"]
    assert [root2.children[a].visit_count for a in case["root_actions"]] == case["root_visits"]
    assert root2.visit_count == case["root_visit_count"] and info2["max_tree_depth"] == case["max_tree_depth"]
    assert abs(root2.value() - case["root_value"]) <= 1e-4 * max(1.0, abs(case["root_value"]))
