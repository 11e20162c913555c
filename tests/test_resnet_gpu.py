"""GPU parity of the residual-network kernels and the step-wise search, in the three tower modes (MZ_TC_MODE):

  "off"   fp32 CUDA-core convs everywhere (reference arithmetic, different summation order)
  "x3"    DEFAULT for 64-channel board nets: wgmma towers on split fp16 operands (x = x_h + x_l/2^11), three partial products, fp32
          accumulation (csrc/conv_x3.cu) - fp32-grade, held to the SAME tolerance as "off"
  "fp16"  opt-in fast mode: plain fp16 operands (csrc/conv_tc.cu), 3x fewer MMAs; per-quantity bounds below

Tolerances (stated here, checked below): logits of "off" / "x3" agree with the reference (oneDNN/ATen on the CPU) to
rtol 2e-4, atol 2e-5; hidden states to rtol 2e-4, atol 5e-5 (the per-channel min-max rescale divides the tower output by
channel ranges down to ~0.05, amplifying its ~2e-6 fp32 noise); scalarised values / rewards to 5e-4 absolute
(support_to_scalar sums 21 softmax terms weighted by up to 10: fp32 logit noise of ~2e-6 is amplified ~100x).  "fp16": logits within 5e-3 absolute,
hidden states (after the per-channel min-max rescale, which divides by ranges as small as 1e-2) within 1.5e-2 for
99.9 % of the elements and 1e-1 for all, scalars within 3e-2."""
import numpy
import pytest

from conftest import golden_json, golden_npz, weights_for
from helpers import oracle_replay, paths_from_trace
from muzero_general_b200.netspec import netspec_from_config
from oracle import mcts as om

pytestmark = pytest.mark.gpu
TOL = dict(rtol=2e-4, atol=2e-5)
SCALAR_ATOL = 5e-4
VALUE_TOL = {"off": 2e-4, "x3": 2e-4, "fp16": 3e-2}


def _uses_tensor_cores(name):
    return name.startswith("connect4")


@pytest.fixture(params=["off", "x3", "fp16"])
def numerics(request, monkeypatch):
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.setenv("MZ_TC_MODE", request.param)
    return request.param


def _skip_redundant(name, numerics):
    if numerics != "off" and not _uses_tensor_cores(name):
        pytest.skip("no tensor-core towers for this net: identical to mode off")


def _close(name, got, want, numerics, kind):
    """kind: 'logits' | 'hidden' | 'scalar'."""
    got, want = numpy.asarray(got), numpy.asarray(want)
    err = numpy.abs(got - want)
    print(f"{name} [{numerics}] {kind}: max abs err {err.max():.3e}, max rel err {(err / (numpy.abs(want) + 1e-3)).max():.3e}")
    if numerics == "fp16":
        if kind == "logits":
            assert err.max() <= 5e-3, name
        elif kind == "hidden":
            assert err.max() <= 1e-1 and numpy.quantile(err, 0.999) <= 1.5e-2, name
        else:
            assert err.max() <= 3e-2, name
    elif kind == "scalar":
        numpy.testing.assert_allclose(got, want, rtol=2e-4, atol=SCALAR_ATOL, err_msg=name)
    elif kind == "hidden":
        numpy.testing.assert_allclose(got, want, rtol=2e-4, atol=5e-5, err_msg=name)
    else:
        numpy.testing.assert_allclose(got, want, err_msg=name, **TOL)


def _engine(cfg, max_games, N):
    from muzero_general_b200.engine import SearchEngine
    return SearchEngine(cfg, max_games=max_games, num_simulations=N)


def _report(name, got, want):
    err = numpy.abs(got - want)
    print(f"{name}: max abs err {err.max():.3e}, max rel err {(err / (numpy.abs(want) + 1e-3)).max():.3e}")


@pytest.mark.parametrize("name", ["tictactoe", "connect4", "breakout", "connect4_b64", "gomoku"])
def test_resnet_network_matches_reference(name, numerics, game_configs):
    _skip_redundant(name, numerics)
    cfg = game_configs[name.split("_")[0]]
    spec = netspec_from_config(cfg)
    g = golden_npz(f"net_{name}.npz")
    n = len(g["obs"])
    eng = _engine(cfg, n, 4)
    eng.load_weights(weights_for(name, spec))
    if _uses_tensor_cores(name):
        assert {"off": "f32 nets", "x3": "f32-grade nets", "fp16": "fp16 operands"}[numerics] in eng.numerics
    tag = f"{name}"
    r0 = eng.initial_inference(g["obs"])
    _close(tag + " init hidden", r0["hidden"], g["init_hidden"].reshape(n, -1), numerics, "hidden")
    _close(tag + " init value logits", r0["value_logits"], g["init_value"], numerics, "logits")
    _close(tag + " init policy logits", r0["policy_logits"], g["init_policy"], numerics, "logits")
    _close(tag + " init value", r0["value"], g["init_value_scalar"], numerics, "scalar")
    assert numpy.isneginf(r0["reward_logits"]).sum() == n * 20 and (r0["reward"] == 0).all()
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(n, -1), g["action"])
    _close(tag + " rec hidden", r1["hidden"], g["rec_hidden"].reshape(n, -1), numerics, "hidden")
    _close(tag + " rec value logits", r1["value_logits"], g["rec_value"], numerics, "logits")
    _close(tag + " rec reward logits", r1["reward_logits"], g["rec_reward"], numerics, "logits")
    _close(tag + " rec policy logits", r1["policy_logits"], g["rec_policy"], numerics, "logits")
    _close(tag + " rec value", r1["value"], g["rec_value_scalar"], numerics, "scalar")
    _close(tag + " rec reward", r1["reward"], g["rec_reward_scalar"], numerics, "scalar")
    r2 = eng.recurrent_inference(g["rec_hidden"].reshape(n, -1), (g["action"] + 1) % spec.action_space)
    _close(tag + " rec2 hidden", r2["hidden"], g["rec2_hidden"].reshape(n, -1), numerics, "hidden")
    _close(tag + " rec2 policy logits", r2["policy_logits"], g["rec2_policy"], numerics, "logits")
    eng.close()


def test_large_configuration_runs_on_the_device(game_configs):
    """games/atari.py (SURVEY.md 8f-4): 32 stacked observations = 131 input planes of 96x96, DownSample stem with 128/256
    channels (row-banded CUDA-core convolutions), 16 blocks x 256 channels, heads of 9216 -> 256 -> 256 -> 601 whose
    weights (9.4 MB per first layer) take the generic heads route.  Network outputs against the reference's, and a
    short search student-forced through the oracle tree."""
    cfg = game_configs["atari"]
    spec = netspec_from_config(cfg)
    assert spec.in_channels == 131 and spec.full_support == 601
    g = golden_npz("net_atari.npz")
    obs = numpy.random.RandomState(int(g["obs_seed"])).random_sample((2, spec.in_channels, 96, 96)).astype(numpy.float32)
    N = 6
    eng = _engine(cfg, 2, N)
    eng.load_weights(weights_for("atari", spec))
    r0 = eng.initial_inference(obs)
    _close("atari init hidden", r0["hidden"], g["init_hidden"].reshape(2, -1), "off", "hidden")
    _close("atari init value logits", r0["value_logits"], g["init_value"], "off", "logits")
    _close("atari init policy logits", r0["policy_logits"], g["init_policy"], "off", "logits")
    numpy.testing.assert_allclose(r0["value"], g["init_value_scalar"], rtol=1e-3, atol=5e-3)
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(2, -1), g["action"])
    _close("atari rec hidden", r1["hidden"], g["rec_hidden"].reshape(2, -1), "off", "hidden")
    _close("atari rec value logits", r1["value_logits"], g["rec_value"], "off", "logits")
    _close("atari rec reward logits", r1["reward_logits"], g["rec_reward"], "off", "logits")
    _close("atari rec policy logits", r1["policy_logits"], g["rec_policy"], "off", "logits")
    numpy.testing.assert_allclose(r1["reward"], g["rec_reward_scalar"], rtol=1e-3, atol=5e-3)
    A = spec.action_space
    rs = numpy.random.RandomState(3)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=2)
    first = rs.randint(0, A, 2).astype(numpy.int32)
    out = eng.search(obs=obs.reshape(2, -1), add_exploration_noise=True, noise=noise, first_index=first, trace=True)
    params = om.SearchParams.from_config(cfg, N)
    for i in range(2):
        tr = out.trace
        res, _ = oracle_replay(params, list(range(A)), 0,
                               (out.root_predicted_value[i], tr["root_reward"][i], list(tr["root_priors_raw"][i])),
                               [(tr["value"][i, s], tr["reward"][i, s], tr["priors"][i, s]) for s in range(N)],
                               list(noise[i]), int(first[i]), seed=cfg.seed, game=i)
        assert [int(v) for v in out.visit_counts[i]] == res.root_visits and out.root_value[i] == res.root_value
    eng.close()


@pytest.mark.parametrize("mode", ["large", "tiny", "overflow"])
def test_tower_range_guard_on_stress_weights(mode, game_configs, monkeypatch):
    """Weights whose tower activations reach ~1e4 ("large"), sit at ~1e-5 inside every block ("tiny") or exceed the fp16
    range ("overflow", ~2e7): the default x3 towers hold the fp32 tolerance on the first two WITHOUT leaving the tensor
    cores, and on the third the range guard notices, the handle switches to the fp32 CUDA-core towers and the call is
    redone - the caller sees reference-accurate numbers either way (fixtures: oracle/gen_golden.py::main_round2)."""
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.setenv("MZ_TC_MODE", "x3")
    name = f"connect4_stress_{mode}"
    cfg = game_configs["connect4"]
    spec = netspec_from_config(cfg)
    g = golden_npz(f"net_{name}.npz")
    info = golden_json("net_connect4_stress_info.json")[mode]
    assert {"large": 1e3 < info["max_activation"] < 65504, "tiny": info["min_layer_peak"] < 6e-5,
            "overflow": info["max_activation"] > 65504}[mode]
    n = len(g["obs"])
    eng = _engine(cfg, n, 4)
    eng.load_weights(weights_for(name, spec))
    assert "f32-grade nets" in eng.numerics
    r0 = eng.initial_inference(g["obs"])
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(n, -1), g["action"])
    if mode == "overflow":
        assert "left after an activation exceeded the fp16 range" in eng.numerics
    else:
        assert "f32-grade nets" in eng.numerics               # still on the tensor cores
    scale = lambda a: max(1.0, float(numpy.abs(a).max()))
    for got, want, what in ((r0["hidden"], g["init_hidden"].reshape(n, -1), "init hidden"),
                            (r0["value_logits"], g["init_value"], "init value logits"),
                            (r0["policy_logits"], g["init_policy"], "init policy logits"),
                            (r1["hidden"], g["rec_hidden"].reshape(n, -1), "rec hidden"),
                            (r1["value_logits"], g["rec_value"], "rec value logits"),
                            (r1["reward_logits"], g["rec_reward"], "rec reward logits"),
                            (r1["policy_logits"], g["rec_policy"], "rec policy logits")):
        err = numpy.abs(got - want)
        print(f"{name} {what}: max abs err {err.max():.3e} (scale {scale(want):.3e})")
        # rtol on the element, atol relative to the tensor's scale (logits of 1e4..1e7 carry fp32 noise of that scale)
        numpy.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-5 * scale(want), err_msg=f"{name} {what}")
    # a whole search still works after the switch / on the stressed towers
    out = eng.search(obs=g["obs"].reshape(n, -1), add_exploration_noise=False)
    assert (out.visit_counts.sum(1) == 4).all()
    eng.close()


@pytest.mark.parametrize("name,N,n", [("tictactoe", 50, 24), ("connect4", 40, 12), ("breakout", 12, 4), ("gomoku", 30, 6)])
def test_resnet_student_forced(name, N, n, numerics, game_configs):
    """Device search with its own residual networks, replayed through the oracle tree."""
    _skip_redundant(name, numerics)
    cfg = game_configs[name]
    spec = netspec_from_config(cfg)
    A, P = spec.action_space, len(cfg.players)
    rs = numpy.random.RandomState(11)
    if name == "breakout":
        obs = rs.random_sample((n, spec.in_channels) + spec.obs_shape[1:]).astype(numpy.float32)
        legal = numpy.ones((n, A), numpy.uint8)
    else:
        obs = rs.randint(0, 2, size=(n, spec.in_channels) + spec.obs_shape[1:]).astype(numpy.float32)
        legal = (rs.uniform(size=(n, A)) < 0.8).astype(numpy.uint8)
        legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    first = numpy.array([rs.randint(0, int(l.sum())) for l in legal], numpy.int32)
    eng = _engine(cfg, n, N)
    eng.load_weights(weights_for(name, spec))
    out = eng.search(obs=obs, legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise,
                     first_index=first, trace=True)
    params = om.SearchParams.from_config(cfg, N)
    for i in range(n):
        acts = [a for a in range(A) if legal[i, a]]
        tr = out.trace
        res, draws = oracle_replay(
            params, acts, int(to_play[i]),
            (out.root_predicted_value[i], tr["root_reward"][i], [tr["root_priors_raw"][i, a] for a in acts]),
            [(tr["value"][i, s], tr["reward"][i, s], tr["priors"][i, s]) for s in range(N)],
            [noise[i, a] for a in acts], int(first[i]), seed=cfg.seed, game=i)
        assert [int(out.visit_counts[i, a]) for a in acts] == res.root_visits
        assert out.root_value[i] == res.root_value
        assert paths_from_trace(tr, i, N) == [s.path_actions for s in res.sims]
        assert int(out.visit_counts[i].sum()) == N
    eng.close()


@pytest.mark.parametrize("name", ["tictactoe", "connect4", "breakout", "connect4_n200", "breakout_n50", "gomoku"])
def test_resnet_closed_loop_matches_reference_counts(name, numerics, game_configs):
    """Own networks + the reference's noise and first pick.  "off" and "x3": the reference's visit counts EXACTLY, at the
    BASELINE simulation counts too (Connect4 N=200, Breakout N=50).  "fp16": counts may move where two children are
    nearly tied, so the bound is on the visit distribution (total variation <= 5 %) and on the root value."""
    _skip_redundant(name, numerics)
    cfg = game_configs[name.split("_")[0]]
    spec = netspec_from_config(cfg)
    A = spec.action_space
    for c in golden_json(f"mcts_{name}.json"):
        eng = _engine(cfg, 1, c["num_simulations"])
        eng.load_weights(weights_for(name, spec))
        obs = numpy.array(c["obs"], numpy.float32).reshape(1, *c["obs_shape"])
        legal = numpy.zeros((1, A), numpy.uint8); legal[0, c["legal"]] = 1
        noise = numpy.zeros((1, A)); noise[0, c["legal"]] = c["noise"]
        out = eng.search(obs=obs, legal_mask=legal, to_play=numpy.array([c["to_play"]], numpy.int32),
                         add_exploration_noise=True, noise=noise, first_index=numpy.array([c["first_index"]], numpy.int32))
        got = [int(out.visit_counts[0, a]) for a in c["root_actions"]]
        if numerics != "fp16":
            assert got == c["root_visits"], (name, numerics)
            if name != "gomoku":
                assert out.max_tree_depth[0] == c["max_tree_depth"]
            else:       # 121 near-uniform priors: one 80-deep chain of near-ties; a 1e-6 logit difference moves its tail
                assert abs(int(out.max_tree_depth[0]) - c["max_tree_depth"]) <= 4
        else:
            tv = 0.5 * sum(abs(x - y) for x, y in zip(got, c["root_visits"])) / c["num_simulations"]
            print(f"{name}/fp16 visit counts {got} vs {c['root_visits']} (TV {tv:.3f})")
            assert tv <= 0.05 and sum(got) == c["num_simulations"]
        vt = VALUE_TOL[numerics]
        # gomoku's N=90 case sends 89 simulations down ONE chain; when its near-tied tail takes another branch (depth
        # differs) the last leaves carry other values: the root mean then agrees to a few percent, not to 2e-4
        rt = 0.05 if name == "gomoku" and int(out.max_tree_depth[0]) != c["max_tree_depth"] else vt
        assert abs(out.root_value[0] - c["root_value"]) <= rt * max(1.0, abs(c["root_value"]))
        assert abs(out.root_predicted_value[0] - c["root_predicted_value"]) <= vt * max(1.0, abs(c["root_predicted_value"]))
        eng.close()


@pytest.mark.parametrize("name,n", [("tictactoe", 700), ("breakout", 37), ("breakout", 200)])
def test_fused_cuda_core_tower_is_bit_identical_to_per_layer_launches(name, n, game_configs, monkeypatch):
    """small_tower.cu keeps conv3x3_kernel's accumulation order: one fused launch == one launch per conv, bit for bit
    (multi-tile grids, ragged last tile, gathered pool input with the action plane are all exercised by the search)."""
    cfg = game_configs[name]
    spec = netspec_from_config(cfg)
    rs = numpy.random.RandomState(5)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    actions = rs.randint(0, spec.action_space, size=n)
    outs = []
    for no_fuse in ("1", "0"):
        monkeypatch.setenv("MZ_TC_MODE", "off")
        monkeypatch.setenv("MZ_NO_FUSE", no_fuse)
        eng = _engine(cfg, n, 6)
        eng.load_weights(weights_for(name, spec))
        l0 = eng.launch_count
        r0 = eng.initial_inference(obs)
        l1 = eng.launch_count
        r1 = eng.recurrent_inference(r0["hidden"], actions)
        l2 = eng.launch_count
        res = eng.search(obs=obs, add_exploration_noise=False)
        outs.append((r0, r1, res, l1 - l0, l2 - l1))
        eng.close()
    (a0, a1, sa, la0, la1), (b0, b1, sb, lb0, lb1) = outs
    for k in ("hidden", "value_logits", "policy_logits", "value"):
        assert numpy.array_equal(a0[k], b0[k]), k
    for k in ("hidden", "value_logits", "policy_logits", "reward_logits", "value", "reward"):
        assert numpy.array_equal(a1[k], b1[k]), k
    assert numpy.array_equal(sa.visit_counts, sb.visit_counts)
    assert numpy.array_equal(sa.root_value, sb.root_value)
    assert lb1 < la1 and lb0 < la0, "fused path must need fewer launches"


@pytest.mark.parametrize("n", [5, 300, 1024])
def test_resident_tower_is_bit_identical_to_streaming_tower(n, game_configs, monkeypatch):
    """conv_tower_resident_kernel (activations stay in shared memory between layers) and conv_tower_tc_kernel
    (activations round-trip through L2) perform the same fp16 x fp16 -> fp32 MMAs and the same epilogue arithmetic."""
    cfg = game_configs["connect4"]
    spec = netspec_from_config(cfg)
    rs = numpy.random.RandomState(11)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    actions = rs.randint(0, spec.action_space, size=n)
    outs = []
    for flag in ("1", "0"):
        monkeypatch.setenv("MZ_TC_MODE", "fp16")
        monkeypatch.setenv("MZ_TC_NO_RESIDENT", flag)
        eng = _engine(cfg, n, 6)
        eng.load_weights(weights_for("connect4", spec))
        r0 = eng.initial_inference(obs)
        r1 = eng.recurrent_inference(r0["hidden"], actions)
        res = eng.search(obs=obs, add_exploration_noise=False)
        outs.append((r0, r1, res))
        eng.close()
    (a0, a1, sa), (b0, b1, sb) = outs
    for k in ("hidden", "value_logits", "policy_logits", "value"):
        assert numpy.array_equal(a0[k], b0[k]), k
    for k in ("hidden", "value_logits", "policy_logits", "reward_logits", "value", "reward"):
        assert numpy.array_equal(a1[k], b1[k]), k
    assert numpy.array_equal(sa.visit_counts, sb.visit_counts)


@pytest.mark.parametrize("name,n,N", [("connect4", 64, 30), ("tictactoe", 200, 25)])
def test_graph_replay_and_dependent_launch_do_not_change_results(name, n, N, game_configs, monkeypatch):
    """CUDA-graph replay and programmatic dependent launch only change WHEN kernels start: a search repeated three
    times (eager, capture, replay) with and without them gives identical visit counts and root values."""
    cfg = game_configs[name]
    spec = netspec_from_config(cfg)
    rs = numpy.random.RandomState(3)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    results = []
    for no_graph, no_pdl in (("1", "1"), ("0", "1"), ("0", "0")):
        monkeypatch.setenv("MZ_TC_MODE", "x3")
        monkeypatch.setenv("MZ_NO_GRAPH", no_graph)
        monkeypatch.setenv("MZ_NO_PDL", no_pdl)
        eng = _engine(cfg, n, N)
        eng.load_weights(weights_for(name, spec))
        runs = [eng.search(obs=obs, add_exploration_noise=False) for _ in range(3)]
        for r in runs[1:]:
            assert numpy.array_equal(r.visit_counts, runs[0].visit_counts)
            assert numpy.array_equal(r.root_value, runs[0].root_value)
        results.append(runs[0])
        eng.close()
    for r in results[1:]:
        assert numpy.array_equal(r.visit_counts, results[0].visit_counts)
        assert numpy.array_equal(r.root_value, results[0].root_value)


@pytest.mark.parametrize("mode", ["x3", "fp16"])
def test_tower_modes_agree_across_batch_sizes(mode, game_configs, monkeypatch):
    """The tensor-core towers pick their kernel / launch count by batch size (fp16: resident <= 1184 boards, streaming
    <= 2368 boards, one launch per conv above; x3: launches of <= 592 boards).  A batch of 2500 boards evaluated at once
    must equal the same boards evaluated in chunks, bit for bit."""
    cfg = game_configs["connect4"]
    spec = netspec_from_config(cfg)
    monkeypatch.setenv("MZ_TC_MODE", mode)
    n = 2500
    rs = numpy.random.RandomState(21)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    actions = rs.randint(0, spec.action_space, size=n)
    eng = _engine(cfg, n, 2)
    eng.load_weights(weights_for("connect4", spec))
    whole0 = eng.initial_inference(obs)
    whole1 = eng.recurrent_inference(whole0["hidden"], actions)
    for lo, hi in ((0, 1000), (1000, 2400), (2400, 2500)):
        part0 = eng.initial_inference(obs[lo:hi])
        part1 = eng.recurrent_inference(part0["hidden"], actions[lo:hi])
        for k in ("hidden", "value_logits", "policy_logits", "value"):
            assert numpy.array_equal(part0[k], whole0[k][lo:hi]), (k, lo)
        for k in ("hidden", "value_logits", "policy_logits", "reward_logits", "value", "reward"):
            assert numpy.array_equal(part1[k], whole1[k][lo:hi]), (k, lo)
    eng.close()


@pytest.mark.parametrize("name,n,N,parts", [("connect4", 300, 24, 2), ("connect4", 520, 12, 4), ("tictactoe", 400, 25, 3)])
def test_partitioned_replay_does_not_change_results(name, n, N, parts, game_configs, monkeypatch):
    """The replayed graph runs the simulations of disjoint game ranges as parallel branches (MZ_PARTS; default 2 for the
    tensor-core towers): the towers of one range overlap the heads and tree steps of the others.  Every game is still
    evaluated by the same arithmetic: visit counts, root values, value ranges and tree depths of the eager, captured
    and replayed searches equal those of a single-chain handle, bit for bit."""
    cfg = game_configs[name]
    spec = netspec_from_config(cfg)
    rs = numpy.random.RandomState(11)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * spec.action_space, size=n)
    monkeypatch.setenv("MZ_TC_MODE", "x3")
    results = []
    for p in (1, parts):
        monkeypatch.setenv("MZ_PARTS", str(p))
        eng = _engine(cfg, n, N)
        eng.load_weights(weights_for(name, spec))
        runs = [eng.search(obs=obs, add_exploration_noise=True, noise=noise) for _ in range(4)]
        assert eng.graph_partitions == p
        for r in runs[1:]:
            assert numpy.array_equal(r.visit_counts, runs[0].visit_counts)
            assert numpy.array_equal(r.root_value, runs[0].root_value)
        results.append(runs[-1])
        eng.close()
    a, b = results
    assert numpy.array_equal(a.visit_counts, b.visit_counts)
    assert numpy.array_equal(a.root_value, b.root_value)
    assert numpy.array_equal(a.value_range, b.value_range)
    assert numpy.array_equal(a.max_tree_depth, b.max_tree_depth)
    assert (b.visit_counts.sum(1) == N).all()


# TicTacToe configs with other boards and action spaces (16 channels, 1 block, heads of 4 reduced channels and 16 hidden
# units, so that several 6x6 games fit in a CTA) for the fused search's instantiations (P, CO, G): G = 4 lanes per game
# for |A| <= 4, 16 up to |A| = 16; P = 3 on 3-wide boards, and on 6-wide ones with CO = 1 (half rows); P = 6 with CO = 4
# on 6-wide boards.  "co4" sizes the batch with the planner: the smallest batch that gets CO = 4 on this device, plus 3.
SEARCH_BOARDS = {"ss_3x3_a9": (3, 3, 9), "ss_3x3_a4": (3, 3, 4), "ss_6x6_a4": (6, 6, 4), "ss_6x6_a16": (6, 6, 16)}
SEARCH_HEADS = dict(reduced_channels_reward=4, reduced_channels_value=4, reduced_channels_policy=4,
                    resnet_fc_reward_layers=[16], resnet_fc_value_layers=[16], resnet_fc_policy_layers=[16])


def _search_board_config(name):
    from netcases import NetCase, make_config
    h, w, a = SEARCH_BOARDS[name]
    return make_config(NetCase(name, "tictactoe", "small_search", dict(observation_shape=(3, h, w), action_space=list(range(a)),
                                                                       channels=16, blocks=1, **SEARCH_HEADS)))


def _small_search_plan(spec, n, S):
    import ctypes
    from muzero_general_b200 import _lib
    from netcases import small_search_inputs
    p = small_search_inputs(spec)
    out = (ctypes.c_int64 * 8)()
    if not _lib.load_library().mz_debug_small_search_plan(p["H"], p["W"], p["C"], p["A"], n, S, p["tower"], p["heads"],
                                                           p["scratch"], p["cap"], out):
        return None
    return tuple(out[:3])          # (P, CO, G)


@pytest.mark.parametrize("name,n,N", [("tictactoe", 1, 25), ("tictactoe", 700, 50), ("tictactoe", 3001, 12), ("tictactoe", 8192, 10),
                                      ("breakout", 5, 20), ("breakout", 300, 12),
                                      ("ss_3x3_a9", 7, 20), ("ss_3x3_a9", "co4", 8), ("ss_3x3_a4", "co4", 8),
                                      ("ss_6x6_a4", 5, 16), ("ss_6x6_a4", "co4", 8), ("ss_6x6_a16", "co4", 8)])
def test_fused_small_search_equals_stepwise_pipeline(name, n, N, game_configs, monkeypatch):
    """Small residual networks run ALL simulations of a search in one launch (csrc/small_search.cu): a CTA takes its
    games through dynamics tower -> reward head + rescale -> prediction tower -> value / policy heads -> tree step with the
    very device functions of the stand-alone kernels.  Visit counts, root values, value ranges, tree depths and the
    exported trees (hidden states included) equal the step-wise pipeline's (MZ_SMALL_SEARCH=0), bit for bit.  The
    ss_* cases reach all six instantiations (P, CO, G) of the kernel; each asserts the one the planner gives it."""
    import torch
    S = torch.cuda.get_device_properties(0).multi_processor_count
    cfg = _search_board_config(name) if name in SEARCH_BOARDS else game_configs[name]
    spec = netspec_from_config(cfg)
    A = spec.action_space
    co4 = n == "co4"
    if co4:
        n = next(m for m in range(1, 20000) if (_small_search_plan(spec, m, S) or (0, 0))[1] == 4) + 3
    inst = _small_search_plan(spec, n, S)
    print(f"[fused small search] {name} n={n}: (P, CO, G) = {inst} on {S} SMs")
    if name in SEARCH_BOARDS:
        G = 4 if A <= 4 else 16
        assert inst == ((spec.hidden_hw[1], 4, G) if co4 else (3, 1, G)), (name, n, inst)
    rs = numpy.random.RandomState(5)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    legal = (rs.uniform(size=(n, A)) < 0.7).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    results, trees = [], []
    for on in ("0", "1"):
        monkeypatch.setenv("MZ_SMALL_SEARCH", on)
        eng = _engine(cfg, n, N)
        eng.load_weights(weights_for(name, spec))
        launches0 = eng.launch_count
        runs = [eng.search(obs=obs, legal_mask=legal, add_exploration_noise=True, noise=noise, keep_tree=True) for _ in range(3)]
        per_search = (eng.launch_count - launches0) // 3
        for r in runs[1:]:
            assert numpy.array_equal(r.visit_counts, runs[0].visit_counts)
            assert numpy.array_equal(r.root_value, runs[0].root_value)
        results.append((runs[-1], per_search))
        trees.append([eng.export_tree(i, with_hidden=True) for i in (0, n // 2, n - 1)])
        eng.close()
    (a, la), (b, lb) = results
    assert la - lb == 5 * N - 1, (la, lb)          # ONE search launch instead of 5 launches per simulation
    assert numpy.array_equal(a.visit_counts, b.visit_counts)
    assert numpy.array_equal(a.root_value, b.root_value)
    assert numpy.array_equal(a.value_range, b.value_range)
    assert numpy.array_equal(a.max_tree_depth, b.max_tree_depth)
    assert numpy.array_equal(a.root_predicted_value, b.root_predicted_value)
    assert (b.visit_counts.sum(1) == N).all()
    for ta, tb in zip(*trees):
        for k in ta:
            assert numpy.array_equal(numpy.asarray(ta[k]), numpy.asarray(tb[k])), k


def test_graph_replay_does_not_depend_on_result_addresses(game_configs, monkeypatch):
    """Device-memory callers get freshly allocated result arrays from the engine on every call; the replayed graph is keyed
    by the INPUT addresses only (results go through the handle's arena and are copied behind the graph), so such a caller
    still replays - seen here as the partitioned graph (2 branches) being in use although every call had new result arrays."""
    import torch
    cfg = game_configs["connect4"]
    spec = netspec_from_config(cfg)
    monkeypatch.setenv("MZ_TC_MODE", "x3")
    monkeypatch.delenv("MZ_PARTS", raising=False)
    n, N = 160, 6
    rs = numpy.random.RandomState(2)
    obs_host = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    obs = torch.from_numpy(obs_host).cuda()
    eng = _engine(cfg, n, N)
    eng.load_weights(weights_for("connect4", spec))
    ref = eng.search(obs=obs_host, add_exploration_noise=False)
    keep = []
    for _ in range(5):
        out = eng.search(obs=obs, add_exploration_noise=False)
        keep.append(out)                                  # keeps the result tensors alive: the next call gets new addresses
        assert numpy.array_equal(out.visit_counts.cpu().numpy(), ref.visit_counts)
        assert numpy.array_equal(out.root_value.cpu().numpy(), ref.root_value)
    assert eng.graph_partitions == 2
    eng.close()
