"""The 128-channel x3 tensor-core towers (csrc/conv_wide.cu behind Runner::wide_tower, MZ_TC_WIDE=1) against an fp64 tower
through mz_debug_wide_tower, and whole Gomoku-shaped nets on that route against the reference's fixtures.

The output and the pool's other slots start as NaN, so a board the tower does not write, or one read from the wrong slot,
fails every comparison.

  exact     sparse small-integer weights, integer biases and inputs, A a power of two with action-plane weights in
            multiples of A: every product and partial sum is exact in fp32 and every activation stays below 65504 (the
            fixtures assert it on the fp64 tower; inputs reach the thousands, so the x_l halves take part), so the device
            tower must EQUAL the fp64 one, and the range guard stays at zero.
  budget    standard-normal operands at gains 1, 1e-4 and 300 against the fp64 tower, inside the error budget of
            test_conv_tower_gpu.py propagated layer by layer at C = 128:
                delta_out = |W| * delta_in + c1 (|W| * |x|) + c2 |y| + delta_res + floor,   c1 = 4e-6, c2 = 2e-6, floor 1e-6 gain
  launches  one launch per tower call (one CTA per board), the plan of mz_debug_wide_tower_plan.

Mutants of csrc/conv_wide.cu, each built and run against test_exact and test_budget (51 tests) on an H100:
  - dropping x_l w_h:                  33 fail - all 30 test_exact cases, test_budget[dynamics-0-(1, 11)] at every gain
  - a dx tap wrapping across the zero column (row stride S = W instead of W + 1):
                                       36 fail - all 30 test_exact cases, test_budget[prediction-1-(5, 5)] and
                                       test_budget[dynamics-0-(1, 11)] at every gain
  - a missing block residual:          31 fail - the 28 test_exact cases with a block, test_budget[prediction-1-(5, 5)]
                                       at every gain
  - the epilogue storing before the neighbouring M-tile's MMAs finished (no CTA barrier after a layer's MMAs):
                                       none fail.  The two-stage weight ring keeps the warpgroups of a CTA within one
                                       stage of each other, and no run overwrote a row another warpgroup still read;
                                       the barrier is kept because the ordering requires it, not because a test shows it."""
import numpy
import pytest
import torch

from conftest import golden_json, golden_npz, weights_for
from muzero_general_b200.netspec import netspec_from_config

pytestmark = pytest.mark.gpu

C = 128
BOARDS = ((1, 1), (1, 11), (11, 1), (5, 5), (8, 11), (11, 11))
SITES = ("representation", "dynamics", "dynamics_pool", "prediction")
STEM = {"representation": 0, "dynamics": 1, "dynamics_pool": 1, "prediction": 0}
C1, C2, FLOOR = 4e-6, 2e-6, 1e-6


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _depths(site):
    return range(0, 7) if STEM[site] else range(1, 7)


def _actions(n, A, rs):
    a = rs.randint(0, A, n)
    a[0], a[-1] = 0, A - 1
    return a.astype(numpy.int32)


def _parents(n, stride, rs):
    p = rs.randint(0, stride, n)
    p[0], p[-1] = 0, stride - 1
    return p.astype(numpy.int32)


def _sparse_int_conv(rs, cin, vmax, two):
    w = numpy.zeros((C, cin, 3, 3), numpy.float32)
    for co in range(C):
        for _ in range(2 if rs.random_sample() < two else 1):
            w[co, rs.randint(cin), rs.randint(3), rs.randint(3)] = rs.choice([-1, 1]) * rs.randint(1, vmax + 1)
    return w


def int_tower(n, H, W, blocks, stem, seed, A=4):
    rs = numpy.random.RandomState(seed)
    ws, bs = [], []
    if stem:
        w = numpy.zeros((C, C + 1, 3, 3), numpy.float32)
        w[:, :C] = _sparse_int_conv(rs, C, 2, 0.3)
        for co in rs.choice(C, 48, replace=False):
            w[co, C, rs.randint(3), rs.randint(3)] = A * rs.choice([-1, 1]) * rs.randint(1, 3)
        ws.append(w)
        bs.append(rs.randint(-3, 4, C).astype(numpy.float32))
    for _ in range(blocks):
        ws.append(_sparse_int_conv(rs, C, 3, 0.3))
        bs.append(rs.randint(-3, 4, C).astype(numpy.float32))
        ws.append(_sparse_int_conv(rs, C, 1, 0.2))
        bs.append(rs.randint(-4, 2, C).astype(numpy.float32))
    act = _actions(n, A, rs) if stem else None
    hi = 16000
    while True:
        x = numpy.random.RandomState(seed + 1).randint(-hi, hi + 1, size=(n, C, H, W)).astype(numpy.float32)
        ref, peak, _ = tower64(x, ws, bs, stem, act, A)
        if peak < 65504 or hi == 1:
            return x, ws, bs, act, A, ref, peak
        hi //= 2


def normal_tower(n, H, W, blocks, stem, gain, seed):
    rs = numpy.random.RandomState(seed)
    A = (7, 128, 1)[seed % 3]
    x = (gain * rs.standard_normal((n, C, H, W))).astype(numpy.float32)
    ws, bs = [], []
    for i in range(stem + 2 * blocks):
        cin = C + 1 if stem and i == 0 else C
        w = rs.standard_normal((C, cin, 3, 3)) / numpy.sqrt(9 * C)
        if cin == C + 1:
            w[:, C] *= gain
        ws.append(w.astype(numpy.float32))
        bs.append((0.1 * gain * rs.standard_normal(C)).astype(numpy.float32))
    return x, ws, bs, (_actions(n, A, rs) if stem else None), A


def _conv(x, w, b=None):
    return torch.nn.functional.conv2d(x, torch.from_numpy(numpy.asarray(w, numpy.float64)),
                                      None if b is None else torch.from_numpy(numpy.asarray(b, numpy.float64)), 1, 1)


def tower64(x, ws, bs, stem, act, A, gain=None, rows=None):
    """The tower in fp64 on the boards `rows` (all by default): (output, largest |activation|, and with `gain` the
    propagated error budget of the output)."""
    idx = numpy.arange(len(x)) if rows is None else numpy.asarray(rows)
    h = torch.from_numpy(x[idx]).double()
    n, _, H, W = h.shape
    peak = float(h.abs().max())
    floor = FLOOR * (gain or 0.0)
    delta = h.abs() * 2.0 ** -22 + floor if gain else None

    def layer(inp, d_in, w, b, res=None, d_res=None):
        y = _conv(inp, w, b)
        if res is not None:
            y = y + res
        d = None
        if gain:
            aw = numpy.abs(w)
            d = _conv(d_in, aw) + C1 * _conv(inp.abs(), aw) + C2 * y.abs() + floor
            if d_res is not None:
                d = d + d_res
        return torch.relu(y), d

    k = 0
    if stem:
        plane = torch.from_numpy(act[idx].astype(numpy.float64) / A)[:, None, None, None].expand(n, 1, H, W)
        d_in = torch.cat([delta, torch.zeros(n, 1, H, W, dtype=torch.float64)], 1) if gain else None
        h, delta = layer(torch.cat([h, plane], 1), d_in, ws[0], bs[0])
        peak = max(peak, float(h.abs().max()))
        k = 1
    while k < len(ws):
        t, dt = layer(h, delta, ws[k], bs[k])
        peak = max(peak, float(t.abs().max()))
        h, delta = layer(t, dt, ws[k + 1], bs[k + 1], h, delta)
        peak = max(peak, float(h.abs().max()))
        k += 2
    return h.numpy(), peak, None if delta is None else delta.numpy()


def run(site, x, ws, bs, act, A, seed=0, parts=1, stride=3):
    from muzero_general_b200.engine import debug_wide_tower
    n, _, H, W = x.shape
    kw = {}
    if site == "dynamics_pool":
        kw = dict(parents=_parents(n, stride, numpy.random.RandomState(seed + 7)), pool_stride=stride, parts=parts)
    out, launches, sat, plan = debug_wide_tower(x, ws, bs, site=site, actions=act, A=A, **kw)
    m_tiles = -(-H * (W + 1) // 64)
    assert plan["m_tiles"] == m_tiles and plan["threads"] == 128 * m_tiles and plan["layers"] == len(ws)
    ranges = -(-n // (((n + parts - 1) // parts + 7) & ~7)) if site == "dynamics_pool" else 1
    assert launches == ranges, (launches, ranges)
    return out, sat


def _cases():
    out = []
    for site in SITES:
        for i, blocks in enumerate(_depths(site)):
            out.append((site, blocks, BOARDS[(i + len(out)) % len(BOARDS)]))
        out.append((site, 6, (11, 11)))
    return out


@pytest.mark.parametrize("site,blocks,board", _cases())
def test_exact(site, blocks, board):
    H, W = board
    stem = STEM[site]
    x, ws, bs, act, A, ref, peak = int_tower(3, H, W, blocks, stem, seed=blocks * 11 + H)
    assert peak < 65504
    got, sat = run(site, x, ws, bs, act, A, seed=blocks)
    assert sat == 0
    assert numpy.array_equal(got, ref.astype(numpy.float32)), numpy.abs(got - ref).max()


@pytest.mark.parametrize("gain", [1.0, 1e-4, 300.0])
@pytest.mark.parametrize("site,blocks,board", [("representation", 6, (11, 11)), ("dynamics", 6, (11, 11)),
                                               ("dynamics_pool", 6, (11, 11)), ("prediction", 6, (11, 11)),
                                               ("dynamics_pool", 2, (8, 11)), ("prediction", 1, (5, 5)),
                                               ("dynamics", 0, (1, 11))])
def test_budget(site, blocks, board, gain):
    H, W = board
    stem = STEM[site]
    x, ws, bs, act, A = normal_tower(2, H, W, blocks, stem, gain, seed=blocks + H)
    ref, _, budget = tower64(x, ws, bs, stem, act, A, gain=gain)
    got, sat = run(site, x, ws, bs, act, A)
    assert sat == 0
    ratio = numpy.abs(got - ref) / budget
    print(f"{site} {blocks} {board} gain {gain}: worst error / budget {ratio.max():.3f}")
    assert ratio.max() <= 1.0


def test_batches_at_the_wave_edges():
    """One board per CTA: 1, one wave - 1, one wave + 1 and several waves, each board inside the budget (checked on the
    boards at the edges) and independent of the batch around it (bit for bit)."""
    from muzero_general_b200.engine import debug_wide_tower_plan
    plan, why = debug_wide_tower_plan(1, C, 11, 11, 1, True, sms())
    wave = plan["wave"]
    x, ws, bs, act, A = normal_tower(3 * wave + 5, 11, 11, 1, 1, 1.0, seed=5)
    full, _ = run("dynamics_pool", x, ws, bs, act, A, seed=1, stride=1)
    rows = [0, wave - 2, wave - 1, wave, 3 * wave + 4]
    ref, _, budget = tower64(x, ws, bs, 1, act, A, gain=1.0, rows=rows)
    assert (numpy.abs(full[rows] - ref) <= budget).all()
    for n in (1, wave - 1, wave + 1):
        got, _ = run("dynamics_pool", x[:n], ws, bs, act[:n], A, seed=1, stride=1)
        assert numpy.array_equal(got, full[:n]), n


@pytest.mark.parametrize("parts", [2, 3, 4])
def test_partitions_equal_one_range(parts):
    n = 2 * sms() + 21
    x, ws, bs, act, A = normal_tower(n, 11, 11, 2, 1, 1.0, seed=9)
    one, _ = run("dynamics_pool", x, ws, bs, act, A, seed=2, parts=1)
    got, _ = run("dynamics_pool", x, ws, bs, act, A, seed=2, parts=parts)
    assert numpy.array_equal(got, one)


@pytest.mark.parametrize("late", [False, True])
def test_range_guard(late):
    """An activation beyond the fp16 range in the last layer bumps the guard; the same tower without it does not."""
    x, ws, bs, act, A = normal_tower(2, 11, 11, 3, 0, 1.0, seed=4)
    if late:
        ws[-1] = ws[-1] * 3e5
    ref, peak, _ = tower64(x, ws, bs, 0, act, A)
    assert (peak > 65504) == late
    _, sat = run("prediction", x, ws, bs, act, A)
    assert (sat > 0) == late


# ---------------------------------------------------------------------------------------------- whole nets
def _engine(cfg, n, N):
    from muzero_general_b200.engine import SearchEngine
    return SearchEngine(cfg, max_games=n, num_simulations=N)


@pytest.fixture
def wide(monkeypatch):
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    monkeypatch.setenv("MZ_TC_WIDE", "1")


def test_gomoku_net_matches_reference(wide, game_configs):
    cfg = game_configs["gomoku"]
    spec = netspec_from_config(cfg)
    g = golden_npz("net_gomoku.npz")
    n = len(g["obs"])
    eng = _engine(cfg, n, 4)
    eng.load_weights(weights_for("gomoku", spec))
    assert "128-channel towers on the tensor cores" in eng.numerics
    tol = dict(rtol=2e-4, atol=2e-5)
    r0 = eng.initial_inference(g["obs"])
    numpy.testing.assert_allclose(r0["hidden"], g["init_hidden"].reshape(n, -1), rtol=2e-4, atol=5e-5)
    numpy.testing.assert_allclose(r0["value_logits"], g["init_value"], **tol)
    numpy.testing.assert_allclose(r0["policy_logits"], g["init_policy"], **tol)
    numpy.testing.assert_allclose(r0["value"], g["init_value_scalar"], rtol=2e-4, atol=5e-4)
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(n, -1), g["action"])
    numpy.testing.assert_allclose(r1["hidden"], g["rec_hidden"].reshape(n, -1), rtol=2e-4, atol=5e-5)
    for k, ref in (("value_logits", "rec_value"), ("reward_logits", "rec_reward"), ("policy_logits", "rec_policy")):
        numpy.testing.assert_allclose(r1[k], g[ref], **tol)
    numpy.testing.assert_allclose(r1["value"], g["rec_value_scalar"], rtol=2e-4, atol=5e-4)
    numpy.testing.assert_allclose(r1["reward"], g["rec_reward_scalar"], rtol=2e-4, atol=5e-4)
    assert "128-channel towers on the tensor cores" in eng.numerics         # the guard did not trip
    eng.close()


def test_gomoku_student_forced(wide, game_configs):
    from helpers import oracle_replay, paths_from_trace
    from oracle import mcts as om
    cfg = game_configs["gomoku"]
    spec = netspec_from_config(cfg)
    n, N, A, P = 6, 30, spec.action_space, len(cfg.players)
    rs = numpy.random.RandomState(11)
    obs = rs.randint(0, 2, size=(n, spec.in_channels) + spec.obs_shape[1:]).astype(numpy.float32)
    legal = (rs.uniform(size=(n, A)) < 0.8).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    first = numpy.array([rs.randint(0, int(l.sum())) for l in legal], numpy.int32)
    eng = _engine(cfg, n, N)
    eng.load_weights(weights_for("gomoku", spec))
    out = eng.search(obs=obs, legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise,
                     first_index=first, trace=True)
    params = om.SearchParams.from_config(cfg, N)
    tr = out.trace
    for i in range(n):
        acts = [a for a in range(A) if legal[i, a]]
        res, _ = oracle_replay(params, acts, int(to_play[i]),
                               (out.root_predicted_value[i], tr["root_reward"][i], [tr["root_priors_raw"][i, a] for a in acts]),
                               [(tr["value"][i, s], tr["reward"][i, s], tr["priors"][i, s]) for s in range(N)],
                               [noise[i, a] for a in acts], int(first[i]), seed=cfg.seed, game=i)
        assert [int(out.visit_counts[i, a]) for a in acts] == res.root_visits
        assert out.root_value[i] == res.root_value
        assert paths_from_trace(tr, i, N) == [s.path_actions for s in res.sims]
    assert "128-channel towers on the tensor cores" in eng.numerics
    eng.close()


def _closed_loop(name, cfg, spec):
    A = spec.action_space
    outs = []
    for c in golden_json(f"mcts_{name}.json"):
        eng = _engine(cfg, 1, c["num_simulations"])
        eng.load_weights(weights_for(name, spec))
        obs = numpy.array(c["obs"], numpy.float32).reshape(1, *c["obs_shape"])
        legal = numpy.zeros((1, A), numpy.uint8); legal[0, c["legal"]] = 1
        noise = numpy.zeros((1, A)); noise[0, c["legal"]] = c["noise"]
        out = eng.search(obs=obs, legal_mask=legal, to_play=numpy.array([c["to_play"]], numpy.int32),
                         add_exploration_noise=True, noise=noise, first_index=numpy.array([c["first_index"]], numpy.int32))
        outs.append((c, out, eng.numerics))
        eng.close()
    return outs


def test_gomoku_closed_loop_matches_reference_counts(wide, game_configs):
    cfg = game_configs["gomoku"]
    spec = netspec_from_config(cfg)
    for c, out, numerics in _closed_loop("gomoku", cfg, spec):
        assert "128-channel towers on the tensor cores" in numerics
        assert [int(out.visit_counts[0, a]) for a in c["root_actions"]] == c["root_visits"]
        assert abs(int(out.max_tree_depth[0]) - c["max_tree_depth"]) <= 4


def test_gomoku15_stays_on_the_cuda_cores(wide):
    """The 6 x 128 net on a 15 x 15 board exceeds the wide towers' shared-memory budget: mcts_gomoku15.json's positions
    run on the CUDA-core towers, and numerics says so."""
    from test_wide_actions_cpu import wide_search_cases
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import synthetic_weights
    cfg = load_game_module("gomoku").MuZeroConfig(board_size=15)
    assert (cfg.blocks, cfg.channels) == (6, 128)
    spec = netspec_from_config(cfg)
    cases = wide_search_cases()
    n, N, A = len(cases), cases[0]["num_simulations"], spec.action_space
    obs = numpy.array([c["obs"] for c in cases], numpy.float32).reshape(n, 3, 15, 15)
    legal = numpy.zeros((n, A), numpy.uint8)
    for i, c in enumerate(cases):
        legal[i, c["legal"]] = 1
    eng = _engine(cfg, n, N)
    eng.load_weights(synthetic_weights(spec, 0))
    assert "128-channel towers stay on the CUDA cores: board too large" in eng.numerics, eng.numerics
    out = eng.search(obs=obs, legal_mask=legal, add_exploration_noise=False)
    assert (out.visit_counts.sum(1) == N).all() and (out.visit_counts[legal == 0] == 0).all()
    eng.close()


def test_graph_replay_equals_eager(wide, game_configs, monkeypatch):
    cfg = game_configs["gomoku"]
    spec = netspec_from_config(cfg)
    n, N = 8, 12
    obs = numpy.random.RandomState(3).randint(0, 2, size=(n, spec.obs_elems)).astype(numpy.float32)
    results = []
    for no_graph in ("1", "0"):
        monkeypatch.setenv("MZ_NO_GRAPH", no_graph)
        eng = _engine(cfg, n, N)
        eng.load_weights(weights_for("gomoku", spec))
        runs = [eng.search(obs=obs, add_exploration_noise=False) for _ in range(3)]
        for r in runs[1:]:
            assert numpy.array_equal(r.visit_counts, runs[0].visit_counts)
            assert numpy.array_equal(r.root_value, runs[0].root_value)
        results.append(runs[0])
        eng.close()
    assert numpy.array_equal(results[0].visit_counts, results[1].visit_counts)
    assert numpy.array_equal(results[0].root_value, results[1].root_value)


def test_stress_weights_fall_back_and_match(wide, game_configs, monkeypatch):
    """Weights whose towers exceed the fp16 range: the guard trips, the handle leaves the wide towers for good (graphs
    captured before are dropped) and the redone calls equal the CUDA-core route bit for bit."""
    from muzero_general_b200.netspec import stress_weights
    cfg = game_configs["gomoku"]
    spec = netspec_from_config(cfg)
    w = stress_weights(spec, 0, "overflow")
    n, N = 4, 6
    obs = numpy.random.RandomState(1).randint(0, 2, size=(n, spec.obs_elems)).astype(numpy.float32)
    eng = _engine(cfg, n, N)
    eng.load_weights(w)
    assert "128-channel towers on the tensor cores" in eng.numerics
    got = [eng.search(obs=obs, add_exploration_noise=False) for _ in range(3)]
    assert "128-channel tensor-core towers left" in eng.numerics
    r_got = eng.initial_inference(obs)
    eng.close()
    monkeypatch.delenv("MZ_TC_WIDE")
    ref_eng = _engine(cfg, n, N)
    ref_eng.load_weights(w)
    ref = ref_eng.search(obs=obs, add_exploration_noise=False)
    r_ref = ref_eng.initial_inference(obs)
    ref_eng.close()
    for g in got:
        assert numpy.array_equal(g.visit_counts, ref.visit_counts) and numpy.array_equal(g.root_value, ref.root_value)
    for k in ("hidden", "value_logits", "policy_logits"):
        assert numpy.array_equal(r_got[k], r_ref[k]), k


def test_device_loop_drains_well_formed_games(wide):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, parse_staged_games
    from muzero_general_b200.games import load_game_module
    mod = load_game_module("gomoku")
    cfg = mod.MuZeroConfig()
    cfg.max_moves = 6
    spec = netspec_from_config(cfg)
    from muzero_general_b200.engine import SearchEngine
    eng = SearchEngine(cfg, max_games=8, num_simulations=6, seed=0)
    eng.load_weights(weights_for("gomoku", spec))
    assert "128-channel towers on the tensor cores" in eng.numerics
    loop = DeviceSelfPlayLoop(eng, "gomoku", cfg.max_moves, temperature_threshold=cfg.temperature_threshold,
                              reward_scale=mod.Game.VECTOR.REWARD_SCALE)
    for _ in range(cfg.max_moves + 1):
        loop.moves(1, 1.0)
    games = parse_staged_games(*loop.drain())            # (the parser checks that the staged blocks add up)
    assert len(games) >= 8
    assert all(1 <= gm["length"] <= cfg.max_moves for gm in games)
    assert "128-channel towers on the tensor cores" in eng.numerics
    eng.close()


def test_unset_keeps_the_cuda_core_route(game_configs, monkeypatch):
    monkeypatch.delenv("MZ_TC_WIDE", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    cfg = game_configs["gomoku"]
    spec = netspec_from_config(cfg)
    eng = _engine(cfg, 4, 4)
    eng.load_weights(weights_for("gomoku", spec))
    assert eng.numerics == "f32 nets + f64 tree statistics"
    eng.kernel_timing(True)                              # process-wide: switched off again before any assert
    eng.search(obs=numpy.zeros((4, spec.obs_elems), numpy.float32), add_exploration_noise=False)
    t = eng.kernel_times()
    eng.kernel_timing(False)
    assert t["conv3x3_kernel"][1] > 0 and t["conv_tower_tc_kernel"][1] == 0
    eng.close()
