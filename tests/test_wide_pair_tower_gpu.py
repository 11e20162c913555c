"""The 128-channel x3 tensor-core towers with each board split across a CTA pair (conv_tower_wide_pair_kernel behind
Runner::wide_tower, MZ_TC_WIDE=2) against an fp64 tower through mz_debug_wide_pair_tower, and Gomoku's 6 x 128 net on 15 x 15
and 16 x 16 boards on that route against the reference's fixtures (oracle/gen_golden_gomoku_pair.py).

The output and the pool's other slots start as NaN, so a board (or a half) the tower does not write, or one read from the
wrong slot, fails every comparison.  The exact and budget checks are test_wide_tower_gpu.py's (sparse integer towers EQUAL
fp64 with the range guard at zero; standard-normal operands at gains 1, 1e-4 and 300 inside the layer-by-layer budget).

Mutants of the pair kernel, each built and run against test_exact, test_budget and test_halo_reaches_the_other_half (47
tests) on an H100:
  - no halo store (the peer's halo row keeps the layer-0 input):
                                       30 fail - the 24 test_exact cases with a block, test_budget[prediction-1-(2, 16)]
                                       at every gain, every halo case
  - the halo written one board row off (into the peer's own boundary row):
                                       the same 30 fail
  - the action table indexed by the local row (y instead of y0 + y):
                                       14 fail - every test_exact case with a dynamics stem
  - the remote row stored with the local row's swizzle phase:
                                       14 fail - the cases on 12 x 12, 13 x 13, 2 x 16 and 3 x 5, where the split shifts
                                       the phase (h S not a multiple of 8); on 15 x 15, 16 x 16 and 16 x 12 it cannot show
The budget cases at 6 blocks do not catch a missing halo: the propagated budget grows with the absolute weights at every
layer, so the integer towers and the halo cases carry the exchange."""
import numpy
import pytest

from conftest import golden_npz, weights_for
from muzero_general_b200.netspec import netspec_from_config
from test_wide_tower_gpu import C, SITES, STEM, _parents, int_tower, normal_tower, sms, tower64

pytestmark = pytest.mark.gpu

BOARDS = ((12, 12), (13, 13), (15, 15), (16, 16), (16, 12), (2, 16))


def _depths(site):
    return range(0, 7) if STEM[site] else range(1, 7)


def run(site, x, ws, bs, act, A, seed=0, parts=1, stride=3, pair=True):
    from muzero_general_b200.engine import debug_wide_pair_tower, debug_wide_tower
    n, _, H, W = x.shape
    kw = {}
    if site == "dynamics_pool":
        kw = dict(parents=_parents(n, stride, numpy.random.RandomState(seed + 7)), pool_stride=stride, parts=parts)
    out, launches, sat, plan = (debug_wide_pair_tower if pair else debug_wide_tower)(x, ws, bs, site=site, actions=act, A=A, **kw)
    if pair:
        h = -(-H // 2)
        m_tiles = -(-h * (W + 1) // 64)
        assert plan["rows0"] == h and plan["m_tiles"] == m_tiles and plan["threads"] == 128 * m_tiles
        assert plan["layers"] == len(ws)
    ranges = -(-n // (((n + parts - 1) // parts + 7) & ~7)) if site == "dynamics_pool" else 1
    assert launches == ranges, (launches, ranges)
    return out, sat


def _cases():
    out = []
    for site in SITES:
        for i, blocks in enumerate(_depths(site)):
            out.append((site, blocks, BOARDS[(i + len(out)) % len(BOARDS)]))
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
@pytest.mark.parametrize("site,blocks,board", [("representation", 6, (16, 12)), ("dynamics", 6, (13, 13)),
                                               ("dynamics_pool", 6, (15, 15)), ("prediction", 6, (16, 16)),
                                               ("dynamics_pool", 2, (12, 12)), ("prediction", 1, (2, 16))])
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


@pytest.mark.parametrize("board", [(15, 15), (16, 16), (3, 5)])
def test_halo_reaches_the_other_half(board):
    """Zero input and biases but one position per board: on CTA 0's last row, one row above it (outside CTA 1's halo), on
    CTA 1's first row and one row below it.  The fp64 tower carries each point into the other half, where the pair gets it
    from the halo rows the epilogues exchange; every element stays inside the budget."""
    H, W = board
    h = -(-H // 2)
    x, ws, bs, act, A = normal_tower(4, H, W, 2, 0, 1.0, seed=3)
    bs = [numpy.zeros_like(b) for b in bs]
    x[:] = 0
    for g, y in enumerate((h - 1, h - 2, h, h + 1)):
        x[g, :, min(max(y, 0), H - 1), W // 2] = numpy.random.RandomState(g).standard_normal(C)
    ref, _, budget = tower64(x, ws, bs, 0, act, A, gain=1.0)
    for g, y in enumerate((h - 1, h - 2, h, h + 1)):
        other = ref[g, :, h:] if y < h else ref[g, :, :h]
        assert numpy.abs(other).max() > 1e-2, (g, y)            # the point reaches the other half
    got, sat = run("prediction", x, ws, bs, act, A)
    assert sat == 0
    assert (numpy.abs(got - ref) <= budget).all(), numpy.abs(got - ref).max()


@pytest.mark.parametrize("board", [(5, 5), (8, 11), (11, 1), (11, 11)])
@pytest.mark.parametrize("site", ["dynamics_pool", "prediction"])
def test_pair_equals_one_cta(site, board):
    """Each output element sees the same operands in the same K order and the same epilogue on both kernels."""
    H, W = board
    stem = STEM[site]
    x, ws, bs, act, A = normal_tower(3, H, W, 3, stem, 1.0, seed=H + W)
    one, _ = run(site, x, ws, bs, act, A, pair=False)
    two, _ = run(site, x, ws, bs, act, A)
    diff = numpy.argwhere(one != two)
    assert len(diff) == 0, f"first differing element {tuple(diff[0])}: one CTA {one[tuple(diff[0])]!r}, pair {two[tuple(diff[0])]!r}"


def test_batches_at_the_wave_edges():
    """One CTA pair per board: 1, one wave - 1, one wave + 1 and several waves, each board inside the budget (checked on
    the boards at the edges) and independent of the batch around it (bit for bit)."""
    from muzero_general_b200.engine import debug_wide_pair_tower_plan
    plan, why = debug_wide_pair_tower_plan(1, C, 15, 15, 1, True, sms())
    wave = plan["wave"]
    x, ws, bs, act, A = normal_tower(3 * wave + 5, 15, 15, 1, 1, 1.0, seed=5)
    full, _ = run("dynamics_pool", x, ws, bs, act, A, seed=1, stride=1)
    rows = [0, wave - 2, wave - 1, wave, 3 * wave + 4]
    ref, _, budget = tower64(x, ws, bs, 1, act, A, gain=1.0, rows=rows)
    assert (numpy.abs(full[rows] - ref) <= budget).all()
    for n in (1, wave - 1, wave + 1):
        got, _ = run("dynamics_pool", x[:n], ws, bs, act[:n], A, seed=1, stride=1)
        assert numpy.array_equal(got, full[:n]), n


@pytest.mark.parametrize("parts", [2, 3, 4])
def test_partitions_equal_one_range(parts):
    n = sms() + 21
    x, ws, bs, act, A = normal_tower(n, 16, 16, 2, 1, 1.0, seed=9)
    one, _ = run("dynamics_pool", x, ws, bs, act, A, seed=2, parts=1)
    got, _ = run("dynamics_pool", x, ws, bs, act, A, seed=2, parts=parts)
    assert numpy.array_equal(got, one)


@pytest.mark.parametrize("half", [None, 0, 1])
def test_range_guard_in_either_half(half):
    """An input activation beyond the fp16 range on a row only CTA `half` reads (its outer board edge) bumps the guard;
    without it the guard stays at zero."""
    x, ws, bs, act, A = normal_tower(2, 15, 15, 1, 0, 1.0, seed=4)
    if half is not None:
        x[1, 5, 0 if half == 0 else 14, 7] = 1e5
    _, peak, _ = tower64(x, ws, bs, 0, act, A)
    assert (peak > 65504) == (half is not None)
    _, sat = run("prediction", x, ws, bs, act, A)
    assert (sat > 0) == (half is not None)


# ---------------------------------------------------------------------------------------------- whole nets
def _gomoku(side):
    from muzero_general_b200.games import load_game_module
    cfg = load_game_module("gomoku").MuZeroConfig(board_size=side)
    assert (cfg.blocks, cfg.channels) == (6, 128)
    return cfg


def _engine(cfg, n, N, **kw):
    from muzero_general_b200.engine import SearchEngine
    return SearchEngine(cfg, max_games=n, num_simulations=N, **kw)


PAIR_ROUTE = "128-channel towers on the tensor cores, boards split across CTA pairs"


@pytest.fixture
def pair(monkeypatch):
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    monkeypatch.setenv("MZ_TC_WIDE", "2")


def _check_net(eng, g, n):
    tol = dict(rtol=2e-4, atol=2e-5)
    r0 = eng.initial_inference(g["obs"])
    numpy.testing.assert_allclose(r0["hidden"], g["init_hidden"].reshape(n, -1), rtol=2e-4, atol=5e-5)
    numpy.testing.assert_allclose(r0["value_logits"], g["init_value"], **tol)
    numpy.testing.assert_allclose(r0["policy_logits"], g["init_policy"], **tol)
    numpy.testing.assert_allclose(r0["value"], g["init_value_scalar"], rtol=2e-4, atol=5e-4)
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(n, -1), g["action"])
    # the dynamics tower's 13 convs, then the min-max rescale: on 16 x 16 one of 98,304 elements of the tensor-core
    # route lands 1.97e-4 from the reference (the fp64 tower checks above are the kernel's contract)
    numpy.testing.assert_allclose(r1["hidden"], g["rec_hidden"].reshape(n, -1), rtol=2e-4, atol=2.5e-4)
    for k, ref in (("value_logits", "rec_value"), ("reward_logits", "rec_reward"), ("policy_logits", "rec_policy")):
        numpy.testing.assert_allclose(r1[k], g[ref], **tol)
    numpy.testing.assert_allclose(r1["value"], g["rec_value_scalar"], rtol=2e-4, atol=5e-4)
    numpy.testing.assert_allclose(r1["reward"], g["rec_reward_scalar"], rtol=2e-4, atol=5e-4)


@pytest.mark.parametrize("route", ["pair", "cuda_cores"])
@pytest.mark.parametrize("side", [15, 16])
def test_gomoku_net_matches_reference(side, route, monkeypatch):
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    if route == "pair":
        monkeypatch.setenv("MZ_TC_WIDE", "2")
    else:
        monkeypatch.delenv("MZ_TC_WIDE", raising=False)
    cfg = _gomoku(side)
    spec = netspec_from_config(cfg)
    g = golden_npz(f"net_gomoku{side}.npz")
    n = len(g["obs"])
    eng = _engine(cfg, n, 4)
    eng.load_weights(weights_for("gomoku", spec))
    assert (PAIR_ROUTE in eng.numerics) == (route == "pair"), eng.numerics
    _check_net(eng, g, n)
    assert (PAIR_ROUTE in eng.numerics) == (route == "pair")             # the guard did not trip
    eng.close()


def test_gomoku15_closed_loop_matches_reference_counts(pair):
    from test_wide_pair_plan_cpu import c128_search_cases
    cfg = _gomoku(15)
    spec = netspec_from_config(cfg)
    A = spec.action_space
    for c in c128_search_cases():
        eng = _engine(cfg, 1, c["num_simulations"])
        eng.load_weights(weights_for("gomoku", spec))
        assert PAIR_ROUTE in eng.numerics
        obs = numpy.array(c["obs"], numpy.float32).reshape(1, *c["obs_shape"])
        legal = numpy.zeros((1, A), numpy.uint8); legal[0, c["legal"]] = 1
        noise = numpy.zeros((1, A)); noise[0, c["legal"]] = c["noise"]
        out = eng.search(obs=obs, legal_mask=legal, to_play=numpy.array([c["to_play"]], numpy.int32),
                         add_exploration_noise=True, noise=noise, first_index=numpy.array([c["first_index"]], numpy.int32))
        assert [int(out.visit_counts[0, a]) for a in c["root_actions"]] == c["root_visits"]
        assert abs(int(out.max_tree_depth[0]) - c["max_tree_depth"]) <= 4
        assert PAIR_ROUTE in eng.numerics
        eng.close()


@pytest.mark.parametrize("side", [15, 16])
def test_gomoku_student_forced(pair, side):
    from helpers import oracle_replay, paths_from_trace
    from oracle import mcts as om
    cfg = _gomoku(side)
    spec = netspec_from_config(cfg)
    n, N, A, P = 4, 20, spec.action_space, len(cfg.players)
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
    assert PAIR_ROUTE in eng.numerics
    eng.close()


def test_graph_replay_equals_eager(pair, monkeypatch):
    cfg = _gomoku(15)
    spec = netspec_from_config(cfg)
    n, N = 8, 12
    obs = numpy.random.RandomState(3).randint(0, 2, size=(n, spec.obs_elems)).astype(numpy.float32)
    results = []
    for no_graph in ("1", "0"):
        monkeypatch.setenv("MZ_NO_GRAPH", no_graph)
        eng = _engine(cfg, n, N)
        eng.load_weights(weights_for("gomoku", spec))
        assert PAIR_ROUTE in eng.numerics
        runs = [eng.search(obs=obs, add_exploration_noise=False) for _ in range(3)]
        for r in runs[1:]:
            assert numpy.array_equal(r.visit_counts, runs[0].visit_counts)
            assert numpy.array_equal(r.root_value, runs[0].root_value)
        results.append(runs[0])
        eng.close()
    assert numpy.array_equal(results[0].visit_counts, results[1].visit_counts)
    assert numpy.array_equal(results[0].root_value, results[1].root_value)


def test_stress_weights_fall_back_and_match(pair, monkeypatch):
    """Weights whose towers exceed the fp16 range: the guard trips, the handle leaves the pair towers for good (graphs
    captured before are dropped) and the redone calls equal the CUDA-core route bit for bit."""
    from muzero_general_b200.netspec import stress_weights
    cfg = _gomoku(15)
    spec = netspec_from_config(cfg)
    w = stress_weights(spec, 0, "overflow")
    n, N = 4, 6
    obs = numpy.random.RandomState(1).randint(0, 2, size=(n, spec.obs_elems)).astype(numpy.float32)
    eng = _engine(cfg, n, N)
    eng.load_weights(w)
    assert PAIR_ROUTE in eng.numerics
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


@pytest.mark.parametrize("side", [15, 16])
def test_device_loop_drains_well_formed_games(pair, side):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, parse_staged_games
    from muzero_general_b200.games import load_game_module
    mod = load_game_module("gomoku")
    cfg = _gomoku(side)
    cfg.max_moves = 6
    spec = netspec_from_config(cfg)
    eng = _engine(cfg, 8, 6, seed=0)
    eng.load_weights(weights_for("gomoku", spec))
    assert PAIR_ROUTE in eng.numerics
    loop = DeviceSelfPlayLoop(eng, "gomoku", cfg.max_moves, temperature_threshold=cfg.temperature_threshold,
                              reward_scale=mod.Game.VECTOR.REWARD_SCALE)
    for _ in range(cfg.max_moves + 1):
        loop.moves(1, 1.0)
    games = parse_staged_games(*loop.drain())            # (the parser checks that the staged blocks add up)
    assert len(games) >= 8
    assert all(1 <= gm["length"] <= cfg.max_moves for gm in games)
    assert PAIR_ROUTE in eng.numerics
    eng.close()


def test_routes_by_switch(monkeypatch, game_configs):
    """MZ_TC_WIDE=2 keeps 11 x 11 on the one-CTA kernel and puts 15 x 15 on pairs; with MZ_TC_WIDE=1 15 x 15 stays on the
    CUDA cores and names the one-CTA reason; a board neither takes names both."""
    from muzero_general_b200.netspec import synthetic_weights
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    for switch, side, want in (("2", 11, "128-channel towers on the tensor cores, split"), ("2", 15, PAIR_ROUTE),
                               ("1", 15, "128-channel towers stay on the CUDA cores: board too large")):
        monkeypatch.setenv("MZ_TC_WIDE", switch)
        cfg = game_configs["gomoku"] if side == 11 else _gomoku(side)
        spec = netspec_from_config(cfg)
        eng = _engine(cfg, 2, 2)
        eng.load_weights(synthetic_weights(spec, 0))
        assert want in eng.numerics and (PAIR_ROUTE in eng.numerics) == (want == PAIR_ROUTE), eng.numerics
        eng.close()
    monkeypatch.setenv("MZ_TC_WIDE", "2")
    cfg = _gomoku(15)
    cfg.observation_shape = (3, 16, 24)                # 8 rows x 25 per CTA: four M-tiles
    spec = netspec_from_config(cfg)
    eng = _engine(cfg, 2, 2)
    eng.load_weights(synthetic_weights(spec, 0))
    assert "one CTA: board too large" in eng.numerics and "CTA pairs: board too large" in eng.numerics, eng.numerics
    eng.close()
