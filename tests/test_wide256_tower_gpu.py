"""The 256-channel x3 tensor-core towers (conv_tower_wide256_kernel behind Runner::wide_tower, MZ_TC_WIDE=3: output
channels split across a CTA pair, boards stacked in M) against an fp64 tower through mz_debug_wide256_tower, and
games/atari.py's 16 x 256 net on that route against the reference's fixtures and the CUDA-core route.

The output and the pool's other slots start as NaN, so a board (or a channel half) the tower does not write, or one read
from the wrong slot, fails every comparison.  The checks are test_wide_tower_gpu.py's at C = 256:

  exact     sparse small-integer weights, integer biases and inputs, A a power of two: every product and partial sum is
            exact in fp32 and every activation stays below 65504, so the device tower must EQUAL the fp64 one with the
            range guard at zero.  Batches of 3 leave the last CTA pair with one real board and one empty slot.
  budget    standard-normal operands at gains 1, 1e-4 and 300 against the fp64 tower, inside the error budget of
            test_conv_tower_gpu.py propagated layer by layer at C = 256:
                delta_out = |W| * delta_in + c1 (|W| * |x|) + c2 |y| + delta_res + floor,   c1 = 4e-6, c2 = 2e-6, floor 1e-6 gain
  packing   1 board per CTA pair equals the planned 2 (and 8 on 1 x 1 boards) bit for bit: an output element sees the
            same operands in the same K order whatever the rows around it hold.

Mutants of csrc/conv_wide256.cu, each built and run against test_exact and test_budget (37 tests) on an H100:
  - no DSMEM store of the peer half (each CTA's planes keep the other half's layer-0 input):
                                       26 fail - the 20 test_exact cases with a block, test_budget[representation-2-(9, 9)]
                                       and test_budget[prediction-1-(3, 5)] at every gain
  - separator rows not zeroed (the row y = H between two stacked boards stored as computed):
                                       25 fail - the 19 test_exact cases that stack boards (all but the three on 9 x 9, one
                                       board per pair), test_budget[dynamics-0-(1, 9)] and [prediction-1-(3, 5)] at every gain
  - the board stride off by one (board b at b H S rows instead of b (H + 1) S: no separator rows):
                                       the same 25 fail
  - dropping x_l w_h:                  25 fail - all 22 test_exact cases, test_budget[dynamics-0-(1, 9)] at every gain
  - a missing block residual:          26 fail - the 20 test_exact cases with a block, test_budget[representation-2-(9, 9)]
                                       and [prediction-1-(3, 5)] at every gain
The budget cases at 16 blocks catch none of them: the propagated budget grows with the absolute weights at every layer,
so the integer towers carry these checks."""
import numpy
import pytest
import torch

from conftest import golden_npz, weights_for
from muzero_general_b200.netspec import netspec_from_config

pytestmark = pytest.mark.gpu

C = 256
SITES = ("representation", "dynamics", "dynamics_pool", "prediction")
STEM = {"representation": 0, "dynamics": 1, "dynamics_pool": 1, "prediction": 0}
BOARDS = ((6, 6), (1, 1), (1, 9), (9, 1), (3, 5), (9, 9), (4, 7))
C1, C2, FLOOR = 4e-6, 2e-6, 1e-6


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


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
        for co in rs.choice(C, 96, replace=False):
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


def run(site, x, ws, bs, act, A, seed=0, parts=1, stride=3, boards=0):
    from muzero_general_b200.engine import debug_wide256_tower, debug_wide256_tower_plan
    n, _, H, W = x.shape
    kw = {}
    if site == "dynamics_pool":
        kw = dict(parents=_parents(n, stride, numpy.random.RandomState(seed + 7)), pool_stride=stride, parts=parts)
    out, launches, sat, plan = debug_wide256_tower(x, ws, bs, site=site, actions=act, A=A, boards=boards, **kw)
    want, why = debug_wide256_tower_plan(n, C, H, W, (len(ws) - STEM[site]) // 2, STEM[site], sms(), boards)
    assert plan == want, (plan, want, why)
    assert plan["layers"] == len(ws) and (boards == 0 or plan["boards"] == boards)
    ranges = -(-n // (((n + parts - 1) // parts + 7) & ~7)) if site == "dynamics_pool" else 1
    assert launches == ranges, (launches, ranges)
    return out, sat


def _cases():
    out = []
    for site in SITES:
        for i, blocks in enumerate((0, 1, 2, 5, 16) if STEM[site] else (1, 2, 5, 16)):
            out.append((site, blocks, BOARDS[(i + len(out)) % len(BOARDS)]))
        out.append((site, 16, (6, 6)))
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
@pytest.mark.parametrize("site,blocks,board", [("dynamics_pool", 16, (6, 6)), ("prediction", 16, (6, 6)),
                                               ("representation", 2, (9, 9)), ("dynamics", 0, (1, 9)),
                                               ("prediction", 1, (3, 5))])
def test_budget(site, blocks, board, gain):
    H, W = board
    stem = STEM[site]
    x, ws, bs, act, A = normal_tower(3, H, W, blocks, stem, gain, seed=blocks + H)
    ref, _, budget = tower64(x, ws, bs, stem, act, A, gain=gain)
    got, sat = run(site, x, ws, bs, act, A)
    assert sat == 0
    ratio = numpy.abs(got - ref) / budget
    print(f"{site} {blocks} {board} gain {gain}: worst error / budget {ratio.max():.3f}")
    assert ratio.max() <= 1.0


@pytest.mark.parametrize("board,planned", [((6, 6), 2), ((1, 1), 8), ((2, 3), 8), ((4, 7), 2)])
@pytest.mark.parametrize("site", ["dynamics_pool", "prediction"])
def test_one_board_per_pair_equals_the_planned_stack(site, board, planned):
    H, W = board
    stem = STEM[site]
    x, ws, bs, act, A = normal_tower(7, H, W, 3, stem, 1.0, seed=H + W)
    stacked, _ = run(site, x, ws, bs, act, A)
    one, _ = run(site, x, ws, bs, act, A, boards=1)
    from muzero_general_b200.engine import debug_wide256_tower_plan
    assert debug_wide256_tower_plan(7, C, H, W, 3, stem, sms())[0]["boards"] == planned
    diff = numpy.argwhere(one != stacked)
    assert len(diff) == 0, f"first differing element {tuple(diff[0])}: 1 board {one[tuple(diff[0])]!r}, stacked {stacked[tuple(diff[0])]!r}"


def test_batches_at_the_wave_edges():
    """One CTA pair per two boards: 1, one wave - 1, one wave + 1 and several waves, each board inside the budget (checked
    on the boards at the edges) and independent of the batch around it (bit for bit)."""
    from muzero_general_b200.engine import debug_wide256_tower_plan
    plan, _ = debug_wide256_tower_plan(1, C, 6, 6, 1, True, sms())
    wave = plan["wave"]
    x, ws, bs, act, A = normal_tower(3 * wave + 5, 6, 6, 1, 1, 1.0, seed=5)
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
    x, ws, bs, act, A = normal_tower(n, 6, 6, 2, 1, 1.0, seed=9)
    one, _ = run("dynamics_pool", x, ws, bs, act, A, seed=2, parts=1)
    got, _ = run("dynamics_pool", x, ws, bs, act, A, seed=2, parts=parts)
    assert numpy.array_equal(got, one)


@pytest.mark.parametrize("where", [None, ("input", 0), ("input", 1), ("bias", 0), ("bias", 1)])
def test_range_guard_in_either_cta_and_either_board(where):
    """An input activation beyond the fp16 range on stacked board 0 or 1 of a pair, or a first-layer output beyond it in
    the channels of CTA 0 or CTA 1 (a bias of 1e5), bumps the guard; without either the guard stays at zero."""
    x, ws, bs, act, A = normal_tower(2, 6, 6, 1, 0, 1.0, seed=4)
    if where and where[0] == "input":
        x[where[1], 5, 3, 2] = 1e5
    elif where:
        bs[0][5 + 128 * where[1]] = 1e5
    _, peak, _ = tower64(x, ws, bs, 0, act, A)
    assert (peak > 65504) == (where is not None)
    _, sat = run("prediction", x, ws, bs, act, A)
    assert (sat > 0) == (where is not None)


# ---------------------------------------------------------------------------------------------- whole nets
WIDE256_ROUTE = "256-channel towers on the tensor cores, output channels split across CTA pairs"


@pytest.fixture
def wide3(monkeypatch):
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    monkeypatch.setenv("MZ_TC_WIDE", "3")


def _atari():
    from muzero_general_b200.games import load_game_module
    cfg = load_game_module("atari").MuZeroConfig()
    assert (cfg.blocks, cfg.channels) == (16, 256)
    return cfg


def _engine(cfg, n, N, **kw):
    from muzero_general_b200.engine import SearchEngine
    return SearchEngine(cfg, max_games=n, num_simulations=N, **kw)


def _obs(spec, n, seed):
    return numpy.random.RandomState(seed).random_sample((n, spec.in_channels) + spec.obs_shape[1:]).astype(numpy.float32)


def test_atari_net_matches_reference(wide3):
    """net_atari.npz against the reference, with two tolerances wider than test_resnet_gpu._close's x3 ones.  The towers
    here are 32 and 33 convs of K = 2304 and the 9216 -> 256 -> 256 -> 601 heads read every hidden element, so the x3
    route's fp32-grade error adds up further than on the 64- and 128-channel nets.  Measured on an H100: 2 of 18,432
    initial hidden-state elements land 1.40e-4 from the reference (atol 2.5e-4 here against 5e-5), and the logits up to
    4.63e-4 (the recurrent reward logits; atol 6e-4 against 2e-5, every logit check); rtol stays 2e-4.  The kernel is
    deterministic, so these are the errors of every run.  test_atari_closed_loop_matches_reference_counts shows that they
    leave the reference's searches unchanged.  The scalars keep test_resnet_gpu's Atari bounds."""
    cfg = _atari()
    spec = netspec_from_config(cfg)
    g = golden_npz("net_atari.npz")
    obs = numpy.random.RandomState(int(g["obs_seed"])).random_sample((2, spec.in_channels, 96, 96)).astype(numpy.float32)
    eng = _engine(cfg, 2, 4)
    eng.load_weights(weights_for("atari", spec))
    assert WIDE256_ROUTE in eng.numerics, eng.numerics
    r0 = eng.initial_inference(obs)
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(2, -1), g["action"])
    checks = [(r0["hidden"], g["init_hidden"].reshape(2, -1), "init hidden", 2.5e-4),
              (r1["hidden"], g["rec_hidden"].reshape(2, -1), "rec hidden", 2.5e-4)]
    checks += [(r[k], g[ref], ref, 6e-4) for r, k, ref in ((r0, "value_logits", "init_value"), (r0, "policy_logits", "init_policy"),
                                                         (r1, "value_logits", "rec_value"), (r1, "reward_logits", "rec_reward"),
                                                         (r1, "policy_logits", "rec_policy"))]
    for got, want, name, _ in checks:
        print(f"atari {name}: max abs err {numpy.abs(got - want).max():.3e}")
    for got, want, name, atol in checks:
        numpy.testing.assert_allclose(got, want, rtol=2e-4, atol=atol, err_msg=name)
    numpy.testing.assert_allclose(r0["value"], g["init_value_scalar"], rtol=1e-3, atol=5e-3)
    numpy.testing.assert_allclose(r1["reward"], g["rec_reward_scalar"], rtol=1e-3, atol=5e-3)
    assert WIDE256_ROUTE in eng.numerics                      # the guard did not trip
    eng.close()


def test_atari_student_forced(wide3):
    from helpers import oracle_replay, paths_from_trace
    from oracle import mcts as om
    cfg = _atari()
    spec = netspec_from_config(cfg)
    n, N, A = 3, 30, spec.action_space
    rs = numpy.random.RandomState(11)
    obs = _obs(spec, n, 12)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    first = rs.randint(0, A, n).astype(numpy.int32)
    eng = _engine(cfg, n, N)
    eng.load_weights(weights_for("atari", spec))
    out = eng.search(obs=obs.reshape(n, -1), add_exploration_noise=True, noise=noise, first_index=first, trace=True)
    params = om.SearchParams.from_config(cfg, N)
    tr = out.trace
    for i in range(n):
        res, _ = oracle_replay(params, list(range(A)), 0,
                               (out.root_predicted_value[i], tr["root_reward"][i], list(tr["root_priors_raw"][i])),
                               [(tr["value"][i, s], tr["reward"][i, s], tr["priors"][i, s]) for s in range(N)],
                               list(noise[i]), int(first[i]), seed=cfg.seed, game=i)
        assert [int(v) for v in out.visit_counts[i]] == res.root_visits
        assert out.root_value[i] == res.root_value
        assert paths_from_trace(tr, i, N) == [s.path_actions for s in res.sims]
    assert WIDE256_ROUTE in eng.numerics
    eng.close()


@pytest.mark.parametrize("route", ["wide256", "cuda_cores"])
def test_atari_closed_loop_matches_reference_counts(route, monkeypatch):
    """The reference's traced N = 50 searches (mcts_atari_n50.json): the device search on the same observations, root noise
    and first pick gives the reference's visit counts on both routes."""
    from test_wide256_plan_cpu import atari_search_cases
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    if route == "wide256":
        monkeypatch.setenv("MZ_TC_WIDE", "3")
    else:
        monkeypatch.delenv("MZ_TC_WIDE", raising=False)
    cfg = _atari()
    spec = netspec_from_config(cfg)
    cases = atari_search_cases()
    n, A = len(cases), spec.action_space
    eng = _engine(cfg, n, cases[0]["num_simulations"])
    eng.load_weights(weights_for("atari", spec))
    assert (WIDE256_ROUTE in eng.numerics) == (route == "wide256"), eng.numerics
    obs = numpy.stack([c["obs"] for c in cases]).reshape(n, -1)
    noise = numpy.array([c["noise"] for c in cases])
    first = numpy.array([c["first_index"] for c in cases], numpy.int32)
    out = eng.search(obs=obs, add_exploration_noise=True, noise=noise, first_index=first)
    for i, c in enumerate(cases):
        assert c["root_actions"] == list(range(A))
        assert [int(v) for v in out.visit_counts[i]] == c["root_visits"], (i, out.visit_counts[i], c["root_visits"])
        assert abs(int(out.max_tree_depth[i]) - c["max_tree_depth"]) <= 4
    assert (WIDE256_ROUTE in eng.numerics) == (route == "wide256")
    eng.close()


def test_graph_replay_equals_eager(wide3, monkeypatch):
    cfg = _atari()
    spec = netspec_from_config(cfg)
    n, N = 3, 8
    obs = _obs(spec, n, 3).reshape(n, -1)
    results = []
    for no_graph in ("1", "0"):
        monkeypatch.setenv("MZ_NO_GRAPH", no_graph)
        eng = _engine(cfg, n, N)
        eng.load_weights(weights_for("atari", spec))
        assert WIDE256_ROUTE in eng.numerics
        runs = [eng.search(obs=obs, add_exploration_noise=False) for _ in range(2)]
        assert numpy.array_equal(runs[1].visit_counts, runs[0].visit_counts)
        assert numpy.array_equal(runs[1].root_value, runs[0].root_value)
        results.append(runs[0])
        eng.close()
    assert numpy.array_equal(results[0].visit_counts, results[1].visit_counts)
    assert numpy.array_equal(results[0].root_value, results[1].root_value)


def test_stress_weights_fall_back_and_match(wide3, monkeypatch):
    """Atari weights whose towers leave the fp16 range: the guard trips, the handle leaves the 256-channel towers for good
    (graphs captured before are dropped) and the redone calls equal the CUDA-core route bit for bit."""
    from muzero_general_b200.netspec import stress_weights
    cfg = _atari()
    spec = netspec_from_config(cfg)
    w = stress_weights(spec, 0, "overflow")
    n, N = 2, 4
    obs = _obs(spec, n, 1).reshape(n, -1)
    eng = _engine(cfg, n, N)
    eng.load_weights(w)
    assert WIDE256_ROUTE in eng.numerics
    got = [eng.search(obs=obs, add_exploration_noise=False) for _ in range(2)]
    assert "256-channel tensor-core towers left" in eng.numerics
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


def test_routes_by_switch(monkeypatch, game_configs):
    """Unset, 1 and 2 keep Atari on the CUDA cores with today's numerics string; 3 takes it to the 256-channel towers and
    routes Gomoku's 128-channel net exactly as 2 does."""
    from muzero_general_b200.netspec import synthetic_weights
    monkeypatch.delenv("MZ_NO_TC", raising=False)
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    strings = {}
    for switch in (None, "1", "2", "3"):
        if switch is None:
            monkeypatch.delenv("MZ_TC_WIDE", raising=False)
        else:
            monkeypatch.setenv("MZ_TC_WIDE", switch)
        for name in ("atari", "gomoku"):
            cfg = game_configs[name]
            spec = netspec_from_config(cfg)
            eng = _engine(cfg, 2, 2)
            eng.load_weights(synthetic_weights(spec, 0))
            strings[switch, name] = eng.numerics
            eng.close()
    for switch in (None, "1", "2"):
        assert strings[switch, "atari"] == "f32 nets + f64 tree statistics", strings[switch, "atari"]
    assert WIDE256_ROUTE in strings["3", "atari"]
    assert strings["3", "gomoku"] == strings["2", "gomoku"]
