"""downsample="CNN" (DownsampleCNN, models.py:278-297) on the device: the stem alone (csrc/cnn_stem.cu through
mz_debug_cnn_stem, output starting as NaN) against fp64, whole CNN nets against the fp64 oracle and the reference, and
searches against the reference's closed loop and against themselves across the pipeline's launch routes.

Exact test: on sparse small-integer operands every partial sum is an integer below 2^24, max pooling is exact and each
average one correctly rounded division of an exact fp32 sum, so the stem EQUALS fp64 rounded to fp32 (rounding twice is
harmless for a division when the wider format has at least 2p + 2 bits).  Budget test: on standard-normal operands the
error stays inside a bound propagated stage by stage: a conv adds gamma_n * (|b| + sum |w||x|), n = cin * k^2 + 1, and
carries its input's bound through sum |w|; ReLU and max are non-expansive; the average adds gamma_cnt * mean|x| and one
rounding."""
import ctypes

import numpy
import pytest
import torch
import torch.nn.functional as F

from cnn_oracle import CnnOracleNet
from cnnstemcases import CASES, exact_operands, plan, unpack
from conftest import golden_json, golden_npz
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
from test_cnn_stem_cpu import cnn_config, stem64

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
gamma = lambda n: n * U / (1 - n * U)
BY_NAME = {c.name: c for c in CASES}
WORST = [0.0]


def _stem_device(case, x, w):
    from muzero_general_b200 import _lib
    lib = _lib.load_library()
    out = numpy.empty((case.n, case.C) + case.hw, numpy.float32)
    pl = (ctypes.c_int64 * 36)()
    p = [numpy.ascontiguousarray(a, numpy.float32) for a in [x] + list(w)]
    assert lib.mz_debug_cnn_stem(0, case.n, case.cin, case.C, case.H, case.W, *[a.ctypes.data for a in p],
                                 out.ctypes.data, pl) == 0, lib.mz_last_error(None)
    got = unpack(list(pl))
    assert got == plan(lib, case.n, case.cin, case.C, case.H, case.W, torch.cuda.get_device_properties(0).multi_processor_count)
    return out


def _bound(case, x, w):
    d = lambda a: torch.from_numpy(numpy.asarray(a)).double()
    x, w1, b1, w2, b2 = map(d, [x] + list(w))
    k = 2 * case.hw[0]
    with torch.no_grad():
        e1 = F.max_pool2d(gamma(case.cin * k * k + 1) * F.conv2d(x.abs(), w1.abs(), b1.abs(), 4, 2), 3, 2)
        p1 = F.max_pool2d(F.relu(F.conv2d(x, w1, b1, 4, 2)), 3, 2)
        e2 = F.conv2d(e1, w2.abs(), None, 1, 2) + gamma(case.mid * 25 + 1) * F.conv2d(p1.abs() + e1, w2.abs(), b2.abs(), 1, 2)
        p2, e2 = F.max_pool2d(F.relu(F.conv2d(p1, w2, b2, 1, 2)), 3, 2), F.max_pool2d(e2, 3, 2)
        cnt = (-(-p2.shape[2] // case.hw[0]) + 1) * (-(-p2.shape[3] // case.hw[1]) + 1)   # a bin's size is at most this
        avg = lambda v: F.adaptive_avg_pool2d(v, case.hw)
        return (avg(e2) + gamma(cnt) * (avg(p2.abs()) + avg(e2)) + U * (avg(p2).abs() + avg(e2))).numpy()


@pytest.mark.parametrize("name", list(BY_NAME))
def test_stem_equals_fp64_on_integer_operands(name):
    case = BY_NAME[name]
    x, w = exact_operands(case, numpy.random.RandomState(17))
    want = stem64(case, x, w)
    assert numpy.abs(want).max() > 0
    assert numpy.array_equal(_stem_device(case, x, w), want.astype(numpy.float32))


@pytest.mark.parametrize("gain", [1.0, 1e-4, 300.0])
@pytest.mark.parametrize("name", list(BY_NAME))
def test_stem_within_propagated_bound(name, gain):
    case = BY_NAME[name]
    rs = numpy.random.RandomState(23)
    k = 2 * case.hw[0]
    x = (rs.standard_normal((case.n, case.cin, case.H, case.W)) * gain).astype(numpy.float32)
    w = [rs.standard_normal((case.mid, case.cin, k, k)) / numpy.sqrt(case.cin * k * k), rs.standard_normal(case.mid) * gain,
         rs.standard_normal((case.C, case.mid, 5, 5)) / numpy.sqrt(case.mid * 25), rs.standard_normal(case.C) * gain]
    w = [a.astype(numpy.float32) for a in w]
    err = numpy.abs(_stem_device(case, x, w).astype(numpy.float64) - stem64(case, x, w))
    bound = _bound(case, x, w)
    WORST[0] = max(WORST[0], float((err / numpy.maximum(bound, 1e-300)).max()))
    print(f"[cnn stem] {name} gain {gain:g}: max err {err.max():.3e}; worst error/bound so far {WORST[0]:.3e}")
    assert (err <= bound).all()


def _engine(cfg, n, N):
    from muzero_general_b200.engine import SearchEngine
    return SearchEngine(cfg, max_games=n, num_simulations=N)


@pytest.mark.parametrize("label,over,n", [("breakout_cnn_b0", dict(blocks=0), 5), ("breakout_cnn_b2", {}, 33),
                                          ("cnn_c64", dict(channels=64, blocks=1), 7)])
def test_initial_inference_matches_fp64_oracle(label, over, n):
    """The sweep's rule (DESIGN.md section 3.6: K = 16, FLOOR = 64 ulps) against CnnOracleNet in fp32 and fp64."""
    from test_net_sweep_gpu import Judge, Ref
    spec = netspec_from_config(cnn_config(**over))
    w = synthetic_weights(spec, 0)
    obs = numpy.random.RandomState(n).random_sample((n, spec.obs_elems)).astype(numpy.float32)
    eng = _engine(cnn_config(**over), n, 2)
    eng.load_weights(w)
    r = eng.initial_inference(obs)
    eng.close()
    oracle = Ref(spec, w)
    oracle.o32, oracle.o64 = CnnOracleNet(spec, w), CnnOracleNet(spec, w, torch.float64)
    ref, j = oracle.initial(obs), Judge(label)
    for i in range(n):
        for k in ("hidden", "value_logits", "policy_logits"):
            j.vector(f"row {i} {k}", r[k][i], ref, k, i)
        j.scalar(f"row {i} value", r["value"][i], ref, "value", i)
    j.finish()


def test_reference_fixture_and_refusal():
    g = golden_npz("net_breakout_cnn.npz")
    spec = netspec_from_config(cnn_config())
    eng = _engine(cnn_config(), 2, 2)
    eng.load_weights(synthetic_weights(spec, 0))
    obs = numpy.random.RandomState(int(g["obs_seed"])).random_sample((2, spec.obs_elems)).astype(numpy.float32)
    r0 = eng.initial_inference(obs)
    r1 = eng.recurrent_inference(g["init_hidden"].reshape(2, -1), g["action"])
    eng.close()
    for got, key in ((r0["hidden"], "init_hidden"), (r1["hidden"], "rec_hidden")):
        numpy.testing.assert_allclose(got, g[key].reshape(2, -1), rtol=2e-4, atol=5e-5)
    for got, key in ((r0["value_logits"], "init_value"), (r0["policy_logits"], "init_policy"),
                     (r1["reward_logits"], "rec_reward"), (r1["policy_logits"], "rec_policy")):
        numpy.testing.assert_allclose(got, g[key], rtol=2e-4, atol=2e-5)
    with pytest.raises(Exception, match="pool2 output is 0 rows"):
        _engine(cnn_config(observation_shape=(3, 20, 24)), 1, 2)


def test_closed_loop_matches_reference_counts():
    cfg = cnn_config()
    spec = netspec_from_config(cfg)
    for c in golden_json("mcts_breakout_cnn_n50.json"):
        eng = _engine(cfg, 1, c["num_simulations"])
        eng.load_weights(synthetic_weights(spec, 0))
        obs = numpy.random.RandomState(c["obs_seed"]).random_sample((1, 3, 96, 96)).astype(numpy.float32)
        noise = numpy.zeros((1, 4)); noise[0, c["legal"]] = c["noise"]
        out = eng.search(obs=obs, legal_mask=numpy.ones((1, 4), numpy.uint8), to_play=numpy.zeros(1, numpy.int32),
                         add_exploration_noise=True, noise=noise, first_index=numpy.array([c["first_index"]], numpy.int32))
        eng.close()
        assert [int(out.visit_counts[0, a]) for a in c["root_actions"]] == c["root_visits"]
        for k in ("root_value", "root_predicted_value"):
            assert abs(getattr(out, k)[0] - c[k]) <= 5e-4 * max(1.0, abs(c[k]))


def test_search_routes_are_bit_identical(monkeypatch):
    """Fused small search, step-wise pipeline, eager (no graph), no PDL, MZ_PARTS = 1..4: the same visit counts, values,
    ranges, depths and root states, each search repeated (capture, replay); Reanalyse's batched initial inference gives
    the roots' hidden states; MCTS.run goes through the host facade."""
    cfg = cnn_config()
    spec = netspec_from_config(cfg)
    n, N = 37, 12
    rs = numpy.random.RandomState(4)
    obs = rs.random_sample((n, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * spec.action_space, size=n)
    w = synthetic_weights(spec, 0)
    results = []
    for env in [dict(MZ_SMALL_SEARCH="1"), dict(MZ_SMALL_SEARCH="0"), dict(MZ_NO_GRAPH="1"), dict(MZ_NO_PDL="1")] + \
               [dict(MZ_PARTS=str(p), MZ_SMALL_SEARCH="0") for p in (1, 2, 3, 4)]:
        for k in ("MZ_SMALL_SEARCH", "MZ_NO_GRAPH", "MZ_NO_PDL", "MZ_PARTS"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng = _engine(cfg, n, N)
        eng.load_weights(w)
        runs = [eng.search(obs=obs, add_exploration_noise=True, noise=noise, keep_tree=True) for _ in range(3)]
        roots = numpy.stack([eng.export_tree(i, with_hidden=True)["hidden"][0] for i in (0, n // 2, n - 1)])
        eng.close()
        for r in runs:
            for k in ("visit_counts", "root_value", "value_range", "max_tree_depth", "root_predicted_value"):
                assert numpy.array_equal(getattr(r, k), getattr((results[0][1] if results else runs[0]), k)), (env, k)
        assert not results or numpy.array_equal(roots, results[0][2]), env
        results.append((env, runs[0], roots))
    assert (results[0][1].visit_counts.sum(1) == N).all()
    from muzero_general_b200.reanalyse import Reanalyse
    re = Reanalyse({"weights": w}, cfg, max_positions=n)
    assert numpy.array_equal(re.engine.initial_inference(obs)["hidden"][[0, n // 2, n - 1]], results[0][2])
    re.close()
    from muzero_general_b200.self_play import MCTS, DeviceModel
    cfg.num_simulations = 8
    model = DeviceModel(cfg)
    model.set_weights(w)
    root, info = MCTS(cfg).run(model, obs[0].reshape(3, 96, 96), [0, 1, 2, 3], 0, True)
    assert root.visit_count == 8 and info["max_tree_depth"] >= 1
