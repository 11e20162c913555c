"""downsample="CNN" (DownsampleCNN, models.py:278-297) without a GPU: the state_dict layout, the CPU oracle against the
reference's outputs, the planner's refusals against the reference's, the reach of the case table, and the mutants the
GPU exact test catches."""
import json

import numpy
import pytest
import torch
import torch.nn.functional as F

from cnn_oracle import CnnOracleNet
from cnnstemcases import CASES, exact_operands, plan
from conftest import golden_npz
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights, weights_spec

torch.set_num_threads(1)          # the fixtures were made single-threaded: the same ATen reduction order


def cnn_config(**over):
    from muzero_general_b200.games import load_game_module
    cfg = load_game_module("breakout").MuZeroConfig()
    cfg.downsample = "CNN"
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


@pytest.fixture(scope="module")
def lib():
    from muzero_general_b200 import _lib
    return _lib.load_library()


def test_weights_spec_and_oracle_reproduce_the_reference():
    g = golden_npz("net_breakout_cnn.npz")
    spec = netspec_from_config(cnn_config())
    assert spec.downsample == 2 and spec.hidden_hw == (6, 6)
    assert [(k, list(s)) for k, s in weights_spec(spec)] == list(zip([str(k) for k in g["keys"]], json.loads(str(g["shapes"]))))
    obs = numpy.random.RandomState(int(g["obs_seed"])).random_sample((2, 3, 96, 96)).astype(numpy.float32)
    net = CnnOracleNet(spec, synthetic_weights(spec, 0))
    v0, _, p0, h0 = net.initial_inference(obs)
    v1, r1, p1, h1 = net.recurrent_inference(h0, torch.from_numpy(g["action"]))
    for got, key in ((v0, "init_value"), (p0, "init_policy"), (h0, "init_hidden"), (v1, "rec_value"), (r1, "rec_reward"),
                     (p1, "rec_policy"), (h1, "rec_hidden")):
        assert numpy.array_equal(got.numpy(), g[key]), key


def test_oracle_reproduces_reference_shapes():
    g = golden_npz("net_cnn_shapes.npz")
    heads = dict(reduced_channels_reward=2, reduced_channels_value=2, reduced_channels_policy=2,
                 resnet_fc_reward_layers=[8], resnet_fc_value_layers=[8], resnet_fc_policy_layers=[8])
    for i, (name, shape, s, ch, blocks) in enumerate((("s24", (3, 24, 24), 0, 8, 1), ("s96x64", (3, 96, 64), 0, 8, 1),
                                                      ("s210", (3, 210, 160), 0, 4, 0), ("stack4", (3, 96, 96), 4, 8, 1))):
        spec = netspec_from_config(cnn_config(observation_shape=shape, stacked_observations=s, channels=ch, blocks=blocks, **heads))
        x = numpy.random.RandomState(i).randint(0, 256, size=(1, spec.in_channels) + shape[1:]).astype(numpy.float32)
        v, _, p, h = CnnOracleNet(spec, synthetic_weights(spec, 0)).initial_inference(x / numpy.float32(255))
        for got, key in ((v, "value"), (p, "policy"), (h, "hidden")):
            assert numpy.array_equal(got.numpy(), g[f"{name}_{key}"]), (name, key)


def test_planner_refuses_exactly_what_the_reference_raises_on(lib):
    g = golden_npz("cnn_geometry.npz")
    table = [(int(H), int(W), g["raises"][i, j]) for i, H in enumerate(g["sizes"]) for j, W in enumerate(g["sizes"])]
    table += [tuple(int(v) for v in row) for row in g["extra"]]
    wrong = [(H, W) for H, W, r in table if (plan(lib, 4, 3, 4, H, W, 132) is None) != bool(r)]
    assert not wrong, wrong[:20]
    assert 0 < g["raises"].sum() < g["raises"].size


@pytest.mark.parametrize("H,W,why", [(20, 24, "pool2 output is 0 rows"), (23, 23, "pool2"), (11, 11, "pool"),
                                     (96, 8, "pool1 output is 0 columns"), (96, 6, "conv1: kernel 12 x 12")])
def test_refusal_names_the_stage(lib, H, W, why):
    assert plan(lib, 1, 3, 16, H, W, 132) is None and why in lib.mz_last_error(None).decode()


def test_plan_geometry(lib):
    p = plan(lib, 8, 3, 16, 210, 160, 132)
    assert (p["h"], p["w"], p["mid"], p["s0"]["k"], p["s1"]["k"]) == (14, 10, 9, 28, 5)
    assert [p["s0"][f] for f in ("Ho", "Wo", "Hp", "Wp")] + [p["s1"]["Hp"], p["s1"]["Wp"]] == [47, 35, 23, 17, 11, 8]
    for H, W, hw in ((96, 96, (6, 6)), (96, 64, (6, 4)), (64, 96, (4, 6)), (24, 24, (2, 2)), (26, 26, (2, 2))):
        assert (plan(lib, 8, 3, 16, H, W, 132)["h"], plan(lib, 8, 3, 16, H, W, 132)["w"]) == hw


@pytest.mark.parametrize("sm_count", [132, 114])
def test_case_table_reaches_every_tile_edge(lib, sm_count):
    seen = set()
    for c in CASES:
        p = plan(lib, c.n, c.cin, c.C, c.H, c.W, sm_count)
        for q, cin, cout in ((p["s0"], c.cin, c.mid), (p["s1"], c.mid, c.C)):
            seen |= {("items", q["items"]), ("chunked", q["cin_chunk"] < cin), ("bands", q["bands"] > 1),
                     ("boards", q["boards"] > 1), ("ragged", c.n % q["boards"] != 0), ("co_tiles", q["grid_y"] > 1),
                     ("partial_tile", cout % q["co_tile"] != 0)}
            assert q["grid_x"] == -(-c.n // q["boards"]) and q["grid_y"] == -(-cout // q["co_tile"])
            assert q["threads"] <= 256 and q["smem"] <= 112 * 1024
    want = {("items", i) for i in (1, 2, 4, 8, 16)}
    want |= {(k, v) for k in ("chunked", "bands", "boards", "ragged", "co_tiles", "partial_tile") for v in (False, True)}
    assert want <= seen, sorted(want - seen)


def stem64(case, x, w, kernel_from_w=False, ceil_mode=False, floor_bins=False, no_bias=False, stride=4, pad=2):
    """The stem in fp64, with one deliberate mistake switched on when asked."""
    t = lambda a: torch.from_numpy(numpy.asarray(a)).double()
    (h, wd), w1 = case.hw, t(w[0])
    if kernel_from_w:                                   # k = 2 ceil(W / 16): crop or zero-pad the kernel to that size
        k = 2 * wd
        w1 = F.pad(w1, (0, max(0, k - w1.shape[3]), 0, max(0, k - w1.shape[2])))[:, :, :k, :k]
    y = F.max_pool2d(F.relu(F.conv2d(t(x), w1, None if no_bias else t(w[1]), stride, pad)), 3, 2, ceil_mode=ceil_mode)
    y = F.max_pool2d(F.relu(F.conv2d(y, t(w[2]), t(w[3]), 1, 2)), 3, 2, ceil_mode=ceil_mode)
    if not floor_bins:
        return F.adaptive_avg_pool2d(y, (h, wd)).numpy()
    Hp, Wp = y.shape[2:]
    end = lambda i, In, Out: max((i + 1) * In // Out, i * In // Out + 1)
    return numpy.stack([numpy.stack([y[:, :, i * Hp // h:end(i, Hp, h), j * Wp // wd:end(j, Wp, wd)].mean((2, 3)).numpy()
                                     for j in range(wd)], -1) for i in range(h)], -2)


MUTANTS = {"kernel width from ceil(W/16)": dict(kernel_from_w=True), "ceil-mode pooling": dict(ceil_mode=True),
           "adaptive bins with a floor end": dict(floor_bins=True), "dropped bias": dict(no_bias=True),
           "stride 3": dict(stride=3), "stride 5": dict(stride=5), "padding 1": dict(pad=1), "padding 3": dict(pad=3)}


def test_every_mutant_changes_an_exact_case():
    """Each mistake changes the integer-operand stem of at least one case; on the device the kernel must EQUAL the
    unmutated fp64 stem on those operands (test_cnn_stem_gpu.py::test_stem_equals_fp64_on_integer_operands)."""
    caught = {m: [] for m in MUTANTS}
    for c in CASES:
        if c.cin > 19:
            continue                                    # the wide stacks: seconds of fp64 convs on a CPU
        c = c._replace(n=min(c.n, 2))
        x, w = exact_operands(c, numpy.random.RandomState(17))
        want = stem64(c, x, w)
        for m, kw in MUTANTS.items():
            try:
                got = stem64(c, x, w, **kw)
            except RuntimeError:                        # the mutant cannot even run this geometry
                got = None
            if got is None or got.shape != want.shape or not numpy.array_equal(got, want):
                caught[m].append(c.name)
    for m, names in caught.items():
        print(f"[cnn stem mutants] {m}: caught by {', '.join(names)}")
    assert all(caught.values()), caught
