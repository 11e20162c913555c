"""CPU checks of the network case table (tests/netcases.py): the fp64 oracle computes the same networks as the fp32
oracle on every case, the table covers every route with shapes that really select it, and the host-side planner of the
fused small-network search accepts exactly the small-search cases and refuses their neighbours."""
import dataclasses

import numpy
import pytest
import torch

from muzero_general_b200.netspec import FC
from netcases import BY_NAME, CASES, ROUTES, SEARCH_CASES, case_spec, edge_weights, make_config, small_search_inputs
from oracle.net import OracleNet, support_to_scalar


def _inputs(spec, n, seed=0):
    rs = numpy.random.RandomState(seed)
    obs = rs.random_sample((n, spec.in_channels) + tuple(spec.obs_shape[1:])).astype(numpy.float32)
    act = (numpy.arange(n) % spec.action_space).astype(numpy.int64).reshape(n, 1)
    act[-1, 0] = spec.action_space - 1
    return obs, act


@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_fp64_oracle_agrees_with_fp32_oracle(name):
    """Same network, two precisions: the fp64 outputs lie within fp32 noise of the fp32 (reference-exact) outputs, so
    the fp64 oracle is a restatement of the reference and a valid yardstick for the kernels."""
    case = BY_NAME[name]
    spec = case_spec(case)
    w = edge_weights(spec, case.weights)
    o32, o64 = OracleNet(spec, w), OracleNet(spec, w, torch.float64)
    obs, act = _inputs(spec, 4)
    S = spec.support_size
    a = o32.initial_inference(obs)
    b = o64.initial_inference(obs)
    assert b[3].dtype == torch.float64
    ra = o32.recurrent_inference(a[3], torch.from_numpy(act))
    rb = o64.recurrent_inference(a[3], torch.from_numpy(act))      # same fp32 input state
    outs = list(zip(("init value", "init policy", "init hidden", "rec value", "rec reward", "rec policy", "rec hidden"),
                    (a[0], a[2], a[3], ra[0], ra[1], ra[2], ra[3]), (b[0], b[2], b[3], rb[0], rb[1], rb[2], rb[3])))
    outs += [("init value scalar", support_to_scalar(a[0], S), support_to_scalar(b[0], S, torch.float64)),
             ("rec value scalar", support_to_scalar(ra[0], S), support_to_scalar(rb[0], S, torch.float64)),
             ("rec reward scalar", support_to_scalar(ra[1], S), support_to_scalar(rb[1], S, torch.float64))]
    for what, x32, x64 in outs:
        x32, x64 = x32.double().numpy(), x64.numpy()
        err = numpy.abs(x32 - x64).max()
        scale = max(1.0, float(numpy.abs(x64).max()))
        # hidden states: the rescale divides by channel ranges down to ~1e-3 on the narrow boards, amplifying fp32 noise
        bound = 2e-3 if "hidden" in what else 1e-4 * scale
        assert err <= bound, (name, what, err, bound)
    # the root reward logits are log(one-hot) in either precision
    assert torch.equal(torch.isinf(a[1]), torch.isinf(b[1]))


def test_case_table_covers_every_route_with_shapes_that_select_it():
    """Each route has a case, and every case has the shape its route needs (tensor cores: C == 64, H <= 6, W <= 7 and
    no DownSample; fused CUDA-core tower: 2 <= W <= 8, H <= 16; per-layer: wider boards or MZ_NO_FUSE; heads_kernel<32>
    versus <128>: C*H*W <= 1024; the fused FC fixed shape: CartPole's exactly)."""
    assert {c.route for c in CASES} == set(ROUTES)
    for c in CASES:
        spec = case_spec(c)
        make_config(c)
        if spec.kind == FC:
            # fc_net.cuh::fc_matches_fixed<CartPoleShape> (the representation network is not part of the search)
            fixed = (spec.encoding, spec.support_size, spec.action_space) == (8, 10, 2) and \
                spec.fc_dynamics == spec.fc_reward == spec.fc_value == spec.fc_policy == [16]
            assert fixed == (c.route == "fc_fixed"), c.name
            assert (spec.action_space > 32) == (c.route == "fc_stepwise"), c.name
            continue
        H, W = spec.hidden_hw
        tc_shape = spec.channels == 64 and H <= 6 and W <= 7 and not spec.downsample
        assert tc_shape == (c.route in ("tc", "tc_heads_left")), c.name
        if c.route == "small_tower":
            assert 2 <= W <= 8 and H <= 16
        if c.route == "per_layer":
            assert W > 8 or c.env.get("MZ_NO_FUSE") == "1" or spec.channels >= 48
        if c.route == "heads_wide":
            assert spec.channels * H * W > 1024
        if c.route == "downsample":
            assert spec.downsample and (H, W) == tuple(-(-x // 16) for x in spec.obs_shape[1:])
    assert any(case_spec(c).blocks == 0 and c.route == "tc" for c in CASES)
    # tensor-core towers: one 8-layer launch (4 blocks) and towers split across launches (the dynamics tower from 4
    # blocks on, every tower from 5), the split in-search dynamics tower inside a partitioned search too
    tc_blocks = {case_spec(c).blocks for c in CASES if c.route == "tc"}
    assert 4 in tc_blocks and max(tc_blocks) >= 5, tc_blocks
    assert any(BY_NAME[name].route == "tc" and case_spec(BY_NAME[name]).blocks >= 5 for name in SEARCH_CASES)
    assert any(case_spec(c).blocks == 0 and c.route != "tc" and case_spec(c).kind != FC for c in CASES)
    narrow_tc = [c for c in CASES if c.route == "tc" and case_spec(c).channels * numpy.prod(case_spec(c).hidden_hw) <= 1024]
    assert narrow_tc, "no tensor-core case takes the narrow heads"


def _plan(lib, H, W, C, A, n, tower, heads, scratch, cap, sms=132):
    import ctypes
    out = (ctypes.c_int64 * 8)()
    return bool(lib.mz_debug_small_search_plan(H, W, C, A, n, sms, tower, heads, scratch, cap, out))


def test_small_search_planner_accepts_the_cases_and_refuses_their_neighbours():
    """mz_debug_small_search_plan (host only) takes every small-search case of the table at the search sizes of the
    GPU sweep, and refuses the same nets with 5..8 actions (no lane-group width) or a 4-wide board."""
    from muzero_general_b200 import _lib
    lib = _lib.load_library()
    cases = [c for c in CASES if c.route == "small_search"]
    assert len(cases) >= 4
    for c in cases:
        p = small_search_inputs(case_spec(c))
        for n in (1, 40, 300):
            assert _plan(lib, p["H"], p["W"], p["C"], p["A"], n, p["tower"], p["heads"], p["scratch"], p["cap"]), (c.name, n)
        for A in (5, 6, 7, 8):
            assert not _plan(lib, p["H"], p["W"], p["C"], A, 40, p["tower"], p["heads"], p["scratch"], p["cap"]), (c.name, A)
        assert not _plan(lib, p["H"], 4, p["C"], p["A"], 40, p["tower"], p["heads"], p["scratch"], p["cap"]), c.name
    # two 32-channel blocks: tower weights beyond shared memory
    big = small_search_inputs(dataclasses.replace(case_spec(BY_NAME["ss_3x3_a16_c20"]), channels=32))
    assert not _plan(lib, big["H"], big["W"], big["C"], big["A"], 40, big["tower"], big["heads"], big["scratch"], big["cap"])
    # the other residual routes of the table are not small-search shapes
    for c in CASES:
        spec = case_spec(c)
        if spec.kind == FC or c.route == "small_search" or spec.blocks < 1:
            continue
        p = small_search_inputs(spec)
        if c.route in ("tc", "tc_heads_left", "heads_big", "heads_wide", "per_layer", "downsample"):
            continue       # not decided by the planner (tensor cores, heads or per-layer convs rule them out first)
        assert not _plan(lib, p["H"], p["W"], p["C"], p["A"], 40, p["tower"], p["heads"], p["scratch"], p["cap"]), c.name
