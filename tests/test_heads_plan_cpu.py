"""Host-side launch planner of the residual heads (Runner::plan_heads in csrc/resnet.cu, through mz_debug_heads_plan): the case
table of tests/headcases.py, sized at 132 SMs (H100 SXM) and 114 SMs (H100 PCIe), reaches every route and edge it claims;
the planner refuses what the routes cannot take, with the reason; and the multiply-high division of heads.cuh is exact for
every divisor and index heads_kernel can be handed."""
import numpy
import pytest

from headcases import BY_NAME, CASES, ROUTES, SITES, SMEM_LIMIT, case_plan, first_range, layer_ks


@pytest.fixture(scope="module")
def plan_fn():
    from muzero_general_b200.engine import debug_heads_plan
    return debug_heads_plan


@pytest.mark.parametrize("S", [132, 114])
def test_case_table_reaches_every_route_and_edge(plan_fn, S):
    plans = {c.name: case_plan(c, S, plan_fn) for c in CASES}
    for c in CASES:
        n, p = plans[c.name]
        assert p["route"] == c.route, (c.name, S, p)
        if c.route != "generic":
            assert p["smem"] <= SMEM_LIMIT and p["grid"] <= S and p["threads"] == p["groups"] * {"warp": 32, "wide": 128}[c.route]
    assert {c.route for c in CASES} == set(ROUTES)
    # groups per CTA cut down by shared memory: fewer than the batch asks for
    shrunk = [k for k, (n, p) in plans.items() if p["route"] == "wide" and p["groups"] < min(8, -(-first_range(n, BY_NAME[k].parts) // S))]
    assert "pred_wide_shrunk_persist" in shrunk, shrunk
    # split-K: every ks at span 32 and at span 16 on the narrow kernel
    ks = {(len(c.heads), k) for c in CASES if c.route == "warp" for head in layer_ks(c, "warp") for k in head}
    assert {k for _, k in ks} == {1, 2, 4, 8}, ks
    assert {(1, 4), (1, 8), (2, 2), (2, 4)} <= ks, ks
    # channels, boards, C*HW on both sides of 1024
    assert {20, 48} <= {c.C for c in CASES} and {16, 32, 64} <= {c.C for c in CASES}
    assert any(c.HW == 1 for c in CASES) and any((c.H, c.W) == (16, 8) and c.layout == "dense" for c in CASES)
    assert any(c.C * c.HW <= 1024 for c in CASES) and any(c.C * c.HW > 1024 for c in CASES)
    # head shapes
    heads = [h for c in CASES for h in c.heads]
    assert {1, 2, 3, 5, 16} <= {rc for rc, _, _ in heads}
    assert {(), (16,), (3, 9), (128,), (256, 256)} <= {hid for _, hid, _ in heads}
    assert {1, 3, 7, 21, 601} <= {o for _, _, o in heads}
    assert any(c.site == "prediction" and len(c.heads[0][1]) != len(c.heads[1][1]) for c in CASES)
    # layouts at every site, batches, partitions
    for s in SITES:
        assert {c.layout for c in CASES if c.site == s} == {"dense", "f16", "split"}, s
    ranges = {k: (first_range(n, BY_NAME[k].parts), p) for k, (n, p) in plans.items()}
    assert any(m == 1 for m, _ in ranges.values())
    assert any(p["groups"] > 1 and m % p["groups"] for m, p in ranges.values() if p["route"] != "generic")
    persistent = {k for k, (m, p) in ranges.items() if p["route"] != "generic" and m > p["grid"] * p["groups"]}
    assert {c.name for c in CASES if c.n == "persist"} <= persistent, persistent
    assert {c.parts for c in CASES if c.site == "dynamics_pool"} >= {2, 3, 4}


def test_forced_routes_plan_where_they_fit(plan_fn):
    """Every dense single-range case takes all three routes when forced, except a forced group whose weights do not fit."""
    for c in CASES:
        if c.layout != "dense" or c.parts != 1:
            continue
        for route in ROUTES:
            p, why = plan_fn(4, c.C, c.H, c.W, c.heads, c.site, c.layout, route, 0, 132)
            if c.route == "generic" and route != "generic":
                assert p is None and "exceed shared memory" in why, (c.name, route, why)
            else:
                assert p is not None and p["route"] == route, (c.name, route, why)


TTT = dict(C=16, H=3, W=3, heads=[(2, [], 21), (3, [], 9)], site="prediction")


@pytest.mark.parametrize("change,reason", [
    (dict(layout="f16", C=64, route="generic"), "dense states only"),
    (dict(layout="split", C=64, route="generic"), "dense states only"),
    (dict(route="generic", g0=8), "partitioned calls are not supported"),
    (dict(heads=[(16, [256, 256], 21), (16, [], 7)], H=16, W=8, g0=8), "partitioned calls are not supported"),
    (dict(heads=[(16, [256, 256], 21), (16, [], 7)], H=16, W=8, route="warp"), "forced group"),
    (dict(heads=[(16, [256, 256], 21), (16, [], 7)], H=16, W=8, route="wide"), "forced group"),
    (dict(layout="f16"), "64 channels"),
    (dict(layout="split", C=64, H=7, W=7), "64 channels"),
    (dict(C=18), "bad shape"),
    (dict(heads=[(2, [], 20), (3, [], 9)]), "2 S + 1"),
])
def test_planner_refuses_what_the_routes_cannot_take(plan_fn, change, reason):
    a = dict(TTT, layout="dense", route="planned", g0=0)
    a.update(change)
    p, why = plan_fn(4, a["C"], a["H"], a["W"], a["heads"], a["site"], a["layout"], a["route"], a["g0"], 132)
    assert p is None and reason in why, (p, why)


def test_generic_route_when_one_group_does_not_fit(plan_fn):
    """The planned route falls back to the generic kernels on a dense state whose tile alone exceeds shared memory, and
    refuses the same state on the board layout (which has no generic route)."""
    p, _ = plan_fn(4, 64, 32, 32, [], "representation", "dense", "planned", 0, 132)
    assert p["route"] == "generic"
    p, _ = plan_fn(4, 64, 6, 7, [(2, [], 21), (4, [], 7)], "prediction", "f16", "planned", 0, 132)
    assert p["route"] == "wide"


def _umulhi_exact(HW, i):
    m = (2 ** 32 + HW - 1) // HW
    return numpy.array_equal((i * numpy.uint64(m)) >> numpy.uint64(32), i // numpy.uint64(HW))


def test_hw_inv_division_is_exact_for_every_index_heads_kernel_takes(plan_fn):
    """heads.cuh divides by HW as __umulhi(i, ceil(2^32 / HW)).  Exhaustively exact for 2 <= HW <= 1024 and i < 2^17.  Beyond,
    by the sufficient condition i * (ceil(2^32 / HW) * HW - 2^32) < 2^32 (the rounding error of the reciprocal stays below one
    step of i / HW) for every i below the largest index: heads_kernel divides only staging / rescale indices i < C * HW and
    conv1x1 items i < HW * ceil(rc / 4) <= rc * HW, and one group's tile of HW * (C + 4) floats plus its rc * HW activations
    must fit in 227 KB, so every index is below 227 KB / 4 bytes."""
    i = numpy.arange(2 ** 17, dtype=numpy.uint64)
    for HW in range(2, 1025):
        assert _umulhi_exact(HW, i), HW
    i_max = SMEM_LIMIT // 4
    assert i_max < 2 ** 17
    for HW in range(1025, i_max // 5 + 1):              # C >= 4: HW * (C + 4) <= i_max
        e = ((2 ** 32 + HW - 1) // HW) * HW - 2 ** 32
        assert i_max * e < 2 ** 32, HW
    # the largest tiles heads_kernel takes are below that index bound; one more position and the planner leaves them
    for C in (4, 16, 64):
        HW = i_max // (C + 4)
        while HW > 1:
            p, _ = plan_fn(1, C, HW, 1, [], "representation", "dense", "planned", 0, 132)
            if p["route"] != "generic":
                break
            HW -= 1
        assert C * HW < i_max and HW * (C + 4) <= i_max, (C, HW)
