"""Host-side launch planner of the fused CUDA-core tower (csrc/small_tower.cu, through mz_debug_small_tower_plan): the case
table of tests/smalltowercases.py, sized at 132 SMs (H100 SXM) and 114 SMs (H100 PCIe), reaches every instantiation and
edge it claims, and the planner refuses the shapes the kernel cannot take, with the reason."""
import pytest

from smalltowercases import BY_NAME, CASES, INSTANTIATIONS, REFUSED, SITES, case_plan, first_range


@pytest.fixture(scope="module")
def plan_fn():
    from muzero_general_b200.engine import debug_small_tower_plan
    return debug_small_tower_plan


@pytest.mark.parametrize("S", [132, 114])
def test_case_table_reaches_every_instantiation_and_edge(plan_fn, S):
    plans = {c.name: case_plan(c, S, plan_fn) for c in CASES}
    for c in CASES:
        n, p = plans[c.name]
        assert (p["P"], p["CO"]) == c.target, (c.name, S, n, p)
        assert p["threads"] <= 704 and p["smem"] <= 226 * 1024 and p["grid"] <= 4 * S
    assert {c.target for c in CASES} == INSTANTIATIONS
    # boards, channels, input planes, sites, depths
    assert {c.W for c in CASES} == set(range(2, 9))
    assert {1, 16} <= {c.H for c in CASES}
    assert {4, 32} <= {c.C for c in CASES} and min(c.C for c in CASES) == 4 and max(c.C for c in CASES) == 32
    assert any(c.stem_cin > c.C for c in CASES if c.site == "representation")        # cap_channels > C: 11 planes, C = 8
    assert {1, 3} <= {c.cin for c in CASES if c.site == "representation"}
    assert set(SITES) == {c.site for c in CASES}
    assert {c.blocks for c in CASES if c.stem} == set(range(5))
    assert {c.blocks for c in CASES if not c.stem} == set(range(1, 6))
    for c in CASES:
        assert c.layers <= 10
        deeper, why = plan_fn(1, c.stem_cin, c.C, c.H, c.W, c.blocks + 1, c.stem, S)
        if c.layers + 2 > 10:
            assert deeper is None and "1 to 10 layers" in why, c.name
    assert {c.parts for c in CASES if c.site == "dynamics_pool"} >= {2, 3, 4}
    # a batch of 1, ragged last tiles, more boards than one round of resident tiles (for the first range of the search)
    ranges = {k: (first_range(n, BY_NAME[k].parts), p) for k, (n, p) in plans.items()}
    assert any(m == 1 for m, _ in ranges.values())
    assert any(m > p["boards"] > 1 and m % p["boards"] for m, p in ranges.values())
    rounds = [k for k, (m, p) in ranges.items() if -(-m // p["boards"]) > p["grid"]]
    assert {"p6_co4_6x6_rounds", "p8_co4_c32_16x8_rounds"} <= set(rounds), rounds
    # a CO = 4 case split into partitions: every range still takes CO = 4 ... except possibly the last, shorter one
    n, p = plans["p2_co4_16x2_parts3"]
    assert p["CO"] == 4 and first_range(n, 3) < n


@pytest.mark.parametrize("args,reason", REFUSED)
def test_planner_refuses_shapes_the_kernel_cannot_take(plan_fn, args, reason):
    p, why = plan_fn(*args, 132)
    assert p is None and reason in why, (p, why)


def test_planner_says_why_it_refuses_large_weights(plan_fn):
    """32 channels and 4 blocks after the dynamics stem: 9 layers of weights exceed shared memory (the network then runs
    one conv per launch); 2 blocks fit."""
    p, why = plan_fn(8, 33, 32, 3, 3, 4, True, 132)
    assert p is None and "shared memory" in why
    assert plan_fn(8, 33, 32, 3, 3, 2, True, 132)[0] is not None
