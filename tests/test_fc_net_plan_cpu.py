"""Launch plans of the fully-connected network routes (fc_infer_plan in csrc/fc_infer.cu and fc_debug_plan in
csrc/fc_search.cu, through mz_debug_fc_net_plan): the case table of tests/fccases.py reaches every fc_inference_kernel<G>,
every path of the search's network call at every lane-group width it runs at, and the near-misses of the fixed shape; the
nets whose shared memory cannot hold the blob and one warp's groups are refused.  Host only."""
import pytest

from fccases import (BY_NAME, CASES, INFER_ROUTES, SEARCH_ROUTES, SMEM_CAP, SMS, blob_floats, edge_case, groups_per_warp,
                     infer_smem, maxw, one_pass, runs)


@pytest.fixture(scope="module")
def plan_fn():
    from muzero_general_b200.engine import debug_fc_net_plan
    return debug_fc_net_plan


def want_threads(case, G):
    return max(t for t in (32, 64, 96, 128) if infer_smem(case, G, t // G) <= SMEM_CAP)


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("name,G,route", runs())
def test_case_plan(plan_fn, name, G, route, sms):
    case = BY_NAME[name]
    for n in sorted({1, groups_per_warp(G) - 1 or 1, groups_per_warp(G) + 1, one_pass(G, sms) - 1, one_pass(G, sms) + 1}):
        p, why = plan_fn(case.spec(), G, route, n, sm_count=sms)
        assert p is not None, (name, G, route, why)
        assert p["G"] == G
        if route in INFER_ROUTES:
            t = want_threads(case, G)
            assert p == {"path": "infer", "G": G, "threads": t, "grid": min(-(-n // (t // G)), 8 * sms),
                         "smem": infer_smem(case, G, t // G)}, (name, n)
        else:
            assert p["path"] == case.search_path(G) and p["threads"] == 32, (name, G, p)
            assert p["grid"] == min(-(-n // (32 // G)), 8 * sms)


def test_table_reaches_every_instantiation_and_path(plan_fn):
    infer, search = set(), set()
    for name, G, route in runs():
        p, _ = plan_fn(BY_NAME[name].spec(), G, route, 100)
        (infer if route in INFER_ROUTES else search).add((G, p["path"]) if route in SEARCH_ROUTES else (G, p["threads"] == 128))
    assert {G for G, _ in infer} == {4, 8, 16, 32}
    assert any(not full for _, full in infer), "no case shrinks fc_inference_kernel's CTA"
    assert {(16, "fixed"), (32, "fixed")} <= search
    for G in (4, 8, 16, 32):
        assert {(G, "fused"), (G, "split")} <= search, G
    # the fixed path with one and two players is the same network call: P only changes the search's backup
    shapes = {(c.E, c.A, c.S, c.obs) for c in CASES}
    assert {e for e, _, _, _ in shapes} >= {1, 3, 5, 8, 32, 36, 64}
    assert {s for _, _, s, _ in shapes} >= {0, 4, 10, 20, 300}
    assert {a for c in CASES for a in [c.A] if c.search_groups()} >= {1, 2, 3, 4, 7, 8, 17, 32}
    assert max(c.A for c in CASES) == 256
    hidden = {tuple(h) for c in CASES for h in (c.rep, c.dyn, c.rew, c.val, c.pol)}
    assert hidden >= {(), (3,), (16,), (33,), (3, 9), (128, 128)}
    for k in range(5):      # every hidden list in every MLP
        assert {(c.rep, c.dyn, c.rew, c.val, c.pol)[k] for c in CASES} >= {(), (3,), (16,), (33,), (3, 9), (128, 128)}, k
    assert any(c.obs > max(c.E, c.F, c.A, *c.rep, *c.dyn, *c.rew, *c.val, *c.pol) for c in CASES), "obs never sets maxw"
    unequal = [c for c in CASES if len(c.rew) == len(c.val) == len(c.pol) and len({c.rew, c.val, c.pol}) > 1]
    assert unequal, "no heads of equal depth and unequal widths"


def test_near_misses_take_the_generic_path(plan_fn):
    assert plan_fn(BY_NAME["cartpole"].spec(), 16, "search_sim", 1)[0]["path"] == "fixed"
    assert plan_fn(BY_NAME["cartpole_rep_none"].spec(), 32, "search_sim", 1)[0]["path"] == "fixed"
    for name in ("cartpole_rew_16_16", "cartpole_a3", "cartpole_s20", "cartpole_e12", "cartpole_h20"):
        for G in (16, 32):
            assert plan_fn(BY_NAME[name].spec(), G, "search_sim", 1)[0]["path"] != "fixed", (name, G)


def test_blob_and_width_restatement_match_the_loader(plan_fn):
    """fccases.blob_floats / maxw restate abi.cu's packing: the planned shared memory agrees byte for byte."""
    for c in CASES:
        p, _ = plan_fn(c.spec(), c.groups[-1], "infer_initial", 1)
        assert p["smem"] == infer_smem(c, c.groups[-1], p["threads"] // c.groups[-1]), c.name
        assert maxw(c) % 4 == 0 and blob_floats(c) > 0


def test_search_refuses_more_actions_than_lanes(plan_fn):
    p, why = plan_fn(BY_NAME["e5_a7_split"].spec(), 4, "search_sim", 1)
    assert p is None and "lane" in why


def test_shared_memory_edge_is_planned_and_refused(plan_fn):
    at = edge_case(0)
    beyond = edge_case(16)          # one 4-float granule of the blob beyond the limit
    p, why = plan_fn(at.spec(), 32, "infer_initial", 1000)
    assert p is not None and p["smem"] == SMEM_CAP and p["threads"] == 32, why
    p, why = plan_fn(beyond.spec(), 32, "infer_initial", 1000)
    assert p is None and str(SMEM_CAP) in why and str(SMEM_CAP + 16) in why
    # G = 4 with support 300: 128 threads would need 32 groups of 2420 floats - the CTA shrinks to 64 threads
    p, _ = plan_fn(BY_NAME["g4_s300_flat"].spec(), 4, "infer_recurrent", 1000)
    assert p["threads"] == 64 and 32 * (4 * 604 + 4) * 4 > SMEM_CAP
