"""The user-environment contract games (tests/user_env_contract_games.py) on the host alone: every source compiles for
sm_90a without spills, the cases reach every launch, layout and rule edge by selfplay.cu's formulas, the fp32 / fp64
contraction cases have draws where the fused and unfused roundings differ, and the Python rules replay their own games
(the bookkeeping the GPU tests rely on)."""
import numpy
import pytest

from user_env_contract_games import (BAD_ROWS, CASES, TEMPERATURES, ContractVector, bad_rows_expected,
                                     contraction_differs, coverage, edges, finished_games, fp32_operands,
                                     fp64_operands, fused32, fused64, moves_per_call, replay, stride_of)


@pytest.mark.parametrize("name", sorted(CASES) + ["bad_rows"])
def test_contract_sources_compile_without_spills(name):
    from muzero_general_b200.engine import debug_user_env_compile
    rc, log, info = debug_user_env_compile(BAD_ROWS if name == "bad_rows" else CASES[name].source)
    assert rc == 0, log
    for kernel in ("reset", "step"):
        regs, frame, spill_stores, spill_loads = info[kernel]
        assert 0 < regs <= 255 and frame >= 0, (kernel, info)
        assert spill_stores == 0 and spill_loads == 0, (kernel, info)


def test_the_cases_reach_every_edge():
    from muzero_general_b200 import _lib
    cases = list(CASES.values())
    e = {c.name: edges(c) for c in cases}
    A = {c.A for c in cases}
    assert {1, 32, 33, 128, 129, 225, _lib.MZ_MAX_ACTIONS} <= A and max(A) == _lib.MZ_MAX_ACTIONS == 256
    # host_act_kernel<128> at its last width and <256> at its first
    assert {(c.A, e[c.name]["act_kernel"]) for c in cases} >= {(128, 128), (129, 256), (256, 256)}
    # observe / start kernels: 32 threads at O_in + A = 4096, 256 at 4097 - reached through stacked observations
    rows = {c.O_in + c.A: (e[c.name]["slot_threads"], c.stack) for c in cases}
    assert rows[4096][0] == 32 and rows[4097][0] == 256 and rows[4097][1] >= 1
    # the wrappers' grid: one partial CTA, two and three CTAs with a partial last one
    assert {c.B for c in cases} >= {1, 127, 129, 300}
    assert {(e[c.name]["wrapper_ctas"], e[c.name]["partial_cta"]) for c in cases} >= {(1, True), (2, True), (3, True)}
    # state: none, one byte, 17 bytes on a 32-byte stride, the limit
    strides = {c.state_bytes: e[c.name]["state_stride"] for c in cases}
    assert strides[0] == 0 and strides[1] == 16 and strides[17] == 32
    assert strides[_lib.MZ_USER_ENV_MAX_STATE_BYTES] == 4096 == _lib.MZ_USER_ENV_MAX_STATE_BYTES
    assert any(c.P == 2 for c in cases) and any(c.P == 1 for c in cases)
    # the rule edges, over the games the GPU tests finish
    total = {}
    for c in cases:
        cov = coverage(c, finished_games(c, len(TEMPERATURES) * moves_per_call(c)))
        for k, v in cov.items():
            total[k] = total.get(k, 0) + v
        if c.P > 1:
            assert cov["opens_1"] > 0 and cov["same_player"] > 0, (c.name, cov)
    assert all(total[k] > 0 for k in total), total


@pytest.mark.parametrize("name", sorted(CASES))
def test_contraction_inputs_round_differently(name):
    """Among the draws of the games the GPU tests finish, some fp32 and some fp64 a * b + c round differently fused and
    unfused, so a source compiled with contraction would write other observations."""
    c = CASES[name]
    gids = finished_games(c, len(TEMPERATURES) * moves_per_call(c))
    assert gids
    assert contraction_differs(11, gids, c.max_moves) == (True, True)


def test_fused_references_round_once():
    """fused32 / fused64 against float64 arithmetic where the exact value is known: operands in [1, 2) make the fp32
    product and sum exact in float64, so fused32 is one rounding; fused64 keeps the product's low bits."""
    a, b, c = fp32_operands(11, 7, 1)
    assert 1 <= a < 2 and 1 <= b < 2 and 1 <= c < 2 and a.dtype == numpy.float32
    exact = numpy.float64(a) * numpy.float64(b) + numpy.float64(c)
    assert exact - numpy.float64(c) == numpy.float64(a) * numpy.float64(b)
    assert fused32(a, b, c) == numpy.float32(exact)
    x, y, z = fp64_operands(11, 7, 1)
    assert abs(fused64(x, y, z) - (x * y + z)) <= 2 * numpy.spacing(x * y + z)


def test_bad_row_counts():
    """The reference counts of BAD_ROWS: a done row without a legal action is not counted."""
    assert bad_rows_expected(0, 40, 5, 2) == 0
    assert bad_rows_expected(1, 40, 5, 2) == 14            # slots 0, 3, .., 39; slots 1, 4, .. end their game
    assert bad_rows_expected(2, 40, 5, 2) == 10
    assert bad_rows_expected(3, 40, 5, 2) == 8


@pytest.mark.parametrize("name", ["single", "turns33", "wide225"])
def test_the_rules_replay_their_own_games(name):
    """The host vector plays random legal moves with the loop's slot schedule; replay() rebuilds every finished game
    from its id, actions and length alone, and its ending list is finished_games'."""
    c = CASES[name]
    first, stride, M = 7, stride_of(c), len(TEMPERATURES) * moves_per_call(c)
    env = ContractVector(c, c.B, 11, first, stride)
    obs = env.reset()
    rs = numpy.random.RandomState(0)
    live = {g: dict(obs=[obs[g].ravel().copy()], action=[], reward=[], to_play=[], first=int(env.to_play()[g]))
            for g in range(c.B)}
    games = {}
    for _ in range(M):
        legal = env.legal_mask()
        actions = numpy.array([rs.choice(numpy.nonzero(legal[g])[0]) for g in range(c.B)])
        obs, reward, done = env.step(actions)
        tp = env.to_play()
        ended = numpy.zeros(c.B, bool)
        for g in range(c.B):
            r = live[g]
            r["action"].append(actions[g]); r["reward"].append(reward[g]); r["to_play"].append(tp[g])
            r["obs"].append(obs[g].ravel().copy())
            if done[g] or len(r["action"]) == c.max_moves:
                games[env.gid[g]] = dict(length=len(r["action"]), action=numpy.array(r["action"]), rec=r)
                ended[g] = True
        if ended.any():
            obs = env.reset(ended)
            for g in numpy.nonzero(ended)[0]:
                live[g] = dict(obs=[obs[g].ravel().copy()], action=[], reward=[], to_play=[], first=int(env.to_play()[g]))
    assert sorted(games) == sorted(finished_games(c, M))
    ref = replay(c, 11, first, stride, games)
    for gid, g in games.items():
        r = ref[gid]
        assert numpy.array_equal(r["obs"], numpy.stack(g["rec"]["obs"])), gid
        assert r["reward"].tobytes() == numpy.array(g["rec"]["reward"], numpy.float32).tobytes()
        assert r["to_play"].tolist() == g["rec"]["to_play"] and r["first_to_play"] == g["rec"]["first"]
