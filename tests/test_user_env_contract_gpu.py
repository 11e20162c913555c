"""The user-environment contract (csrc/user_env.cuh, mz_selfplay_begin_user) at its edges, against a plain Python
restatement of each test game (tests/user_env_contract_games.py): 1 to 256 actions (host_act_kernel<128> / <256>),
search inputs of O_in + A = 4096 and 4097 (the 32- and 256-thread observe / start kernels, the latter through stacked
observations), 1, 127, 129 and 300 slots (one to three wrapper CTAs, the last one partial), state of 0, 1, 17 and
4096 bytes kept across games, the MzEnvCtx values, irregular turn order, every kind of ending, partial row writes, and
fp32 / fp64 expressions whose fused and unfused roundings differ.

* Replay: every game a case finishes over three calls (temperatures 1, 0 and 0.5, new weights each call) is its
  rules' game bit for bit - observations, rewards, to_play, first_to_play, length - with every action legal under the
  rules' mask and no root visit on an illegal action.
* Parity: the same plug-in without DEVICE_SOURCE plays the host-stepped route ("device-host-env", the rules' vector
  game) and gives identical games.
* Priorities: the PER priorities of irregular-turn games equal reanalyse.initial_priorities.
* Bad rows: mz_env_check counts the rows the loop cannot play, and only those; the handle begins again without a new
  compile.
* SelfPlay: play_moves takes the "device-user-env" route and its counters agree with the replay.

Mutants, each applied alone to the library and run on an H100 (only runs that change values, or that a launch refuses,
were made):

| mutant | caught by |
|---|---|
| the NVRTC options without `-fmad=false` (user_env.cu) | `test_user_games_replay_through_the_python_rules`, every case: the fp32 / fp64 `a * b + c` observations |
| reset's `ctx.game_id` without `+ id_stride` (user_env.cuh) | `test_user_games_replay_through_the_python_rules`, every case |
| step's `ctx.move` one too large (user_env.cuh) | `test_user_games_replay_through_the_python_rules`, every case; `test_bad_rows_are_counted_and_the_handle_begins_again` |
| `mz_env_check` counting a done row without a legal action (user_env.cuh) | `test_user_games_replay_through_the_python_rules`, every case (the call fails); `test_bad_rows_are_counted_and_the_handle_begins_again` (the allowed terminal rows are counted too) |
| the wrapper grid `B / 128` in place of `(B + 127) / 128` (selfplay.cu) | `test_user_games_replay_through_the_python_rules[single]` and `[narrow32]`: B = 1 and 127 launch no CTA, which the launch refuses. Run only on those two cases: with B = 129 or 300 the slots past the last CTA would search rows no reset wrote |
| `initial_priority` signing the bootstrap and rewards by move parity in place of comparing `to_play` (selfplay.cu) | `test_priorities_under_irregular_turn_order`; the host-stepped parity tests pass, as both routes share the packing warp |
"""
import numpy
import pytest

from muzero_general_b200 import _lib
from muzero_general_b200.engine import SearchEngine, UserEnvSelfPlayLoop, parse_staged_games
from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
from user_env_contract_games import (BAD_ROWS, CASES, FIRST_GAME_ID, SEED, TEMPERATURES, Case, bad_rows_expected,
                                     finished_games, make_config, make_game, moves_per_call, replay, stride_of)

pytestmark = pytest.mark.gpu

MZ_EINVAL = -1        # include/mzb200.h


def _engine(case, **over):
    cfg = make_config(case, **over)
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=case.B, num_simulations=cfg.num_simulations, seed=SEED)
    eng.load_weights(synthetic_weights(spec, 0))
    return cfg, spec, eng


def _loop(eng, case, **kw):
    return UserEnvSelfPlayLoop(eng, case.source, case.state_bytes, case.shape, case.max_moves,
                               first_game_id=FIRST_GAME_ID, game_id_stride=stride_of(case),
                               stacked_observations=case.stack, **kw)


def _play(case, eng, spec, loop):
    """Three calls of moves_per_call moves, one temperature each, new weights before each -> {game id: record}."""
    games = {}
    for i, T in enumerate(TEMPERATURES):
        eng.load_weights(synthetic_weights(spec, i))
        loop.moves(moves_per_call(case), T)
        for g in parse_staged_games(*loop.drain()):
            assert g["game_id"] not in games
            games[g["game_id"]] = g
    return games


def _check_replay(case, games):
    """Every record equals its rules' game; returns the replay."""
    ref = replay(case, SEED, FIRST_GAME_ID, stride_of(case), games)
    for gid, g in games.items():
        r = ref[gid]
        assert g["slot"] == (gid - FIRST_GAME_ID) % stride_of(case), gid
        assert (g["length"], g["first_to_play"]) == (len(r["reward"]), r["first_to_play"]), gid
        assert g["obs"].tobytes() == r["obs"].astype(numpy.float32).tobytes(), (gid, "obs")
        assert g["reward"].tobytes() == r["reward"].tobytes(), (gid, "reward")
        assert g["to_play"].tolist() == r["to_play"].tolist(), (gid, "to_play")
        visits = g["visits"]
        assert (visits[r["legal"] == 0] == 0).all(), (gid, "visits on illegal actions")
        assert (visits.sum(1) > 0).all(), gid
    return ref


@pytest.mark.parametrize("name", sorted(CASES))
def test_user_games_replay_through_the_python_rules(name):
    """Every game the case finishes is the Python rules' game bit for bit, and the loop finishes exactly the games the
    rules' lengths predict (no game lost, none extra)."""
    case = CASES[name]
    cfg, spec, eng = _engine(case)
    loop = _loop(eng, case)
    games = _play(case, eng, spec, loop)
    assert loop.compiles == 1
    M = len(TEMPERATURES) * moves_per_call(case)
    assert sorted(games) == sorted(finished_games(case, M))
    ref = _check_replay(case, games)
    # the whole batch moved every move: finished moves plus the moves of the games in flight
    assert loop.stats.env_steps == sum(g["length"] for g in games.values()) + int(loop.peek()["move_index"].sum())
    if case.P > 1:
        tp = [numpy.concatenate([[r["first_to_play"]], r["to_play"]]) for r in ref.values()]
        assert any(t[0] == 1 for t in tp) and any((t[1:] == t[:-1]).any() for t in tp)
    eng.close()


# the host-stepped route steps the same rules on the host: one case above 128 actions, one above 4096 input floats
@pytest.mark.parametrize("name", ["wide129", "row4097"])
def test_user_games_equal_the_host_stepped_route(name):
    """SelfPlay with DEVICE_SOURCE ("device-user-env") and with the same rules as a host vector game
    ("device-host-env"), same seed, weights, first_game_id and stride: the same games finish, and they are identical -
    id, first_to_play, root values, visit counts, actions, rewards, to_play, PER priorities, observations."""
    from muzero_general_b200 import self_play as sp
    case = CASES[name]
    got, steps = {}, {}
    for user in (True, False):
        cfg = make_config(case, host_env_device_loop=not user)
        spec = netspec_from_config(cfg)
        Game = make_game(case, FIRST_GAME_ID, stride_of(case), user=user)
        w = sp.SelfPlay({"weights": synthetic_weights(spec, 0)}, Game, cfg, seed=SEED, first_game_id=FIRST_GAME_ID,
                        game_id_stride=stride_of(case))
        assert w.loop_path == ("device-user-env" if user else "device-host-env")
        games = {}
        for i, T in enumerate(TEMPERATURES):
            w.model.set_weights(synthetic_weights(spec, i))
            out = w.play_moves(moves_per_call(case), T)
            games.update({g["game_id"]: g for buf, index in out._chunks for g in parse_staged_games(buf, index)})
        got[user], steps[user] = games, w.env_steps
        w.close()
    usr, hst = got[True], got[False]
    assert set(usr) == set(hst) and steps[True] == steps[False] and len(usr) >= case.B
    for gid in usr:
        a, b = usr[gid], hst[gid]
        assert (a["length"], a["first_to_play"]) == (b["length"], b["first_to_play"]), gid
        assert a["root_value"].tobytes() == b["root_value"].tobytes(), gid
        for key in ("visits", "action", "reward", "to_play", "priority", "obs"):
            assert a[key].tobytes() == b[key].tobytes(), (gid, key)
    assert any(g["priority"].any() for g in usr.values())


PRIORITY_SWEEP = [(1.0, 1, 1.0), (1.0, 3, 0.997), (1.0, "long", 1.0), (0.5, 1, 0.997), (0.5, 3, 1.0),
                  (0.5, "long", 0.997)]


def _parity_signed(gh, cfg):
    """initial_priorities with to_play taken from move parity (first_to_play, then alternating): what a kernel that
    signs rewards and the bootstrap by parity would compute."""
    from muzero_general_b200 import reanalyse as ra
    first = gh.to_play_history[0]
    alt = type("Alt", (), dict(root_values=gh.root_values, reward_history=gh.reward_history,
                               reanalysed_predicted_root_values=None,
                               to_play_history=[(first + i) % 2 for i in range(len(gh.to_play_history))]))()
    return ra.initial_priorities(alt, cfg)[0]


def test_priorities_under_irregular_turn_order():
    """turns33 (player 1 opens about half the games, 30 % of the moves let the same player move again): the packing
    warp's PER priorities equal reanalyse.initial_priorities - bit for bit at alpha = 1, within one float32 ulp at
    alpha = 0.5 (an exact sqrt on the device, numpy's ** 0.5 on the host) - for td_steps 1, 3 and longer than any game,
    discount 1 and 0.997.  Signing by move parity would give other priorities on these games."""
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200.self_play import PackedGameHistory
    case = CASES["turns33"]
    cfg, spec, eng = _engine(case)
    for alpha, td, discount in PRIORITY_SWEEP:
        td_steps = case.max_moves + 5 if td == "long" else td
        cfg.td_steps, cfg.discount, cfg.PER_alpha = td_steps, discount, alpha
        loop = _loop(eng, case, td_steps=td_steps, per_alpha=alpha, discount=discount)
        assert loop.with_priorities
        records = _play(case, eng, spec, loop)
        _check_replay(case, records)
        games = [PackedGameHistory(g, case.shape, numpy.float32, float, True) for g in records.values()]
        parity_differs = 0
        for gh in games:
            want, _ = ra.initial_priorities(gh, cfg)
            assert gh.priorities.dtype == numpy.float32 and gh.priorities.shape == want.shape
            if alpha == 1.0:
                assert numpy.array_equal(gh.priorities, want), (gh.game_id, alpha, td, discount)
            else:
                numpy.testing.assert_allclose(gh.priorities, want, rtol=2e-7, atol=0)
            parity_differs += not numpy.allclose(_parity_signed(gh, cfg), want, rtol=1e-6, atol=0)
        assert parity_differs > len(games) // 10, (parity_differs, len(games))
    assert loop.compiles == 1
    eng.close()


def test_bad_rows_are_counted_and_the_handle_begins_again():
    """BAD_ROWS (one source: the game id's thousands pick which rows misbehave): a reset with an empty mask fails
    mz_selfplay_begin_user, a step that leaves games in play without a legal action or writes to_play = num_players
    fails the call, each with the count the reference predicts - terminal rows without a legal action are not counted.
    Every time the same handle begins again, plays, and compiles nothing new."""
    case = Case("bad_rows", 5, (1, 1, 4), 0, 40, 0, 2, 6)
    cfg, spec, eng = _engine(case)

    def begin(mode):
        return UserEnvSelfPlayLoop(eng, BAD_ROWS, 0, case.shape, case.max_moves, first_game_id=1000 * mode)

    for mode in (3, 1, 2):
        k = bad_rows_expected(mode, case.B, case.A, case.P)
        assert k > 0
        with pytest.raises(_lib.MzError) as e:
            loop = begin(mode)
            loop.moves(2, 1.0)
        assert e.value.code == MZ_EINVAL
        what = "mz_env_reset left %d slots" if mode == 3 else "wrote %d rows"
        assert what % k in str(e.value), (mode, k, str(e.value))
        loop = begin(0)
        st = loop.moves(case.max_moves, 1.0)
        assert st.games_finished == case.B and st.env_steps == case.B * case.max_moves
        assert loop.compiles == 1
    eng.close()


@pytest.mark.parametrize("name", ["wide256", "row4097"])
def test_selfplay_api_on_user_games(name):
    """SelfPlay.play_moves on a wide case and a stacked case: the "device-user-env" route, PackedGames out, the games
    the rules' replay expects, and played_games / env_steps equal to what those games and the games in flight moved."""
    from muzero_general_b200 import self_play as sp
    case = CASES[name]
    cfg = make_config(case)
    spec = netspec_from_config(cfg)
    Game = make_game(case, FIRST_GAME_ID, stride_of(case))
    w = sp.SelfPlay({"weights": synthetic_weights(spec, 0)}, Game, cfg, seed=SEED, first_game_id=FIRST_GAME_ID,
                    game_id_stride=stride_of(case))
    assert w.loop_path == "device-user-env"
    games = {}
    for i, T in enumerate(TEMPERATURES):
        w.model.set_weights(synthetic_weights(spec, i))
        out = w.play_moves(moves_per_call(case), T)
        assert isinstance(out, sp.PackedGames)
        games.update({g["game_id"]: g for buf, index in out._chunks for g in parse_staged_games(buf, index)})
    assert sorted(games) == sorted(finished_games(case, len(TEMPERATURES) * moves_per_call(case)))
    _check_replay(case, games)
    in_flight = int(w._device_loop.loop.peek()["move_index"].sum())
    assert w.played_games == len(games)
    assert w.played_steps == sum(g["length"] for g in games.values())
    assert w.env_steps == w.played_steps + in_flight
    w.close()
