"""Stacked observations (config.stacked_observations > 0) in the device self-play loop (csrc/selfplay.cu::stack_fill):
the input every search sees against GameHistory.get_stacked_observations (oracle.mcts.stacked_observation, pinned to the
reference by tests/golden/kat.json), the loop against host compositions of search + sampling (+ opponent), the
SelfPlay API on stacked configs, the refusals of mz_selfplay_begin, and the stacked networks against the fp64 oracle.
Everything goes through the C ABI."""
import ctypes as C

import numpy
import pytest

from conftest import weights_for
from muzero_general_b200 import _lib
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from oracle import mcts as om
from oracle import philox

pytestmark = pytest.mark.gpu

MZ_EINVAL = -1                                  # include/mzb200.h
SMALL_GOMOKU = dict(blocks=1, channels=16)      # loop tests: the stack is under test, not the 128-channel towers
ENVS = ["cartpole", "tictactoe", "connect4", "gomoku", "twentyone", "simple_grid"]


def _cfg(name, s, **over):
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.stacked_observations = s
    for k, v in ({**SMALL_GOMOKU, **over} if name == "gomoku" else over).items():
        setattr(cfg, k, v)
    return mod, cfg


def _loop(name, s, B, N, seed=0, first_game_id=0, opponent="self", muzero_player=0, **over):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    mod, cfg = _cfg(name, s, **over)
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    eng.load_weights(weights_for(name, spec))
    loop = DeviceSelfPlayLoop(eng, name, cfg.max_moves, temperature_threshold=cfg.temperature_threshold,
                              reward_scale=getattr(getattr(mod.Game, "VECTOR", None), "REWARD_SCALE", 1),
                              first_game_id=first_game_id, opponent=opponent, muzero_player=muzero_player,
                              stacked_observations=s)
    return mod, cfg, spec, eng, loop


def _drain(loop):
    from muzero_general_b200.engine import parse_staged_games
    return parse_staged_games(*loop.drain())


def _peek(loop, peeked):
    """Peeks the loop and keys every slot's search input by (game id, move index)."""
    pk = loop.peek()
    for g in range(len(pk["game_id"])):
        peeked[(int(pk["game_id"][g]), int(pk["move_index"][g]))] = pk["obs"][g].copy()
    return pk


def _reference_stack(rec, t, s, A, shape):
    """get_stacked_observations(t, s, A) of the drained game's history: the float64 observations and action_history
    (dummy first entry 0) the reference keeps, made float32 like torch.tensor(obs).float()."""
    obs = [numpy.asarray(o, numpy.float64).reshape(shape) for o in rec["obs"]]
    actions = [0] + [int(a) for a in rec["action"]]
    return om.stacked_observation(obs, actions, t, s, A).astype(numpy.float32).ravel()


def _check_stacks(peeked, recs, s, A, shape, searched=None):
    """Every peeked input of the drained games (at every move, or where searched(rec, t)), bit for bit against the
    reference's stack.  Returns (inputs checked, action ids that appeared in a checked stack)."""
    n, seen = 0, set()
    for rec in recs:
        gid = rec["game_id"]
        for t in range(rec["length"]):
            if searched is not None and not searched(rec, t):
                continue
            want = _reference_stack(rec, t, s, A, shape)
            got = peeked[(gid, t)]
            assert got.shape == want.shape and got.tobytes() == want.tobytes(), (gid, t, numpy.nonzero(got != want)[0][:8])
            seen |= {int(rec["action"][p]) for p in range(max(0, t - s), t)}
            n += 1
    return n, seen


# ------------------------------------------------------------------------------------------ the stacked input
MAX_MOVES = dict(cartpole=30, connect4=16, gomoku=12)
STACK_CASES = [(name, s) for name in ENVS for s in (1, 3)] + [("simple_grid", 8), ("tictactoe", 12)]


@pytest.mark.parametrize("name,s", STACK_CASES)
def test_search_input_is_the_reference_stack(name, s, monkeypatch):
    """Every slot plays until it has finished at least one game and restarted.  The first half of the slots play host-
    chosen actions that run through every action id in their first moves; the other half sample on the device.  Every
    input a search saw, keyed by (game id, move), equals the reference's stack of the drained game bit for bit, with
    stacks deeper than the game so far (zero planes) and, for Simple Grid s = 8 and TicTacToe s = 12, deeper than any
    game.  Every action id's plane value a / A appears in a checked stack (Twenty-One: only 0, since a stand ends the
    game)."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    B = 64 if name == "gomoku" else 32
    over = {"max_moves": MAX_MOVES[name]} if name in MAX_MOVES else {}
    mod, cfg, spec, eng, loop = _loop(name, s, B, 2, seed=11, **over)
    A, shape = spec.action_space, tuple(cfg.observation_shape)
    assert eng.obs_elems == (shape[0] * (s + 1) + s) * shape[1] * shape[2]
    half = B // 2
    peeked, recs = {}, []
    for _ in range(2 * cfg.max_moves + 2):
        pk = _peek(loop, peeked)
        forced = numpy.full(B, -1, numpy.int32)
        for g in range(half):
            legal = numpy.nonzero(pk["legal_mask"][g])[0]
            target = (g + int(pk["move_index"][g]) * half) % A
            forced[g] = legal[numpy.searchsorted(legal, target) % len(legal)]
        loop.moves(1, 1.0, forced_action=forced)
        recs += _drain(loop)
    eng.close()
    assert {r["slot"] for r in recs} == set(range(B)) and len(recs) >= 2 * B
    n, seen = _check_stacks(peeked, recs, s, A, shape)
    assert n == sum(r["length"] for r in recs)
    assert seen == (set(range(A)) - {1} if name == "twentyone" else set(range(A)))


# ------------------------------------------------------------------------------------------ the loop
# name, s, B, N, moves, config overrides
COMPOSITION_CASES = [("cartpole", 2, 32, 12, 14, dict(max_moves=10)), ("tictactoe", 2, 32, 8, 12, {}),
                     ("connect4", 2, 24, 8, 16, dict(max_moves=12)), ("gomoku", 2, 16, 6, 12, dict(max_moves=10)),
                     ("twentyone", 2, 32, 8, 8, {}), ("simple_grid", 2, 32, 8, 10, {}),
                     ("connect4", 8, 24, 8, 16, dict(max_moves=12))]


@pytest.mark.parametrize("name,s,B,N,moves,over", COMPOSITION_CASES)
def test_device_loop_equals_host_composition_with_injected_draws(name, s, B, N, moves, over, monkeypatch):
    """One move at a time with the host's draws injected (root noise, action uniforms): the visit counts, root values
    and actions the device records equal [mz_search on the peeked stacked input] + [select_action with numpy's choice
    rule], and the peeked inputs are the reference's stacks."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    mod, cfg, spec, eng, loop = _loop(name, s, B, N, seed=5, **over)
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=5)
    ref.load_weights(weights_for(name, spec))
    A = spec.action_space
    rs = numpy.random.RandomState(17)
    expected, delivered, peeked = {}, [], {}
    for _ in range(moves):
        pk = _peek(loop, peeked)
        legal = pk["legal_mask"]
        gam = rs.standard_gamma(cfg.root_dirichlet_alpha, size=(B, A)) * (legal > 0)
        noise = gam / gam.sum(1, keepdims=True)
        u = rs.random_sample(B)
        out = ref.search(obs=pk["obs"], legal_mask=legal, to_play=pk["to_play"], add_exploration_noise=True, noise=noise,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        want = numpy.array([om.select_action([int(a) for a in numpy.nonzero(legal[g])[0]],
                                             out.visit_counts[g][legal[g] > 0], 1.0, om.InjectedDraws(uniform=u[g]))
                            for g in range(B)])
        for g in range(B):
            expected.setdefault(int(pk["game_id"][g]), []).append((out.visit_counts[g].copy(), out.root_value[g], int(want[g])))
        loop.moves(1, 1.0, uniform=u, noise=noise)
        delivered += _drain(loop)
    eng.close(); ref.close()
    assert len(delivered) >= B // 2
    for rec in delivered:
        exp = expected[rec["game_id"]]
        assert rec["length"] == len(exp)
        for t, (visits, root_value, action) in enumerate(exp):
            assert rec["visits"][t].tolist() == visits.tolist() and rec["root_value"][t] == root_value, (rec["game_id"], t)
            assert rec["action"][t] == action, (rec["game_id"], t)
    n, _ = _check_stacks(peeked, delivered, s, A, tuple(cfg.observation_shape))
    assert n == sum(r["length"] for r in delivered)


TEST_MODE_CASES = [(name, opponent, mp) for name in ("tictactoe", "connect4") for opponent in ("expert", "random")
                   for mp in (0, 1)]


@pytest.mark.parametrize("name,opponent,muzero_player", TEST_MODE_CASES)
def test_test_mode_games_equal_host_composition(name, opponent, muzero_player, monkeypatch):
    """Test-mode games with s = 2: MuZero's moves equal [search of the peeked stacked input] +
    [uniform53(seed, game, move, 0, TAG_ACTION)] + [numpy's choice rule], the opponent's moves replay on the host
    (tests/test_eval_gpu.py::_check_record), and the input at each of MuZero's turns is the reference's stack of the
    whole history, the opponent's moves (and its opening move when muzero_player = 1) included."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    from test_eval_gpu import _check_record
    s, B, N, T, seed = 2, 32, 6, 1.0, 0x5EED_0000_0051 + muzero_player
    over = dict(max_moves=12 - muzero_player) if name == "connect4" else {}
    mod, cfg, spec, eng, loop = _loop(name, s, B, N, seed=seed, opponent=opponent, muzero_player=muzero_player, **over)
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    ref.load_weights(weights_for(name, spec))
    expected, recs, peeked = {}, {}, {}
    for _ in range(16 if name == "connect4" else 12):
        pk = _peek(loop, peeked)
        assert (pk["to_play"] == muzero_player).all()
        out = ref.search(obs=pk["obs"], legal_mask=pk["legal_mask"], to_play=pk["to_play"], add_exploration_noise=True,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        for g in range(B):
            gid, mv = int(pk["game_id"][g]), int(pk["move_index"][g])
            u = philox.uniform53(seed, gid, mv, 0, philox.TAG_ACTION)
            idx = [int(a) for a in numpy.nonzero(pk["legal_mask"][g])[0]]
            expected[(gid, mv)] = (out.visit_counts[g].copy(), out.root_value[g],
                                   om.select_action(idx, out.visit_counts[g][idx], T, om.InjectedDraws(uniform=float(u))))
        loop.moves(1, T)
        for rec in _drain(loop):
            recs[rec["game_id"]] = rec
    eng.close(); ref.close()
    assert len(recs) >= B
    for rec in recs.values():
        _check_record(mod, cfg, rec, expected, seed, opponent, muzero_player)
    # MuZero moves at even t when it opens, at odd t when the opponent does
    mine = lambda rec, t: t % 2 == muzero_player
    n, _ = _check_stacks(peeked, recs.values(), s, spec.action_space, tuple(cfg.observation_shape), mine)
    assert n == sum(int((~numpy.isnan(r["root_value"])).sum()) for r in recs.values())


@pytest.mark.parametrize("name,max_moves", [("tictactoe", 9), ("cartpole", 20)])
def test_histories_are_batch_and_rank_invariant(name, max_moves):
    """With s = 2, global games 16..31 have the same histories as slots 16..31 of a 32-game batch and as slots 0..15 of
    a 16-game batch whose first id is 16."""
    def games(B, first):
        mod, cfg, spec, eng, loop = _loop(name, 2, B, 6, seed=3, first_game_id=first, max_moves=max_moves)
        out = {}
        for _ in range(max_moves + 2):
            loop.moves(1, 1.0)
            for rec in _drain(loop):
                out[rec["game_id"]] = rec
        eng.close()
        return out
    a, b = games(32, 0), games(16, 16)
    common = [g for g in range(16, 32) if g in a and g in b]
    assert len(common) == 16
    for g in common:
        for key in ("action", "visits", "root_value", "reward", "obs"):
            assert numpy.array_equal(a[g][key], b[g][key]), (g, key)


# ------------------------------------------------------------------------------------------ the SelfPlay API
@pytest.mark.parametrize("name", ENVS)
def test_selfplay_api_on_stacked_configs(name, monkeypatch):
    """SelfPlay with rng_mode="philox" and stacked_observations = 2 takes the device loop.  Its histories keep the raw
    observations in observation_shape, get_stacked_observations builds the network's input from them, the device PER
    priorities equal reanalyse.initial_priorities, Reanalyse's batched values run on them, and play_test_games
    works."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200 import self_play as sp
    over = {"max_moves": 14} if name in ("connect4", "gomoku") else {"max_moves": 30} if name == "cartpole" else {}
    mod, cfg = _cfg(name, 2, **over)
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations = 24, "philox", 6
    spec = netspec_from_config(cfg)
    w = weights_for(name, spec)
    worker = sp.SelfPlay({"weights": w}, mod.Game, cfg, seed=0)
    assert worker.loop_path == "device"
    games = []
    for _ in range(8):
        games += list(worker.play_moves(4, 1.0))
    assert games and worker.env_steps == 24 * 32 and worker.played_games == len(games)
    A = spec.action_space
    for gh in games[:16]:
        T = len(gh.action_history) - 1
        assert len(gh.observation_history) == T + 1 and len(gh.root_values) == T
        assert all(o.shape == tuple(cfg.observation_shape) for o in gh.observation_history)
        stacked = gh.get_stacked_observations(-1, 2, A)
        assert numpy.asarray(stacked).size == spec.obs_elems
        if gh.priorities is not None:
            want, _ = ra.initial_priorities(gh, cfg)
            numpy.testing.assert_allclose(gh.priorities, want, rtol=2e-7, atol=0)
    re = ra.Reanalyse({"weights": w}, cfg, max_positions=512)
    values = re.fresh_root_values(games[:8])
    re.close()
    for gh, v in zip(games[:8], values):
        assert numpy.atleast_1d(v).shape == (len(gh.root_values),) and numpy.isfinite(v).all()
    worker.reset_stream()
    tests, summary = worker.play_test_games(10)
    assert len(tests) == 10 == summary["games"]
    assert all(o.shape == tuple(cfg.observation_shape) for gh in tests for o in gh.observation_history)
    worker.close()


def test_begin_refuses_a_mismatched_stack():
    """MZ_EINVAL with a message naming the environment, s and the obs_c it needs: a handle built for s = 2 begun with
    s = 1, a negative s, and s = 2 on a handle built for s = 0."""
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine

    def begin(eng, s):
        d = _lib.MzSelfPlayDesc()
        d.env, d.max_moves, d.reward_scale, d.stacked_observations = _lib.MZ_ENV_TICTACTOE, 9, 20, s
        return eng.lib.mz_selfplay_begin(eng._h, C.byref(d)), eng.lib.mz_last_error(eng._h).decode()

    eng2 = SearchEngine(_cfg("tictactoe", 2)[1], max_games=4, num_simulations=2)
    rc, msg = begin(eng2, 1)
    assert rc == MZ_EINVAL and "TicTacToe" in msg and "stacked_observations = 1" in msg and "obs_c = 7" in msg, msg
    rc, msg = begin(eng2, -1)
    assert rc == MZ_EINVAL and "stacked_observations must be >= 0" in msg, msg
    assert begin(eng2, 2)[0] == 0
    eng2.close()
    eng0 = SearchEngine(_cfg("tictactoe", 0)[1], max_games=4, num_simulations=2)
    rc, msg = begin(eng0, 2)
    assert rc == MZ_EINVAL and "stacked_observations = 2" in msg and "obs_c = 11" in msg and "27 input values" in msg, msg
    with pytest.raises(_lib.MzError, match="obs_c = 11") as err:
        DeviceSelfPlayLoop(eng0, "tictactoe", 9, stacked_observations=2)
    assert err.value.code == MZ_EINVAL
    eng0.close()


# ------------------------------------------------------------------------------------------ networks on stacked inputs
@pytest.mark.parametrize("name", ENVS)
def test_stacked_networks_match_the_fp64_oracle(name, monkeypatch):
    """Each environment's net built for s = 2 (CartPole's and Simple Grid's FC nets, TicTacToe's small net, Connect4's
    default towers, Twenty-One's and the small Gomoku net), on whatever route its wider stem takes: initial inference,
    and the root and expansions of one untraced search, within tests/test_net_sweep_gpu.py's budget against
    oracle/net.py in fp64 (the x3 budget where the net runs on the x3 towers)."""
    from muzero_general_b200.engine import SearchEngine
    from test_net_sweep_gpu import Judge, Ref, _pools
    monkeypatch.delenv("MZ_TC_MODE", raising=False)
    _, cfg = _cfg(name, 2)
    spec = netspec_from_config(cfg)
    w = weights_for(name, spec)
    n, N = 40, 8
    eng = SearchEngine(cfg, max_games=n, num_simulations=N)
    eng.load_weights(w)
    A = spec.action_space
    obs, _, _ = _pools(spec, n, seed=7)
    mode = "x3" if "f32-grade nets" in eng.numerics else None
    judge = Judge(f"stacked {name} [{eng.numerics}]", mode)
    ref = Ref(spec, w)
    ri = ref.initial(obs)
    d0 = eng.initial_inference(obs)
    for r in range(n):
        judge.vector(f"row {r} init hidden", d0["hidden"][r], ri, "hidden", r)
        judge.vector(f"row {r} init value logits", d0["value_logits"][r], ri, "value_logits", r)
        judge.vector(f"row {r} init policy logits", d0["policy_logits"][r], ri, "policy_logits", r)
        judge.scalar(f"row {r} init value", d0["value"][r], ri, "value", r)
    out = eng.search(obs=obs, add_exploration_noise=False, keep_tree=True)
    for g in (0, n // 2, n - 1):
        tree = eng.export_tree(g, with_hidden=True)
        assert tree["n_expansions"] == N + 1
        judge.vector(f"game {g} root hidden", tree["hidden"][0], ri, "hidden", g)
        judge.scalar(f"game {g} root value", out.root_predicted_value[g], ri, "value", g)
        judge.vector(f"game {g} root priors", out.root_priors[g], ri, "priors", g)
        slot_of = {int(e): s for s, e in enumerate(tree["child_expansion"]) if e >= 0}
        exps = [1, 2, N]
        rr = ref.recurrent(tree["hidden"][[slot_of[e] // A for e in exps]], [slot_of[e] % A for e in exps])
        for k, e in enumerate(exps):
            judge.vector(f"game {g} expansion {e} hidden", tree["hidden"][e], rr, "hidden", k)
            judge.scalar(f"game {g} expansion {e} edge reward", tree["child_reward"][slot_of[e]], rr, "reward", k)
            judge.vector(f"game {g} expansion {e} child priors", tree["child_prior"][e * A:(e + 1) * A], rr, "priors", k)
    judge.finish()
    eng.close()
