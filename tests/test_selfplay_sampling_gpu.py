"""The device self-play loop's random decisions (csrc/selfplay.cu, csrc/common.cuh) against host oracles.

* Action sampling at every temperature: the played action is select_action's (self_play.py:222-245) with numpy's
  choice rule (oracle/mcts.py::numpy_choice_index) for the same uniform, including uniforms placed exactly on the
  rule's boundaries; T = 0 and moves past temperature_threshold take the first maximum; T = inf takes
  floor(u * n_legal).
* The production path (mz_selfplay_enqueue / wait, several moves per call, device-drawn noise and uniforms) against a
  host composition of [search of the peeked state] + [oracle.philox.uniform53] + [numpy's choice rule].
* Device-drawn root noise, element for element, against oracle.philox.gamma in every kernel that draws it.
* PER priorities computed while packing, against reanalyse.initial_priorities, over alpha, td_steps and discount.
Everything goes through the C ABI."""
import math

import numpy
import pytest

from conftest import weights_for
from helpers import random_teacher
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from oracle import mcts as om
from oracle import philox

pytestmark = pytest.mark.gpu

INF = float("inf")
ONE_MINUS = math.nextafter(1.0, 0.0)


def _setup(name, B, N, seed=0, threshold=None, td_steps=0, per_alpha=1.0, **over):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    for k, v in over.items():
        setattr(cfg, k, v)
    spec = netspec_from_config(cfg)
    w = weights_for(name, spec)
    vec = getattr(mod.Game, "VECTOR", None)

    def make_loop(staging_bytes=0):
        eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
        eng.load_weights(w)
        loop = DeviceSelfPlayLoop(eng, name, cfg.max_moves, temperature_threshold=threshold,
                                  reward_scale=getattr(vec, "REWARD_SCALE", 1), staging_bytes=staging_bytes,
                                  td_steps=td_steps, per_alpha=per_alpha, discount=cfg.discount)
        return eng, loop

    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    ref.load_weights(w)
    return mod, cfg, spec, ref, make_loop


def _drain(loop):
    from muzero_general_b200.engine import parse_staged_games
    return parse_staged_games(*loop.drain())


def _effective_temperature(T, threshold, move):
    return T if not threshold or move + 1 < threshold else 0.0


def _oracle_action(visits, legal, T, u):
    idx = [int(a) for a in numpy.nonzero(legal)[0]]
    return om.select_action(idx, visits[idx], T, om.InjectedDraws(uniform=float(u)))


def _boundaries(visits, legal, T):
    """(normalised cdf, unnormalised cdf, p) of select_action's distribution over the legal actions."""
    d = numpy.asarray(visits[numpy.nonzero(legal)[0]], dtype="int32") ** (1 / T)
    p = d / sum(d)
    raw = numpy.cumsum(p)
    return raw / raw[-1], raw, p


def _pick_uniform(rs, visits, legal, T, kind):
    """A uniform on an edge of the rule for this slot: numpy's boundary cdf_k / cdf[-1], one ulp below or above it,
    or the unnormalised boundary cdf_k; at T = inf the boundary k / n and its neighbours; a plain draw otherwise.
    Interior boundaries where the two cdfs differ are preferred.  Returns (u, exact): exact is False where the
    device's pow (non-integer 1/T) could move a boundary within 1e-12 of u."""
    n = int(legal.sum())
    if T == INF:
        b = rs.randint(0, n) / n
        return min(max([b, math.nextafter(b, 0.0), math.nextafter(b, 1.0)][kind % 3], 0.0), ONE_MINUS), True
    if T == 0 or n == 1:
        return rs.random_sample(), True
    cdf, raw, p = _boundaries(visits, legal, T)
    if T not in (1.0, 0.5, 0.25):
        u = rs.random_sample()
        return u, bool(numpy.abs(numpy.concatenate([cdf, raw]) - u).min() > 1e-12)
    interior = [k for k in range(n - 1) if p[k] > 0 and cdf[k] < 1.0]
    if not interior:
        return rs.random_sample(), True
    differing = [k for k in interior if cdf[k] != raw[k]]
    k = int(rs.choice(differing or interior))
    u = [cdf[k], math.nextafter(cdf[k], 0.0), math.nextafter(cdf[k], 2.0), raw[k]][kind % 4]
    return min(max(float(u), 0.0), ONE_MINUS), True


# ------------------------------------------------------------------------------------------ sampling, injected draws
@pytest.mark.parametrize("name,B,N,moves,over", [("tictactoe", 64, 5, 30, {}), ("connect4", 48, 6, 30, {}),
                                                 ("cartpole", 64, 4, 30, dict(max_moves=12))])
def test_device_sampler_equals_numpy_choice_at_every_temperature(name, B, N, moves, over, monkeypatch):
    """One move per call with injected noise and uniforms; the temperature cycles through 1, 0.5, 0.25, 0, inf and
    0.7.  Per slot the uniform sits on a boundary of numpy's rule (or next to it) for the visit counts a reference
    search of the peeked state returns.  The played action equals select_action with numpy's choice rule; for
    1/T = 1/0.7 the device's pow is within 2 ulps of the host's, so equality is asserted only where u is more than
    1e-12 from every boundary."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    mod, cfg, spec, ref, make_loop = _setup(name, B, N, seed=11, **over)
    eng, loop = make_loop()
    A = spec.action_space
    rs = numpy.random.RandomState(5)
    temps = [1.0, 0.5, 0.25, 0.0, INF, 0.7]
    expected, delivered = {}, []
    checked = {T: 0 for T in temps}
    informative = 0                    # slots where the unnormalised cumulative sum would pick another action
    for t in range(moves):
        T = temps[t % len(temps)]
        pk = loop.peek()
        legal = pk["legal_mask"]
        gam = rs.standard_gamma(cfg.root_dirichlet_alpha, size=(B, A)) * (legal > 0)
        noise = gam / gam.sum(1, keepdims=True)
        out = ref.search(obs=pk["obs"], legal_mask=legal, to_play=pk["to_play"], add_exploration_noise=True, noise=noise,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        u = numpy.zeros(B)
        want = numpy.zeros(B, numpy.int64)
        exact = numpy.zeros(B, bool)
        for g in range(B):
            u[g], exact[g] = _pick_uniform(rs, out.visit_counts[g], legal[g], T, t * B + g)
            want[g] = _oracle_action(out.visit_counts[g], legal[g], T, u[g])
            if 0 < T < INF and exact[g]:
                cdf, raw, _ = _boundaries(out.visit_counts[g], legal[g], T)
                informative += int(numpy.searchsorted(raw, u[g], side="right")) != int(numpy.searchsorted(cdf, u[g], side="right"))
            expected.setdefault(int(pk["game_id"][g]), []).append(
                (out.visit_counts[g].copy(), out.root_value[g], int(want[g]), bool(exact[g])))
        loop.moves(1, T, uniform=u, noise=noise)
        after = loop.peek()
        kept = (after["move_index"] != 0) & exact
        assert (after["last_action"][kept] == want[kept]).all(), (name, T, t)
        checked[T] += int(kept.sum())
        delivered += _drain(loop)
    assert delivered and all(checked[T] > 0 for T in temps), checked
    if name == "tictactoe":            # where these searches leave counts whose cumulative sum misses 1
        assert informative > 0
    for rec in delivered:
        exp = expected[rec["game_id"]]
        assert rec["length"] == len(exp)
        for t, (visits, root_value, action, exact) in enumerate(exp):
            assert rec["visits"][t].tolist() == visits.tolist()
            assert rec["root_value"][t] == root_value
            if exact:
                assert rec["action"][t] == action, (rec["game_id"], t)
    eng.close(); ref.close()


def test_temperature_threshold_switches_to_the_first_maximum(monkeypatch):
    """TicTacToe with temperature_threshold = 3: moves with t + 1 >= 3 are the first maximum of the visit counts over
    the legal actions, whatever the uniform; earlier moves sample.  The uniform is chosen so that sampling would
    often pick another action."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    B, N = 64, 6
    mod, cfg, spec, ref, make_loop = _setup("tictactoe", B, N, seed=2, threshold=3)
    eng, loop = make_loop()
    A = spec.action_space
    rs = numpy.random.RandomState(8)
    would_differ = 0
    for t in range(12):
        pk = loop.peek()
        legal = pk["legal_mask"]
        gam = rs.standard_gamma(cfg.root_dirichlet_alpha, size=(B, A)) * (legal > 0)
        noise = gam / gam.sum(1, keepdims=True)
        out = ref.search(obs=pk["obs"], legal_mask=legal, to_play=pk["to_play"], add_exploration_noise=True, noise=noise,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        u = numpy.where(rs.random_sample(B) < 0.5, ONE_MINUS, rs.random_sample(B))
        want = numpy.zeros(B, numpy.int64)
        for g in range(B):
            mv = int(pk["move_index"][g])
            T = _effective_temperature(1.0, 3, mv)
            want[g] = _oracle_action(out.visit_counts[g], legal[g], T, u[g])
            if T == 0:
                masked = numpy.where(legal[g] > 0, out.visit_counts[g], -1)
                assert want[g] == int(numpy.argmax(masked))
                would_differ += _oracle_action(out.visit_counts[g], legal[g], 1.0, u[g]) != want[g]
        loop.moves(1, 1.0, uniform=u, noise=noise)
        after = loop.peek()
        kept = after["move_index"] != 0
        assert (after["last_action"][kept] == want[kept]).all(), t
        for rec in _drain(loop):
            assert rec["length"] >= 5
    assert would_differ > 20
    eng.close(); ref.close()


# ------------------------------------------------------------------------------------------ production path
def _replay_board(mod, rec):
    """The record's actions on the host environment: same observations and rewards, and the game ends on the last."""
    env = mod.Game(0)
    env.reset()
    for t in range(rec["length"]):
        assert int(rec["action"][t]) in env.legal_actions()
        obs, reward, done = env.step(int(rec["action"][t]))
        assert numpy.array_equal(numpy.asarray(obs, numpy.float32).ravel(), rec["obs"][t + 1])
        assert float(reward) == float(rec["reward"][t])
        assert done == (t + 1 == rec["length"])


@pytest.mark.parametrize("name,B,N,T,threshold,moves,max_moves,staging", [
    ("tictactoe", 32, 6, 1.0, None, 20, None, 3 * 2048),
    ("tictactoe", 32, 6, 0.5, 4, 20, None, 0),
    ("connect4", 16, 5, 0.25, 8, 30, None, 0),
    ("cartpole", 32, 5, 1.0, None, 30, 14, 0),
    ("cartpole", 32, 5, 0.5, 6, 30, 14, 0),
])
def test_production_loop_equals_host_composition(name, B, N, T, threshold, moves, max_moves, staging, monkeypatch):
    """No injection.  Run A plays one move per call; before each move the host composes [search of the peeked state
    with device-drawn noise and ties] + [uniform53(seed, game, move, 0, TAG_ACTION)] + [numpy's choice rule], and
    every delivered record's visits, root values and actions equal it bit for bit; rewards and observations replay
    on the host environment (CartPole: the first observation is float32(-0.05 + 0.1 * uniform53(..., TAG_RESET))).
    Run B plays the same seeded loop through mz_selfplay_enqueue / wait in chunks of 1, 3 and 8 moves (with a
    staging area that parks games, where given) until it has finished every game run A finished: each is identical."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    over = {} if max_moves is None else dict(max_moves=max_moves)
    seed = 0x1234_5678_9ABC
    mod, cfg, spec, ref, make_loop = _setup(name, B, N, seed=seed, threshold=threshold, **over)
    eng_a, loop_a = make_loop()
    expected, recs_a = {}, {}
    for _ in range(moves):
        pk = loop_a.peek()
        out = ref.search(obs=pk["obs"], legal_mask=pk["legal_mask"], to_play=pk["to_play"], add_exploration_noise=True,
                         game_id=pk["game_id"], move_index=pk["move_index"])
        for g in range(B):
            gid, mv = int(pk["game_id"][g]), int(pk["move_index"][g])
            u = philox.uniform53(seed, gid, mv, 0, philox.TAG_ACTION)
            a = _oracle_action(out.visit_counts[g], pk["legal_mask"][g], _effective_temperature(T, threshold, mv), u)
            expected.setdefault(gid, []).append((out.visit_counts[g].copy(), out.root_value[g], a))
        loop_a.moves(1, T)
        for rec in _drain(loop_a):
            recs_a[rec["game_id"]] = rec
    eng_a.close(); ref.close()
    assert len(recs_a) >= B // 2
    for gid, rec in recs_a.items():
        exp = expected[gid]
        assert rec["length"] == len(exp)
        for t, (visits, root_value, action) in enumerate(exp):
            assert rec["visits"][t].tolist() == visits.tolist(), (gid, t)
            assert rec["root_value"][t] == root_value, (gid, t)
            assert rec["action"][t] == action, (gid, t)
        if name == "cartpole":
            first = [numpy.float32(-0.05 + 0.1 * philox.uniform53(seed, gid, 0, k, philox.TAG_RESET)) for k in range(4)]
            assert rec["obs"][0].tolist() == first, gid
            assert (rec["reward"] == 1.0).all()
        else:
            _replay_board(mod, rec)

    eng_b, loop_b = make_loop(staging)
    # parked games hold their slots back (a 3-game staging area delivers at most 3 games per call), so run B may need
    # more calls than run A to finish the same games; every slot plays its ids first + slot + j * B in order, whatever
    # the parking, so it eventually finishes each of them
    recs_b, played, parked, i = {}, 0, 0, 0
    while played < moves or (not set(recs_a) <= set(recs_b) and i < 400):
        k = [1, 3, 8][i % 3]
        loop_b.enqueue(k, T)
        st = loop_b.wait()
        parked = max(parked, st.parked_slots)
        for rec in _drain(loop_b):
            assert rec["game_id"] not in recs_b
            recs_b[rec["game_id"]] = rec
        played += k
        i += 1
    eng_b.close()
    if staging:
        assert parked > 0
    assert set(recs_a) <= set(recs_b)
    for gid in sorted(recs_a):
        for key in ("length", "slot", "first_to_play", "action", "visits", "root_value", "reward", "to_play", "obs"):
            assert numpy.array_equal(recs_a[gid][key], recs_b[gid][key]), (gid, key)



# ------------------------------------------------------------------------------------------ device-drawn root noise
def _check_noise(nz, legal, seed, gid, mv, alpha):
    """Row by row: the device's noise equals the restated Gamma draws normalised over the legal actions within 1e-12
    relative; rows where a draw's accept / reject decision lies within 1e-12 of its threshold are skipped (the
    device's log / cospi / pow are not correctly rounded).  Returns the number of rows checked."""
    checked = 0
    for i in range(nz.shape[0]):
        want, margin = philox.dirichlet_noise(seed, int(gid[i]), int(mv[i]), [bool(x) for x in legal[i]], alpha)
        if margin < 1e-12:
            continue
        want = numpy.array(want)
        assert ((nz[i] == 0) == (want == 0)).all(), i
        numpy.testing.assert_allclose(nz[i], want, rtol=1e-12, atol=0, err_msg=f"row {i}")
        checked += 1
    assert checked >= 0.99 * nz.shape[0]
    return checked


def _noise_case(cfg, n, N, rs, all_legal=False):
    A, P = len(cfg.action_space), len(cfg.players)
    legal = numpy.ones((n, A), numpy.uint8) if all_legal else (rs.uniform(size=(n, A)) < 0.6).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    t = random_teacher(rs, n, N, A, reward_scale=1.0 if P == 1 else 0.0, legal=legal)
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    gid = rs.randint(0, 1 << 40, n).astype(numpy.int64)
    mv = rs.randint(0, 300, n).astype(numpy.int32)
    return legal, t, to_play, gid, mv


@pytest.mark.parametrize("game,alpha", [("tictactoe", None), ("connect4", None), ("cartpole", None),
                                        ("connect4", 0.25), ("tictactoe", 0.3)])
def test_device_noise_narrow_root_equals_restated_gamma(game, alpha, game_configs):
    """Teacher-forced searches with noise=None: trace["noise"] of the fused kernel (tree.cuh) and of the step-wise
    root (A <= 32) are identical, and equal the restated draws element for element, at each game's own alpha and at
    the reference alphas 0.25 and 0.3."""
    from muzero_general_b200.engine import SearchEngine
    import copy
    cfg = copy.copy(game_configs[game])
    if alpha is not None:
        cfg.root_dirichlet_alpha = alpha
    n, N = 512, 6
    rs = numpy.random.RandomState(31)
    legal, t, to_play, gid, mv = _noise_case(cfg, n, N, rs)
    eng = SearchEngine(cfg, max_games=n, num_simulations=N, seed=0xA5A5_0000_1111)
    kw = dict(legal_mask=legal, to_play=to_play, add_exploration_noise=True, game_id=gid, move_index=mv, teacher=t,
              trace=True, n_games=n)
    a = eng.search(**kw)
    b = eng.search(stepwise=True, **kw)
    eng.close()
    assert numpy.array_equal(a.trace["noise"], b.trace["noise"])
    assert numpy.array_equal(a.visit_counts, b.visit_counts)
    _check_noise(a.trace["noise"], legal, 0xA5A5_0000_1111, gid, mv, cfg.root_dirichlet_alpha)


@pytest.mark.parametrize("A,alpha", [(33, 0.25), (64, 0.3), (121, 0.3), (128, 0.25)])
def test_device_noise_wide_root_equals_restated_gamma(A, alpha, game_configs):
    """The wide kernel (tree_wide.cu, 32 < A <= 128) draws action k = lane + 32 j with counter k: equal to the
    restated draws over a restricted legal set."""
    from muzero_general_b200.engine import SearchEngine
    import copy
    cfg = copy.copy(game_configs["gomoku" if A == 121 else "cartpole"])
    cfg.action_space = list(range(A))
    cfg.root_dirichlet_alpha = alpha
    n, N = 96, 4
    rs = numpy.random.RandomState(A)
    legal, t, to_play, gid, mv = _noise_case(cfg, n, N, rs)
    eng = SearchEngine(cfg, max_games=n, num_simulations=N, seed=77)
    out = eng.search(legal_mask=legal, to_play=to_play, add_exploration_noise=True, game_id=gid, move_index=mv,
                     teacher=t, trace=True, n_games=n)
    eng.close()
    _check_noise(out.trace["noise"], legal, 77, gid, mv, alpha)


@pytest.mark.parametrize("name", ["tictactoe", "cartpole"])
def test_device_noise_of_an_imported_root_equals_restated_gamma(name, monkeypatch):
    """A search continued from an imported tree (mz_import_tree + MZ_FLAG_CONTINUE, tree_adopt_root_kernel) draws the
    noise over the whole action space: equal to the restated draws."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    spec = netspec_from_config(cfg)
    A, N, seed = spec.action_space, 8, 4242
    eng = SearchEngine(cfg, max_games=1, num_simulations=N, seed=seed, extra_expansions=N + 1)
    eng.load_weights(weights_for(name, spec))
    rs = numpy.random.RandomState(3)
    checked = 0
    for trial in range(12):
        obs = rs.randint(0, 2, size=(1, spec.obs_elems)).astype(numpy.float32) if name != "cartpole" else \
            rs.uniform(-0.05, 0.05, size=(1, 4)).astype(numpy.float32)
        eng.search(obs=obs, legal_mask=numpy.ones((1, A), numpy.uint8), to_play=numpy.zeros(1, numpy.int32),
                   add_exploration_noise=True, keep_tree=True)
        eng.import_tree(0, eng.export_tree(0, with_hidden=True))
        gid = numpy.array([rs.randint(0, 1 << 40)], numpy.int64)
        mv = numpy.array([rs.randint(0, 50)], numpy.int32)
        out = eng.search(legal_mask=numpy.ones((1, A), numpy.uint8), to_play=numpy.zeros(1, numpy.int32),
                         add_exploration_noise=True, keep_tree=True, continue_tree=True, n_games=1, trace=True,
                         game_id=gid, move_index=mv)
        want, margin = philox.dirichlet_noise(seed, int(gid[0]), int(mv[0]), [True] * A, cfg.root_dirichlet_alpha)
        if margin < 1e-12:
            continue
        numpy.testing.assert_allclose(out.trace["noise"][0], want, rtol=1e-12, atol=0)
        checked += 1
    eng.close()
    assert checked >= 10


# ------------------------------------------------------------------------------------------ PER priorities
PRIORITY_SWEEP = [(1.0, 1, 1.0), (1.0, 3, 0.997), (1.0, "long", 1.0), (0.5, 1, 0.997), (0.5, 3, 1.0),
                  (0.5, "long", 0.997)]


@pytest.mark.parametrize("alpha,td,discount", PRIORITY_SWEEP)
@pytest.mark.parametrize("name,B,N,moves,max_moves", [("cartpole", 32, 4, 40, 12), ("tictactoe", 32, 4, 30, None),
                                                      ("connect4", 16, 4, 45, None)])
def test_device_priorities_sweep(name, B, N, moves, max_moves, alpha, td, discount, monkeypatch):
    """PackedGameHistory.priorities (computed by the packing warp) against reanalyse.initial_priorities, which is
    pinned to the reference's ReplayBuffer: bit for bit at alpha = 1; at alpha = 0.5 the device takes an exact sqrt
    and the host numpy's ** 0.5, one float32 ulp apart in about 1 case of 1000.  td_steps 1, 3 and max_moves + 5
    (never a bootstrap value), discount 1 and 0.997; CartPole games cut by max_moves, board games won or drawn."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200 import reanalyse as ra
    from muzero_general_b200.self_play import PackedGameHistory
    over = dict(discount=discount, PER_alpha=alpha)
    if max_moves:
        over["max_moves"] = max_moves
    mod = load_game_module(name)
    cfg0 = mod.MuZeroConfig()
    td_steps = (max_moves or cfg0.max_moves) + 5 if td == "long" else td
    mod, cfg, spec, ref, make_loop = _setup(name, B, N, seed=9, td_steps=td_steps, per_alpha=alpha, **over)
    cfg.td_steps = td_steps
    ref.close()
    eng, loop = make_loop()
    assert loop.with_priorities
    vec = getattr(mod.Game, "VECTOR", None)
    args = (cfg.observation_shape, getattr(vec, "OBS_DTYPE", numpy.float32), int if vec is not None else float, True)
    games = []
    for _ in range(moves):
        loop.moves(1, 1.0)
        games += [PackedGameHistory(rec, *args) for rec in _drain(loop)]
    eng.close()
    assert len(games) >= B
    ends = {"cut": 0, "won": 0, "drawn": 0}
    for gh in games:
        want, top = ra.initial_priorities(gh, cfg)
        assert gh.priorities.dtype == numpy.float32 and gh.priorities.shape == want.shape
        if alpha == 1.0:
            assert numpy.array_equal(gh.priorities, want), gh.game_id
        else:
            numpy.testing.assert_allclose(gh.priorities, want, rtol=2e-7, atol=0)
        T = len(gh)
        if name == "cartpole":
            ends["cut"] += T == cfg.max_moves
        elif gh.reward_history[-1] != 0:
            ends["won"] += 1
        else:
            ends["drawn"] += 1
    if name == "cartpole":
        assert ends["cut"] > 0
    else:
        assert ends["won"] > 0
        if name == "tictactoe":
            assert ends["drawn"] > 0
