"""Device-resident self-play (mz_selfplay_*, csrc/selfplay.cu) against the reference's recorded environment
trajectories, the host loop and the search it wraps.  Everything goes through the C ABI."""
import pickle

import numpy
import pytest

from conftest import golden_json, weights_for
from muzero_general_b200.games import load_game_module
from muzero_general_b200.netspec import netspec_from_config
from oracle import mcts as om

pytestmark = pytest.mark.gpu


def _loop(name, B, N, seed=0, first_game_id=0, staging_bytes=0, **over):
    from muzero_general_b200.engine import DeviceSelfPlayLoop, SearchEngine
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    for k, v in over.items():
        setattr(cfg, k, v)
    spec = netspec_from_config(cfg)
    eng = SearchEngine(cfg, max_games=B, num_simulations=N, seed=seed)
    eng.load_weights(weights_for(name, spec))
    vec = getattr(mod.Game, "VECTOR", None)
    loop = DeviceSelfPlayLoop(eng, name, cfg.max_moves, temperature_threshold=cfg.temperature_threshold,
                              reward_scale=getattr(vec, "REWARD_SCALE", 1), first_game_id=first_game_id,
                              staging_bytes=staging_bytes)
    return mod, cfg, spec, eng, loop


def _drain(loop):
    from muzero_general_b200.engine import parse_staged_games
    return parse_staged_games(*loop.drain())


@pytest.mark.parametrize("name", ["tictactoe", "connect4"])
def test_board_environments_replay_the_reference_trajectories(name, monkeypatch):
    """Slot g is driven through the reference's recorded game g (tests/golden/env_*.json) with forced actions: the
    device observation planes, legal masks, side to move, rewards and terminations are the reference's, bit for bit."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    fx = golden_json(f"env_{name}.json")
    games = fx["games"]
    B = len(games)
    mod, cfg, spec, eng, loop = _loop(name, B, 2)
    A = spec.action_space
    longest = max(len(g) for g in games)
    finished = {}
    pk = loop.peek()
    assert (pk["move_index"] == 0).all() and (pk["game_id"] == numpy.arange(B)).all() and (pk["to_play"] == 0).all()
    for t in range(longest):
        forced = numpy.zeros(B, numpy.int32)
        for g in range(B):
            if t < len(games[g]):
                forced[g] = games[g][t]["action"]
            else:                                   # the slot already plays its next game: any legal action
                forced[g] = int(numpy.nonzero(pk["legal_mask"][g])[0][0])
        loop.moves(1, 1.0, forced_action=forced)
        pk = loop.peek()
        for g in range(B):
            if t < len(games[g]):
                s = games[g][t]
                assert int(pk["last_action"][g]) in (s["action"], -1)
                if not s["done"]:
                    assert pk["obs"][g].astype(numpy.int8).tolist() == s["obs"], (name, g, t)
                    assert numpy.nonzero(pk["legal_mask"][g])[0].tolist() == s["legal"]
                    assert int(pk["to_play"][g]) == s["to_play"] and int(pk["move_index"][g]) == t + 1
                else:                               # packed and restarted within the same move
                    assert int(pk["move_index"][g]) == 0 and int(pk["game_id"][g]) == g + B
        for rec in _drain(loop):
            if rec["game_id"] < B:
                finished[rec["game_id"]] = rec
    assert sorted(finished) == list(range(B))
    for g, rec in finished.items():
        steps = games[g]
        assert rec["length"] == len(steps) and rec["slot"] == g and rec["first_to_play"] == 0
        assert rec["action"].tolist() == [s["action"] for s in steps]
        assert rec["reward"].tolist() == [float(s["reward"]) for s in steps]
        assert rec["to_play"].tolist() == [s["to_play"] for s in steps]
        assert rec["obs"][1:].astype(numpy.int8).tolist() == [s["obs"] for s in steps]
        first = numpy.zeros(spec.obs_elems, numpy.float32)
        first[2 * (spec.obs_elems // 3):] = 1.0                         # empty board, player +1 to move
        assert rec["obs"][0].tolist() == first.tolist()
        assert (rec["visits"].sum(1) == 2).all()                        # every move was searched (N = 2)
    eng.close()


def test_cartpole_physics_one_step_at_a_time():
    """Every recorded transition obeys the host environment's equations (games/cartpole.py here; gym's CartPole-v1 is
    not vendored in the reference - parity unpinned): stepping the host physics from observation t with the recorded
    action reproduces observation t+1 to fp32 rounding; +1 reward per move; episodes end by the rule."""
    from muzero_general_b200.games import cartpole as cp
    B = 64
    mod, cfg, spec, eng, loop = _loop("cartpole", B, 3, max_moves=60)
    recs = []
    for _ in range(70):
        loop.moves(1, 1.0)
        recs += _drain(loop)
    assert len(recs) >= B
    checked = 0
    for rec in recs:
        T = rec["length"]
        assert 1 <= T <= 60 and (rec["reward"] == 1.0).all() and (rec["to_play"] == 0).all()
        assert (numpy.abs(rec["obs"][0]) <= 0.05).all()
        env = cp.CartPoleVector(1, 0)
        for t in range(T):
            env.state = rec["obs"][t].astype(numpy.float64)[None]
            env.steps[:] = t
            obs, _, done = env.step(numpy.array([rec["action"][t]]))
            numpy.testing.assert_allclose(obs.ravel(), rec["obs"][t + 1], rtol=2e-6, atol=2e-7)
            checked += 1
        x, th = float(rec["obs"][T][0]), float(rec["obs"][T][2])
        ended = abs(x) > 2.4 or abs(th) > cp._THETA_LIMIT
        assert ended or T == 60
    assert checked > 500
    # fresh ids per slot: first_game_id + slot + k * B
    for rec in recs:
        assert rec["game_id"] % B == rec["slot"]
    eng.close()


@pytest.mark.parametrize("name,B,N,moves", [("cartpole", 48, 20, 14), ("tictactoe", 40, 16, 12), ("connect4", 24, 12, 30)])
def test_device_loop_equals_host_composition_with_injected_draws(name, B, N, moves, monkeypatch):
    """One move at a time with the host's draws injected (root noise, action uniforms): the action the device plays and
    the record it keeps equal [mz_search on the peeked observation] + [select_action with numpy's choice rule for the
    injected uniform (oracle/mcts.py::numpy_choice_index)]."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200.engine import SearchEngine
    mod, cfg, spec, eng, loop = _loop(name, B, N, seed=5)
    ref = SearchEngine(cfg, max_games=B, num_simulations=N, seed=5)
    ref.load_weights(weights_for(name, spec))
    A = spec.action_space
    rs = numpy.random.RandomState(17)
    expected = {}                                    # game id -> list of (visits, root_value, action)
    delivered = []
    for t in range(moves):
        pk = loop.peek()
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
        after = loop.peek()
        restarted = after["move_index"] == 0
        assert (after["last_action"][~restarted] == want[~restarted]).all()
        delivered += _drain(loop)
    assert delivered
    for rec in delivered:
        exp = expected[rec["game_id"]]
        assert rec["length"] == len(exp)
        for t, (visits, root_value, action) in enumerate(exp):
            assert rec["visits"][t].tolist() == visits.tolist()
            assert rec["root_value"][t] == root_value
            assert rec["action"][t] == action
    eng.close(); ref.close()


def test_histories_are_batch_and_rank_invariant():
    """Global game 21 has the same history whether it is slot 21 of a 32-game batch on 'rank 0' or slot 5 of a 16-game
    batch whose first id is 16 ('rank 1' of two): every draw is keyed by (seed, global game id, move)."""
    def games(B, first):
        mod, cfg, spec, eng, loop = _loop("cartpole", B, 12, seed=3, first_game_id=first, max_moves=40)
        out = {}
        for _ in range(45):
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


def test_backpressure_parks_finished_games_until_the_host_drains():
    """A staging area of three games: finished games that do not fit wait in their slots (parked, not searched into
    the records) and are delivered after the next drain; no game is lost or duplicated."""
    from muzero_general_b200.engine import parse_staged_games
    B = 32
    mod, cfg, spec, eng, loop = _loop("tictactoe", B, 4, staging_bytes=3 * 2048, num_simulations=4)
    seen, parked_max = {}, 0
    for _ in range(80):
        st = loop.moves(1, 1.0)
        parked_max = max(parked_max, st.parked_slots)
        buf, index = loop.drain()
        assert len(buf) <= 3 * 2048
        for rec in parse_staged_games(buf, index):
            assert rec["game_id"] not in seen
            seen[rec["game_id"]] = rec["length"]
    assert parked_max > 0
    assert len(seen) > B                                        # slots did restart
    ids = sorted(seen)
    for slot in range(B):                                       # per slot: consecutive games first+slot+k*B, no gaps
        mine = [g for g in ids if g % B == slot]
        assert mine == [slot + k * B for k in range(len(mine))]
    assert all(5 <= n <= 9 for n in seen.values())
    eng.close()


@pytest.mark.parametrize("name", ["cartpole", "tictactoe"])
def test_selfplay_api_on_the_device_loop(name, monkeypatch):
    """SelfPlay.play_moves with rng_mode="philox": PackedGameHistory objects with the reference's attribute set and
    types; they pickle as plain GameHistory; continuous_self_play feeds a buffer from the device loop."""
    monkeypatch.setenv("MZ_TC_MODE", "off")
    from muzero_general_b200 import self_play as sp
    mod = load_game_module(name)
    cfg = mod.MuZeroConfig()
    cfg.num_parallel_games, cfg.rng_mode, cfg.num_simulations, cfg.max_moves = 24, "philox", 6, min(cfg.max_moves, 30)
    cfg.training_steps, cfg.ratio, cfg.moves_per_weight_refresh = 8, None, 4
    spec = netspec_from_config(cfg)
    w = weights_for(name, spec)
    worker = sp.SelfPlay({"weights": w}, mod.Game, cfg, seed=0)
    assert worker.loop_path == "device"
    games = []
    for _ in range(12):
        batch = worker.play_moves(3, 1.0)
        assert len(batch.lengths()) == len(batch) and batch.total_moves == int(batch.lengths().sum())
        games += list(batch)
    assert games and worker.env_steps == 24 * 36 and worker.played_games == len(games)
    assert worker.played_steps == sum(len(g.root_values) for g in games)
    for gh in games[:10]:
        T = len(gh.action_history) - 1
        assert isinstance(gh, sp.GameHistory) and T == len(gh) >= 1
        assert len(gh.child_visits) == T == len(gh.root_values) and len(gh.observation_history) == T + 1
        assert gh.action_history[0] == 0 and gh.reward_history[0] == 0
        assert gh.observation_history[0].shape == tuple(cfg.observation_shape)
        assert all(abs(sum(c) - 1) < 1e-12 for c in gh.child_visits)
        assert isinstance(gh.root_values[0], float) and gh.priorities is not None
        assert gh.get_stacked_observations(-1, 0, len(cfg.action_space)).shape == tuple(cfg.observation_shape)
        plain = pickle.loads(pickle.dumps(gh))
        assert type(plain) is sp.GameHistory and plain.child_visits == gh.child_visits
        # PER priorities computed by the packing warp == the reference's save_game loop (restated in reanalyse.py and
        # pinned bit for bit to the unmodified ReplayBuffer in tests/test_reanalyse_cpu.py); alpha = 0.5 is an exact sqrt
        # on the device and numpy's pow on the host: one float32 ulp of slack
        from muzero_general_b200 import reanalyse as ra
        want, top = ra.initial_priorities(gh, cfg)
        assert gh.priorities.dtype == numpy.float32 and gh.priorities.shape == want.shape
        numpy.testing.assert_allclose(gh.priorities, want, rtol=2e-7, atol=0)
        assert gh.game_priority == gh.priorities.max()
        if name == "tictactoe":
            assert gh.observation_history[0].dtype == numpy.int32 and isinstance(gh.reward_history[-1], int)

    class Storage:
        def __init__(self):
            self.d = dict(weights=w, training_step=0, terminate=False, num_played_steps=0, num_played_games=0)
        def get_info(self, k):
            if k == "training_step":
                self.d["training_step"] += 2
            return self.d[k]
        def set_info(self, k, v=None):
            self.d.update(k if isinstance(k, dict) else {k: v})

    class Buffer:
        def __init__(self):
            self.games = []
        def save_game(self, gh, storage=None):
            self.games.append(gh)

    buf = Buffer()
    worker.continuous_self_play(Storage(), buf)
    assert buf.games and all(len(g.child_visits) == len(g.action_history) - 1 for g in buf.games)


def test_multi_rank_entry_point_is_world_size_invariant(tmp_path):
    """python -m muzero_general_b200.parallel: 32 CartPole games on one rank and 2 x 16 games on two ranks (torchrun;
    the ranks share the GPU and talk over gloo when the box has a single one, NCCL otherwise) finish the SAME games -
    every global game id both runs completed has the same content hash; counters add up over the ranks."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    common = ["--game", "cartpole", "--games", "32", "--reports", "3", "--moves-per-report", "12", "--simulations", "10"]
    env = dict(os.environ, PYTHONPATH=root)
    one = tmp_path / "one"
    subprocess.run([sys.executable, "-m", "muzero_general_b200.parallel", *common, "--dump-histories", str(one)],
                   check=True, cwd=root, env=env, timeout=600)
    two = tmp_path / "two"
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                    "127.0.0.1", "--master-port", "29731", "-m", "muzero_general_b200.parallel", *common,
                    "--dump-histories", str(two)], check=True, cwd=root, env=env, timeout=600)
    a = json.load(open(one / "rank0.json"))
    b0, b1 = json.load(open(two / "rank0.json")), json.load(open(two / "rank1.json"))
    assert a["summary"]["num_played_steps"] == 32 * 36 == b0["summary"]["num_played_steps"]
    assert b0["summary"]["world"] == 2 and len(b0["lines"][0]["per_rank"]) == 2
    merged = dict(b0["digests"], **b1["digests"])
    assert not set(b0["digests"]) & set(b1["digests"])
    # first games of every slot carry the ids 0..31 in both runs
    first = [str(g) for g in range(32) if str(g) in a["digests"] and str(g) in merged]
    assert len(first) >= 16
    for g in first:
        assert a["digests"][g] == merged[g], g
