"""Multi-level selection of the fused FC search kernel (tree.cuh::tree_select_lookahead).

With MZ_FC_SELECT_LEVELS=1 the kernel resolves one tree level per selection round (tree_select); by default it scores
D levels per round, D the largest with A + A^2 + ... + A^D <= G.  Both must select the same leaves: visit counts, root
values, value ranges, tie counts, depths and every traced path are compared bit for bit, here between the two settings
and, for injected network outputs, against the C oracle."""
import copy

import numpy
import pytest

from conftest import golden_npz
from helpers import random_teacher
from oracle import mcts as om
from oracle import philox

pytestmark = pytest.mark.gpu


def _levels(A, G):
    D, lanes, w = 1, 0, 1
    for d in range(1, 5):
        w *= max(A, 2)
        if lanes + w > G:
            break
        lanes += w
        D = d
    return D


def _search_both(monkeypatch, eng, **kw):
    """The same search with one level per round and with the default; asserts the fused kernel ran (one launch)."""
    outs = []
    for lv in ("1", None):
        if lv is None:
            monkeypatch.delenv("MZ_FC_SELECT_LEVELS", raising=False)
        else:
            monkeypatch.setenv("MZ_FC_SELECT_LEVELS", lv)
        n0 = eng.launch_count
        outs.append(eng.search(trace=True, **kw))
        assert eng.launch_count == n0 + 1
    return outs


def _assert_same(a, b):
    assert numpy.array_equal(a.visit_counts, b.visit_counts)
    assert numpy.array_equal(a.root_value, b.root_value)
    assert numpy.array_equal(a.value_range, b.value_range)
    assert numpy.array_equal(a.tie_count, b.tie_count)
    assert numpy.array_equal(a.max_tree_depth, b.max_tree_depth)
    assert numpy.array_equal(a.trace["depth"], b.trace["depth"])
    D = a.trace["actions"].shape[-1]
    mask = numpy.arange(D)[None, None, :] < a.trace["depth"][:, :, None]
    assert numpy.array_equal(numpy.where(mask, a.trace["actions"], 0), numpy.where(mask, b.trace["actions"], 0))


@pytest.mark.parametrize("weights", ["synthetic", "pretrained"])
@pytest.mark.parametrize("restricted", [False, True])
def test_cartpole_full_size_one_level_vs_default(weights, restricted, monkeypatch, game_configs):
    """The headline workload (CartPole, 4096 games, N = 50) through the fixed-shape kernel, D = 3 against D = 1;
    `restricted`: partial root legal masks and host-supplied first-simulation tie picks."""
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.netspec import netspec_from_config, synthetic_weights
    cfg = game_configs["cartpole"]
    spec = netspec_from_config(cfg)
    n, N, A = 4096, 50, spec.action_space
    eng = SearchEngine(cfg, max_games=n, num_simulations=N)
    eng.load_weights(synthetic_weights(spec, 0) if weights == "synthetic" else golden_npz("weights_cartpole_pretrained.npz"))
    rs = numpy.random.RandomState(7)
    obs = rs.uniform(-0.05, 0.05, size=(n, spec.obs_elems)).astype(numpy.float32)
    noise = rs.dirichlet([cfg.root_dirichlet_alpha] * A, size=n)
    kw = dict(obs=obs, add_exploration_noise=True, noise=noise, game_id=numpy.arange(n, dtype=numpy.int64),
              trace_depth=N + 1)
    if restricted:
        legal = (rs.uniform(size=(n, A)) < 0.8).astype(numpy.uint8)
        legal[numpy.arange(n), rs.randint(0, A, n)] = 1
        kw.update(legal_mask=legal, first_index=rs.randint(0, A, n).astype(numpy.int32))
    a, b = _search_both(monkeypatch, eng, **kw)
    _assert_same(a, b)
    assert a.max_tree_depth.max() > 3           # deep enough for several rounds per selection
    eng.close()


def _teacher_case(A, P, n, N, seed):
    """Injected outputs quantised so that siblings tie exactly below the root: priors from small integer weights, values
    and rewards on a coarse grid (equal visit counts and equal values give equal scores)."""
    rs = numpy.random.RandomState(seed)
    legal = (rs.uniform(size=(n, A)) < 0.7).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    t = random_teacher(rs, n, N, A, reward_scale=1.0 if P == 1 else 0.0, legal=legal)
    w = rs.randint(1, 3, size=(n, N, A)).astype(numpy.float32)
    quant = rs.uniform(size=n) < 0.5                  # half the games quantised, half continuous
    t["priors"][quant] = (w / w.sum(-1, keepdims=True)).astype(numpy.float32)[quant]
    t["value"][quant] = (rs.randint(-2, 3, size=(n, N)) / 2).astype(numpy.float32)[quant]
    if P == 1:
        t["reward"][quant] = (rs.randint(0, 2, size=(n, N)) / 2).astype(numpy.float32)[quant]
    noise = rs.dirichlet([0.25] * A, size=n)
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    gid = rs.randint(0, 1 << 40, n).astype(numpy.int64)
    mv = rs.randint(0, 400, n).astype(numpy.int32)
    first = rs.randint(0, A, n).astype(numpy.int32)
    return t, legal, noise, to_play, gid, mv, first


def _tie_depths(cfg, N, A, t, legal, noise, to_play, gid, mv, first, games):
    """Depths of the parents of every exact tie the Python oracle draws for, over the given games."""
    params = om.SearchParams.from_config(cfg, N)
    depths = []
    for i in games:
        acts = [a for a in range(A) if legal[i, a]]
        ev = om.TableEvaluator((t["root_value"][i], t["root_reward"][i], [t["root_priors"][i, a] for a in acts]),
                               [(t["value"][i, s], t["reward"][i, s], t["priors"][i, s]) for s in range(N)])

        def tie_fn(n_tied, ctx, i=i):
            if ctx == (0, 0):                         # the supplied pick, clamped like the kernel's first_index
                return min(int(first[i]), n_tied - 1)
            if n_tied > 1:
                depths.append(ctx[1])
            return philox.tie_index(cfg.seed, int(gid[i]), int(mv[i]), ctx[0], ctx[1], n_tied)

        draws = om.InjectedDraws([noise[i, a] for a in acts], None, tie_fn=tie_fn)
        om.TreeSearch(params).run(ev, None, acts, int(to_play[i]), True, draws)
    return depths


@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("A,G", [(2, 16), (3, 16), (4, 16), (5, 16), (8, 16), (2, 32)])
def test_teacher_forced_one_level_vs_default_vs_c_oracle(A, G, P, monkeypatch, game_configs):
    """Injected outputs for A actions in groups of G lanes (D = 3, 2, 1, 1, 1 at G = 16, D = 4 for A = 2 at G = 32),
    partial root legal masks, supplied first-simulation picks: D = 1, the default and the C oracle select the same
    leaves, with exact ties drawn below the root."""
    from muzero_general_b200.engine import SearchEngine
    from oracle import build_c
    cfg = copy.copy(game_configs["cartpole"])
    cfg.action_space = list(range(A))
    cfg.players = list(range(P))
    n, N = 2048, 50
    t, legal, noise, to_play, gid, mv, first = _teacher_case(A, P, n, N, seed=1000 * A + 10 * G + P)
    monkeypatch.setenv("MZ_FC_GROUP", str(G))
    eng = SearchEngine(cfg, max_games=n, num_simulations=N)
    a, b = _search_both(monkeypatch, eng, legal_mask=legal, to_play=to_play, add_exploration_noise=True, noise=noise,
                        first_index=first, game_id=gid, move_index=mv, teacher=t, trace_depth=N + 1, n_games=n)
    eng.close()
    _assert_same(a, b)
    ref = build_c.tree_search(n, N, A, P, cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction,
                              legal, to_play, noise, first, cfg.seed, gid, mv, t, D=N + 1)
    assert (b.visit_counts == ref["visit_counts"]).all()
    assert (b.root_value == ref["root_value"]).all()
    assert (b.max_tree_depth == ref["max_depth"]).all()
    assert (b.tie_count == ref["ties"]).all()
    assert (b.value_range == ref["range"]).all()
    assert (b.trace["depth"] == ref["depth"]).all()
    mask = numpy.arange(N + 1)[None, None, :] < ref["depth"][:, :, None]
    assert (numpy.where(mask, b.trace["actions"], 0) == numpy.where(mask, ref["actions"], 0)).all()
    assert b.tie_count.sum() > 0
    depths = _tie_depths(cfg, N, A, t, legal, noise, to_play, gid, mv, first, range(16))
    D = _levels(A, G)
    assert {d % D for d in depths if d > 0} == set(range(D))    # ties at every level of a round, not only its first
