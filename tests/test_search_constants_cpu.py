"""The tree search at search constants no shipped game uses: two-player rewards under a discount below 1, other pb_c
constants and root exploration fractions, value ranges that stay flat at a nonzero value.

The fixtures (tests/golden/mcts_constants.json.gz) are reference searches at the constant sets K1..K4 of
oracle/gen_golden_search_constants.py.  Here oracle/mcts.py and oracle/tree_oracle.c replay every one of them bit for
bit, and the C oracle equals the Python oracle on signed synthetic teachers at every set, both player modes and action
spaces from 2 to 225.  tests/test_search_constants_gpu.py holds the device to the C oracle on the same teachers."""
import copy
import hashlib
import os

import numpy
import pytest

from conftest import GOLDEN, golden_json
from helpers import oracle_replay, teacher_from_cases
from oracle import build_c
from oracle import mcts as om
from oracle.gen_golden_search_constants import CONSTANTS, OVERRIDE_KEYS, load_fixture

KEYS = sorted(CONSTANTS)
FIXTURE = [(k, g) for k in KEYS for g in CONSTANTS[k][4]]


def constants_config(base, key, A=None, P=None):
    """A copy of a game config with set `key`'s search constants (and optionally A actions, P players)."""
    cfg = copy.copy(base)
    cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction = CONSTANTS[key][:4]
    if A is not None:
        cfg.action_space = list(range(A))
    if P is not None:
        cfg.players = list(range(P))
    return cfg


def flat_point(discount, P):
    """(reward r, value v), v != 0, with every backed-up node value equal to v at this discount: r + d * v == v for one
    player, r - d * v == v and -r + d * v == -v for two, all exact in fp64 on fp32 inputs.  A game whose every simulation
    returns (v, r), with root reward r, keeps its value range at lo == hi == v for the whole search, so MinMaxStats.normalize
    must hand back v itself (self_play.py:566-570).  v >= 64 outweighs any exploration term of these searches."""
    for v in range(64, 1024):
        r = v * (1 - discount) if P == 1 else v * (1 + discount)
        r32, v32 = float(numpy.float32(r)), float(numpy.float32(v))
        dv = discount * v32
        if P == 1 and r32 + dv == v32:
            return r32, v32
        if P == 2 and r32 - dv == v32 and -r32 + dv == -v32:
            return r32, v32
    raise AssertionError(f"no exact fixed point at discount {discount}")


N_FLAT = 3          # games 0..2: the flat value range (lo == hi == v != 0), game 0 with priors peaked on one action
N_QUANT = 4         # games 3..6: quantised priors, values and rewards (exact ties below the root)


def signed_teacher(rs, n, N, A, discount, P, legal):
    """Injected network outputs over the whole range the tree must take: rewards of both signs (root rewards too),
    values up to +-50, games with a flat nonzero value range, games quantised for exact ties."""
    def soft(x):
        e = numpy.exp(x - x.max(-1, keepdims=True)).astype(numpy.float32)
        return (e / e.sum(-1, keepdims=True)).astype(numpy.float32)
    scale = rs.choice([1.0, 10.0, 50.0], size=(n, 1)).astype(numpy.float32)
    t = dict(root_value=rs.uniform(-50, 50, n).astype(numpy.float32),
             root_reward=rs.uniform(-1, 1, n).astype(numpy.float32),
             value=(scale * rs.uniform(-1, 1, (n, N))).astype(numpy.float32),
             reward=(scale * rs.uniform(-1, 1, (n, N)) / 5).astype(numpy.float32),
             priors=soft(rs.standard_normal((n, N, A)).astype(numpy.float32)))
    logits = numpy.where(legal > 0, rs.standard_normal((n, A)), -numpy.inf).astype(numpy.float32)
    t["root_priors"] = soft(logits)
    t["root_reward"][-2:] = [0.75, -0.625]            # both signs at the root in every batch
    r, v = flat_point(discount, P)
    t["value"][:N_FLAT], t["reward"][:N_FLAT], t["root_reward"][:N_FLAT] = v, r, r
    # game 0 follows its visited child every simulation: with lo == hi that child's score carries +v, more than any
    # exploration term, so the path grows one level per simulation and the backup leaves the shuffle recurrence once it
    # is a lane group deep
    peaked = numpy.full(A, -8.0, numpy.float32)
    peaked[0] = 8.0
    t["priors"][0] = soft(peaked)
    q = slice(N_FLAT, N_FLAT + N_QUANT)
    w = rs.randint(1, 3, size=(N_QUANT, N, A)).astype(numpy.float32)
    t["priors"][q] = (w / w.sum(-1, keepdims=True)).astype(numpy.float32)
    t["value"][q] = (rs.randint(-4, 5, size=(N_QUANT, N)) / 2).astype(numpy.float32)
    t["reward"][q] = (rs.randint(-2, 3, size=(N_QUANT, N)) / 2).astype(numpy.float32)
    return t


def signed_case(A, P, key, n, N, seed):
    """One batch: legal masks (game 0 keeps action 0 legal), noise, sides to move, Philox keys and the teacher."""
    discount = CONSTANTS[key][0]
    rs = numpy.random.RandomState(seed)
    legal = (rs.uniform(size=(n, A)) < 0.7).astype(numpy.uint8)
    legal[numpy.arange(n), rs.randint(0, A, n)] = 1
    legal[0, 0] = 1
    t = signed_teacher(rs, n, N, A, discount, P, legal)
    noise = rs.dirichlet([0.3] * A, size=n) * legal
    noise /= noise.sum(1, keepdims=True)
    to_play = rs.randint(0, P, n).astype(numpy.int32)
    gid = rs.randint(0, 1 << 40, n).astype(numpy.int64)
    mv = rs.randint(0, 300, n).astype(numpy.int32)
    return t, legal, noise, to_play, gid, mv


def test_fixture_matches_its_manifest():
    m = golden_json("MANIFEST_constants.json")
    for name, digest in m["files"].items():
        assert hashlib.sha256(open(os.path.join(GOLDEN, name), "rb").read()).hexdigest() == digest, name


@pytest.mark.parametrize("key,game", FIXTURE)
def test_fixtures_cover_signed_rewards_at_off_default_constants(key, game, game_configs):
    cfg = game_configs[game]
    runs = load_fixture()[key][game]
    rewards = [s["reward"] for r in runs for s in r["sims"]]
    assert min(rewards) < 0 < max(rewards)
    assert CONSTANTS[key][:4] != (cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction)


@pytest.mark.parametrize("key,game", FIXTURE)
def test_python_oracle_reproduces_reference(key, game, game_configs):
    """Teacher-forced from the reference's own outputs: visit counts, root value, depth, child value sums, every path."""
    cfg = constants_config(game_configs[game], key)
    for c in load_fixture()[key][game]:
        params = om.SearchParams.from_config(cfg, c["num_simulations"])
        ev = om.TableEvaluator((c["root_predicted_value"], c["root_reward"], c["root_priors_raw"]),
                               [(s["value"], s["reward"], s["priors"]) for s in c["sims"]])
        draws = om.InjectedDraws(c["noise"], c["first_index"])
        res = om.TreeSearch(params).run(ev, None, c["legal"], c["to_play"], c["add_noise"], draws)
        assert draws.later_ties == c["later_ties"] == 0
        assert res.root_actions == c["root_actions"] and res.root_visits == c["root_visits"]
        assert res.root_value == c["root_value"] and res.max_tree_depth == c["max_tree_depth"]
        assert res.root_priors == c["root_priors"]
        _, slots = res.tree.children(0)
        assert [res.tree.vsum[s] for s in slots] == c["root_child_value_sums"]
        assert res.tree.vsum[0] == c["root_value_sum"]
        assert [s.path_actions for s in res.sims] == [s["actions"] for s in c["sims"]]


@pytest.mark.parametrize("key,game", FIXTURE)
def test_c_oracle_reproduces_reference(key, game, game_configs):
    cfg = constants_config(game_configs[game], key)
    A, P = len(cfg.action_space), len(cfg.players)
    for c in load_fixture()[key][game]:
        N = c["num_simulations"]
        t, legal, noise, first, to_play = teacher_from_cases([c], A, N)
        r = build_c.tree_search(1, N, A, P, cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction,
                                legal, to_play, noise, first, cfg.seed, None, None, t)
        assert [int(r["visit_counts"][0, a]) for a in c["root_actions"]] == c["root_visits"]
        assert r["root_value"][0] == c["root_value"] and r["max_depth"][0] == c["max_tree_depth"]
        assert r["ties"][0] == 0
        assert [[int(a) for a in r["actions"][0, s, :r["depth"][0, s]]] for s in range(N)] == [s["actions"] for s in c["sims"]]


@pytest.mark.parametrize("key", OVERRIDE_KEYS)
def test_override_fixture_is_a_continued_search(key):
    """The override_root_with cases: the imported subtree's visits are part of the continued root's."""
    fx = load_fixture()["override"][key]
    case = fx["cases"][0]
    assert case["root_visit_count"] == case["pre_visits"] + fx["first"]["num_simulations"]
    assert case["pre_visits"] > 0 and sum(case["root_visits"]) == case["root_visit_count"] - 1


@pytest.mark.parametrize("A", [2, 3, 7, 9, 121, 225])
@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("key", KEYS)
def test_c_oracle_matches_python_oracle_on_signed_teachers(key, P, A, game_configs):
    """Every field of both oracles, game by game, with Philox ties; and the coverage each batch claims."""
    cfg = constants_config(game_configs["cartpole"], key, A, P)
    n, N = (10, 40) if A <= 9 else (7, 36)
    t, legal, noise, to_play, gid, mv = signed_case(A, P, key, n, N, seed=97 * A + 7 * P + KEYS.index(key))
    r = build_c.tree_search(n, N, A, P, cfg.discount, cfg.pb_c_base, cfg.pb_c_init, cfg.root_exploration_fraction,
                            legal, to_play, noise, None, cfg.seed, gid, mv, t, D=N)
    params = om.SearchParams.from_config(cfg, N)
    ties = 0
    for i in range(n):
        acts = [a for a in range(A) if legal[i, a]]
        res, draws = oracle_replay(params, acts, int(to_play[i]),
                                   (t["root_value"][i], t["root_reward"][i], [t["root_priors"][i, a] for a in acts]),
                                   [(t["value"][i, s], t["reward"][i, s], t["priors"][i, s]) for s in range(N)],
                                   [noise[i, a] for a in acts], None, seed=cfg.seed, game=int(gid[i]), move=int(mv[i]))
        assert [int(r["visit_counts"][i, a]) for a in acts] == res.root_visits, i
        assert r["root_value"][i] == res.root_value and r["max_depth"][i] == res.max_tree_depth
        assert r["ties"][i] == draws.later_ties
        assert (r["range"][i, 0], r["range"][i, 1]) == (res.range_lo, res.range_hi)
        assert [[int(a) for a in r["actions"][i, s, :r["depth"][i, s]]] for s in range(N)] == [s.path_actions for s in res.sims]
        ties += draws.later_ties
    _, v = flat_point(cfg.discount, P)
    assert (r["range"][:N_FLAT, 0] == v).all() and (r["range"][:N_FLAT, 1] == v).all()
    assert r["max_depth"][0] == N                     # the peaked flat game descends one level per simulation
    assert ties > 0
