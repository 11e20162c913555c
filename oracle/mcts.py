"""ORACLE (test infrastructure, never shipped or measured as the product).

CPU restatement of the reference's per-move tree search, ``MCTS.run`` and friends
(``self_play.py:249-476,553-570``), on flat Python lists instead of ``Node`` objects.
All tree arithmetic is Python float (IEEE fp64) in exactly the reference's operation
order, because the device kernels are required to match it bit for bit:

* UCB score                  self_play.py:380-404
* argmax with tie list       self_play.py:363-378
* expansion / prior softmax  self_play.py:451-465
* root Dirichlet mixing      self_play.py:467-476
* backup, both player modes  self_play.py:406-430
* min-max statistics         self_play.py:553-570
* action selection           self_play.py:222-245

Randomness is injected through a ``draws`` object so the same search can be driven by the
reference's legacy global ``numpy.random`` stream (to reproduce the golden fixtures made
by ``oracle/gen_golden.py`` from the reference itself) or by the counter-based Philox
stream the device uses (``oracle/philox.py``).

Pinned against: ``tests/golden/*.json`` (reference outputs; see ``oracle/gen_golden.py``).
Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import
this file.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy


# ----------------------------------------------------------------------------- parameters
@dataclass
class SearchParams:
    num_simulations: int
    action_space: Sequence[int]
    players: Sequence[int]
    discount: float
    pb_c_base: float
    pb_c_init: float
    root_dirichlet_alpha: float
    root_exploration_fraction: float

    @classmethod
    def from_config(cls, config, num_simulations=None):
        return cls(
            num_simulations=config.num_simulations if num_simulations is None else num_simulations,
            action_space=list(config.action_space),
            players=list(config.players),
            discount=config.discount,
            pb_c_base=config.pb_c_base,
            pb_c_init=config.pb_c_init,
            root_dirichlet_alpha=config.root_dirichlet_alpha,
            root_exploration_fraction=config.root_exploration_fraction,
        )


# ----------------------------------------------------------------------------- random draws
class LegacyNumpyDraws:
    """The reference's draw order on a legacy numpy stream (self_play.py:22,371,473,236,243).

    ``rs=None`` uses the process-global ``numpy.random`` exactly like the reference.
    """

    def __init__(self, rs=None):
        self.rs = numpy.random if rs is None else rs

    def dirichlet(self, alpha, n, ctx=None):
        return self.rs.dirichlet([alpha] * n)

    def tie_index(self, n_tied, ctx=None):
        # numpy.random.choice(list) == list[randint(0, len(list))]; no state consumed for n=1
        return int(self.rs.choice(n_tied))

    def sample_index(self, probabilities, ctx=None):
        return int(self.rs.choice(len(probabilities), p=probabilities))

    def uniform_index(self, n, ctx=None):
        return int(self.rs.choice(n))


class InjectedDraws:
    """Draws supplied by the caller (what the C-ABI accepts as host-provided draws).

    ``noise``        Dirichlet sample for this search (length = number of legal actions)
    ``first_index``  index into the root's child list picked at the first simulation
    ``tie_fn``       called for any later exact tie: tie_fn(n_tied, ctx) -> index
    ``uniform``      the uniform in [0, 1) behind the action choice: ``numpy_choice_index`` at a finite temperature,
                     ``floor(uniform * n)`` at T = inf (the device's documented rule)
    """

    def __init__(self, noise=None, first_index=None, tie_fn=None, uniform=None):
        self.noise = noise
        self.first_index = first_index
        self.tie_fn = tie_fn
        self.uniform = uniform
        self.later_ties = 0

    def sample_index(self, probabilities, ctx=None):
        assert self.uniform is not None, "no uniform supplied for the action choice"
        return numpy_choice_index(probabilities, self.uniform)

    def uniform_index(self, n, ctx=None):
        assert self.uniform is not None, "no uniform supplied for the action choice"
        return min(int(self.uniform * n), n - 1)

    def dirichlet(self, alpha, n, ctx=None):
        assert self.noise is not None and len(self.noise) == n
        return self.noise

    def tie_index(self, n_tied, ctx=None):
        sim, depth = ctx
        if sim == 0 and depth == 0 and self.first_index is not None:
            return int(self.first_index)
        if n_tied > 1 and not (sim == 0 and depth == 0):     # the first simulation's all-way tie is expected
            self.later_ties += 1
        if self.tie_fn is None:
            assert n_tied == 1, "unexpected exact tie and no tie_fn supplied"
            return 0
        return int(self.tie_fn(n_tied, ctx))


# ----------------------------------------------------------------------------- statistics
class RunningRange:
    """self_play.py:553-570"""

    def __init__(self):
        self.hi = -float("inf")
        self.lo = float("inf")

    def update(self, v):
        self.hi = max(self.hi, v)
        self.lo = min(self.lo, v)

    def normalize(self, v):
        if self.hi > self.lo:
            return (v - self.lo) / (self.hi - self.lo)
        return v


# ----------------------------------------------------------------------------- the tree
@dataclass
class Tree:
    """Flat storage. Slot 0 is the root; every expansion appends one block of child slots."""
    visit: List[int] = field(default_factory=lambda: [0])
    vsum: List[float] = field(default_factory=lambda: [0])
    prior: List[float] = field(default_factory=lambda: [0])
    reward: List[float] = field(default_factory=lambda: [0])
    to_play: List[int] = field(default_factory=lambda: [-1])
    block: List[int] = field(default_factory=lambda: [-1])   # slot -> expansion id or -1
    state: List[object] = field(default_factory=lambda: [None])
    # per expansion
    base: List[int] = field(default_factory=list)            # first child slot
    acts: List[List[int]] = field(default_factory=list)      # actions of the children, in order

    def value(self, s):
        if self.visit[s] == 0:
            return 0
        return self.vsum[s] / self.visit[s]

    def expand(self, s, actions, to_play, reward, priors, state):
        self.to_play[s] = to_play
        self.reward[s] = reward
        self.state[s] = state
        e = len(self.base)
        self.block[s] = e
        self.base.append(len(self.visit))
        self.acts.append(list(actions))
        for p in priors:
            self.visit.append(0)
            self.vsum.append(0)
            self.prior.append(p)
            self.reward.append(0)
            self.to_play.append(-1)
            self.block.append(-1)
            self.state.append(None)
        return e

    def children(self, s):
        e = self.block[s]
        b = self.base[e]
        return self.acts[e], range(b, b + len(self.acts[e]))


@dataclass
class SimRecord:
    path_actions: List[int]
    path_slots: List[int]
    value: float
    reward: float
    priors: List[float]
    leaf_to_play: int


@dataclass
class SearchResult:
    tree: Tree
    root_actions: List[int]
    root_visits: List[int]
    root_value: float
    max_tree_depth: int
    root_predicted_value: Optional[float]
    root_priors: List[float]           # after noise
    root_priors_raw: List[float]       # before noise
    noise: Optional[List[float]]
    sims: List[SimRecord]
    range_lo: float = float("inf")
    range_hi: float = -float("inf")


class TreeSearch:
    def __init__(self, params: SearchParams):
        self.p = params

    # self_play.py:380-404
    def _score(self, tree, parent, child, rng):
        p = self.p
        c = math.log((tree.visit[parent] + p.pb_c_base + 1) / p.pb_c_base) + p.pb_c_init
        c *= math.sqrt(tree.visit[parent]) / (tree.visit[child] + 1)
        u = c * tree.prior[child]
        if tree.visit[child] > 0:
            q = tree.value(child)
            v = rng.normalize(tree.reward[child] + p.discount * (q if len(p.players) == 1 else -q))
        else:
            v = 0
        return u + v

    # self_play.py:363-378
    def _pick(self, tree, s, rng, draws, ctx):
        acts, slots = tree.children(s)
        scores = [self._score(tree, s, c, rng) for c in slots]
        best = max(scores)
        tied = [i for i, x in enumerate(scores) if x == best]
        i = tied[draws.tie_index(len(tied), ctx)]
        return acts[i], slots[i]

    # self_play.py:406-430
    def _backup(self, tree, path, value, to_play, rng):
        p = self.p
        if len(p.players) == 1:
            for s in reversed(path):
                tree.vsum[s] += value
                tree.visit[s] += 1
                rng.update(tree.reward[s] + p.discount * tree.value(s))
                value = tree.reward[s] + p.discount * value
        elif len(p.players) == 2:
            for s in reversed(path):
                tree.vsum[s] += value if tree.to_play[s] == to_play else -value
                tree.visit[s] += 1
                rng.update(tree.reward[s] + p.discount * -tree.value(s))
                value = (-tree.reward[s] if tree.to_play[s] == to_play else tree.reward[s]) \
                    + p.discount * value
        else:
            raise NotImplementedError("More than two player mode not implemented.")

    # self_play.py:260-361
    def run(self, evaluator, observation, legal_actions, to_play, add_exploration_noise, draws):
        p = self.p
        tree = Tree()
        value0, reward0, priors0, state0 = evaluator.root(observation, legal_actions)
        assert legal_actions, f"Legal actions should not be an empty array. Got {legal_actions}."
        assert set(legal_actions).issubset(set(p.action_space)), \
            "Legal actions should be a subset of the action space."
        tree.expand(0, legal_actions, to_play, reward0, priors0, state0)
        raw = list(priors0)
        noise = None
        if add_exploration_noise:
            noise = draws.dirichlet(p.root_dirichlet_alpha, len(legal_actions))
            f = p.root_exploration_fraction
            _, slots = tree.children(0)
            for c, n in zip(slots, noise):
                tree.prior[c] = tree.prior[c] * (1 - f) + n * f      # self_play.py:476
            noise = [float(n) for n in noise]

        rng = RunningRange()
        deepest = 0
        sims = []
        for sim in range(p.num_simulations):
            vtp = to_play
            s = 0
            path = [0]
            acts_taken = []
            depth = 0
            while tree.block[s] >= 0:
                a, s = self._pick(tree, path[-1], rng, draws, (sim, depth))
                depth += 1
                path.append(s)
                acts_taken.append(a)
                vtp = p.players[vtp + 1] if vtp + 1 < len(p.players) else p.players[0]
            parent = path[-2]
            value, reward, priors, state = evaluator.step(tree.state[parent], acts_taken[-1])
            tree.expand(s, p.action_space, vtp, reward, priors, state)
            self._backup(tree, path, value, vtp, rng)
            deepest = max(deepest, depth)
            sims.append(SimRecord(acts_taken, list(path), value, reward, list(priors), vtp))

        acts, slots = tree.children(0)
        return SearchResult(
            tree=tree,
            root_actions=list(acts),
            root_visits=[tree.visit[c] for c in slots],
            root_value=tree.value(0),
            max_tree_depth=deepest,
            root_predicted_value=value0,
            root_priors=[tree.prior[c] for c in slots],
            root_priors_raw=raw,
            noise=noise,
            sims=sims,
            range_lo=rng.lo,
            range_hi=rng.hi,
        )


# ----------------------------------------------------------------------------- evaluators
class ModelEvaluator:
    """Batch-1 network calls + scalarisation exactly like self_play.py:279-295,339-351."""

    def __init__(self, net, support_size):
        from oracle.net import prior_softmax, support_to_scalar
        self.net = net
        self.S = support_size
        self._s2s = support_to_scalar
        self._soft = prior_softmax
        self.calls = 0

    def root(self, observation, legal_actions):
        import torch
        obs = torch.tensor(numpy.asarray(observation)).float().unsqueeze(0)
        v, r, pol, h = self.net.initial_inference(obs)
        self.calls += 1
        return (self._s2s(v, self.S).item(), self._s2s(r, self.S).item(),
                self._soft(pol[0], legal_actions), h)

    def step(self, state, action):
        import torch
        v, r, pol, h = self.net.recurrent_inference(state, torch.tensor([[action]]))
        self.calls += 1
        acts = list(range(pol.shape[1]))
        return (self._s2s(v, self.S).item(), self._s2s(r, self.S).item(),
                self._soft(pol[0], acts), h)


class TableEvaluator:
    """Teacher forcing: per-simulation outputs come from a table, independent of the path.

    table["root"] = (value, reward, priors); table["sims"][i] = (value, reward, priors).
    """

    def __init__(self, root, sims):
        self._root = root
        self._sims = sims
        self._i = 0

    def root(self, observation, legal_actions):
        v, r, pri = self._root
        return float(v), float(r), [float(x) for x in pri], None

    def step(self, state, action):
        v, r, pri = self._sims[self._i]
        self._i += 1
        return float(v), float(r), [float(x) for x in pri], None


# ----------------------------------------------------------------------------- action choice
def numpy_choice_index(p, u):
    """The index ``numpy.random.RandomState.choice(len(p), p=p)`` returns when its one uniform draw is ``u``.

    Legacy ``choice`` with ``p`` consumes exactly one ``random_sample()`` double and computes
    ``cdf = p.cumsum(); cdf /= cdf[-1]; cdf.searchsorted(u, side="right")``.  The division by ``cdf[-1]`` matters:
    the sequential cumulative sum of ``dist / sum(dist)`` often ends one ulp away from 1, which moves interior
    boundaries by an ulp."""
    cdf = numpy.cumsum(numpy.asarray(p, dtype=numpy.float64))
    cdf /= cdf[-1]
    return int(cdf.searchsorted(u, side="right"))


def select_action(actions, visit_counts, temperature, draws, ctx=None):
    """self_play.py:222-245 on the root's (actions, visit counts) in child order."""
    counts = numpy.array(visit_counts, dtype="int32")
    if temperature == 0:
        return actions[int(numpy.argmax(counts))]
    if temperature == float("inf"):
        return actions[draws.uniform_index(len(actions), ctx)]
    dist = counts ** (1 / temperature)
    dist = dist / sum(dist)
    return actions[draws.sample_index(dist, ctx)]


def child_visit_policy(action_space, actions, visit_counts):
    """self_play.py:496-507"""
    total = sum(visit_counts)
    lut = dict(zip(actions, visit_counts))
    return [lut[a] / total if a in lut else 0 for a in action_space]


def stacked_observation(observations, actions, index, num_stacked, action_space_size):
    """self_play.py:513-550 - current frame, then (frame, action plane) pairs, newest first."""
    index = index % len(observations)
    out = [numpy.asarray(observations[index]).copy()]
    like = out[0][0]
    for past in range(index - 1, index - num_stacked - 1, -1):
        if past >= 0:
            out.append(numpy.asarray(observations[past]))
            out.append(numpy.asarray([numpy.ones_like(like) * actions[past + 1] / action_space_size]))
        else:
            out.append(numpy.zeros_like(out[0]))
            out.append(numpy.asarray([numpy.zeros_like(like)]))
    return numpy.concatenate(out)
