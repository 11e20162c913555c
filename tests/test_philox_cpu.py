"""The CPU restatements of the device's random draws (oracle/philox.py) and of numpy's weighted choice
(oracle/mcts.py::numpy_choice_index), pinned to published known answers, to scipy's Gamma distribution and to numpy
itself.  The GPU tests replay the device's draws through these functions, so they must be right on their own."""
import math

import numpy
import pytest
import scipy.stats

from oracle import mcts as om
from oracle import philox


@pytest.mark.parametrize("counter,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox4x32_10_known_answers(counter, key, want):
    """Random123's kat_vectors for philox4x32_10."""
    assert philox.philox4x32_10(counter, key) == want


def test_uniform53_bit_recipe():
    """Words 0 and 1 of the block at (game_lo, move, c2, game_hi) under key (seed_lo, seed_hi ^ tag), combined like
    numpy's random_sample: (a >> 5) * 2**26 + (b >> 6), over 2**53.  Every tag gives its own stream."""
    seed, game, move = 0x0123456789ABCDEF, 0x1_0000_0007, 11
    for tag in (philox.TAG_ACTION, philox.TAG_RESET):
        for c2 in range(4):
            w = philox.philox4x32_10((game & 0xFFFFFFFF, move, c2, game >> 32), (seed & 0xFFFFFFFF, (seed >> 32) ^ tag))
            u = philox.uniform53(seed, game, move, c2, tag)
            assert u == ((w[0] >> 5) * 2.0 ** 26 + (w[1] >> 6)) * 2.0 ** -53
            assert 0.0 <= u < 1.0 and (u * 2.0 ** 53).is_integer()
    assert philox.uniform53(seed, game, move, 0, philox.TAG_ACTION) != philox.uniform53(seed, game, move, 0, philox.TAG_RESET)
    assert philox.TAG_RESET == 0x7169E004
    # uniform: the mean and the spread of 20 000 draws
    us = numpy.array([philox.uniform53(7, g, 3, 0, philox.TAG_ACTION) for g in range(20000)])
    assert scipy.stats.kstest(us, "uniform").pvalue > 1e-3


@pytest.mark.parametrize("alpha", [0.1, 0.25, 0.3, 1.0, 2.5])
def test_gamma_restatement_is_gamma_distributed(alpha):
    """20 000 draws of the restated philox_gamma (distinct games, moves and counters) pass a Kolmogorov-Smirnov test
    against scipy.stats.gamma(alpha); every decision margin is finite and small margins are rare."""
    draws, margins = [], []
    for i in range(20000):
        v, m = philox.gamma(0x5EED, i // 64, (i // 8) % 8, i % 8, alpha)
        draws.append(v)
        margins.append(m)
    draws = numpy.array(draws)
    assert (draws > 0).all() and numpy.isfinite(draws).all()
    assert scipy.stats.kstest(draws, scipy.stats.gamma(alpha).cdf).pvalue > 1e-3
    assert numpy.mean(numpy.array(margins) < 1e-12) < 1e-3


def test_gamma_boost_uses_counter_word_0xffff():
    """alpha < 1: gamma(alpha) = gamma(alpha + 1) * U ** (1 / alpha) with U from the block whose 4th counter word is
    0xFFFF."""
    for k in range(50):
        base, _ = philox.gamma(3, 9, 2, k, 1.3)
        boosted, _ = philox.gamma(3, 9, 2, k, 0.3)
        w = philox.philox4x32_10((9, 2, k, 0xFFFF), (3, philox.TAG_NOISE))
        assert boosted == base * ((w[0] + 0.5) / 4294967296.0) ** (1.0 / 0.3)


def test_dirichlet_noise_is_normalised_over_the_legal_actions():
    legal = [1, 0, 1, 1, 0, 1, 1]
    noise, margin = philox.dirichlet_noise(1, 2, 3, legal, 0.3)
    assert [n == 0.0 for n in noise] == [not x for x in legal]
    assert abs(sum(noise) - 1.0) < 1e-15 and margin > 0
    for k, ok in enumerate(legal):
        if ok:
            assert noise[k] == philox.gamma(1, 2, 3, k, 0.3)[0] / sum(philox.gamma(1, 2, 3, j, 0.3)[0]
                                                                     for j in range(7) if legal[j])


def _dist(counts, temperature):
    """_sample_action's distribution: visit_counts ** (1 / T) / sum (builtin sum, left to right)."""
    d = numpy.array(counts, dtype="int32") ** (1 / temperature)
    return d / sum(d)


def test_numpy_choice_index_equals_numpy_choice():
    """For many seeds and distributions: numpy_choice_index(p, RandomState(s).random_sample())
    == RandomState(s).choice(len(p), p=p), i.e. legacy choice with p consumes exactly one double and the rule is
    numpy's.  Includes distributions whose sequential cumulative sum does not end at exactly 1."""
    rs = numpy.random.RandomState(0)
    unnormalised_end = 0
    for s in range(3000):
        n = int(rs.choice([2, 7, 9, 33, 121]))
        counts = rs.randint(0, 9, n)
        counts[rs.randint(n)] += 1
        p = _dist(counts, float(rs.choice([1.0, 0.5, 0.25, 0.7])))
        unnormalised_end += numpy.cumsum(p)[-1] != 1.0
        u = numpy.random.RandomState(s).random_sample()
        assert om.numpy_choice_index(p, u) == numpy.random.RandomState(s).choice(n, p=p), (s, p, u)
    assert unnormalised_end > 100


def _boundary_cases():
    """(p, u) pairs on the edges of numpy's rule: u exactly on a normalised boundary cdf_k / cdf[-1], one ulp either
    side, and on the unnormalised boundary cdf_k, for distributions whose cumulative sum does not end at 1."""
    rs = numpy.random.RandomState(1)
    out = []
    while len(out) < 400:
        n = int(rs.choice([7, 9, 121]))
        p = _dist(rs.randint(0, 6, n) + (numpy.arange(n) == 0), float(rs.choice([1.0, 0.5, 0.25])))
        raw = numpy.cumsum(p)
        if raw[-1] == 1.0:
            continue
        cdf = raw / raw[-1]
        for k in range(n - 1):
            if raw[k] != cdf[k] and p[k] > 0:
                for u in (cdf[k], numpy.nextafter(cdf[k], 0), numpy.nextafter(cdf[k], 2), raw[k]):
                    if u < 1.0:
                        out.append((p, float(u)))
    return out


def test_numpy_choice_index_on_boundaries():
    """On every boundary case the restated rule is numpy's own choice.  numpy is driven through a RandomState whose
    next random_sample() is u (a generator with a one-value stream), so the comparison is with numpy's code, not a
    restatement of it."""
    differs = 0
    for p, u in _boundary_cases():
        want = _numpy_choice_with_uniform(p, u)
        assert om.numpy_choice_index(p, u) == want, (p, u)
        raw = numpy.cumsum(p)
        differs += int(numpy.searchsorted(raw, u, side="right")) != want
    assert differs > 0          # the unnormalised rule would pick differently on some of them


def _numpy_choice_with_uniform(p, u):
    """numpy.random.RandomState.choice(len(p), p=p) with its single uniform replaced by u.  Legacy choice draws that
    uniform with self.random_sample(); the subclass returns u from it."""
    class Fixed(numpy.random.RandomState):
        def random_sample(self, size=None):
            return numpy.full(size, u) if size is not None else u
    return int(Fixed(0).choice(len(p), p=p))


def test_injected_draws_choose_like_the_device():
    """select_action with InjectedDraws(uniform=u): numpy's rule at a finite temperature, the first maximum at T = 0,
    floor(u * n) at T = inf."""
    actions, counts = [0, 2, 3, 5], [3, 0, 3, 1]
    assert om.select_action(actions, counts, 0, om.InjectedDraws(uniform=0.9)) == 0
    for u, want in ((0.0, 0), (0.2499999, 0), (0.25, 2), (0.5, 3), (0.75, 5), (math.nextafter(1.0, 0), 5)):
        assert om.select_action(actions, counts, float("inf"), om.InjectedDraws(uniform=u)) == want
    for T in (1.0, 0.5, 0.25):
        p = _dist(counts, T)
        for u in numpy.linspace(0, 1, 41)[:-1]:
            assert om.select_action(actions, counts, T, om.InjectedDraws(uniform=float(u))) == \
                actions[_numpy_choice_with_uniform(p, float(u))]
