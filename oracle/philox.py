"""ORACLE (test infrastructure). Philox4x32-10 counter-based generator in plain Python.

Restates the published algorithm (Salmon et al., "Parallel random numbers: as easy as
1, 2, 3", SC'11; constants M0=0xD2511F53, M1=0xCD9E8D57, W0=0x9E3779B9, W1=0xBB67AE85)
that ``muzero_general_b200/csrc/common.cuh`` implements on the device, and the draws the device
builds from it (``common.cuh``: tie indices, ``philox_gamma``; ``csrc/selfplay.cu``:
``philox_uniform53``), so that every random decision of the GPU can be replayed on the CPU.
Known-answer vectors from the Random123 distribution, the uniform's bit recipe and the gamma
sampler's distribution are checked in ``tests/test_philox_cpu.py``.
"""
import math

M0 = 0xD2511F53
M1 = 0xCD9E8D57
W0 = 0x9E3779B9
W1 = 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(counter, key):
    c0, c1, c2, c3 = (int(x) & MASK for x in counter)
    k0, k1 = (int(x) & MASK for x in key)
    for _ in range(10):
        p0 = M0 * c0
        p1 = M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & MASK, p1 & MASK, ((p0 >> 32) ^ c3 ^ k1) & MASK, p0 & MASK
        k0 = (k0 + W0) & MASK
        k1 = (k1 + W1) & MASK
    return c0, c1, c2, c3


# Stream tags (key word 1 is seed_hi ^ tag); must match csrc/common.cuh and csrc/selfplay.cu (kTagReset)
TAG_TIE = 0x7169E001
TAG_NOISE = 0x7169E002
TAG_ACTION = 0x7169E003
TAG_RESET = 0x7169E004


def tie_index(seed, game, move, sim, depth, n_tied):
    """Index in [0, n_tied) used by the device for an exact UCB tie (mulhi of word 0)."""
    w = philox4x32_10((game & MASK, move, sim, depth), (seed & MASK, ((seed >> 32) & MASK) ^ TAG_TIE))
    return (w[0] * n_tied) >> 32


def uniform53(seed, game, move, c2, tag):
    """``philox_uniform53``: a double in [0, 1) with 53 random bits, built like numpy's ``random_sample`` from words
    0 and 1 of the block at counter (game_lo, move, c2, game_hi), key (seed_lo, seed_hi ^ tag).  Exact: every step
    is an integer below 2**53 or a power-of-two scaling."""
    w = philox4x32_10((game & MASK, move, c2, (game >> 32) & MASK), (seed & MASK, ((seed >> 32) & MASK) ^ tag))
    return ((w[0] >> 5) * 67108864 + (w[1] >> 6)) / 9007199254740992.0


def _open_unit(word):
    return (word + 0.5) * (1.0 / 4294967296.0)


def gamma(seed, game, move, counter, alpha):
    """``philox_gamma`` (csrc/common.cuh): a Gamma(alpha, 1) draw -> (value, margin).

    Marsaglia & Tsang (2000) on a = alpha (alpha + 1 when alpha < 1); iteration ``it`` takes the block at counter
    (game_lo, move, counter, it) under TAG_NOISE: word 0 and 1 give a Box-Muller normal, word 2 the acceptance
    uniform.  After 64 rejections the device returns d = a - 1/3.  For alpha < 1 the result is multiplied by
    U ** (1 / alpha), U from word 0 of the block at counter word 3 = 0xFFFF.

    The device's ``log``, ``cospi`` and ``pow`` are not correctly rounded, and Python's ``cos(2 pi u)`` is not
    ``cospi(2 u)``, so the value agrees to a few ulps, and an accept / reject decision taken within such an error of
    its threshold could go the other way.  ``margin`` is the smallest relative distance of any decision made from
    its threshold; callers skip draws whose margin is below ~1e-12."""
    a = alpha + 1.0 if alpha < 1.0 else alpha
    d = a - 1.0 / 3.0
    c = 1.0 / math.sqrt(9.0 * d)
    key = (seed & MASK, ((seed >> 32) & MASK) ^ TAG_NOISE)
    out = d
    margin = math.inf
    for it in range(64):
        w = philox4x32_10((game & MASK, move, counter, it), key)
        u1, u2, u3 = _open_unit(w[0]), _open_unit(w[1]), _open_unit(w[2])
        x = math.sqrt(-2.0 * math.log(u1)) * math.cos(2.0 * math.pi * u2)
        t = 1.0 + c * x
        margin = min(margin, abs(t))
        if t <= 0.0:
            continue
        v = t * t * t
        lhs, rhs = math.log(u3), 0.5 * x * x + d - d * v + d * math.log(v)
        margin = min(margin, abs(lhs - rhs) / max(1.0, abs(lhs), abs(rhs)))
        if lhs < rhs:
            out = d * v
            break
    if alpha < 1.0:
        w = philox4x32_10((game & MASK, move, counter, 0xFFFF), key)
        out *= _open_unit(w[0]) ** (1.0 / alpha)
    return out, margin


def dirichlet_noise(seed, game, move, legal, alpha):
    """Root noise as the device draws it when the host passes none: Gamma draws keyed by the action index,
    normalised over the legal actions (zero elsewhere) -> (noise list, smallest margin)."""
    draws = [gamma(seed, game, move, k, alpha) if ok else (0.0, math.inf) for k, ok in enumerate(legal)]
    total = sum(v for v, _ in draws)
    return [v / total for v, _ in draws], min(m for _, m in draws)
