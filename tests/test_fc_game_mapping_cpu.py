"""Which games share a warp and an SM in the fused FC search (fc_search.cu: warp_first, the persistent loop's stride, and
the grid of prepare_one), restated in Python from the plan the library makes (host arithmetic only).

At the headline batch every game starts in the one pass, each exactly once, and no SM holds more games than an even
spread over the SMs would give it: re-mapping games to SMs cannot shorten the launch."""
import math

import pytest

from test_fc_plan_cpu import H100, plan


def games_of_cta(b, groups, G, grid, n):
    """Games each lane group of CTA b searches, in the kernel's order (the warp loop runs while its first group has a game)."""
    out = []
    for w in range(groups * G // 32):
        per_warp = 32 // G
        warp_first = b * groups + w * per_warp
        for g0 in range(warp_first, n, grid * groups):
            out += [g0 + k for k in range(per_warp) if g0 + k < n]
    return out


@pytest.mark.parametrize("n", [1, 31, 1000, 3696, 4096, 4224])
def test_every_game_is_searched_once_in_one_pass(n):
    p = plan(n)
    grid = min(math.ceil(n / p["groups"]), p["ctas_per_sm"] * H100["sms"])
    seen = []
    for b in range(grid):
        seen += games_of_cta(b, p["groups"], 16, grid, n)
    assert sorted(seen) == list(range(n))
    assert p["passes"] == 1 and grid * p["groups"] >= n


def test_headline_batch_fills_no_sm_beyond_an_even_spread():
    """4096 games: 512 CTAs of 8 games, at most 4 resident per SM, so no SM holds more than 32 = ceil(4096 / 132) games;
    the 132 SMs split as 116 x 32 + 16 x 24 games."""
    n, sms = 4096, H100["sms"]
    p = plan(n)
    grid = math.ceil(n / p["groups"])
    assert grid <= p["ctas_per_sm"] * sms
    assert p["ctas_per_sm"] * p["groups"] == math.ceil(n / sms) == 32
    full = grid - (p["ctas_per_sm"] - 1) * sms
    assert (full, sms - full) == (116, 16)
