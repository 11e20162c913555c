"""Case table of the residual heads (csrc/heads.cuh::heads_one_sample run by heads_kernel<32> and heads_kernel<128>, and the
generic big_*_kernel route, reached through mz_debug_heads / mz_debug_heads_plan).  Importable without a GPU.

The planner takes heads_kernel<32> (one warp per sample; two heads of the prediction site share it, 16 lanes each) when
C*H*W <= 1024, heads_kernel<128> otherwise, min(groups, ceil(n / SMs)) groups per CTA, fewer while the head weights and the
groups' tiles exceed 227 KB, and the generic route when even one group does not fit.  Every case names the route it
targets; the batches marked "persist" hold more samples than grid x groups, so they depend on the SM count.
tests/test_heads_plan_cpu.py asserts at 132 and 114 SMs what the table reaches:

  * the three routes, and a case whose groups per CTA are cut down by shared memory
  * one head at span 32 and two heads sharing a warp at span 16; split-K ks = 1, 2, 4 and 8 (``ks_of`` restates the rule)
  * C a power of two and not (20, 48); H*W = 1; boards up to 16 x 8 dense; C*H*W on both sides of 1024
  * reduced channels 1, 2, 3, 5, 16; hidden layers [], [16], [3, 9], [128], [256, 256], value and policy of different
    depths in one launch; logits 1, 3, 7, 21 (S = 10) and 601 (S = 300)
  * the three layouts at every site that uses them; batches of 1, ragged last groups, more samples than grid x groups;
    parts 2..4 at the in-search site
"""
from __future__ import annotations

from dataclasses import dataclass

SITES = ("representation", "dynamics", "dynamics_pool", "prediction")
ROUTES = ("warp", "wide", "generic")
SMEM_LIMIT = 227 * 1024
GROUP_THREADS = {"warp": 32, "wide": 128}


@dataclass(frozen=True)
class HeadsCase:
    name: str
    site: str
    C: int
    H: int
    W: int
    layout: str
    heads: tuple           # ((reduced channels, hidden widths, logits), ...) of the site's heads
    n: object              # samples: an int or "persist"
    route: str             # the planned route
    parts: int = 1
    pool_stride: int = 3
    out_slot: int = 1

    @property
    def HW(self):
        return self.H * self.W

    @property
    def S(self):
        return (self.heads[0][2] - 1) // 2 if self.heads else 0


def _c(name, site, C, H, W, layout, heads, n, route, parts=1):
    return HeadsCase(name, site, C, H, W, layout, tuple((rc, tuple(h), o) for rc, h, o in heads), n, route, parts)


CASES = [
    # rescale only
    _c("rep_warp_c16_3x3_n1", "representation", 16, 3, 3, "dense", [], 1, "warp"),
    _c("rep_wide_c48_5x5", "representation", 48, 5, 5, "dense", [], 37, "wide"),
    _c("rep_warp_c20_5x5_persist", "representation", 20, 5, 5, "dense", [], "persist", "warp"),
    _c("rep_wide_c16_16x8", "representation", 16, 16, 8, "dense", [], 5, "wide"),
    _c("rep_f16_6x7", "representation", 64, 6, 7, "f16", [], 45, "wide"),
    _c("rep_split_3x3", "representation", 64, 3, 3, "split", [], 7, "warp"),
    # reward head + rescale (one head, span 32 on the narrow kernel)
    _c("dyn_warp_ks4_c16_3x3", "dynamics", 16, 3, 3, "dense", [(16, [], 7)], 29, "warp"),
    _c("dyn_warp_ks8_c20_5x5", "dynamics", 20, 5, 5, "dense", [(16, [], 3)], 133, "warp"),
    _c("dyn_wide_c32_16x8_rc5", "dynamics", 32, 16, 8, "dense", [(5, [16], 21)], 9, "wide"),
    _c("dyn_hw1_s0", "dynamics", 16, 1, 1, "dense", [(3, [], 1)], 5, "warp"),
    _c("dyn_f16_6x7", "dynamics", 64, 6, 7, "f16", [(2, [], 21)], 11, "wide"),
    _c("dyn_split_6x7", "dynamics", 64, 6, 7, "split", [(1, [16], 21)], 3, "wide"),
    _c("pool_warp_c16_3x3_parts2", "dynamics_pool", 16, 3, 3, "dense", [(16, [], 21)], 301, "warp", 2),
    _c("pool_split_6x7_parts3", "dynamics_pool", 64, 6, 7, "split", [(2, [], 21)], 67, "wide", 3),
    _c("pool_f16_3x3_parts4", "dynamics_pool", 64, 3, 3, "f16", [(3, [], 7)], 29, "warp", 4),
    _c("pool_wide_c48_5x5_parts4", "dynamics_pool", 48, 5, 5, "dense", [(5, [16], 21)], 100, "wide", 4),
    # value + policy heads (two heads: span 16 each on the narrow kernel)
    _c("pred_warp_shared_depths", "prediction", 16, 3, 3, "dense", [(2, [], 21), (3, [3, 9], 7)], 40, "warp"),
    _c("pred_warp_ks2_c16_4x4", "prediction", 16, 4, 4, "dense", [(5, [], 3), (2, [16], 7)], 23, "warp"),
    _c("pred_warp_ks4_c16_8x8_persist", "prediction", 16, 8, 8, "dense", [(2, [], 3), (16, [16], 1)], "persist", "warp"),
    _c("pred_warp_s300", "prediction", 16, 3, 3, "dense", [(1, [], 601), (2, [], 3)], 9, "warp"),
    _c("pred_wide_s300_c48", "prediction", 48, 5, 5, "dense", [(2, [16], 601), (16, [], 7)], 13, "wide"),
    _c("pred_generic_256x256", "prediction", 16, 16, 8, "dense", [(16, [256, 256], 21), (16, [], 7)], 6, "generic"),
    _c("pred_wide_shrunk_persist", "prediction", 32, 16, 8, "dense", [(4, [32], 21), (4, [], 7)], "persist", "wide"),
    _c("pred_f16_6x7", "prediction", 64, 6, 7, "f16", [(2, [], 21), (4, [], 7)], 50, "wide"),
    _c("pred_split_3x3", "prediction", 64, 3, 3, "split", [(3, [16], 21), (5, [128], 7)], 17, "warp"),
    _c("pred_hw1_n1", "prediction", 16, 1, 1, "dense", [(5, [], 1), (3, [], 3)], 1, "warp"),
]

BY_NAME = {c.name: c for c in CASES}


def ks_of(span, in_width, out_width, group=32):
    """Split-K width of one FC layer (heads.cuh): adjacent lanes that share one output's dot product, narrow kernel only."""
    ks = 1
    if group == 32:
        in4, out4 = (in_width + 3) // 4, (out_width + 3) // 4 * 4
        while ks < 8 and 2 * ks * out4 <= span and in4 >= 16 * ks:
            ks *= 2
    return ks


def layer_ks(case, route):
    """[[ks of each FC layer] per head] of the case on ``route``."""
    if route == "generic" or not case.heads:
        return [[1] * (len(h[1]) + 1) for h in case.heads]
    group = GROUP_THREADS[route]
    span = group // len(case.heads)
    out = []
    for rc, hidden, n_out in case.heads:
        widths = [rc * case.HW, *hidden, n_out]
        out.append([ks_of(span, widths[i], widths[i + 1], group) for i in range(len(widths) - 1)])
    return out


def partition_games(n, parts):
    """Samples per range of the partitioned replay (pipeline.h::partition_games): the last range may hold fewer."""
    return ((n + parts - 1) // parts + 7) & ~7


def first_range(n, parts):
    return min(n, partition_games(n, parts))


def batch(case, S):
    """Samples of the case on S SMs: "persist" holds more than twice the most samples one wave of CTAs can take."""
    if isinstance(case.n, int):
        return case.n
    return 2 * (1024 // GROUP_THREADS[case.route]) * S + 3


def case_plan(case, S, plan_fn, route="planned"):
    """(samples, plan of the launch of the first range); ``plan_fn`` is engine.debug_heads_plan."""
    n = batch(case, S)
    p, why = plan_fn(first_range(n, case.parts), case.C, case.H, case.W, case.heads, case.site, case.layout, route, 0, S)
    assert p is not None, (case.name, S, why)
    return n, p
