"""Case table of the fused CUDA-core tower (csrc/small_tower.cu: small_tower_kernel<P, CO> and its planner, reached through
mz_debug_small_tower / mz_debug_small_tower_plan).  Importable without a GPU.

The planner picks CO (output channels per thread) = 4 once n * (C / 4) * H reaches 384 threads per SM, else 1; P (pixels
per thread) = W, or W / 2 for CO = 1 on even boards of width >= 4 when twice the threads still fit in a CTA; then boards per
CTA, CTAs per SM and a persistent grid.  Every case names the (P, CO) it targets.  The batches of the CO = 4 cases and of
the cases that take more than one round of resident tiles depend on the SM count, so they are chosen through the plan
query at run time (``batch``); tests/test_small_tower_plan_cpu.py asserts at 132 and 114 SMs what the table reaches:

  * all 14 instantiations, P in 2..8 x CO in {1, 4}
  * boards of W = 2..8 and H = 1..16; C = 4..32, C = 8 with 11 input planes (cap_channels > C); in_channels 1 and 3
  * 0..4 blocks after a stem and 1..5 without (one more is refused: the 10-layer cap)
  * batches of 1, ragged last tiles, more boards than one round of resident tiles
  * the four call sites of resnet_inference, parts 2..4 at the in-search site
"""
from __future__ import annotations

from dataclasses import dataclass

SITES = ("representation", "dynamics", "dynamics_pool", "prediction")
INSTANTIATIONS = {(P, CO) for P in range(2, 9) for CO in (1, 4)}


@dataclass(frozen=True)
class TowerCase:
    name: str
    site: str
    C: int
    H: int
    W: int
    blocks: int
    target: tuple          # (P, CO)
    n: object              # boards: an int, "co4" (+ extra) or "rounds"
    extra: int = 0
    cin: int = 0           # observation planes at the representation site
    parts: int = 1

    @property
    def stem(self):
        return self.site != "prediction"

    @property
    def in_channels(self):
        """Planes of the tower input as stored (x's second dimension)."""
        return self.cin if self.site == "representation" else self.C

    @property
    def stem_cin(self):
        """Planes the first conv reads (the plan query's in_channels)."""
        return {"representation": self.cin, "prediction": self.C}.get(self.site, self.C + 1)

    @property
    def layers(self):
        return self.stem + 2 * self.blocks


def _case(name, site, C, H, W, blocks, target, n, extra=0, cin=3, parts=1):
    return TowerCase(name, site, C, H, W, blocks, target, n, extra, cin if site == "representation" else 0, parts)


CASES = [
    # CO = 1 (small batches)
    _case("p2_co1_1x2_n1", "representation", 16, 1, 2, 0, (2, 1), 1, cin=1),
    _case("p2_co1_c4_half_rows", "dynamics", 4, 5, 4, 2, (2, 1), 7),
    _case("p3_co1_3x3_parts2", "dynamics_pool", 16, 3, 3, 2, (3, 1), 701, parts=2),
    _case("p4_co1_8x8_half_rows", "prediction", 16, 8, 8, 1, (4, 1), 5),
    _case("p5_co1_5x5", "dynamics", 12, 5, 5, 3, (5, 1), 23),
    _case("p6_co1_c24_15x6", "prediction", 24, 15, 6, 1, (6, 1), 3),
    _case("p7_co1_c8_11_planes", "representation", 8, 6, 7, 2, (7, 1), 9, cin=11),
    _case("p8_co1_c24_16x8", "representation", 24, 16, 8, 1, (8, 1), 2, cin=3),
    # CO = 4 (from n (C / 4) H >= 384 S on)
    _case("p2_co4_16x2_parts3", "dynamics_pool", 32, 16, 2, 1, (2, 4), "co4", 5, parts=3),
    _case("p3_co4_16x3", "prediction", 16, 16, 3, 2, (3, 4), "co4", 1),
    _case("p4_co4_16x4", "representation", 16, 16, 4, 1, (4, 4), "co4", 0, cin=3),
    _case("p5_co4_c32_8x5", "dynamics", 32, 8, 5, 1, (5, 4), "co4", 2),
    _case("p6_co4_6x6_rounds", "dynamics_pool", 16, 6, 6, 4, (6, 4), "rounds"),
    _case("p7_co4_c32_6x7", "prediction", 32, 6, 7, 2, (7, 4), "co4", 9),
    _case("p8_co4_c32_16x8_rounds", "prediction", 32, 16, 8, 1, (8, 4), "rounds"),
    # every depth: 0..4 blocks after a stem, 1..5 without (5 blocks = 10 layers, the cap)
    *[_case(f"depth_rep_b{b}", "representation", 16, 3, 3, b, (3, 1), 1 + 4 * b, cin=3) for b in range(5)],
    *[_case(f"depth_dyn_b{b}", "dynamics", 8, 4, 6, b, (3, 1), 11 + b) for b in range(5)],
    _case("depth_pool_b4_parts4", "dynamics_pool", 8, 4, 6, 4, (3, 1), 29, parts=4),
    *[_case(f"depth_pred_b{b}", "prediction", 16, 3, 3, b, (3, 1), 2 + 3 * b) for b in range(1, 5)],
    _case("depth_pred_b5_boards", "prediction", 16, 3, 3, 5, (3, 1), 301),
]

BY_NAME = {c.name: c for c in CASES}

# shapes the fused tower refuses, with the reason the plan query gives: (n, in_channels, C, H, W, blocks, stem)
REFUSED = [
    ((4, 17, 16, 6, 9, 1, True), "rows x 2..8 columns"),          # W = 9
    ((4, 17, 16, 17, 3, 1, True), "rows x 2..8 columns"),         # H = 17
    ((4, 7, 6, 3, 3, 1, True), "multiple of 4"),                  # C % 4 != 0
    ((4, 17, 16, 3, 3, 5, True), "1 to 10 layers"),               # 11 layers after a stem
    ((4, 16, 16, 3, 3, 6, False), "1 to 10 layers"),              # 12 layers without
]


def partition_games(n, parts):
    """Boards per range of the partitioned replay (pipeline.h::partition_games): the last range may hold fewer."""
    return ((n + parts - 1) // parts + 7) & ~7


def first_range(n, parts):
    return min(n, partition_games(n, parts))


def plan_of(plan_fn, case, n, S):
    p, why = plan_fn(n, case.stem_cin, case.C, case.H, case.W, case.blocks, case.stem, S)
    assert p is not None, (case.name, n, S, why)
    return p


def batch(case, S, plan_fn):
    """Boards of the case on S SMs; ``plan_fn`` is engine.debug_small_tower_plan."""
    if isinstance(case.n, int):
        return case.n
    # the smallest first range that gets CO = 4 (CO only grows with n)
    lo, hi = 1, 1 << 20
    while lo < hi:
        mid = (lo + hi) // 2
        if plan_of(plan_fn, case, mid, S)["CO"] == 4:
            hi = mid
        else:
            lo = mid + 1
    if case.n == "co4":
        return case.parts * lo + case.extra
    # "rounds": grow the batch until its tiles outnumber the resident CTAs, then make the last tile ragged
    n = lo
    while True:
        p = plan_of(plan_fn, case, n, S)
        if -(-n // p["boards"]) > p["grid"]:
            break
        n = n * 3 // 2 + 1
    while n % plan_of(plan_fn, case, n, S)["boards"] == 0:
        n += 1
    return n


def case_plan(case, S, plan_fn):
    """(boards, plan of the launch of the first range)."""
    n = batch(case, S, plan_fn)
    return n, plan_of(plan_fn, case, first_range(n, case.parts), S)
