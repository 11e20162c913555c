"""Cases of the DownsampleCNN stem (csrc/cnn_stem.cu) shared by its CPU and GPU tests: (name, n boards, in planes, C, H, W),
mid = (in + C) // 2.  At 132 and at 114 SMs they reach 1, 2, 4, 8 and 16 conv pixels per thread, whole and chunked cin,
one and several bands, boards per CTA and channel tiles, ragged last CTAs and partial channel tiles
(test_cnn_stem_cpu.py::test_case_table_reaches_every_tile_edge)."""
import ctypes
from typing import NamedTuple

import numpy

FIELDS = ("k", "stride", "Ho", "Wo", "Hp", "Wp", "co_tile", "band", "bands", "boards", "cin_chunk", "items", "threads",
          "grid_x", "grid_y", "smem")          # per stage, at plan[3 + 16 * stage]


class StemCase(NamedTuple):
    name: str
    n: int
    cin: int
    C: int
    H: int
    W: int
    mid = property(lambda c: (c.cin + c.C) // 2)
    hw = property(lambda c: (-(-c.H // 16), -(-c.W // 16)))


CASES = [StemCase(*c) for c in (
    ("breakout_b1", 1, 3, 16, 96, 96), ("breakout_b37", 37, 3, 16, 96, 96),
    ("breakout_b701", 701, 3, 16, 96, 96),              # more than one wave; 2 boards per CTA, ragged
    ("atari_210x160", 2, 3, 16, 210, 160),              # k = 28
    ("wide_96x64", 5, 3, 16, 96, 64), ("tall_64x96", 5, 3, 16, 64, 96),     # W != H: the kernel comes from H
    ("small_24", 9, 3, 16, 24, 24), ("small_26", 3, 3, 16, 26, 26),         # pooled 1 x 1, averaged UP to 2 x 2
    ("in1_c4", 3, 1, 4, 48, 48), ("stack4_c16", 3, 19, 16, 96, 96),
    ("c64_b130", 130, 3, 64, 96, 96),                   # mid 33: a partial channel tile
    ("c64_210x160", 1, 3, 64, 210, 160),                # 16 pixels per thread
    ("atari_in131_c256", 1, 131, 256, 96, 96), ("in131_c64_b2", 2, 131, 64, 96, 96))]   # chunked cin, mid 193 / 97


def unpack(v):
    d = dict(h=v[0], w=v[1], mid=v[2])
    for s in range(2):
        d[f"s{s}"] = {f: int(v[3 + 16 * s + i]) for i, f in enumerate(FIELDS)}
    return d


def plan(lib, n, cin, C, H, W, sm_count):
    """The planner's plan as a dict, or None (the refusal is in mz_last_error(NULL))."""
    out = (ctypes.c_int64 * 36)()
    return unpack(list(out)) if lib.mz_debug_cnn_stem_plan(n, cin, C, H, W, sm_count, out) else None


def sparse_ints(rs, shape, density=0.1, lo=-3, hi=3):
    return (rs.randint(lo, hi + 1, size=shape) * (rs.uniform(size=shape) < density)).astype(numpy.float32)


def exact_operands(case, rs):
    """Sparse small-integer input and features.{0,3} weights / biases: every partial sum an integer below 2^24."""
    k = 2 * case.hw[0]
    x = sparse_ints(rs, (case.n, case.cin, case.H, case.W), density=0.3, lo=0, hi=3)
    return x, [sparse_ints(rs, s) for s in ((case.mid, case.cin, k, k), (case.mid,), (case.C, case.mid, 5, 5), (case.C,))]
