"""Case table of the DownSample stem (downsample="resnet", models.py:233-275; csrc/resnet.cu Runner::downsample behind
mz_debug_downsample).  Importable without a GPU.

The stem halves the frame four times (conv1 and conv2 at stride 2, then two 3 x 3 / stride-2 average pools), each
halving rounding up, so a frame of H x W ends as ceil(H / 16) x ceil(W / 16).  The cases cover:

  * frames where each of the four halvings is odd or even: 1 x 1, 1 x W, H x 1, 17 x 33, 20 x 24, 96 x 96 (the
    reference's breakout and atari frames), 210 x 160 (a raw Atari frame), and 96 x 129 / 96 x 130, whose first convs at
    C / 2 >= 64 channels a 64-channel cout tile cannot hold (P = 1 on a 65-wide output row: 16 x 65 items)
  * C = 8 (C / 2 = 4, the narrowest stem), 16 (breakout), 96 (a 32-channel last cout tile), 128 and 256 (atari)
  * 3 and 131 input planes (131: conv1 stages its input planes a chunk at a time, the chunk not dividing 131)
  * batches of 1, exactly the boards one CTA holds, one more, and frames split into several row bands

tests/test_downsample_cpu.py asserts what the table reaches through the launch planner.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy


@dataclass(frozen=True)
class DsCase:
    name: str
    n: int
    cin: int
    C: int
    H: int
    W: int

    @property
    def hw(self):
        return -(-self.H // 16), -(-self.W // 16)


CASES = [
    DsCase("c8_1x1_n1", 1, 3, 8, 1, 1),
    DsCase("c8_1x1_n32", 32, 3, 8, 1, 1),              # 32 boards per CTA in every conv: exactly one CTA
    DsCase("c8_1x1_n33", 33, 3, 8, 1, 1),              # one more: a second CTA of one board
    DsCase("c8_200x1", 3, 3, 8, 200, 1),
    DsCase("c16_1x200", 2, 3, 16, 1, 200),
    DsCase("c16_17x33_in131", 2, 131, 16, 17, 33),
    DsCase("c96_20x24", 5, 3, 96, 20, 24),
    DsCase("c16_96x96_breakout", 3, 3, 16, 96, 96),
    DsCase("c16_210x160", 2, 3, 16, 210, 160),
    DsCase("c8_12x56", 9, 3, 8, 12, 56),               # P = 7 at both strides (28, 14 and 7 columns)
    DsCase("c128_96x129", 1, 3, 128, 96, 129),
    DsCase("c256_96x130_in131", 1, 131, 256, 96, 130),
    DsCase("c256_96x96_atari", 1, 131, 256, 96, 96),
]

BY_NAME = {c.name: c for c in CASES}


def conv_shapes(c: DsCase):
    """(stage, cin, cout, H, W, stride) of the stem's five distinct conv shapes, as resnet.cu plans them."""
    out = lambda x: (x - 1) // 2 + 1
    h1, w1 = out(c.H), out(c.W)
    h2, w2 = out(h1), out(w1)
    return [("conv1", c.cin, c.C // 2, c.H, c.W, 2), ("resblocks1", c.C // 2, c.C // 2, h1, w1, 1),
            ("conv2", c.C // 2, c.C, h1, w1, 2), ("resblocks2", c.C, c.C, h2, w2, 1),
            ("resblocks3", c.C, c.C, out(h2), out(w2), 1)]


def conv_list(c: DsCase):
    """(name, cin, cout, stride) of the 18 convs in execution order, the layout of mz_debug_downsample's weights."""
    h = c.C // 2
    convs = [("conv1", c.cin, h, 2)]
    convs += [(f"resblocks1.{i}.conv{k}", h, h, 1) for i in range(2) for k in (1, 2)]
    convs += [("conv2", h, c.C, 2)]
    convs += [(f"resblocks{s}.{i}.conv{k}", c.C, c.C, 1) for s in (2, 3) for i in range(3) for k in (1, 2)]
    return convs


def exact_operands(c: DsCase, rs):
    """Sparse small-integer operands on which the stem is exact in fp32: x in {-1, 0, 1}; conv weights in {-1, 0, 1}
    (about 1.5 nonzero taps per output), conv1's times 81 and every bias before the first pool a multiple of 81, so
    each value the first pool averages is a multiple of 81 and its average a multiple of 9; resblocks3's biases are
    multiples of 9, so the second pool's averages are integers as well."""
    x = rs.randint(-1, 2, (c.n, c.cin, c.H, c.W)).astype(numpy.float32)
    ws, bs = [], []
    for name, cin, cout, _ in conv_list(c):
        keep = rs.random_sample((cout, cin, 3, 3)) < 1.5 / (9 * cin)
        w = rs.randint(-1, 2, (cout, cin, 3, 3)) * keep
        step = 9 if name.startswith("resblocks3") else 81
        b = rs.randint(-2, 3, cout) * step
        if name in ("conv1", "conv2"):
            b = numpy.zeros(cout)
        if name == "conv1":
            w = w * 81
        ws.append(w.astype(numpy.float32))
        bs.append(b.astype(numpy.float32))
    return x, ws, bs


def normal_operands(c: DsCase, rs, gain):
    """Standard-normal operands: x and the biases scaled by `gain`, weights by 1 / sqrt(fan-in) so the activations keep
    their scale through the 18 convs."""
    x = (rs.standard_normal((c.n, c.cin, c.H, c.W)) * gain).astype(numpy.float32)
    ws, bs = [], []
    for name, cin, cout, _ in conv_list(c):
        ws.append((rs.standard_normal((cout, cin, 3, 3)) / numpy.sqrt(9 * cin)).astype(numpy.float32))
        b = numpy.zeros(cout) if name in ("conv1", "conv2") else rs.standard_normal(cout) * gain
        bs.append(b.astype(numpy.float32))
    return x, ws, bs
