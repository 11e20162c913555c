"""Case table of the CUDA-core conv3x3 kernel (csrc/resnet.cu: conv3x3_kernel<P, STRIDE, MAX_ITEMS> and its host
planner conv3x3_plan, reached through mz_debug_conv3x3 / mz_debug_conv3x3_plan).  Importable without a GPU.

The planner picks P (pixels per thread) from the output width (the first of 8, 7, 6, 4, 3, 2 that divides Wo, else 1),
MAX_ITEMS (accumulator tiles per thread: 4 when a CTA holds more than 256 items of 4 channels x P pixels), row bands
for large images, boards per CTA for small ones, a cin chunk when the staged planes do not fit in shared memory, and
cout tiles of 64 channels (the last one narrower when 64 does not divide Cout), halved down to 4 channels while one
output row of a tile is more than the 4 x 256 items a CTA holds.  The cases were taken from the
planner, not guessed; tests/test_conv_plan_cpu.py asserts what they reach:

  * all 28 instantiations: P in {1, 2, 3, 4, 6, 7, 8} x stride {1, 2} x MAX_ITEMS {1, 4}
  * several row bands with a shorter last band (s1_p2_m4, s1_p4_m4, s1_p8_m4_atari_rb); one band per row (s1_p1_m4_67)
  * several boards per CTA with a partial last CTA; batches of 1, exactly the boards per CTA, one more, and 300
  * a cin chunk smaller than Cin that does not divide it: games/atari.py's 131 -> 128 stride-2 stem at 96 x 96
  * Cout 4, 12, 48, 64, 68, 96, 128, 160 and 256; Cin != Cout, Cin 3, 33 and 131
  * boards of 1 x 1, 1 x W and H x 1, prime widths (5, 13, 43, 67, 131, 521)
  * cout tiles of 32, 16 and 4 channels on rows too wide for 64 (ct32_*, ct16_*, ct4_*), a narrower last tile behind them
  * one shape the planner refuses (REFUSED)
"""
from __future__ import annotations

from dataclasses import dataclass


@dataclass(frozen=True)
class ConvCase:
    name: str
    n: int
    cin: int
    cout: int
    H: int
    W: int
    stride: int = 1

    @property
    def out_hw(self):
        return (self.H - 1) // self.stride + 1, (self.W - 1) // self.stride + 1


CASES = [
    # one accumulator tile per thread
    ConvCase("s1_p1_m1_1x1", 1, 3, 4, 1, 1),
    ConvCase("s1_p1_m1_9x1", 4, 5, 256, 9, 1),
    ConvCase("s1_p2_m1_1x2", 2, 33, 12, 1, 2),
    ConvCase("s1_p3_m1_3x3", 300, 3, 16, 3, 3),
    ConvCase("s1_p4_m1_6x4", 3, 64, 64, 6, 4),
    ConvCase("s1_p6_m1_6x6", 7, 16, 96, 6, 6),
    ConvCase("s1_p7_m1_6x7", 131, 65, 64, 6, 7),
    ConvCase("s1_p8_m1_16x8", 9, 16, 16, 16, 8),
    ConvCase("s2_p1_m1_1x1", 33, 4, 12, 1, 1, 2),
    ConvCase("s2_p2_m1_5x4", 5, 16, 48, 5, 4, 2),
    ConvCase("s2_p3_m1_7x5", 6, 12, 4, 7, 5, 2),
    ConvCase("s2_p4_m1_1x7", 16, 4, 68, 1, 7, 2),
    ConvCase("s2_p6_m1_11x11", 4, 33, 48, 11, 11, 2),
    ConvCase("s2_p7_m1_13x13", 12, 8, 12, 13, 13, 2),
    ConvCase("s2_p8_m1_3x15", 9, 4, 160, 3, 15, 2),
    # four accumulator tiles per thread
    ConvCase("s1_p1_m4_67", 2, 32, 32, 67, 67),
    ConvCase("s1_p2_m4", 3, 48, 96, 5, 26),
    ConvCase("s1_p3_m4", 2, 4, 16, 5, 39),
    ConvCase("s1_p4_m4", 2, 64, 64, 23, 20),
    ConvCase("s1_p6_m4", 4, 64, 128, 9, 12),
    ConvCase("s1_p7_m4", 3, 64, 68, 9, 14),
    ConvCase("s1_p8_m4", 2, 33, 96, 9, 16),
    ConvCase("s1_p8_m4_atari_rb", 1, 128, 128, 48, 48),
    ConvCase("s2_p1_m4", 2, 131, 64, 3, 33, 2),
    ConvCase("s2_p2_m4", 2, 16, 48, 3, 43, 2),
    ConvCase("s2_p3_m4", 2, 3, 48, 9, 29, 2),
    ConvCase("s2_p4_m4", 2, 12, 48, 9, 39, 2),
    ConvCase("s2_p6_m4", 2, 32, 64, 12, 35, 2),
    ConvCase("s2_p7_m4", 2, 16, 160, 12, 41, 2),
    ConvCase("s2_p8_m4_atari_stem", 1, 131, 128, 96, 96, 2),
    # cout tiles narrower than 64: P = 1 and one output row of a 64-channel tile is more than 1024 items
    ConvCase("ct32_s1_6x67", 4, 64, 64, 6, 67),                 # 16 x 67 items; 32 channels: 8 x 67
    ConvCase("ct32_s2_ds129", 3, 16, 128, 7, 129, 2),           # DownSample conv1 of a 256-channel net, 129-wide frame
    ConvCase("ct16_s1_3x131", 2, 8, 68, 3, 131),                # 16-channel tiles, the fifth one of 4 channels
    ConvCase("ct4_s1_2x521", 1, 4, 12, 2, 521),                 # three 4-channel tiles
]

BY_NAME = {c.name: c for c in CASES}

# a board 1031 wide: 1031 is prime, so P = 1, and one output row alone is 1031 items even in a 4-channel cout tile,
# beyond the 4 x 256 a CTA holds
REFUSED = ConvCase("refused_1x1031", 2, 4, 8, 1, 1031)
REFUSED_REASON = "image too large for the item budget"


def net_conv_shapes(spec):
    """(cin, cout, H, W, stride) of every distinct conv3x3 of a residual net, as resnet.cu runs them: the
    representation stem (or the DownSample convs and blocks), the dynamics stem with its action plane, and the
    blocks of the towers."""
    C, (h, w) = spec.channels, spec.hidden_hw
    H, W = spec.obs_shape[1], spec.obs_shape[2]
    out = lambda x, s: (x - 1) // s + 1
    if spec.downsample:
        h1, w1 = out(H, 2), out(W, 2)
        h2, w2 = out(h1, 2), out(w1, 2)
        shapes = [(spec.in_channels, C // 2, H, W, 2), (C // 2, C // 2, h1, w1, 1), (C // 2, C, h1, w1, 2),
                  (C, C, h2, w2, 1), (C, C, out(h2, 2), out(w2, 2), 1)]
    else:
        shapes = [(spec.in_channels, C, H, W, 1)]
    shapes.append((C + 1, C, h, w, 1))
    if spec.blocks > 0:
        shapes.append((C, C, h, w, 1))
    return shapes
