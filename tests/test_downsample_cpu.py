"""The DownSample stem's convs through the launch planner (csrc/resnet.cu::conv3x3_plan, behind mz_debug_conv3x3_plan;
the plan does not depend on the GPU's SM count): the case table of tests/downsamplecases.py reaches every launch feature
at the stem's own shapes, and every frame of 1..256 x 1..256 has a plan for each of its convs at the widths the tests
run (mz_create plans the same shapes and refuses a net whose conv has none)."""
import ctypes

import numpy
import pytest

from downsamplecases import CASES, DsCase, conv_shapes

FIELDS = ("P", "stride", "max_items", "bands", "band_rows", "boards", "cin_chunk", "gx", "gy", "gz", "smem", "cout_tile")
WIDTHS = (8, 16, 96, 128, 256)


@pytest.fixture(scope="module")
def lib():
    from muzero_general_b200 import _lib
    return _lib.load_library()


def _plan(lib, n, cin, cout, H, W, stride):
    out = (ctypes.c_int64 * len(FIELDS))()
    if not lib.mz_debug_conv3x3_plan(n, cin, cout, H, W, stride, out):
        return None
    return dict(zip(FIELDS, out))


def test_case_table_reaches_every_launch_feature(lib):
    plans = [(c, st, cin, _plan(lib, c.n, cin, cout, H, W, s)) for c in CASES for st, cin, cout, H, W, s in conv_shapes(c)]
    assert all(p for *_, p in plans), [(c.name, st) for c, st, _, p in plans if p is None]
    # every pixels-per-thread at both strides, both accumulator counts
    assert {(p["P"], p["stride"]) for *_, p in plans} == {(P, s) for P in (1, 2, 3, 4, 6, 7, 8) for s in (1, 2)}
    assert {p["max_items"] for *_, p in plans} == {1, 4}
    # several row bands, one row per band; several boards per CTA with a partial last CTA
    assert any(p["bands"] > 1 for *_, p in plans) and any(p["band_rows"] == 1 for *_, p in plans)
    assert any(p["boards"] > 1 and c.n % p["boards"] for c, _, _, p in plans)
    # batches of 1, exactly the boards of one CTA, one more
    assert any(c.n == 1 for c, *_ in plans)
    assert any(c.n == p["boards"] > 1 and p["gx"] == 1 for c, _, _, p in plans)
    assert any(c.n == p["boards"] + 1 and p["gx"] == 2 for c, _, _, p in plans)
    # conv1 stages 131 input planes a chunk at a time, the chunk not dividing 131
    assert any(st == "conv1" and cin == 131 and 131 % p["cin_chunk"] for c, st, cin, p in plans)
    # the first convs of the 96 x 129 / 96 x 130 frames at 128 / 256 channels: 32-channel cout tiles
    for name in ("c128_96x129", "c256_96x130_in131"):
        tiles = {st: p["cout_tile"] for c, st, _, p in plans if c.name == name}
        assert tiles["conv1"] == tiles["resblocks1"] == 32 and tiles["conv2"] == 64, (name, tiles)
    # every halving odd somewhere and even somewhere (H, then W)
    for dim in ("H", "W"):
        sizes = [getattr(c, dim) for c in CASES]
        for k in range(4):
            halves = {-(-s // 2 ** k) % 2 for s in sizes if -(-s // 2 ** k) > 1}
            assert halves == {0, 1}, (dim, k, halves)
    assert {c.C for c in CASES} == set(WIDTHS) and {c.cin for c in CASES} == {3, 131}
    assert {(1, 1), (96, 96), (210, 160), (96, 129), (96, 130)} <= {(c.H, c.W) for c in CASES}
    assert any(c.H == 1 < c.W for c in CASES) and any(c.W == 1 < c.H for c in CASES)


def _refused_before(cout, H, W, stride):
    """The planner before cout tiles could be narrower than min(cout, 64), restated on arrays of H and W: a shape was
    refused when one output row of that tile was more than 1024 items."""
    Wo = (W - 1) // stride + 1
    P = numpy.ones_like(Wo)
    for c in (2, 3, 4, 6, 7, 8):          # the first of 8, 7, 6, 4, 3, 2 dividing Wo wins: assign in reverse
        P = numpy.where(Wo % c == 0, c, P)
    return min(cout, 64) // 4 * (Wo // P) > 1024


def test_every_frame_up_to_256_has_a_plan_for_each_conv(lib):
    """Every DownSample geometry of 1..256 x 1..256 at 8, 16, 96, 128 and 256 channels, conv1 reading 3 or 131 planes,
    64 boards: each of the stem's conv shapes has a launch plan.  Before the planner could narrow the cout tile, 9728 of
    these frames were refused at 128 and 256 channels and 6144 at 96 (the first convs at C / 2 channels, P = 1 on an
    output row of more than 64 columns), none at 8 and 16."""
    out = lambda x: (x - 1) // 2 + 1
    H, W = numpy.meshgrid(numpy.arange(1, 257), numpy.arange(1, 257), indexing="ij")
    for C in WIDTHS:
        before = numpy.zeros(H.shape, bool)
        shapes = set()
        for Hi in range(1, 257):
            for Wi in range(1, 257):
                for _, cin, cout, h, w, s in conv_shapes(DsCase("grid", 64, 3, C, Hi, Wi)):
                    shapes.add((cin, cout, h, w, s))
                shapes.add((131, C // 2, Hi, Wi, 2))
        refused = [s for s in sorted(shapes) if _plan(lib, 64, *s) is None]
        assert not refused, (C, len(refused), refused[:5], lib.mz_last_error(None).decode())
        h1, w1 = out(H), out(W)
        for cout, h, w, s in ((C // 2, H, W, 2), (C // 2, h1, w1, 1), (C, h1, w1, 2), (C, out(h1), out(w1), 1),
                              (C, out(out(h1)), out(out(w1)), 1)):
            before |= _refused_before(cout, h, w, s)
        assert int(before.sum()) == {8: 0, 16: 0, 96: 6144, 128: 9728, 256: 9728}[C], (C, int(before.sum()))
        if C >= 128:
            assert before[95, 128] and not before[95, 127]        # 96 x 129 refused, 96 x 128 not

