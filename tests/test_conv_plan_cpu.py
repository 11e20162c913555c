"""Host-side launch planner of the CUDA-core conv3x3 kernel (csrc/resnet.cu::conv3x3_plan, through
mz_debug_conv3x3_plan): the case table of tests/convcases.py reaches every feature it claims, the planner refuses the
shape it cannot launch and says why, and the plans of the bundled games' layers are the ones the launcher used before
the cout tiles were allowed a narrower last tile, or narrower tiles on rows too wide for 64 channels."""
import ctypes

import pytest

from convcases import BY_NAME, CASES, REFUSED, REFUSED_REASON, net_conv_shapes

FIELDS = ("P", "stride", "max_items", "bands", "band_rows", "boards", "cin_chunk", "gx", "gy", "gz", "smem", "cout_tile")


@pytest.fixture(scope="module")
def lib():
    from muzero_general_b200 import _lib
    return _lib.load_library()


def _plan(lib, n, cin, cout, H, W, stride):
    out = (ctypes.c_int64 * len(FIELDS))()
    if not lib.mz_debug_conv3x3_plan(n, cin, cout, H, W, stride, out):
        return None
    return dict(zip(FIELDS, out))


def _case_plan(lib, c):
    return _plan(lib, c.n, c.cin, c.cout, c.H, c.W, c.stride)


def _earlier_plan(n, cin, cout, H, W, stride):
    """The launcher's arithmetic before this planner existed, restated, with its grid.y = cout // 64 (which dropped the
    last cout % 64 channels) and its one cout tile width, min(cout, 64); None where one output row of that tile was
    more than a CTA's 1024 items (the shape was refused).  Only shapes with cout <= 64 or a multiple of 64 are compared
    with it."""
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    P = next((c for c in (8, 7, 6, 4, 3, 2) if Wo % c == 0), 1)
    ct = min(cout, 64)
    bands = 1
    while bands < Ho and (ct // 4) * -(-Ho // bands) * (Wo // P) > 1024:
        bands += 1
    band_rows = -(-Ho // bands)
    bands = -(-Ho // band_rows)
    items = (ct // 4) * band_rows * (Wo // P)
    boards = min(256 // items if items < 256 else 1, 32, n)
    if items * boards > 1024:
        return None
    plane = ((band_rows - 1) * stride + 3) * (W + 2)
    chunk = cin
    while chunk > 1 and chunk * 9 * ct + boards * chunk * plane > 200 * 1024 // 4:
        chunk = (chunk + 1) // 2
    return dict(P=P, stride=stride, max_items=4 if items * boards > 256 else 1, bands=bands, band_rows=band_rows,
                boards=boards, cin_chunk=chunk, gx=-(-n // boards), gy=cout // ct, gz=bands,
                smem=(chunk * 9 * ct + boards * chunk * plane) * 4, cout_tile=ct)


def test_case_table_reaches_every_planner_feature(lib):
    plans = {c.name: _case_plan(lib, c) for c in CASES}
    assert all(plans.values()), [k for k, p in plans.items() if p is None]
    # all 28 instantiations
    inst = {(p["P"], p["stride"], p["max_items"]) for p in plans.values()}
    want = {(P, s, m) for P in (1, 2, 3, 4, 6, 7, 8) for s in (1, 2) for m in (1, 4)}
    assert inst == want, sorted(want - inst)
    for c in CASES:
        p, (Ho, Wo) = plans[c.name], c.out_hw
        assert (p["stride"], p["gx"], p["gy"], p["gz"]) == (c.stride, -(-c.n // p["boards"]), -(-c.cout // p["cout_tile"]),
                                                             p["bands"])
        assert p["bands"] == -(-Ho // p["band_rows"]) and p["cin_chunk"] <= c.cin and p["smem"] <= 200 * 1024
        # a tile narrower than min(cout, 64) only where one output row of the wider tile exceeds the 1024 items, and
        # then the widest multiple-of-4 halving that fits
        ct = min(c.cout, 64)
        while ct > 4 and ct // 4 * (Wo // p["P"]) > 1024:
            ct = (ct // 2 + 3) // 4 * 4
        assert p["cout_tile"] == ct and p["cout_tile"] // 4 * p["band_rows"] * (Wo // p["P"]) * p["boards"] <= 1024, c.name
    # several bands with a shorter last band; one band per output row of a tall image
    assert any(p["bands"] > 1 and BY_NAME[k].out_hw[0] % p["band_rows"] for k, p in plans.items())
    assert any(p["bands"] == BY_NAME[k].out_hw[0] > 1 for k, p in plans.items())
    assert plans["s1_p1_m4_67"]["bands"] == 67
    # several boards per CTA with a partial last CTA; batches of 1, exactly the boards per CTA, one more, a few hundred
    assert any(p["boards"] > 1 and BY_NAME[k].n % p["boards"] for k, p in plans.items())
    ns = {(BY_NAME[k].n, p["boards"]) for k, p in plans.items()}
    assert any(n == 1 for n, _ in ns)
    assert any(n == b > 1 for n, b in ns)
    assert any(n == b + 1 and b > 1 for n, b in ns)
    assert any(n >= 200 for n, _ in ns)
    # a cin chunk smaller than Cin that does not divide it: the atari stem stages 17 of its 131 input planes at a time
    assert plans["s2_p8_m4_atari_stem"]["cin_chunk"] == 17
    assert any(p["cin_chunk"] < BY_NAME[k].cin and BY_NAME[k].cin % p["cin_chunk"] for k, p in plans.items())
    # channel counts, including cout tiles narrower than 64 behind full ones (68, 96, 160)
    couts = {c.cout for c in CASES}
    assert {4, 12, 48, 64, 68, 96, 128, 160, 256} <= couts
    assert {c.cout % 64 for c in CASES if c.cout > 64} >= {4, 32}
    assert any(c.cin != c.cout for c in CASES) and {3, 33, 131} <= {c.cin for c in CASES}
    # boards of 1 x 1, 1 x W, H x 1 and prime widths
    shapes = {(c.H, c.W) for c in CASES}
    assert (1, 1) in shapes and any(h == 1 < w for h, w in shapes) and any(w == 1 < h for h, w in shapes)
    assert {5, 13, 43, 67} <= {w for _, w in shapes}
    # cout tiles of 32, 16 and 4 channels, each behind a last tile of fewer channels or a full one
    tiles = {p["cout_tile"] for p in plans.values()}
    assert {4, 16, 32, 64} <= tiles, tiles
    assert any(p["cout_tile"] < 64 and BY_NAME[k].cout % p["cout_tile"] for k, p in plans.items())
    assert any(p["cout_tile"] < 64 and p["stride"] == 2 for p in plans.values())


def test_row_no_cout_tile_holds_is_refused_with_its_reason(lib):
    c = REFUSED
    assert _case_plan(lib, c) is None
    assert REFUSED_REASON in lib.mz_last_error(None).decode()
    # the same board one column narrower (1030 = 2 x 515: P = 2) launches, in 4-channel tiles
    assert _plan(lib, c.n, c.cin, c.cout, c.H, c.W - 1, c.stride)["cout_tile"] == 4
    # the 64-channel board 67 wide that a 64-channel tile cannot hold (one row is 16 x 67 = 1072 items) launches in
    # 32-channel tiles, a band per row; the planner refused it before the tiles could be narrower
    p = _plan(lib, 4, 64, 64, 6, 67, 1)
    assert (p["cout_tile"], p["gy"], p["band_rows"]) == (32, 2, 1)
    assert _earlier_plan(4, 64, 64, 6, 67, 1) is None


@pytest.mark.parametrize("args,reason", [((1, 4, 6, 3, 3, 1), "multiple of 4"), ((1, 4, 0, 3, 3, 1), "multiple of 4"),
                                         ((1, 4, 8, 3, 3, 3), "stride"), ((0, 4, 8, 3, 3, 1), "empty"),
                                         ((1, 0, 8, 3, 3, 1), "empty")])
def test_planner_refuses_shapes_the_kernel_cannot_take(lib, args, reason):
    assert _plan(lib, *args) is None
    assert reason in lib.mz_last_error(None).decode()


def _bundled_shapes():
    from muzero_general_b200.games import load_game_module
    from muzero_general_b200.netspec import RESNET, netspec_from_config
    out = []
    for game in ("tictactoe", "connect4", "gomoku", "breakout", "atari"):
        spec = netspec_from_config(load_game_module(game).MuZeroConfig())
        assert spec.kind == RESNET
        out += [(game, s) for s in net_conv_shapes(spec)]
    return out


def test_bundled_games_and_earlier_shapes_keep_their_launch_plans(lib):
    """Every shape that launched before keeps its plan: the layers of the bundled games at batches of 1 to 8192, and
    the cases of the table whose cout is at most 64 or a multiple of 64.  The other cases differ only in grid.y, which
    now covers the last cout % 64 channels."""
    shapes = _bundled_shapes()
    assert {g for g, _ in shapes} == {"tictactoe", "connect4", "gomoku", "breakout", "atari"}
    for game, (cin, cout, H, W, stride) in shapes:
        for n in (1, 7, 64, 1024, 8192):
            assert _plan(lib, n, cin, cout, H, W, stride) == _earlier_plan(n, cin, cout, H, W, stride), (game, cin, cout, H, W)
    for c in CASES:
        p, old = _case_plan(lib, c), _earlier_plan(c.n, c.cin, c.cout, c.H, c.W, c.stride)
        if old is None:
            assert p["cout_tile"] < min(c.cout, 64), c.name         # refused before: launches in narrower tiles now
        elif c.cout <= 64 or c.cout % 64 == 0:
            assert p == old, c.name
        else:
            assert p == dict(old, gy=old["gy"] + 1), c.name
