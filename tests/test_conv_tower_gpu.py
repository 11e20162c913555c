"""Whole 64-channel tensor-core towers (csrc/conv_x3.cu, csrc/conv_tc.cu behind Runner::tower_tc) against an fp64 tower,
through mz_debug_conv_tower: every call site of the network (representation, dynamics as an API call and in search,
prediction), every depth the launch packing treats differently, batches at the launch, tile and CTA edges, and the
partitioned replay.  The single-conv tests (test_conv_gpu.py) cannot see what happens between layers: activations
rewritten in place, the fp32 residual kept in registers, the weight refill of the next layer, the action table parked in
the residual registers, the fp16 resident kernel and the workspace rotation between launches.

Workspaces, the pool's other slots and the output start as NaN, so a layer that reads a board nobody wrote fails.

  exact     sparse small-integer weights, integer biases and inputs, A a power of two with action-plane weights in
            multiples of A: every product and partial sum is exact in fp32, so the device tower must EQUAL the fp64 one
            while every activation stays below 65504 (x3: x_h + x_l hold 22 bits) or 2048 (fp16 stores).  The fixtures
            assert those ranges on the fp64 tower.
  budget    standard-normal operands at gains 1, 1e-4 and 300 against the fp64 tower, with an error budget propagated
            layer by layer in fp64 from the single-conv contract (ReLU is 1-Lipschitz, convolutions of absolute values):
                delta_out = |W| * delta_in + c1 (|W| * |x|) + c2 |y| + delta_res + floor
            x3: c1 = 4e-6, c2 = 2e-6, floor 1e-6 gain; fp16: c1 = 2e-3, c2 = 1e-3, floor 1e-5.
  launches  the packing restated: the first launch holds the stem and floor((8 - stem) / 2) blocks, every later one 4
            blocks, times conv_x3_launches(n) per range in x3; one launch per conv on the fp16 per-conv path (n > 16 S).

S is the device's SM count: 4 S boards fill one x3 launch, 8 S one fp16 resident launch, 16 S one fused fp16 launch."""
import numpy
import pytest
import torch

pytestmark = pytest.mark.gpu

C = 64
BOARDS = ((1, 1), (1, 7), (6, 1), (3, 3), (5, 4), (6, 6), (6, 7))
SITES = ("representation", "dynamics", "dynamics_pool", "prediction")
STEM = {"representation": 0, "dynamics": 1, "dynamics_pool": 1, "prediction": 0}
CONTRACT = {"x3": (4e-6, 2e-6, 1e-6), "fp16": (2e-3, 1e-3, 1e-5)}       # c1, c2, absolute floor (x3: times the gain)
LIMIT = {"x3": 65504.0, "fp16": 2048.0}                                  # largest |activation| of the exact fixtures
SMALL_X3 = (1, 2, 3, 4, 5, 7)


def _depths(site):
    return range(0, 7) if STEM[site] else range(1, 7)


_SMS = []


def sms():
    if not _SMS:
        _SMS.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _SMS[0]


def x3_batches(S):
    return SMALL_X3 + (4 * S - 1, 4 * S, 4 * S + 1, 8 * S + 3)


def fp16_batches(S):
    return (8 * S, 8 * S + 1, 16 * S, 16 * S + 1)


# ---------------------------------------------------------------------------------------------- fixtures
def _actions(n, A, rs):
    a = rs.randint(0, A, n)
    a[0] = 0
    a[-1] = A - 1
    return a.astype(numpy.int32)


def _parents(n, stride, rs):
    p = rs.randint(0, stride, n)
    p[0] = 0
    p[-1] = stride - 1
    return p.astype(numpy.int32)


def _sparse_int_conv(rs, cin, vmax, two=0.5):
    """[64, cin, 3, 3] with one or two nonzero taps of +-1..+-vmax per output channel."""
    w = numpy.zeros((C, cin, 3, 3), numpy.float32)
    for co in range(C):
        for _ in range(2 if rs.random_sample() < two else 1):
            w[co, rs.randint(cin), rs.randint(3), rs.randint(3)] = rs.choice([-1, 1]) * rs.randint(1, vmax + 1)
    return w


def int_tower(mode, n, H, W, blocks, stem, seed, A=4):
    """Operands of the exact test: integers, A a power of two, action-plane weights in multiples of A.  The inputs start
    at +-4000 (x3: the x_l halves of the activations are not zero) or +-8 (fp16) and are halved until the fp64 tower
    stays inside the exact range on every board.  Returns the operands and the fp64 tower's output and peak."""
    ws, bs, act = _int_weights(n, blocks, stem, numpy.random.RandomState(seed), A)
    hi = 4000 if mode == "x3" else 8
    while True:
        x = numpy.random.RandomState(seed + 1).randint(-hi, hi + 1, size=(n, C, H, W)).astype(numpy.float32)
        ref, peak, _, _ = tower64(x, ws, bs, stem, act, A)
        if peak < LIMIT[mode] or hi == 1:
            return x, ws, bs, act, A, ref, peak
        hi //= 2


def _int_weights(n, blocks, stem, rs, A):
    ws, bs = [], []
    if stem:
        w = numpy.zeros((C, C + 1, 3, 3), numpy.float32)
        w[:, :C] = _sparse_int_conv(rs, C, 2, two=0.3)
        for co in rs.choice(C, 24, replace=False):          # the action plane reaches 24 channels through one tap each
            w[co, C, rs.randint(3), rs.randint(3)] = A * rs.choice([-1, 1]) * rs.randint(1, 3)
        ws.append(w)
        bs.append(rs.randint(-3, 4, C).astype(numpy.float32))
    for _ in range(blocks):
        ws.append(_sparse_int_conv(rs, C, 3, two=0.3))
        bs.append(rs.randint(-3, 4, C).astype(numpy.float32))
        ws.append(_sparse_int_conv(rs, C, 1, two=0.2))
        bs.append(rs.randint(-4, 2, C).astype(numpy.float32))
    return ws, bs, _actions(n, A, rs) if stem else None


def normal_tower(n, H, W, blocks, stem, gain, seed, A=None):
    """Standard-normal operands scaled by `gain` (inputs, biases, the action plane's weights): the tower is positively
    homogeneous, so every activation scales with it."""
    rs = numpy.random.RandomState(seed)
    A = A or (7, 128, 1)[seed % 3]
    x = (gain * rs.standard_normal((n, C, H, W))).astype(numpy.float32)
    ws, bs = [], []
    for i in range(stem + 2 * blocks):
        cin = C + 1 if stem and i == 0 else C
        w = rs.standard_normal((C, cin, 3, 3)) / numpy.sqrt(9 * C)
        if cin == C + 1:
            w[:, C] *= gain
        ws.append(w.astype(numpy.float32))
        bs.append((0.1 * gain * rs.standard_normal(C)).astype(numpy.float32))
    act = _actions(n, A, rs) if stem else None
    return x, ws, bs, act, A


# ---------------------------------------------------------------------------------------------- fp64 tower
def _conv(x, w, b=None):
    return torch.nn.functional.conv2d(x, torch.from_numpy(numpy.asarray(w, numpy.float64)),
                                      None if b is None else torch.from_numpy(numpy.asarray(b, numpy.float64)), 1, 1)


def tower64(x, ws, bs, stem, act, A, mode=None, gain=1.0, rows=None):
    """The tower in fp64 on the boards `rows` (all by default): (output, largest |activation| anywhere, per-layer peaks
    and, with `mode`, the propagated error budget of the output)."""
    idx = numpy.arange(len(x)) if rows is None else numpy.asarray(rows)
    h = torch.from_numpy(x[idx]).double()
    n, _, H, W = h.shape
    peaks = [float(h.abs().max())]
    c1 = c2 = floor = 0.0
    delta = None
    if mode:
        c1, c2, floor = CONTRACT[mode]
        if mode == "x3":
            floor *= gain
        # the input boards are stored as fp16 (fp16 mode) or x_h + x_l (22 bits, x3)
        delta = h.abs() * (2.0 ** -11 if mode == "fp16" else 2.0 ** -22) + floor

    def layer(inp, d_in, w, b, res=None, d_res=None):
        y = _conv(inp, w, b)
        if res is not None:
            y = y + res
        d = None
        if mode:
            aw = numpy.abs(w)
            d = _conv(d_in, aw) + c1 * _conv(inp.abs(), aw) + c2 * y.abs() + floor
            if d_res is not None:
                d = d + d_res
        return torch.relu(y), d

    k = 0
    if stem:
        plane = torch.from_numpy(act[idx].astype(numpy.float64) / A)[:, None, None, None].expand(n, 1, H, W)
        inp = torch.cat([h, plane], 1)
        d_in = torch.cat([delta, torch.zeros(n, 1, H, W, dtype=torch.float64)], 1) if mode else None
        h, delta = layer(inp, d_in, ws[0], bs[0])
        peaks.append(float(h.abs().max()))
        k = 1
    while k < len(ws):
        t, dt = layer(h, delta, ws[k], bs[k])
        peaks.append(float(t.abs().max()))
        h, delta = layer(t, dt, ws[k + 1], bs[k + 1], h, delta)
        peaks.append(float(h.abs().max()))
        k += 2
    return h.numpy(), max(peaks), peaks, None if delta is None else delta.numpy()


# ---------------------------------------------------------------------------------------------- launch packing
def partition_ranges(n, parts):
    per = ((n + parts - 1) // parts + 7) & ~7
    return [min(per, n - p * per) for p in range(parts) if n - p * per > 0]


def expected_launches(mode, n, blocks, stem, S, parts=1):
    if mode == "fp16" and n > 16 * S:
        return stem + 2 * blocks                       # one launch per conv
    first = (8 - stem) // 2
    towers = 1 + max(0, -(-(blocks - first) // 4))
    if mode == "fp16":
        return towers
    return sum(towers * -(-m // (4 * S)) for m in partition_ranges(n, parts))


def run(mode, site, x, ws, bs, act, A, seed=0, parts=1, stride=None):
    from muzero_general_b200.engine import debug_conv_tower
    n = len(x)
    kw = {}
    if site == "dynamics_pool":
        stride = stride or 3
        kw = dict(parents=_parents(n, stride, numpy.random.RandomState(seed + 7)), pool_stride=stride, parts=parts)
    out, launches, sat = debug_conv_tower(x, ws, bs, mode=mode, site=site, actions=act, A=A, **kw)
    stem = STEM[site]
    assert launches == expected_launches(mode, n, (len(ws) - stem) // 2, stem, sms(), parts), (mode, site, n, len(ws), launches)
    return out, sat


def _rows(n, S, seed):
    """Boards at the launch, tile and CTA edges plus a few random ones."""
    rows = {0, 1, 2, 3, n - 1, n - 2}
    for b in (4 * S, 8 * S, 16 * S):
        rows |= {b - 1, b, b + 1}
    rows |= set(int(r) for r in numpy.random.RandomState(seed).randint(0, n, 4))
    return sorted(r for r in rows if 0 <= r < n)


# ---------------------------------------------------------------------------------------------- a. exact on integers
def _check_exact(mode, site, n, H, W, blocks, seed, rows=None, A=4):
    stem = STEM[site]
    x, ws, bs, act, A, ref, peak = int_tower(mode, n, H, W, blocks, stem, seed, A)
    assert peak < LIMIT[mode], f"fixture left the exact range: {peak} ({mode} {site} {H}x{W} blocks {blocks})"
    # x3: some activations need more than fp16's 11 bits, so the x_l halves take part
    assert (peak > 2048 if mode == "x3" else ref.any()), f"fixture too tame to test: {peak}"
    got, sat = run(mode, site, x, ws, bs, act, A, seed)
    dev, ref = (got, ref) if rows is None else (got[rows], ref[rows])
    bad = numpy.argwhere(dev != ref)
    assert len(bad) == 0, f"{mode} {site} {H}x{W} n={n} blocks {blocks}: {len(bad)} differences, first at {bad[0]}: " \
                          f"{dev[tuple(bad[0])]} vs {ref[tuple(bad[0])]}"
    assert sat == 0


@pytest.mark.parametrize("mode", ["x3", "fp16"])
@pytest.mark.parametrize("H,W", BOARDS)
def test_tower_exact_on_integers_every_site_and_depth(H, W, mode):
    """The full cross of board, call site and depth at small batches (odd ones leave a CTA's second tile one board)."""
    i = 0
    for site in SITES:
        for blocks in _depths(site):
            n = SMALL_X3[i % len(SMALL_X3)]
            # (fp16: a * table of A = 128 grows past 2048 within a few blocks; the budget test takes A = 128 there)
            A = ((1, 4, 128) if mode == "x3" else (1, 4))[i % (3 if mode == "x3" else 2)] if STEM[site] else 4
            _check_exact(mode, site, n, H, W, blocks, seed=100 * H + 10 * W + i, A=A)
            i += 1


@pytest.mark.parametrize("site", SITES)
@pytest.mark.parametrize("mode", ["x3", "fp16"])
def test_tower_exact_on_integers_at_launch_edges(mode, site):
    """Batches at the x3 launch edges (4 S - 1 .. 8 S + 3) and the fp16 kernel switches (resident / streaming / per conv),
    deep towers split across launches; the fp64 tower on the edge boards only."""
    S = sms()
    batches = x3_batches(S)[len(SMALL_X3):] if mode == "x3" else fp16_batches(S)
    for j, n in enumerate(batches):
        H, W = ((6, 7), (5, 4), (6, 7), (3, 3))[j % 4]
        blocks = (6, 4, 5, 6)[j % 4]
        _check_exact(mode, site, n, H, W, blocks, seed=7 + j, rows=_rows(n, S, j))


# ---------------------------------------------------------------------------------------------- b. propagated budget
def _check_budget(mode, site, n, H, W, blocks, gain, seed, rows=None, stride=None):
    stem = STEM[site]
    x, ws, bs, act, A = normal_tower(n, H, W, blocks, stem, gain, seed)
    got, sat = run(mode, site, x, ws, bs, act, A, seed, stride=stride)
    ref, peak, _, delta = tower64(x, ws, bs, stem, act, A, mode=mode, gain=gain, rows=rows)
    assert peak < 65504.0
    dev = got if rows is None else got[rows]
    err = numpy.abs(dev.astype(numpy.float64) - ref)
    worst = float((err / delta).max())
    assert numpy.isfinite(dev).all() and worst <= 1.0, f"{mode} {site} {H}x{W} n={n} blocks {blocks} gain {gain}: " \
                                                       f"error / budget {worst:.3f}"
    assert sat == 0
    return worst


@pytest.mark.parametrize("mode", ["x3", "fp16"])
@pytest.mark.parametrize("H,W", BOARDS)
def test_tower_within_propagated_budget(H, W, mode):
    worst = {}
    i = 0
    for gain in (1.0, 1e-4, 300.0):
        for site in SITES:
            for blocks in ((0, 3, 4, 6) if STEM[site] else (1, 4, 5, 6)):
                n = SMALL_X3[i % len(SMALL_X3)]
                r = _check_budget(mode, site, n, H, W, blocks, gain, seed=1000 + i)
                worst[gain] = max(worst.get(gain, 0.0), r)
                i += 1
    print(f"[tower budget] {mode} {H}x{W}: worst error / budget " + ", ".join(f"gain {g:g}: {r:.3f}" for g, r in worst.items()))


@pytest.mark.parametrize("mode", ["x3", "fp16"])
def test_tower_within_propagated_budget_at_launch_edges(mode):
    S = sms()
    batches = x3_batches(S)[len(SMALL_X3):] if mode == "x3" else fp16_batches(S)
    worst = 0.0
    for j, n in enumerate(batches):
        for k, site in enumerate(SITES):
            gain = (1.0, 300.0, 1e-4)[(j + k) % 3]
            worst = max(worst, _check_budget(mode, site, n, 6, 7, 6, gain, seed=j * 4 + k, rows=_rows(n, S, j)))
    print(f"[tower budget] {mode} launch edges: worst error / budget {worst:.3f}")


# ---------------------------------------------------------------------------------------------- c. launch counts
@pytest.mark.parametrize("site", SITES)
@pytest.mark.parametrize("mode", ["x3", "fp16"])
def test_tower_launch_counts(mode, site):
    """Every depth packs as restated in expected_launches (asserted inside run()): the in-search dynamics tower, whose
    input is a read-only pool, included."""
    S = sms()
    for n in ((5, 4 * S + 1) if mode == "x3" else (5, 16 * S + 1)):
        for blocks in _depths(site):
            x, ws, bs, act, A = normal_tower(n, 3, 3, blocks, STEM[site], 1.0, seed=blocks)
            run(mode, site, x, ws, bs, act, A)
    # the split dynamics tower of a search holds four blocks per launch after the first
    assert expected_launches("x3", 5, 5, 1, S) == 2 and expected_launches("x3", 5, 6, 1, S) == 2


# ---------------------------------------------------------------------------------------------- d. partitions
@pytest.mark.parametrize("blocks", [3, 6])
def test_partitioned_tower_is_bit_identical(blocks):
    """The ranges of the partitioned replay, each with its own first-game offset, give the whole batch's results."""
    S = sms()
    for n in (37, 4 * S + 1, 8 * S + 3):
        x, ws, bs, act, A = normal_tower(n, 6, 7, blocks, 1, 1.0, seed=n)
        base, _ = run("x3", "dynamics_pool", x, ws, bs, act, A, seed=n, stride=5)
        for parts in (2, 3, 4):
            got, _ = run("x3", "dynamics_pool", x, ws, bs, act, A, seed=n, parts=parts, stride=5)
            assert numpy.array_equal(got, base), (n, blocks, parts)


# ---------------------------------------------------------------------------------------------- e. range guard
@pytest.mark.parametrize("site", ["prediction", "dynamics_pool"])
def test_range_guard_sees_a_late_layer_of_a_split_tower(site):
    """Activations beyond 65504 only in the last block of a 6-block tower (the second launch): the guard counts them;
    the same tower without that bias stays in range and leaves the count at zero."""
    S = sms()
    stem = STEM[site]
    for n in (3, 4 * S + 1):
        x, ws, bs, act, A, _, _ = int_tower("x3", n, 6, 7, 6, stem, seed=n)
        _, _, peaks, _ = tower64(x, ws, bs, stem, act, A)
        assert max(peaks) < 65504.0
        _, sat = run("x3", site, x, ws, bs, act, A, seed=n)
        assert sat == 0
        bs = [b.copy() for b in bs]
        bs[-1][5] = 70000.0
        _, _, peaks, _ = tower64(x, ws, bs, stem, act, A)
        assert max(peaks[:-1]) < 65504.0 < peaks[-1], peaks
        _, sat = run("x3", site, x, ws, bs, act, A, seed=n)
        assert sat > 0
