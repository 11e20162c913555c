"""Whole fused CUDA-core towers (csrc/small_tower.cu: small_tower_kernel<P, CO>, whose small_tower_tile the fused
small-network search shares) through mz_debug_small_tower: the four call sites of resnet_inference (representation with its
stem from the observation planes, dynamics as an API call and in search with the gathered pool and partitions, prediction),
every instantiation, every depth up to the 10-layer cap, batches of 1, ragged last tiles and more than one round of tiles.
The case table is tests/smalltowercases.py, sized from the SM count read at run time; every run asserts that the launch took
the plan the planner gives for the case (mz_debug_small_tower_plan) and the (P, CO) the case targets.

The output and the pool's other slots start as NaN, so a board the tower does not write, or reads from the wrong slot, fails.

  exact       integer inputs, sparse small-integer weights, integer biases, A a power of two with action-plane weights in
              multiples of A.  The fixture asserts on the fp64 side that every partial sum stays below 2^24 (each layer's
              |W| * |x| + |b| + |residual|), so every fp32 operation is exact and the device tower must EQUAL the fp64 one.
  per-layer   standard-normal operands at gains 1, 1e-4 and 300, A not a power of two: the fused tower equals, bit for bit,
              the chain of single conv3x3_kernel launches (mz_debug_conv3x3) with bias, residual and ReLU, the action plane
              passed as float32(action) / float32(A).  test_conv_cuda_core_gpu.py pins conv3x3_kernel to fp64 with the
              rigorous gamma_n bound of its FMA chain, so this pins the tower's rounding without a propagated budget."""
import time

import numpy
import pytest
import torch

from smalltowercases import BY_NAME, CASES, case_plan, first_range

pytestmark = pytest.mark.gpu

_SMS = []


def sms():
    if not _SMS:
        _SMS.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _SMS[0]


def _plan_fn():
    from muzero_general_b200.engine import debug_small_tower_plan
    return debug_small_tower_plan


# ---------------------------------------------------------------------------------------------- fixtures
def _ends(n, hi, rs):
    a = rs.randint(0, hi, n)
    a[0] = 0
    a[-1] = hi - 1
    return a.astype(numpy.int32)


def _sparse_int_conv(rs, C, cin, vmax, two=0.5):
    """[C, cin, 3, 3] with one or two nonzero taps of +-1..+-vmax per output channel."""
    w = numpy.zeros((C, cin, 3, 3), numpy.float32)
    for co in range(C):
        for _ in range(2 if rs.random_sample() < two else 1):
            w[co, rs.randint(cin), rs.randint(3), rs.randint(3)] = rs.choice([-1, 1]) * rs.randint(1, vmax + 1)
    return w


def int_operands(case, n, seed):
    """Operands of the exact test (see the module docstring).  The inputs start at +-64 and are halved until the fp64
    tower's partial-sum bound stays below 2^24.  Returns (x, weights, biases, actions, A, fp64 output)."""
    rs = numpy.random.RandomState(seed)
    C, dyn = case.C, case.site in ("dynamics", "dynamics_pool")
    A = (2, 4, 8, 16)[seed % 4] if dyn else 1
    ws, bs = [], []
    if case.stem:
        w = numpy.zeros((C, case.stem_cin, 3, 3), numpy.float32)
        w[:, :case.in_channels] = _sparse_int_conv(rs, C, case.in_channels, 2, two=0.3)
        if dyn:             # the action plane reaches 3/8 of the channels through one tap each
            for co in rs.choice(C, max(1, 3 * C // 8), replace=False):
                w[co, C, rs.randint(3), rs.randint(3)] = A * rs.choice([-1, 1]) * rs.randint(1, 3)
        ws.append(w)
        bs.append(rs.randint(-3, 4, C).astype(numpy.float32))
    for _ in range(case.blocks):
        ws.append(_sparse_int_conv(rs, C, C, 3, two=0.3))
        bs.append(rs.randint(-3, 4, C).astype(numpy.float32))
        ws.append(_sparse_int_conv(rs, C, C, 1, two=0.2))
        bs.append(rs.randint(-4, 2, C).astype(numpy.float32))
    act = _ends(n, A, rs) if dyn else None
    hi = 64
    while True:
        x = numpy.random.RandomState(seed + 1).randint(-hi, hi + 1, (n, case.in_channels, case.H, case.W)).astype(numpy.float32)
        ref, bound = tower64(x, ws, bs, case.site, act, A)
        if bound < 2.0 ** 24:
            return x, ws, bs, act, A, ref
        assert hi > 1, f"{case.name}: no integer fixture stays below 2^24"
        hi //= 2


def normal_operands(case, n, gain, seed):
    """Standard-normal operands scaled by `gain` (inputs, biases, the action plane's weights), A not a power of two."""
    rs = numpy.random.RandomState(seed)
    C, dyn = case.C, case.site in ("dynamics", "dynamics_pool")
    A = (3, 7, 12)[seed % 3] if dyn else 1
    x = (gain * rs.standard_normal((n, case.in_channels, case.H, case.W))).astype(numpy.float32)
    ws, bs = [], []
    for i in range(case.layers):
        cin = case.stem_cin if case.stem and i == 0 else C
        w = rs.standard_normal((C, cin, 3, 3)) / numpy.sqrt(9 * cin)
        if dyn and i == 0:
            w[:, C] *= gain
        ws.append(w.astype(numpy.float32))
        bs.append((0.1 * gain * rs.standard_normal(C)).astype(numpy.float32))
    return x, ws, bs, _ends(n, A, rs) if dyn else None, A


# ---------------------------------------------------------------------------------------------- references
def _conv(x, w, b=None):
    return torch.nn.functional.conv2d(x, torch.from_numpy(numpy.asarray(w, numpy.float64)),
                                      None if b is None else torch.from_numpy(numpy.asarray(b, numpy.float64)), 1, 1)


def tower64(x, ws, bs, site, act, A):
    """The tower in fp64 (ReLU after every conv, the block input added before the second ReLU of a block): (output,
    largest bound on any partial sum, |W| * |x| + |b| + |residual| over every layer)."""
    h = torch.from_numpy(x).double()
    bound = 0.0

    def layer(inp, w, b, res=None):
        nonlocal bound
        y = _conv(inp, w, b)
        s = _conv(inp.abs(), numpy.abs(w), numpy.abs(b))
        if res is not None:
            y, s = y + res, s + res.abs()
        bound = max(bound, float(s.max()))
        return torch.relu(y)

    k = 0
    if site != "prediction":
        inp = h
        if site != "representation":
            n, _, H, W = h.shape
            plane = torch.from_numpy(act.astype(numpy.float64) / A)[:, None, None, None].expand(n, 1, H, W)
            inp = torch.cat([h, plane], 1)
        h = layer(inp, ws[0], bs[0])
        k = 1
    while k < len(ws):
        t = layer(h, ws[k], bs[k])
        h = layer(t, ws[k + 1], bs[k + 1], h)
        k += 2
    return h.numpy(), bound


def per_layer_chain(x, ws, bs, site, act, A):
    """The same tower as one mz_debug_conv3x3 launch per conv (the network's per-layer route)."""
    from muzero_general_b200.engine import debug_conv3x3
    h, k = x, 0
    if site != "prediction":
        if site != "representation":
            n, _, H, W = x.shape
            plane = act.astype(numpy.float32) / numpy.float32(A)
            h = numpy.concatenate([x, numpy.broadcast_to(plane[:, None, None, None], (n, 1, H, W))], 1)
        h = debug_conv3x3(h, ws[0], bs[0], relu=True)
        k = 1
    while k < len(ws):
        t = debug_conv3x3(h, ws[k], bs[k], relu=True)
        h = debug_conv3x3(t, ws[k + 1], bs[k + 1], residual=h, relu=True)
        k += 2
    return h


def run(case, n, x, ws, bs, act, A, seed):
    """The device tower; asserts the plan of the launch (that of the first range when partitioned)."""
    from muzero_general_b200.engine import debug_small_tower
    kw = {}
    if case.site == "dynamics_pool":
        stride = 3
        kw = dict(parents=_ends(n, stride, numpy.random.RandomState(seed + 7)), pool_stride=stride, parts=case.parts)
    out, plan = debug_small_tower(x, ws, bs, site=case.site, actions=act, A=A, **kw)
    want, why = _plan_fn()(first_range(n, case.parts), case.stem_cin, case.C, case.H, case.W, case.blocks, case.stem, sms())
    assert plan == want, (case.name, n, plan, want, why)
    assert (plan["P"], plan["CO"]) == case.target, (case.name, plan)
    return out, plan


NAMES = [c.name for c in CASES]


@pytest.mark.parametrize("name", NAMES)
def test_small_tower_exact_on_integers(name):
    case = BY_NAME[name]
    S = sms()
    n, _ = case_plan(case, S, _plan_fn())
    t0 = time.perf_counter()
    x, ws, bs, act, A, ref = int_operands(case, n, seed=sum(map(ord, name)))
    assert numpy.count_nonzero(ref) > ref.size // 20, f"{name}: fixture too tame to test"
    got, plan = run(case, n, x, ws, bs, act, A, seed=1)
    bad = numpy.argwhere(got != ref)
    assert len(bad) == 0, f"{name} n={n} {plan}: {len(bad)} differences, first at {bad[0]}: " \
                          f"{got[tuple(bad[0])]} vs {ref[tuple(bad[0])]}"
    print(f"[small tower exact] {name}: n={n} P={plan['P']} CO={plan['CO']} boards/CTA={plan['boards']} "
          f"grid={plan['grid']} ({time.perf_counter() - t0:.2f} s)")


@pytest.mark.parametrize("name", NAMES)
def test_small_tower_equals_per_layer_chain(name):
    case = BY_NAME[name]
    n, _ = case_plan(case, sms(), _plan_fn())
    for k, gain in enumerate((1.0, 1e-4, 300.0)):
        seed = 3 * sum(map(ord, name)) + k
        x, ws, bs, act, A = normal_operands(case, n, gain, seed)
        got, _ = run(case, n, x, ws, bs, act, A, seed)
        want = per_layer_chain(x, ws, bs, case.site, act, A)
        assert numpy.isfinite(want).all() and numpy.count_nonzero(want) > want.size // 20
        bad = numpy.argwhere(got.view(numpy.uint32) != want.view(numpy.uint32))
        assert len(bad) == 0, f"{name} n={n} gain {gain}: {len(bad)} differences, first at {bad[0]}: " \
                              f"{got[tuple(bad[0])]!r} vs {want[tuple(bad[0])]!r}"


def test_debug_small_tower_refuses_what_the_planner_refuses():
    """A 9-column board has no fused launch: the entry says so instead of running another route."""
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import debug_small_tower
    x = numpy.zeros((2, 16, 3, 9), numpy.float32)
    ws = [numpy.zeros((16, 16, 3, 3), numpy.float32)] * 2
    with pytest.raises(_lib.MzError, match="refuses the shape.*2..8 columns"):
        debug_small_tower(x, ws, site="prediction")
