"""The residual heads (csrc/heads.cuh::heads_one_sample in heads_kernel<32> / heads_kernel<128>, and the generic big_*_kernel
route of csrc/resnet.cu) against plain references, case by case over tests/headcases.py, through mz_debug_heads, which runs
the network's own call-site helpers with every output, the pool's other slots and the board layouts' padding starting as
NaN bytes.  Every run asserts the plan of its launch.

  * rescale (models.py:530-553): bit for bit equal to a numpy float32 restatement, in every layout and at every site
  * logits: on integer operands (partial sums below 2^24, hidden units >= 0 or <= -104 for every sample) EQUAL to fp64;
    on standard-normal operands at gains 1, 1e-4 and 300 inside a bound propagated layer by layer with
    gamma_n = n u / (1 - n u), u = 2^-24, which holds for any summation order (split-K, 16-lane reductions)
  * support_to_scalar (models.py:645-666): one-hot and two-hot logits give the numpy float32 restatement of
    inverse_value_transform bit for bit at every support index; otherwise inside a first-order budget of fp64
  * forced routes agree inside the same bounds, and bit for bit where they add in the same order; a 22-bit input in the
    split layout gives the dense input's logits; partitioned ranges equal one range
"""
import zlib

import numpy
import pytest

from headcases import BY_NAME, CASES, HeadsCase, batch, case_plan, first_range, layer_ks

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ELU = 5.0       # device ELU expf(x) - 1 for x <= 0: expf within 2 ulp (<= 4u since expf(x) <= 1), the subtraction rounds once (<= u)
F32 = numpy.float32
WORST = {}


def gamma(n):
    return n * U / (1.0 - n * U)


@pytest.fixture(scope="module")
def eng():
    from muzero_general_b200 import engine
    from muzero_general_b200.engine import debug_heads, debug_heads_plan  # noqa: F401
    return engine


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def report(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))


def teardown_module(module):
    if WORST:
        print("\nworst measured error / bound:", {k: "%.3g" % v for k, v in sorted(WORST.items())})


# ---------------------------------------------------------------------------------------------------- references
def f16_split(x):
    """(x_h, x_l) of the split layout: x_h = fp16(x), x_l = fp16(float32(x - x_h) * 2048)."""
    x = numpy.asarray(x, F32)
    h = x.astype(numpy.float16)
    lo = ((x - h.astype(F32)) * F32(2048.0)).astype(numpy.float16)
    return h, lo


def staged(x, layout):
    """The fp32 values heads_kernel stages from x in ``layout``: x_h + x_l 2^-11 joined by one rounding."""
    if layout == "dense":
        return numpy.asarray(x, F32)
    h, lo = f16_split(x)
    if layout == "f16":
        return h.astype(F32)
    return (h.astype(numpy.float64) + lo.astype(numpy.float64) / 2048.0).astype(F32)


def rescale_ref(x):
    """models.py:530-553 in float32: per (sample, channel) min / max over the positions, scale < 1e-5 gets 1e-5 added."""
    n, C = x.shape[:2]
    v = x.reshape(n, C, -1)
    lo, hi = v.min(2, keepdims=True), v.max(2, keepdims=True)
    scale = hi - lo
    scale[scale < F32(1e-5)] += F32(1e-5)
    return ((v - lo) / scale).reshape(x.shape)


def board_index(C, H, W):
    """[C, H*W] offsets (in halves) of (channel, position) inside one board of the P64S layout, and the padding mask."""
    c = numpy.arange(C)[:, None]
    p = numpy.arange(H * W)[None, :]
    pos = (p // W + 1) * 8 + p % W
    idx = pos * 64 + (((c >> 3) ^ (pos & 7)) << 3) + (c & 7)
    pad = numpy.ones(4096, bool)
    pad[idx.ravel()] = False
    return idx, pad


def check_layout_state(stored, v, layout, C, H, W, what):
    """stored [n, floats] in the board layout equals fp16 / split fp16 of v [n, C, H, W]; the padding keeps its NaN bytes."""
    n = v.shape[0]
    halves = stored.reshape(n, -1).view(numpy.uint16)
    idx, pad = board_index(C, H, W)
    h, lo = f16_split(v.reshape(n, C, H * W))
    assert numpy.array_equal(halves[:, idx], h.view(numpy.uint16)), what + ": x_h"
    assert (halves[:, :4096][:, pad] == 0xFFFF).all(), what + ": padding written"
    if layout == "split":
        assert numpy.array_equal(halves[:, 4096 + idx], lo.view(numpy.uint16)), what + ": x_l"
        assert (halves[:, 4096:][:, pad] == 0xFFFF).all(), what + ": padding written (x_l)"


def head_forward(x, head, want_bound=False):
    """fp64 conv1x1 -> flatten -> MLP (ELU between layers) of x [n, C, HW] (the staged fp32 values), and with
    ``want_bound`` the propagated bound on the device's error."""
    n, C, HW = x.shape
    xd = x.astype(numpy.float64)
    W1, b1 = head["conv_w"].astype(numpy.float64), head["conv_b"].astype(numpy.float64)
    h = (numpy.einsum("rk,nkp->nrp", W1, xd) + b1[None, :, None]).reshape(n, -1)
    mag = (numpy.einsum("rk,nkp->nrp", numpy.abs(W1), numpy.abs(xd)) + numpy.abs(b1)[None, :, None]).reshape(n, -1)
    delta = gamma(C + 1) * mag
    sums = [mag]
    fc = head["fc"]
    for l, (w, b) in enumerate(fc):
        w, b = w.astype(numpy.float64), b.astype(numpy.float64)
        aw = numpy.abs(w)
        pre = h @ w.T + b
        mag = (numpy.abs(h) + delta) @ aw.T + numpy.abs(b)
        sums.append(numpy.abs(h) @ aw.T + numpy.abs(b))
        delta = delta @ aw.T + gamma(w.shape[1] + 1) * mag
        if l < len(fc) - 1:
            h = numpy.where(pre > 0, pre, numpy.expm1(numpy.minimum(pre, 0.0)))
            delta = delta + C_ELU * U
        else:
            h = pre
    return (h, delta, sums) if want_bound else h


def ivt32(x):
    """common.cuh::inverse_value_transform restated in float32 (every operation correctly rounded)."""
    x = numpy.asarray(x, F32)
    eps = F32(0.001)
    t = (numpy.abs(x) + F32(1.0)) + eps
    t = F32(1.0) + (F32(4.0) * eps) * t
    t = numpy.sqrt(t) - F32(1.0)
    t = t / (F32(2.0) * eps)
    t = t * t - F32(1.0)
    return numpy.sign(x).astype(F32) * t


def ivt64(x):
    return numpy.sign(x) * (((numpy.sqrt(1 + 4 * 0.001 * (numpy.abs(x) + 1 + 0.001)) - 1) / (2 * 0.001)) ** 2 - 1)


def ivt64_slope(x):
    a = numpy.abs(x)
    r = numpy.sqrt(1 + 4 * 0.001 * (a + 1 + 0.001))
    return 2 * ((r - 1) / 0.002) / 0.002 * (2 * 0.001 / r)


# ---------------------------------------------------------------------------------------------------- operands
def make_heads(case, rs, kind, gain=1.0):
    heads = []
    for rc, hidden, n_out in case.heads:
        widths = [rc * case.HW, *hidden, n_out]
        if kind == "int":
            h = {"conv_w": rs.randint(-2, 3, (rc, case.C)).astype(F32), "conv_b": rs.randint(-4, 5, rc).astype(F32), "fc": []}
            for i in range(len(widths) - 1):
                dens = min(1.0, 8.0 / widths[i])
                w = (rs.randint(-1, 2, (widths[i + 1], widths[i])) * (rs.rand(widths[i + 1], widths[i]) < dens)).astype(F32)
                h["fc"].append([w, rs.randint(-3, 4, widths[i + 1]).astype(F32)])
        else:
            h = {"conv_w": (rs.randn(rc, case.C) * gain).astype(F32), "conv_b": (rs.randn(rc) * gain).astype(F32), "fc": []}
            for i in range(len(widths) - 1):
                h["fc"].append([(rs.randn(widths[i + 1], widths[i]) / numpy.sqrt(widths[i])).astype(F32),
                                rs.randn(widths[i + 1]).astype(F32)])
        heads.append(h)
    return heads


def fix_int_biases(heads, x, rs):
    """Hidden biases that keep every hidden unit >= 0 for every sample or <= -104 for every sample (ELU exact: the
    identity, or expf underflowed and exactly -1)."""
    for head in heads:
        n = x.shape[0]
        W1, b1 = head["conv_w"].astype(numpy.float64), head["conv_b"].astype(numpy.float64)
        h = (numpy.einsum("rk,nkp->nrp", W1, x.reshape(n, x.shape[1], -1).astype(numpy.float64)) + b1[None, :, None]).reshape(n, -1)
        for l, (w, b) in enumerate(head["fc"][:-1]):
            z = h @ w.astype(numpy.float64).T
            up = rs.rand(len(b)) < 0.6
            b[:] = numpy.where(up, -z.min(0) + rs.randint(0, 3, len(b)), -z.max(0) - 104 - rs.randint(0, 3, len(b)))
            pre = z + b
            assert ((pre >= 0).all(0) | (pre <= -104).all(0)).all()
            h = numpy.where(pre > 0, pre, -1.0)


def run(eng, case, x, heads, route="planned", parts=None, layout=None, sm=None):
    out = eng.debug_heads(x, heads, case.site, layout or case.layout, route, parts or case.parts, case.pool_stride, case.out_slot)
    if sm is not None:
        n = x.shape[0]
        _, want = case_plan(case, sm, eng.debug_heads_plan, route) if n == batch(case, sm) else (None, None)
        if want is not None:
            assert out["plan"] == want, (case.name, route, out["plan"], want)
        if route != "planned":
            assert out["plan"]["route"] == route
    return out


def check_rescale(case, x, out):
    """Every rescaling output of a run against the float32 restatement; the pool's other slots keep their NaN bytes."""
    if case.site == "prediction":
        return
    want = rescale_ref(staged(x, case.layout))
    assert numpy.array_equal(out["rescaled"].view(numpy.uint32), want.view(numpy.uint32)), case.name + ": rescaled"
    pool = out["pool"]
    others = [s for s in range(case.pool_stride) if s != case.out_slot]
    assert (pool[:, others].view(numpy.uint32) == 0xFFFFFFFF).all(), case.name + ": another pool slot written"
    if case.layout == "dense":
        assert numpy.array_equal(pool[:, case.out_slot].reshape(want.shape).view(numpy.uint32), want.view(numpy.uint32))
    else:
        check_layout_state(pool[:, case.out_slot], want, case.layout, case.C, case.H, case.W, case.name + ": pool")
        check_layout_state(out["state"], want, case.layout, case.C, case.H, case.W, case.name + ": state")


def int_input(case, rs, n):
    x = rs.randint(-3, 4, (n, case.C, case.H, case.W)).astype(F32)
    # a constant channel and a channel spanning ~1e-6 (the 1e-5 rule), in every sample
    x[:, 0] = 2.0
    return x


# ---------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_heads_exact_on_integer_operands(eng, sm_count, name):
    """Rescale bit for bit; logits EQUAL to fp64 (every partial sum an integer below 2^24)."""
    case = BY_NAME[name]
    rs = numpy.random.RandomState(zlib.crc32(name.encode()))
    n = batch(case, sm_count)
    x = int_input(case, rs, n)
    heads = make_heads(case, rs, "int")
    fix_int_biases(heads, x, rs)
    out = run(eng, case, x, heads, sm=sm_count)
    check_rescale(case, x, out)
    xs = staged(x, case.layout).reshape(n, case.C, -1)
    for h, head in enumerate(heads):
        want, _, sums = head_forward(xs, head, want_bound=True)
        assert max(float(s.max()) for s in sums) < 2 ** 24, name
        got = out["logits"][h]
        assert numpy.array_equal(got.astype(numpy.float64), want), (name, h, numpy.abs(got - want).max())
    if case.heads:
        assert not numpy.isnan(out["scalar"][0]).any()
        if case.site == "prediction":
            assert (out["scalar"][1].view(numpy.uint32) == 0xFFFFFFFF).all(), "the policy head has no scalar"


def check_budget(case, xs, heads, out, key):
    for h, head in enumerate(heads):
        want, delta, _ = head_forward(xs, head, want_bound=True)
        err = numpy.abs(out["logits"][h].astype(numpy.float64) - want)
        assert (err <= delta).all(), (case.name, key, h, float((err / delta).max()))
        report(key, (err / numpy.maximum(delta, 1e-300)).max())
    if case.heads:
        check_scalar_budget(case, out, key)


def check_scalar_budget(case, out, key):
    """support_to_scalar of the device's own logits against fp64: the max is exact; each exp(l - m) carries the rounding of
    the difference (u |d|) and expf's 2 ulp (4u); the sums gamma_F; the division u; then the slope of the transform over
    the interval, plus the transform's own float32 rounding measured at the interval's ends and at its centre."""
    logits = out["logits"][0].astype(numpy.float64)
    S = case.S
    k = numpy.arange(-S, S + 1, dtype=numpy.float64)
    m = logits.max(1, keepdims=True)
    d = logits - m
    e = numpy.exp(d)
    rel = numpy.abs(d) * U + 4 * U
    den, num = e.sum(1), (k * e).sum(1)
    F = 2 * S + 1
    dden = (e * rel).sum(1) + gamma(F) * den
    dnum = (numpy.abs(k) * e * rel).sum(1) + gamma(F) * (numpy.abs(k) * e).sum(1)
    x = num / den
    tiny = F * 2.0 ** -149                          # an exp that underflows into the subnormals loses its relative bound
    dden, dnum = dden + tiny, dnum + S * tiny
    dx = (dnum + numpy.abs(x) * dden) / (den - dden) + U * numpy.abs(x)
    want = ivt64(x)
    ends = [numpy.clip(x - dx, -S, S), x, numpy.clip(x + dx, -S, S)]
    own = numpy.max([numpy.abs(ivt32(F32(y)).astype(numpy.float64) - ivt64(F32(y).astype(numpy.float64))) for y in ends], 0)
    bound = ivt64_slope(numpy.abs(x) + dx) * (dx + numpy.abs(x) * U) + 2 * own + 1e-300
    err = numpy.abs(out["scalar"][0].astype(numpy.float64) - want)
    assert (err <= bound).all(), (case.name, key, float((err / bound).max()))
    report(key + " scalar", (err / bound).max())


@pytest.mark.parametrize("gain", [1.0, 1e-4, 300.0])
@pytest.mark.parametrize("name", [c.name for c in CASES if c.heads])
def test_heads_inside_fp64_budget(eng, sm_count, name, gain):
    case = BY_NAME[name]
    rs = numpy.random.RandomState(zlib.crc32(f"{name} {gain}".encode()))
    n = min(batch(case, sm_count), 300)
    x = (rs.randn(n, case.C, case.H, case.W) * gain).astype(F32)
    x[:, 0] = F32(gain)                                                     # a constant channel
    x[:, 1] = F32(gain) * (1 + rs.rand(n, case.H, case.W) * 1e-6)           # a channel spanning ~1e-6 (the 1e-5 rule)
    heads = make_heads(case, rs, "normal", gain)
    out = run(eng, case, x, heads)
    check_rescale(case, x, out)
    check_budget(case, staged(x, case.layout).reshape(n, case.C, -1), heads, out, "logits")


@pytest.mark.parametrize("name", ["pred_warp_s300", "pred_wide_s300_c48"])
def test_scalar_budget_on_saturated_logits(eng, name):
    """The last value layer scaled by 40 (netcases.py `sat`): logits spread over ~100, support_to_scalar near its ends."""
    case = BY_NAME[name]
    rs = numpy.random.RandomState(5)
    x = rs.randn(64, case.C, case.H, case.W).astype(F32)
    heads = make_heads(case, rs, "normal")
    heads[0]["fc"][-1] = [w * F32(40.0) for w in heads[0]["fc"][-1]]
    out = run(eng, case, x, heads)
    assert numpy.ptp(out["logits"][0], 1).max() > 50
    check_budget(case, x.reshape(64, case.C, -1), heads, out, "sat")


def one_hot_case(S, site):
    """TicTacToe-sized heads whose first head writes support index o = a B + b (B = ceil(sqrt(2 S + 1))) as the digits a
    and b: conv1x1 passes the first 6 channels through (6 x 9 >= 2 B inputs), one FC layer puts 110 on inputs a and B + b."""
    heads = [(6, (), 2 * S + 1)] + ([(1, (), 3)] if site == "prediction" else [])
    return HeadsCase("onehot", site, 16, 3, 3, "dense", tuple(heads), 1, "warp")


@pytest.mark.parametrize("S,site", [(10, "dynamics"), (10, "prediction"), (300, "dynamics"), (300, "prediction")])
@pytest.mark.parametrize("route", ["warp", "wide", "generic"])
def test_inverse_value_transform_bit_for_bit(eng, S, site, route):
    """Logits one-hot after float32 exp (the hot entry 220, the others 110 or 0) at every support index, and two-hot ties
    (an exact half-integer expectation): the scalar equals the float32 restatement of inverse_value_transform(k - S) bit
    for bit."""
    case = one_hot_case(S, site)
    F = 2 * S + 1
    B = int(numpy.ceil(numpy.sqrt(F)))
    rs = numpy.random.RandomState(S)
    pairs = [(o1, o2) for o1, o2 in rs.randint(0, F, (256, 2)) if o1 // B == o2 // B and o1 != o2][:48]
    n = F + len(pairs)
    flat = numpy.zeros((n, case.C * case.HW), F32)
    for j, hot in enumerate([(o,) for o in range(F)] + pairs):
        for o in hot:
            flat[j, o // B] = flat[j, B + o % B] = 1.0
    w = numpy.zeros((F, 6 * case.HW), F32)
    w[numpy.arange(F), numpy.arange(F) // B] = 110.0
    w[numpy.arange(F), B + numpy.arange(F) % B] = 110.0
    heads = [{"conv_w": numpy.eye(6, case.C, dtype=F32), "conv_b": numpy.zeros(6, F32), "fc": [[w, numpy.zeros(F, F32)]]}]
    if site == "prediction":
        heads.append({"conv_w": numpy.ones((1, case.C), F32), "conv_b": numpy.zeros(1, F32),
                      "fc": [[numpy.ones((3, case.HW), F32), numpy.zeros(3, F32)]]})
    out = run(eng, case, flat.reshape(n, case.C, case.H, case.W), heads, route=route)
    logits = out["logits"][0]
    assert (numpy.sort(logits, 1)[:, -3] <= logits.max(1) - 104).all()           # one- or two-hot after exp
    k = numpy.concatenate([numpy.arange(F) - S, [(o1 + o2 - 2 * S) / 2.0 for o1, o2 in pairs]]).astype(F32)
    assert numpy.array_equal(out["scalar"][0].view(numpy.uint32), ivt32(k).view(numpy.uint32)), (S, site, route)


@pytest.mark.parametrize("name", [c.name for c in CASES if c.layout == "dense" and c.parts == 1 and c.heads])
def test_forced_routes_agree(eng, name):
    """warp, wide and generic on the same head: inside the same fp64 bounds; bit-identical rescale always, logits where every
    layer adds with ks = 1 on both routes, scalars where both reduce with 32 lanes."""
    case = BY_NAME[name]
    rs = numpy.random.RandomState(11)
    n = 37
    x = rs.randn(n, case.C, case.H, case.W).astype(F32)
    heads = make_heads(case, rs, "normal")
    outs = {}
    for route in ("warp", "wide", "generic"):
        p, _ = eng.debug_heads_plan(n, case.C, case.H, case.W, case.heads, case.site, "dense", route)
        if p is None:
            continue
        outs[route] = run(eng, case, x, heads, route=route)
        check_rescale(case, x, outs[route])
        check_budget(case, x.reshape(n, case.C, -1), heads, outs[route], "routes")
    ref = outs.get("generic") or outs["wide"]
    for route, o in outs.items():
        if case.site != "prediction":
            assert numpy.array_equal(o["rescaled"].view(numpy.uint32), ref["rescaled"].view(numpy.uint32))
        ks1 = all(k == 1 for head in layer_ks(case, route) for k in head)
        for h in range(len(case.heads)):
            if ks1:
                assert numpy.array_equal(o["logits"][h].view(numpy.uint32), ref["logits"][h].view(numpy.uint32)), (name, route, h)
        lanes32 = route != "warp" or len(case.heads) == 1
        if lanes32 and ks1:
            assert numpy.array_equal(o["scalar"][0].view(numpy.uint32), ref["scalar"][0].view(numpy.uint32)), (name, route)


@pytest.mark.parametrize("name", [c.name for c in CASES if c.layout == "split"])
def test_split_layout_equals_dense_on_22_bit_inputs(eng, name):
    case = BY_NAME[name]
    rs = numpy.random.RandomState(3)
    n = 19
    x = (rs.randint(-2 ** 21, 2 ** 21, (n, case.C, case.H, case.W)) / 2048.0).astype(F32)
    assert numpy.array_equal(staged(x, "split"), x)
    heads = make_heads(case, rs, "normal")
    dense = run(eng, case, x, heads, layout="dense", parts=1)
    split = run(eng, case, x, heads, layout="split", parts=1)
    assert dense["plan"]["route"] == split["plan"]["route"]
    for h in range(len(case.heads)):
        assert numpy.array_equal(dense["logits"][h].view(numpy.uint32), split["logits"][h].view(numpy.uint32)), (name, h)
    assert numpy.array_equal(dense["scalar"].view(numpy.uint32), split["scalar"].view(numpy.uint32))
    if case.site != "prediction":
        assert numpy.array_equal(dense["rescaled"].view(numpy.uint32), split["rescaled"].view(numpy.uint32))


@pytest.mark.parametrize("name", [c.name for c in CASES if c.parts > 1])
def test_partitions_equal_one_range(eng, sm_count, name):
    case = BY_NAME[name]
    rs = numpy.random.RandomState(4)
    n = batch(case, sm_count)
    assert first_range(n, case.parts) < n
    x = rs.randn(n, case.C, case.H, case.W).astype(F32)
    heads = make_heads(case, rs, "normal")
    one = run(eng, case, x, heads, parts=1)
    split = run(eng, case, x, heads)
    for key in ("scalar", "rescaled", "pool") + (("state",) if "state" in one else ()):
        assert numpy.array_equal(one[key].view(numpy.uint32), split[key].view(numpy.uint32)), (name, key)
    assert numpy.array_equal(one["logits"][0].view(numpy.uint32), split["logits"][0].view(numpy.uint32))
