"""downsample="resnet" (DownSample, models.py:233-275) on the device: the stem alone (csrc/resnet.cu Runner::downsample
through mz_debug_downsample, every device buffer but the input starting as NaN) at every case of
tests/downsamplecases.py, its output and its six stage outputs (conv1, resblocks1, conv2, resblocks2, the first pool,
resblocks3), in three checks:

  exact    sparse small-integer operands (downsamplecases.exact_operands): every partial sum is an integer below 2^24
           (asserted on the fp64 side) and every average an exact division, so the stem EQUALS a float64 restatement
           (F.conv2d, F.avg_pool2d(3, 2, 1) counting the padding).
  chain    standard-normal operands: the stem equals, bit for bit, a chain of mz_debug_conv3x3 launches (the bias,
           residual and ReLU of each conv as the reference has them) and a float32 restatement of avgpool3x3s2_kernel
           (the valid taps summed in row-major order from 0, then one correctly rounded division by 9).  Sharp at any
           depth, where the bound below loosens over 18 convs.
  budget   standard-normal operands at gains 1, 1e-4 and 300: each stage within a bound propagated stage by stage.  A conv
           adds (gamma_n + gamma64_n) * (|b| + |r| + sum |w| (|x| + e_x)), n = 9 Cin + 2 (the bound of
           tests/test_conv_cuda_core_gpu.py), and carries its input's bound e_x through sum |w| (and the residual's);
           ReLU is non-expansive; a pool carries the average of its input's bound and adds (gamma_9 + 2u) times the
           average of |x| + e_x (at most 8 rounded additions and one rounded division).

Mutants of csrc/resnet.cu, each built into the library and run against this file's tests on the cases c8_1x1_n33,
c16_17x33_in131, c96_20x24 and c16_210x160 on one H100 (failing tests out of 20):

  pool divisor = valid taps                 11: exact and chain on all four; budget on c8_1x1_n33
  pool padding off by one                    6: exact and chain on the three frames larger than 1 x 1
  resblocks2 / resblocks3 packed swapped    11: exact and chain on all four; budget on c8_1x1_n33
  resblocks3.0 without its residual         10: exact on three, chain on all four; budget on c8_1x1_n33
  conv1 with ReLU                           19: exact on three, chain and budget on all four
  H / W not updated after conv2              6: exact and chain on the three frames larger than 1 x 1 (every buffer of
                                               this build 8x as large, so the stale shapes stay inside them)
  Runner::blocks leaving the wrong workspace 20: every test
The budget alone misses five of them on the larger frames, where 18 convs loosen it; the chain test catches each.
"""
import numpy
import pytest
import torch
import torch.nn.functional as F

from downsamplecases import BY_NAME, conv_list, exact_operands, normal_operands

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
gamma = lambda n, u=U: n * u / (1 - n * u)
STAGES = ("conv1", "resblocks1", "conv2", "resblocks2", "pool1", "resblocks3", "output")
WORST = [0.0, ""]


def _device(case, x, ws, bs):
    """The seven stage outputs of the device stem, in STAGES order."""
    from muzero_general_b200 import _lib
    lib = _lib.load_library()
    out = lambda v: (v - 1) // 2 + 1
    h1, w1 = out(case.H), out(case.W)
    h2, w2 = out(h1), out(w1)
    shapes = [(case.C // 2, h1, w1)] * 2 + [(case.C, h2, w2)] * 2 + [(case.C, out(h2), out(w2))] * 2
    shapes = [(case.n,) + s for s in shapes]
    stages = numpy.empty(sum(int(numpy.prod(s)) for s in shapes), numpy.float32)
    res = numpy.empty((case.n, case.C) + case.hw, numpy.float32)
    x = numpy.ascontiguousarray(x, numpy.float32)
    w = numpy.ascontiguousarray(numpy.concatenate([a.ravel() for a in ws]), numpy.float32)
    b = numpy.ascontiguousarray(numpy.concatenate(bs), numpy.float32)
    rc = lib.mz_debug_downsample(0, case.n, case.cin, case.C, case.H, case.W, x.ctypes.data, w.ctypes.data, b.ctypes.data,
                                 res.ctypes.data, stages.ctypes.data)
    assert rc == 0, lib.mz_last_error(None).decode()
    got, at = [], 0
    for s in shapes:
        size = int(numpy.prod(s))
        got.append(stages[at:at + size].reshape(s))
        at += size
    return got + [res]


def _stem64(case, x, ws, bs, bound):
    """The stem in float64 (on the GPU: exact for the integer operands, ~1e-16 relative otherwise), per stage; with
    `bound`, also the propagated error bound of the fp32 device stem per stage, else the largest partial-sum magnitude
    of any conv (the integer operands must keep it below 2^24)."""
    dev = "cuda"
    t = lambda a: torch.from_numpy(numpy.asarray(a, numpy.float64)).to(dev)
    W, B = [t(w) for w in ws], [t(b) for b in bs]
    big = [0.0]

    def conv(i, v, e, stride, res=None, relu=False):
        n = 9 * ws[i].shape[1] + 2
        y = F.conv2d(v, W[i], B[i], stride, 1)
        size = F.conv2d(v.abs() + e, W[i].abs(), B[i].abs(), stride, 1)
        ey = F.conv2d(e, W[i].abs(), None, stride, 1)
        if res is not None:
            y, size, ey = y + res[0], size + res[0].abs() + res[1], ey + res[1]
        big[0] = max(big[0], float(size.max()))
        ey = ey + (gamma(n) + gamma(n, 2.0 ** -53)) * size if bound else ey
        return (F.relu(y) if relu else y), ey

    def blocks(v, e, first, count):
        for k in range(count):
            i = first + 2 * k
            h, eh = conv(i, v, e, 1, relu=True)
            v, e = conv(i + 1, h, eh, 1, res=(v, e), relu=True)
        return v, e

    def pool(v, e):
        P = lambda a: F.avg_pool2d(a, 3, 2, 1)
        g = gamma(9) + 2 * U + gamma(9, 2.0 ** -53) if bound else 0.0
        return P(v), P(e) + g * P(v.abs() + e)

    v = t(x)
    e = torch.zeros_like(v)
    out = []
    # no cuDNN: the native fp64 convolution sums each output directly (no FFT or Winograd transform of the operands)
    with torch.backends.cudnn.flags(enabled=False):
        v, e = conv(0, v, e, 2); out.append((v, e))
        v, e = blocks(v, e, 1, 2); out.append((v, e))
        v, e = conv(5, v, e, 2); out.append((v, e))
        v, e = blocks(v, e, 6, 3); out.append((v, e))
        v, e = pool(v, e); out.append((v, e))
        v, e = blocks(v, e, 12, 3); out.append((v, e))
        v, e = pool(v, e); out.append((v, e))
    return [(a.cpu().numpy(), b.cpu().numpy()) for a, b in out], big[0]


def _pool32(v):
    """avgpool3x3s2_kernel restated in float32: the valid taps of each window summed in row-major order starting from
    0 (a padding tap adds an exact 0), then one correctly rounded division by 9."""
    n, C, H, W = v.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    p = numpy.zeros((n, C, 2 * Ho + 1, 2 * Wo + 1), numpy.float32)
    p[:, :, 1:H + 1, 1:W + 1] = v
    s = numpy.zeros((n, C, Ho, Wo), numpy.float32)
    for dy in range(3):
        for dx in range(3):
            s = s + p[:, :, dy:dy + 2 * Ho:2, dx:dx + 2 * Wo:2]
    return s / numpy.float32(9)


def _chain(x, ws, bs):
    from muzero_general_b200.engine import debug_conv3x3
    conv = lambda v, i, stride, res=None, relu=False, bias=True: debug_conv3x3(v, ws[i], bs[i] if bias else None, res,
                                                                               relu, stride=stride)

    def blocks(v, first, count):
        for k in range(count):
            i = first + 2 * k
            v = conv(conv(v, i, 1, relu=True), i + 1, 1, res=v, relu=True)
        return v

    out = [conv(x, 0, 2, bias=False)]
    out.append(blocks(out[-1], 1, 2))
    out.append(conv(out[-1], 5, 2, bias=False))
    out.append(blocks(out[-1], 6, 3))
    out.append(_pool32(out[-1]))
    out.append(blocks(out[-1], 12, 3))
    out.append(_pool32(out[-1]))
    return out


def _first_difference(stage, got, want):
    bad = numpy.argwhere(~(got == want))
    return f"{stage}: {len(bad)} of {got.size} differ, first at {tuple(bad[0])}: {got[tuple(bad[0])]} != {want[tuple(bad[0])]}"


@pytest.mark.parametrize("name", list(BY_NAME))
def test_stem_equals_fp64_on_integer_operands(name):
    case = BY_NAME[name]
    x, ws, bs = exact_operands(case, numpy.random.RandomState(sum(map(ord, name))))
    want, big = _stem64(case, x, ws, bs, bound=False)
    assert big < 2 ** 24, big
    assert numpy.abs(want[-1][0]).max() > 0
    for stage, got, (w64, _) in zip(STAGES, _device(case, x, ws, bs), want):
        assert numpy.array_equal(got, w64.astype(numpy.float32)), _first_difference(stage, got, w64.astype(numpy.float32))


@pytest.mark.parametrize("name", list(BY_NAME))
def test_stem_equals_its_conv_chain_bit_for_bit(name):
    case = BY_NAME[name]
    x, ws, bs = normal_operands(case, numpy.random.RandomState(5 + len(name)), 1.0)
    for stage, got, want in zip(STAGES, _device(case, x, ws, bs), _chain(x, ws, bs)):
        assert got.shape == want.shape and numpy.array_equal(got, want), _first_difference(stage, got, want)


@pytest.mark.parametrize("gain", [1.0, 1e-4, 300.0])
@pytest.mark.parametrize("name", list(BY_NAME))
def test_stem_within_propagated_bound(name, gain):
    case = BY_NAME[name]
    x, ws, bs = normal_operands(case, numpy.random.RandomState(23 + len(name)), gain)
    ref, _ = _stem64(case, x, ws, bs, bound=True)
    for stage, got, (w64, bound) in zip(STAGES, _device(case, x, ws, bs), ref):
        err = numpy.abs(got.astype(numpy.float64) - w64)
        ok = err <= bound                       # NaN (a plane nobody wrote) compares False
        assert ok.all(), f"{name} gain {gain} {stage}: {int((~ok).sum())} beyond the bound, first at {tuple(numpy.argwhere(~ok)[0])}"
        ratio = float((err / numpy.maximum(bound, numpy.finfo(numpy.float64).tiny)).max())
        if ratio > WORST[0]:
            WORST[:] = [ratio, f"{name} gain {gain:g} {stage}"]
    print(f"[downsample] {name} gain {gain:g}: worst error/bound so far {WORST[0]:.3e} ({WORST[1]})")


def test_refusals_name_their_stage():
    """A frame whose conv1 output row is 1031 columns (prime, so one pixel per thread) is more than a CTA's items even in
    4-channel tiles: the stem is refused before any launch, naming the stage; a net with that frame is refused at
    creation the same way.  A conv1 or conv2 bias is refused (the reference's convs have none)."""
    from muzero_general_b200 import _lib
    lib = _lib.load_library()
    case = BY_NAME["c8_1x1_n1"]
    x = numpy.zeros((1, 3, 1, 2062), numpy.float32)
    ws = [numpy.zeros((co, ci, 3, 3), numpy.float32) for _, ci, co, _ in conv_list(case)]
    bs = [numpy.zeros(co, numpy.float32) for _, _, co, _ in conv_list(case)]
    w, b = numpy.concatenate([a.ravel() for a in ws]), numpy.concatenate(bs)
    res = numpy.empty((1, 8, 1, 129), numpy.float32)
    rc = lib.mz_debug_downsample(0, 1, 3, 8, 1, 2062, x.ctypes.data, w.ctypes.data, b.ctypes.data, res.ctypes.data, None)
    msg = lib.mz_last_error(None).decode()
    assert rc == _lib.MZ_EUNSUPPORTED and "DownSample conv1" in msg and "item budget" in msg, (rc, msg)
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    cfg = load_game_module("breakout").MuZeroConfig()
    cfg.observation_shape, cfg.channels = (3, 1, 2062), 8
    with pytest.raises(_lib.MzError, match="DownSample conv1"):
        SearchEngine(cfg, max_games=1, num_simulations=2)
    x = numpy.zeros((1, 3, 1, 1), numpy.float32)
    b[0] = 1.0
    rc = lib.mz_debug_downsample(0, 1, 3, 8, 1, 1, x.ctypes.data, w.ctypes.data, b.ctypes.data, res.ctypes.data, None)
    assert rc != 0 and "no bias" in lib.mz_last_error(None).decode()

