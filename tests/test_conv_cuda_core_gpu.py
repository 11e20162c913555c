"""The CUDA-core conv3x3 kernel (csrc/resnet.cu: conv3x3_kernel, the "strict" path every other conv is checked
against) at every launch shape of tests/convcases.py, against an fp64 convolution.  Each case runs without and with
the bias + residual + ReLU epilogue, in two checks:

  exact      x in [-2, 2], w in [-1, 1], bias in [-3, 3], residual in [-5, 5], all integers: every partial sum is an
             integer below 2^24, so any fp32 summation order is exact and the result must EQUAL the fp64 conv.  Any
             wrong tap, band, stride, padding, cin chunk, board offset or cout tile shows.
  rounding   standard-normal operands at gains 1, 1e-4 and 300 (x, bias and residual scaled):
             |dev - ref| <= (gamma_n + gamma64_n) * (sum |w||x| + |b| + |r|), n = 9 Cin + 2, gamma_n = n u / (1 - n u),
             u = 2^-24.  That is the rigorous bound of a chain of n fp32 roundings (9 Cin FMAs, the bias add, the
             residual add; ReLU does not increase it), plus the same bound at u = 2^-53 for the fp64 reference.

mz_debug_conv3x3 fills its device output with NaN before the launch, so an element the kernel does not write fails
both checks."""
import numpy
import pytest
import torch

from convcases import BY_NAME, CASES, REFUSED, REFUSED_REASON

pytestmark = pytest.mark.gpu

EPILOGUES = {"plain": (False, False, False), "bias_res_relu": (True, True, True)}
GAINS = (1.0, 1e-4, 300.0)


def _gamma(n, u):
    return n * u / (1 - n * u)


def _conv64(x, w, stride):
    return torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, stride, 1).numpy()


def _operands(c, rs, gain=None):
    Ho, Wo = c.out_hw
    xs, ws, rs_shape = (c.n, c.cin, c.H, c.W), (c.cout, c.cin, 3, 3), (c.n, c.cout, Ho, Wo)
    if gain is None:        # small integers
        x, w = rs.randint(-2, 3, xs), rs.randint(-1, 2, ws)
        b, r = rs.randint(-3, 4, c.cout), rs.randint(-5, 6, rs_shape)
    else:
        x, w = rs.standard_normal(xs) * gain, rs.standard_normal(ws)
        b, r = rs.standard_normal(c.cout) * gain, rs.standard_normal(rs_shape) * gain
    return [a.astype(numpy.float32) for a in (x, w, b, r)]


def _run(c, x, w, b, r, epilogue):
    from muzero_general_b200.engine import debug_conv3x3
    use_b, use_r, relu = EPILOGUES[epilogue]
    b, r = (b if use_b else None), (r if use_r else None)
    got = debug_conv3x3(x, w, b, r, relu, tensor_cores=False, stride=c.stride)
    assert got.shape == (c.n, c.cout) + c.out_hw
    ref = _conv64(x, w, c.stride)
    size = _conv64(numpy.abs(x), numpy.abs(w), c.stride)
    if b is not None:
        ref = ref + b.astype(numpy.float64)[None, :, None, None]
        size = size + numpy.abs(b).astype(numpy.float64)[None, :, None, None]
    if r is not None:
        ref = ref + r
        size = size + numpy.abs(r)
    if relu:
        ref = numpy.maximum(ref, 0.0)
    return got, ref, size


@pytest.mark.parametrize("epilogue", list(EPILOGUES))
@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_cuda_core_conv_against_fp64(name, epilogue):
    c = BY_NAME[name]
    rs = numpy.random.RandomState(sum(map(ord, name)) + len(epilogue))
    # exact on small integers
    got, ref, size = _run(c, *_operands(c, rs), epilogue)
    assert size.max() < 2 ** 24
    bad = numpy.argwhere(got != ref)
    assert len(bad) == 0, f"{name} {epilogue}: {len(bad)} of {got.size} elements differ, first at {tuple(bad[0])}: " \
                          f"{got[tuple(bad[0])]} != {ref[tuple(bad[0])]}"
    # rounding bound on standard-normal operands
    n = 9 * c.cin + 2
    gamma = _gamma(n, 2.0 ** -24) + _gamma(n, 2.0 ** -53)
    worst = 0.0
    for gain in GAINS:
        got, ref, size = _run(c, *_operands(c, rs, gain), epilogue)
        err = numpy.abs(got - ref)
        bound = gamma * size
        ok = err <= bound                       # NaN (an unwritten element) compares False
        assert ok.all(), f"{name} {epilogue} gain {gain}: {int((~ok).sum())} elements beyond the bound, first at " \
                         f"{tuple(numpy.argwhere(~ok)[0])}"
        worst = max(worst, float((err / numpy.maximum(bound, numpy.finfo(numpy.float64).tiny)).max()))
    print(f"[conv3x3] {name} {epilogue}: worst err / bound {worst:.2e}")


def test_row_no_cout_tile_holds_is_refused_before_any_launch():
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import debug_conv3x3
    c = REFUSED
    x, w, b, r = _operands(c, numpy.random.RandomState(0))
    with pytest.raises(_lib.MzError, match=REFUSED_REASON):
        debug_conv3x3(x, w, b, r, True, stride=c.stride)


def test_create_refuses_a_net_whose_row_no_cout_tile_holds():
    """An 8-channel net on a 1 x 1031 board: its stem's launch plan is refused, so mz_create fails and names the reason
    and the stage (rather than the first search failing part-way).  The same net one column narrower is created, and
    so is the 64-channel net on a 6 x 67 board that was refused before the cout tiles could be narrower than 64."""
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import SearchEngine
    from muzero_general_b200.games import load_game_module
    cfg = load_game_module("connect4").MuZeroConfig()
    cfg.observation_shape, cfg.action_space, cfg.channels, cfg.blocks = (3, 1, 1031), list(range(4)), 8, 1
    with pytest.raises(_lib.MzError, match=REFUSED_REASON) as e:
        SearchEngine(cfg, max_games=4, num_simulations=2)
    assert "representation stem: 3 -> 8 channels" in str(e.value) and "1 x 1031" in str(e.value)
    cfg.observation_shape = (3, 1, 1030)
    SearchEngine(cfg, max_games=4, num_simulations=2).close()
    cfg.observation_shape, cfg.channels = (3, 6, 67), 64
    SearchEngine(cfg, max_games=4, num_simulations=2).close()


@pytest.mark.parametrize("mode", ["fp16", "x3"])
def test_tensor_core_modes_take_only_64_to_64_at_stride_1(mode):
    from muzero_general_b200 import _lib
    from muzero_general_b200.engine import debug_conv3x3
    rs = numpy.random.RandomState(1)
    for cin, cout, stride in ((64, 68, 1), (32, 64, 1), (64, 64, 2)):
        x = rs.standard_normal((2, cin, 6, 7)).astype(numpy.float32)
        w = rs.standard_normal((cout, cin, 3, 3)).astype(numpy.float32)
        with pytest.raises(_lib.MzError) as e:
            debug_conv3x3(x, w, tensor_cores=mode, stride=stride)
        assert e.value.code == _lib.MZ_EUNSUPPORTED, (cin, cout, stride, str(e.value))
