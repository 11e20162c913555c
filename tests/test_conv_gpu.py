"""conv3x3 kernels against torch's fp32 conv2d (a floating-point kernel: torch fp32 is the reference).

Tolerances stated here: the CUDA-core path accumulates in fp32 (rtol 1e-4); the wgmma "fp16" mode multiplies
fp16 operands (10-bit mantissa, like tf32) with fp32 accumulation and stores fp16:
|err| <= 2e-3 * (|w| . |x|) + 1e-3 * |out| per output; the wgmma "x3" mode (split fp16 operands (x = x_h + x_l/2^11), three partial
products, csrc/conv_x3.cu) is fp32-grade: |err| <= 4e-6 * (|w| . |x|) + 2e-6 * |out| + 1e-6 - two orders of magnitude
inside the CUDA-core path's own tolerance."""
import numpy
import pytest
import torch

pytestmark = pytest.mark.gpu


def _case(n, C, H, W, seed, with_res):
    rs = numpy.random.RandomState(seed)
    x = rs.standard_normal((n, C, H, W)).astype(numpy.float32)
    w = (rs.standard_normal((C, C, 3, 3)) / numpy.sqrt(9 * C)).astype(numpy.float32)
    b = (0.1 * rs.standard_normal(C)).astype(numpy.float32)
    r = rs.standard_normal((n, C, H, W)).astype(numpy.float32) if with_res else None
    return x, w, b, r


def _ref(x, w, b, r, relu):
    y = torch.nn.functional.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), 1, 1)
    if r is not None:
        y = y + torch.from_numpy(r)
    return (torch.relu(y) if relu else y).numpy()


@pytest.mark.parametrize("n,C,H,W", [(5, 64, 6, 7), (9, 16, 3, 3), (3, 16, 6, 6), (2, 8, 48, 48), (2, 16, 24, 24), (2, 16, 12, 12)])
def test_cuda_core_conv_matches_torch(n, C, H, W):
    from muzero_general_b200.engine import debug_conv3x3
    for relu, with_res in ((False, False), (True, True)):
        x, w, b, r = _case(n, C, H, W, 1, with_res)
        got = debug_conv3x3(x, w, b, r, relu, tensor_cores=False)
        numpy.testing.assert_allclose(got, _ref(x, w, b, r, relu), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("n,H,W", [(1, 6, 7), (2, 6, 7), (7, 6, 7), (300, 6, 7), (5, 6, 6), (4, 3, 3), (3, 5, 4)])
def test_tensor_core_conv_matches_torch(n, H, W):
    from muzero_general_b200.engine import debug_conv3x3
    C = 64
    for relu, with_res in ((False, False), (True, True), (True, False)):
        x, w, b, r = _case(n, C, H, W, 2 + n, with_res)
        got = debug_conv3x3(x, w, b, r, relu, tensor_cores="fp16")
        ref = _ref(x, w, b, r, relu)
        # error budget: fp16 operand rounding (2^-11 each) on sum |w||x|, fp16 rounding of the stored result
        bound = torch.nn.functional.conv2d(torch.from_numpy(numpy.abs(x)), torch.from_numpy(numpy.abs(w)), None, 1, 1).numpy()
        err = numpy.abs(got - ref)
        assert (err <= 2e-3 * bound + 1e-3 * numpy.abs(ref) + 1e-5).all(), float((err / (bound + 1e-6)).max())
        # and it is not accidentally exact garbage: correlates with the reference
        assert numpy.abs(got - ref).mean() < 5e-3


@pytest.mark.parametrize("n,H,W", [(1, 6, 7), (2, 6, 7), (3, 6, 7), (4, 6, 7), (7, 6, 7), (300, 6, 7), (1200, 6, 7), (5, 6, 6), (4, 3, 3), (3, 5, 4)])
def test_split_operand_conv_is_fp32_grade(n, H, W):
    """x3 mode against an fp64 convolution: the error budget of 3 partial products of split 16-bit operands."""
    from muzero_general_b200.engine import debug_conv3x3
    C = 64
    for relu, with_res, gain in ((False, False, 1.0), (True, True, 1.0), (True, False, 300.0), (False, True, 1e-4)):
        x, w, b, r = _case(n, C, H, W, 2 + n, with_res)
        x = (x * gain).astype(numpy.float32)
        if r is not None:
            r = (r * gain).astype(numpy.float32)
        b = (b * gain).astype(numpy.float32)
        got = debug_conv3x3(x, w, b, r, relu, tensor_cores="x3")
        y = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), 1, 1)
        if r is not None:
            y = y + torch.from_numpy(r).double()
        ref = (torch.relu(y) if relu else y).numpy()
        bound = torch.nn.functional.conv2d(torch.from_numpy(numpy.abs(x)).double(), torch.from_numpy(numpy.abs(w)).double(), None, 1, 1).numpy()
        err = numpy.abs(got - ref)
        worst = float((err / (4e-6 * bound + 2e-6 * numpy.abs(ref) + 1e-6 * gain)).max())
        print(f"x3 conv n={n} {H}x{W} gain={gain}: max err / budget = {worst:.3f}, max abs err {err.max():.3e}")
        assert worst <= 1.0


def test_split_operand_conv_exact_on_small_integers():
    """Small integer operands are exact in the hi parts (lo parts are zero): the x3 result equals the fp32 reference
    exactly - tiling, tap shifts, padding, in-place update and the register residual are right."""
    from muzero_general_b200.engine import debug_conv3x3
    rs = numpy.random.RandomState(0)
    for n in (1, 3, 11, 600):
        C, H, W = 64, 6, 7
        x = rs.randint(-2, 3, size=(n, C, H, W)).astype(numpy.float32)
        w = rs.randint(-1, 2, size=(C, C, 3, 3)).astype(numpy.float32)
        b = rs.randint(-3, 4, size=C).astype(numpy.float32)
        r = rs.randint(-5, 6, size=(n, C, H, W)).astype(numpy.float32)
        got = debug_conv3x3(x, w, b, r, True, tensor_cores="x3")
        numpy.testing.assert_array_equal(got, _ref(x, w, b, r, True))


def test_tensor_core_conv_exact_on_fp16_representable_inputs():
    """With small integer operands (exact in fp16, results below 2048 so the fp16 store is exact too) the
    tensor-core result equals the fp32 reference exactly: proves tiling, tap shifts and padding are right."""
    from muzero_general_b200.engine import debug_conv3x3
    rs = numpy.random.RandomState(0)
    n, C, H, W = 11, 64, 6, 7
    x = rs.randint(-2, 3, size=(n, C, H, W)).astype(numpy.float32)
    w = rs.randint(-1, 2, size=(C, C, 3, 3)).astype(numpy.float32)
    b = rs.randint(-3, 4, size=C).astype(numpy.float32)
    r = rs.randint(-5, 6, size=(n, C, H, W)).astype(numpy.float32)
    got = debug_conv3x3(x, w, b, r, True, tensor_cores="fp16")
    numpy.testing.assert_array_equal(got, _ref(x, w, b, r, True))
