"""The backup's division by a visit count (tree.cuh::div_by_count) against IEEE division, bit for bit.

div_by_count(s, n, y) with y = RN(1/n) computes q0 = RN(s*y), r = fma(-q0, n, s), q = fma(r, y, q0) and claims RN(s/n)
for every double s (the subnormal, zero and non-finite numerators go to the IEEE division).  A C restatement with libm's
fma() runs it on tens of millions of numerators for every n <= 4096: random magnitudes over the whole normal range, values
next to powers of two, sums of discounted returns like the ones a search accumulates, and the special values.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy
import pytest

C_SRC = r"""
#include <math.h>
#include <float.h>
#include <stdint.h>
/* tree.cuh::div_by_count; y = 1.0 / n is the correctly rounded reciprocal (__drcp_rn on the device) */
static double div_by_count(double s, int n, double y) {
    if (!(fabs(s) >= 0x1p-990 && fabs(s) < INFINITY)) return s / (double)n;
    const double q0 = s * y;
    const double r = fma(-q0, (double)n, s);
    return fma(r, y, q0);
}
/* every s[i] against every n in [n0, n1]: returns the number of results that differ from s / n in any bit */
int64_t mismatches(const double* s, int64_t m, int n0, int n1) {
    int64_t bad = 0;
    for (int n = n0; n <= n1; ++n) {
        const double y = 1.0 / (double)n;
        for (int64_t i = 0; i < m; ++i) {
            const double a = div_by_count(s[i], n, y), b = s[i] / (double)n;
            union { double d; uint64_t u; } ua = {a}, ub = {b};
            bad += ua.u != ub.u;
        }
    }
    return bad;
}
"""


@pytest.fixture(scope="module")
def lib():
    d = tempfile.mkdtemp(prefix="mz_divexact_")
    src, so = os.path.join(d, "div.c"), os.path.join(d, "div.so")
    with open(src, "w") as f:
        f.write(C_SRC)
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so, src, "-lm"])
    lib = ctypes.CDLL(so)
    lib.mismatches.restype = ctypes.c_int64
    lib.mismatches.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int]
    return lib


def run(lib, s, n0, n1):
    s = numpy.ascontiguousarray(s, dtype=numpy.float64)
    return lib.mismatches(s.ctypes.data, s.size, n0, n1)


def numerators(rs, m):
    """m numerators of both signs: log-uniform over 1e-300 .. 1e300, and next to powers of two"""
    mag = 10.0 ** rs.uniform(-300, 300, m // 2)
    p2 = numpy.ldexp(1.0, rs.randint(-990, 1000, m - m // 2))
    steps = rs.randint(-4, 5, p2.size)
    near = numpy.array([numpy.nextafter(p, numpy.inf if k > 0 else -numpy.inf) if k else p for p, k in zip(p2, steps)])
    s = numpy.concatenate([mag, near])
    return s * numpy.where(rs.rand(s.size) < 0.5, -1.0, 1.0)


def test_random_numerators_every_count_up_to_4096(lib):
    # 2500 numerators x 4096 counts = 1.0e7 divisions
    rs = numpy.random.RandomState(7)
    assert run(lib, numerators(rs, 2500), 1, 4096) == 0


def test_value_sums_of_a_search(lib):
    # what a node's value_sum looks like: sums of up to 50 discounted returns of per-step rewards around 1 (CartPole)
    # and of signed values in (-1, 1) (board games)
    rs = numpy.random.RandomState(11)
    ret = numpy.cumsum(rs.uniform(0.0, 1.2, (400, 50)) * 0.997 ** numpy.arange(50), axis=1).ravel()
    signed = numpy.cumsum(rs.uniform(-1.0, 1.0, (400, 50)), axis=1).ravel()
    assert run(lib, numpy.concatenate([ret, signed, -ret]), 1, 256) == 0


def test_special_numerators(lib):
    tiny = numpy.array([0.0, -0.0, 5e-324, -5e-324, 9 * 5e-324, 2.2250738585072014e-308, -2.2250738585072014e-308,
                        2.0 ** -990, numpy.nextafter(2.0 ** -990, 0.0), 1e-305, numpy.inf, -numpy.inf, numpy.nan,
                        numpy.finfo(numpy.float64).max, -numpy.finfo(numpy.float64).max])
    assert run(lib, tiny, 1, 4096) == 0
