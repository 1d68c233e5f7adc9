"""The deterministic transcendentals (regard3d_b200/csrc/detmath.cuh) that every AC-RANSAC decision passes through,
compiled as plain C++ with g++ (as the library's host code is: no FMA contraction): accuracy against mpmath, and the
monotonicity of log10_det across its range-reduction seams, on which the slack of the tier-1 NFA lower bound rests
(acransac_fused.cu subtracts 1e-9 (1 + |LB|) besides the table error)."""
import math
import os
import subprocess
import textwrap

import mpmath
import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

DRIVER = textwrap.dedent(r'''
    #include <cmath>
    #include <cstdio>
    #include <cstdlib>
    #include <vector>
    #include "regard3d_b200/csrc/detmath.cuh"

    static double eval(int fn, double x) {
      using namespace r3d::dm;
      return fn == 0 ? log10_det(x) : fn == 1 ? cbrt_det(x) : fn == 2 ? cos_det(x) : acos_det(x);
    }

    int main(int argc, char** argv) {
      if (argc < 2) return 1;
      if (argv[1][0] == 'e') {  // eval <fn>: n doubles on stdin -> n doubles on stdout (raw)
        const int fn = std::atoi(argv[2]);
        std::vector<double> x;
        double v;
        while (std::fread(&v, sizeof v, 1, stdin) == 1) x.push_back(eval(fn, v));
        std::fwrite(x.data(), sizeof(double), x.size(), stdout);
        return 0;
      }
      // mono <ulps> <e0> <e1>: walk log10_det over +-ulps steps around every 2^e and sqrt(1/2) 2^e, e = e0 .. e1; print
      // the number of steps, of decreasing steps, the largest decrease and the largest in ulp of the value
      const long n = std::atol(argv[2]);
      const int e0 = std::atoi(argv[3]), e1 = std::atoi(argv[4]);
      long steps = 0, drops = 0;
      double worst = 0.0, worst_ulp = 0.0;
      for (int e = e0; e <= e1; ++e)
        for (double s : {std::ldexp(1.0, e), std::ldexp(0.70710678118654752440, e)}) {
          double x = s;
          for (long i = 0; i < n; ++i) x = std::nextafter(x, 0.0);
          double prev = eval(0, x);
          for (long i = 0; i < 2 * n && x < 1.7e308; ++i) {
            x = std::nextafter(x, INFINITY);
            const double y = eval(0, x);
            ++steps;
            if (y < prev) {
              ++drops;
              worst = std::fmax(worst, prev - y);
              worst_ulp = std::fmax(worst_ulp, (prev - y) / (std::nextafter(std::fabs(prev), INFINITY) - std::fabs(prev)));
            }
            prev = y;
          }
        }
      std::printf("%ld %ld %.17g %.17g\n", steps, drops, worst, worst_ulp);
      return 0;
    }
''')


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("detmath")
    src = d / "detmath_driver.cpp"
    src.write_text(DRIVER)
    exe = d / "detmath_driver"
    p = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror", "-I", ROOT, str(src),
                        "-o", str(exe)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]

    def run(*args, data=None):
        r = subprocess.run([str(exe)] + [str(a) for a in args], input=None if data is None else data.tobytes(),
                           capture_output=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        return r.stdout
    return run


def _eval(driver, fn, x):
    return np.frombuffer(driver("e", fn, data=np.ascontiguousarray(x, np.float64)), np.float64)


def _ulp_errors(got, exact):
    """|got - exact| in units of the last place of the exact value (mpmath at 50 digits)."""
    out = []
    for g, ex in zip(got, exact):
        ulp = math.ulp(float(ex)) if float(ex) != 0 else math.ulp(0.0)
        out.append(float(abs(mpmath.mpf(g) - ex) / ulp))
    return np.array(out)


mpmath.mp.dps = 50
RNG = np.random.default_rng(11)
SEAMS = np.concatenate([[math.ldexp(1.0, e), math.ldexp(math.sqrt(0.5), e)] for e in range(-60, 61)])

# written-down accuracy bounds (ulp of the exact result), each a little above what these inputs show
LOG10_ULP = 4.0
CBRT_ULP = 2.0
COS_ULP = 4.0   # where |cos t| >= 1/2; near its zero at pi / 2 the error is absolute: the reduced argument pi / 2 - |t|
COS_ABS = 4 * 2.0 ** -53  # carries the rounding of pi, so the relative error grows as 1 / |cos t|
ACOS_ULP = 8.0


def test_log10_accuracy(driver):
    x = np.r_[10.0 ** RNG.uniform(-300, 300, 3000), RNG.uniform(0.5, 2.0, 1000), SEAMS,
              SEAMS * (1 + 2.0 ** -52), SEAMS * (1 - 2.0 ** -53)]
    got = _eval(driver, 0, x)
    err = _ulp_errors(got, [mpmath.log10(mpmath.mpf(v)) for v in x])
    assert err.max() <= LOG10_ULP, (err.max(), x[err.argmax()])


def test_cbrt_accuracy(driver):
    # the seven-point cubic takes cube roots of |R| + sqrt(R^2 - Q^3) over many decades
    x = np.r_[10.0 ** RNG.uniform(-250, 250, 3000), RNG.uniform(0, 8, 1000), np.ldexp(1.0, np.arange(-90, 91))]
    got = _eval(driver, 1, x)
    assert got[x == 0].tolist() == [0.0] * int((x == 0).sum())
    nz = x > 0
    err = _ulp_errors(got[nz], [mpmath.cbrt(mpmath.mpf(v)) for v in x[nz]])
    assert err.max() <= CBRT_ULP, (err.max(), x[nz][err.argmax()])


def test_cos_accuracy(driver):
    # cos(theta / 3), cos((theta +- 2 pi) / 3) with theta = acos(..) in [0, pi]: arguments in [-pi / 3, pi]
    x = np.r_[RNG.uniform(-math.pi, math.pi, 4000), np.linspace(-math.pi, math.pi, 1001)]
    got = _eval(driver, 2, x)
    exact = [mpmath.cos(mpmath.mpf(v)) for v in x]
    away = np.abs(np.cos(x)) >= 0.5
    err = _ulp_errors(got[away], [exact[i] for i in np.nonzero(away)[0]])
    assert err.max() <= COS_ULP, (err.max(), x[away][err.argmax()])
    absolute = np.array([float(abs(mpmath.mpf(g) - ex)) for g, ex in zip(got, exact)])
    assert absolute.max() <= COS_ABS, absolute.max()


def test_acos_accuracy(driver):
    x = np.r_[RNG.uniform(-1, 1, 4000), 1 - 10.0 ** -RNG.uniform(1, 16, 500), -1 + 10.0 ** -RNG.uniform(1, 16, 500),
              -1.0, 0.0, 1.0]
    got = _eval(driver, 3, x)
    exact = [mpmath.acos(mpmath.mpf(v)) for v in x]
    nz = x < 1.0
    err = _ulp_errors(got[nz], [exact[i] for i in np.nonzero(nz)[0]])
    assert err.max() <= ACOS_ULP, (err.max(), x[nz][err.argmax()])
    assert got[x == 1.0].tolist() == [0.0]
    assert np.isnan(_eval(driver, 3, np.array([1.0 + 2.0 ** -52, -1.0 - 2.0 ** -52]))).all()


@pytest.mark.parametrize("e0,e1,ulps", [(-60, 60, 200000), (-1022, -61, 20000), (61, 1023, 20000)])
def test_log10_monotone_at_seams(driver, e0, e1, ulps):
    """log10_det is not exactly monotone where frexp's range reduction switches branch.  The NFA takes it of
    residual + FLT_EPSILON, anywhere in [2^-23, DBL_MAX] (with an infinite precision the resection model's residuals
    reach far above 2^60), and of the bins' lower edges.  Its largest drop d around the seams 2^e and sqrt(1/2) 2^e of
    every binade (+-200 000 ulp for |e| <= 60, +-20 000 ulp beyond, down to subnormal-free 2^-1022) is what a residual's
    logalpha can fall below its bin's lower-edge value.  The NFA multiplies it by k - NS < 2^24, so the bound can be off
    by at most 2^24 d, which must stay far inside the fixed 1e-4 that the tier-1 bound subtracts."""
    steps, drops, worst, worst_ulp = driver("mono", ulps, e0, e1).split()
    steps, drops, worst, worst_ulp = int(steps), int(drops), float(worst), float(worst_ulp)
    assert steps >= 2 * (e1 - e0 + 1) * 2 * ulps - 2 * ulps
    assert worst_ulp <= 2, (drops, worst, worst_ulp)          # measured: 1 ulp of log10 x, wherever x lies
    assert worst * 2 ** 24 <= 1e-5, worst
