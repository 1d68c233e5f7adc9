"""The Levenberg-Marquardt trust-region controller shared by the GPU least-squares solvers
(regard3d_b200/csrc/lm_trust_region.cuh), compiled as plain C++ with g++ and driven through scripted step sequences.
Every decision, radius and decrease factor is held bit for bit to a Python statement of Ceres' rules; the small dense
Cholesky solve of the same header is held to numpy."""
import math
import os
import random
import subprocess
import textwrap

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

DRIVER = textwrap.dedent(r'''
    #include <cstdio>
    #include <cstdlib>
    #include <cstring>
    #include <vector>
    #include "regard3d_b200/csrc/lm_trust_region.cuh"

    // lm: params, start cost and gradient, then one scripted outcome per iteration; prints the state after each one
    static int run_lm() {
      r3d::LmParams p;
      double cost, gmax0;
      int n;
      if (std::scanf("%u %lf %lf %lf %lf %lf %lf %lf %d", &p.max_iterations, &p.huber_a, &p.function_tolerance,
                     &p.gradient_tolerance, &p.parameter_tolerance, &p.initial_radius, &cost, &gmax0, &n) != 9) return 1;
      struct Step { int pd; double mcc, dn2, xn2, new_cost, gmax; };
      std::vector<Step> steps(n);
      for (Step& s : steps)
        if (std::scanf("%d %lf %lf %lf %lf %lf", &s.pd, &s.mcc, &s.dn2, &s.xn2, &s.new_cost, &s.gmax) != 6) return 1;
      r3d::LmTrustRegion lm(p);
      if (!lm.start(gmax0))
        for (uint32_t iter = 1; iter <= p.max_iterations; ++iter) {
          lm.iterations = iter;
          const Step& s = steps[iter - 1];
          bool accepted = false, stop = false;
          if (lm.step_usable(s.pd != 0, s.mcc)) {
            stop = lm.step_too_small(s.dn2, s.xn2);
            if (!stop && (accepted = lm.accept(cost, s.new_cost, s.mcc))) {
              cost = s.new_cost;
              stop = lm.converged(s.gmax);
            }
          }
          if (!stop && !accepted) stop = lm.reject();
          std::printf("step %.17g %.17g\n", lm.radius, lm.decrease_factor);
          if (stop) break;
        }
      std::printf("end %u %u %d\n", lm.iterations, lm.successful, lm.termination);
      return 0;
    }

    template <int N>
    static int run_chol() {
      double A[N * N], b[N];
      for (double& a : A) if (std::scanf("%lf", &a) != 1) return 1;
      for (double& v : b) if (std::scanf("%lf", &v) != 1) return 1;
      const bool ok = r3d::chol_solve_small<N>(A, b);
      std::printf("%d", (int)ok);
      for (double v : b) std::printf(" %.17g", v);
      for (int i = 0; i < N; ++i)
        for (int j = 0; j <= i; ++j) std::printf(" %.17g", A[N * i + j]);
      std::printf("\n");
      return 0;
    }

    int main(int argc, char** argv) {
      if (argc < 2) return 2;
      if (!std::strcmp(argv[1], "lm")) return run_lm();
      if (!std::strcmp(argv[1], "chol6")) return run_chol<6>();
      if (!std::strcmp(argv[1], "chol12")) return run_chol<12>();
      return 2;
    }
''')


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("lm")
    src = d / "lm_driver.cpp"
    src.write_text(DRIVER)
    exe = d / "lm_driver"
    p = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror", "-I", ROOT, str(src),
                        "-o", str(exe)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]

    def run(mode, text):
        r = subprocess.run([str(exe), mode], input=text, capture_output=True, text=True, timeout=60)
        assert r.returncode == 0, r.stderr[-2000:]
        return r.stdout
    return run


PRM = dict(max_iterations=50, huber_a=16.0, function_tolerance=1e-6, gradient_tolerance=1e-10, parameter_tolerance=1e-8,
           initial_radius=1e4)


def reference(prm, cost, gmax0, steps):
    """Ceres' trust-region LM decisions, stated directly: ([(radius, decrease_factor) after each iteration],
    (iterations, successful steps, termination))."""
    radius, df, successful, trace = prm["initial_radius"], 2.0, 0, []
    if gmax0 <= prm["gradient_tolerance"]:
        return trace, (0, 0, 2)
    ptol = prm["parameter_tolerance"]
    it = 0
    for it in range(1, prm["max_iterations"] + 1):
        pd, mcc, dn2, xn2, new_cost, gmax = steps[it - 1]
        if pd and mcc > 0.0 and math.isfinite(mcc):
            if math.sqrt(dn2) <= ptol * (math.sqrt(xn2) + ptol):
                trace.append((radius, df))
                return trace, (it, successful, 3)
            rho = (cost - new_cost) / mcc
            if rho > 1e-3:
                t = 2.0 * rho - 1.0
                radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - t * t * t))
                df = 2.0
                successful += 1
                small = abs(cost - new_cost) < prm["function_tolerance"] * cost
                cost = new_cost
                trace.append((radius, df))
                if small:
                    return trace, (it, successful, 1)
                if gmax <= prm["gradient_tolerance"]:
                    return trace, (it, successful, 2)
                continue
        radius = radius / df
        df = df * 2.0
        trace.append((radius, df))
        if radius < 1e-32:
            return trace, (it, successful, 4)
    return trace, (it, successful, 0)


def run_both(driver, steps, prm=PRM, cost=100.0, gmax0=1.0):
    steps = list(steps) + [(0, 0.0, 0.0, 0.0, 0.0, 0.0)] * (prm["max_iterations"] - len(steps))
    text = "%d %r %r %r %r %r %r %r %d\n" % (prm["max_iterations"], prm["huber_a"], prm["function_tolerance"],
                                             prm["gradient_tolerance"], prm["parameter_tolerance"],
                                             prm["initial_radius"], cost, gmax0, len(steps))
    text += "".join("%d %r %r %r %r %r\n" % s for s in steps)
    lines = driver("lm", text).split("\n")
    trace = [tuple(float(v) for v in ln.split()[1:]) for ln in lines if ln.startswith("step")]
    end = tuple(int(v) for v in next(ln for ln in lines if ln.startswith("end")).split()[1:])
    ref_trace, ref_end = reference(prm, cost, gmax0, steps)
    assert end == ref_end
    assert trace == ref_trace  # exact: the same IEEE operations in the same order
    return trace, end


def good(cost, new_cost, mcc=None, gmax=1.0):
    """a usable step from cost to new_cost (relative decrease 1 unless mcc is given), far above the parameter tolerance"""
    return (1, cost - new_cost if mcc is None else mcc, 1.0, 1.0, new_cost, gmax)


def test_gradient_stop_at_start(driver):
    trace, end = run_both(driver, [], gmax0=1e-11)
    assert end == (0, 0, 2) and trace == []


def test_function_tolerance_wins_over_gradient_tolerance(driver):
    # the second accepted step changes the cost by less than 1e-6 of the old cost, and the gradient is below its
    # tolerance too: termination 1
    _, end = run_both(driver, [good(100.0, 50.0), good(50.0, 50.0 - 1e-6, gmax=0.0)])
    assert end == (2, 2, 1)
    _, end = run_both(driver, [good(100.0, 50.0, gmax=0.0)])
    assert end == (1, 1, 2)


def test_parameter_tolerance(driver):
    _, end = run_both(driver, [good(100.0, 90.0), (1, 5.0, 1e-20, 1.0, 80.0, 1.0)])
    assert end == (2, 1, 3)


@pytest.mark.parametrize("pd,mcc", [(1, 0.0), (1, -1.0), (1, float("nan")), (1, float("inf")), (0, 5.0)])
def test_unusable_steps_are_rejected(driver, pd, mcc):
    # the trial cost would be accepted if the step were taken: only the step test stands in the way
    trace, end = run_both(driver, [(pd, mcc, 1.0, 1.0, 1.0, 1.0)] * 3, prm=dict(PRM, max_iterations=3))
    assert end == (3, 0, 0)
    assert trace == [(1e4 / 2, 4.0), (1e4 / 8, 8.0), (1e4 / 64, 16.0)]


def test_repeated_rejection_collapses_the_trust_region(driver):
    # radius 1e4 / 2^(k (k + 1) / 2) after k rejections: 2.5e-28 after 14, 7.5e-33 < 1e-32 after 15
    trace, end = run_both(driver, [(1, 1.0, 1.0, 1.0, 200.0, 1.0)] * 20)
    assert end == (15, 0, 4)
    assert trace[-1][0] == 1e4 / 2.0 ** 120


def test_rejection_after_acceptance_restarts_the_decrease_factor(driver):
    bad = (1, 1.0, 1.0, 1.0, 200.0, 1.0)
    trace, _ = run_both(driver, [bad, bad, good(100.0, 90.0, mcc=20.0), bad], prm=dict(PRM, max_iterations=4))
    assert [df for _, df in trace] == [4.0, 8.0, 2.0, 4.0]


def test_radius_grows_to_the_cap(driver):
    # relative decrease 1: the radius triples, 1e4 * 3^26 > 1e16
    steps = [good(1000.0 - k, 999.0 - k) for k in range(30)]
    trace, end = run_both(driver, steps, prm=dict(PRM, max_iterations=30), cost=1000.0)
    assert end == (30, 30, 0)
    assert trace[24][0] == 1e4 * 3.0 ** 25 and trace[25][0] == 1e16 and trace[-1][0] == 1e16


def test_running_out_of_iterations(driver):
    steps = [good(100.0 - k, 99.0 - k, mcc=3.0) for k in range(5)]
    _, end = run_both(driver, steps, prm=dict(PRM, max_iterations=5))
    assert end == (5, 5, 0)


def test_random_sequences(driver):
    rng = random.Random(7)
    for _ in range(200):
        steps, cost = [], 100.0
        for _ in range(PRM["max_iterations"]):
            kind = rng.random()
            mcc = rng.choice([0.0, -1.0, float("nan"), float("inf")]) if kind < 0.1 else rng.uniform(1e-3, 10.0)
            new_cost = cost - mcc * rng.uniform(-0.5, 1.5)
            dn2 = 1e-30 if rng.random() < 0.02 else rng.uniform(1e-6, 1.0)
            steps.append((int(rng.random() > 0.05), mcc, dn2, rng.uniform(0.0, 10.0), new_cost,
                          rng.choice([1.0, 1.0, 1.0, 1e-12])))
            cost = min(cost, new_cost)
        run_both(driver, steps, cost=100.0)


def chol(driver, A, b):
    n = len(b)
    out = driver("chol%d" % n, " ".join("%r" % float(v) for v in list(A.ravel()) + list(b)) + "\n").split()
    vals = [float(v) for v in out[1:]]
    L = np.zeros((n, n))
    L[np.tril_indices(n)] = vals[n:]
    return out[0] == "1", np.array(vals[:n]), L


@pytest.mark.parametrize("n", [6, 12])
def test_chol_solve_small(driver, n):
    rng = np.random.default_rng(n)
    J = rng.standard_normal((3 * n, n))
    A = J.T @ J + np.diag(rng.uniform(0.1, 1.0, n))
    b = rng.standard_normal(n)
    ok, x, L = chol(driver, A, b)
    assert ok
    np.testing.assert_allclose(L, np.linalg.cholesky(A), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(x, np.linalg.solve(A, b), rtol=1e-10, atol=1e-12)
    # indefinite: a negative eigenvalue; the right-hand side comes back untouched
    w, V = np.linalg.eigh(A)
    w[n // 2] = -1.0
    ok, x, _ = chol(driver, (V * w) @ V.T, b)
    assert not ok
    np.testing.assert_array_equal(x, b)
