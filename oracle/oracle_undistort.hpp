// oracle_undistort.hpp -- CPU ORACLE (test infrastructure; see oracle.h).
//
// get_ud_pixel of every camera model by a fixed number of Newton steps on the distortion map, restated statement for
// statement from regard3d_b200/csrc/p3p.cuh (p3p::undistort_pixel).  The resection oracle undistorts with it, and the
// triangulation oracle (oracle_sfm.cpp) does for Brown T2 and fisheye observations.
// model: openMVG EINTRINSIC 1..5; disto: k1 k2 k3 t1 t2 for the polynomial models, k1 k2 k3 k4 for the fisheye.
#pragma once
#include "oracle_detmath.hpp"

#include <cmath>

namespace orc {

constexpr int kUndistortIters = 10;

inline void undistort_newton(int model, double f, double ppx, double ppy, const double* disto, double x, double y, double* xo,
                             double* yo) {
  const double xd = (x - ppx) / f, yd = (y - ppy) / f;
  double xu = xd, yu = yd;
  if (model == 5) {
    const double rd = std::sqrt(xd * xd + yd * yd);
    if (rd > 1e-8) {
      double th = rd;
      for (int it = 0; it < kUndistortIters; ++it) {
        const double t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
        const double g = th * (1.0 + disto[0] * t2 + disto[1] * t4 + disto[2] * t6 + disto[3] * t8) - rd;
        const double dg = 1.0 + 3.0 * disto[0] * t2 + 5.0 * disto[1] * t4 + 7.0 * disto[2] * t6 + 9.0 * disto[3] * t8;
        th = th - g / dg;
      }
      const double ru = det::cos(0.5 * det::kPi - th) / det::cos(th);  // tan(theta)
      const double s = ru / rd;
      xu = xd * s;
      yu = yd * s;
    }
  } else if (model >= 2) {
    const double k1 = disto[0], k2 = model >= 3 ? disto[1] : 0.0, k3 = model >= 3 ? disto[2] : 0.0;
    const double t1 = model == 4 ? disto[3] : 0.0, t2 = model == 4 ? disto[4] : 0.0;
    for (int it = 0; it < kUndistortIters; ++it) {
      const double r2 = xu * xu + yu * yu, r4 = r2 * r2, r6 = r4 * r2;
      const double c = 1.0 + k1 * r2 + k2 * r4 + k3 * r6;
      const double dc = k1 + 2.0 * k2 * r2 + 3.0 * k3 * r4;
      const double fx = xu * c + t2 * (r2 + 2.0 * xu * xu) + 2.0 * t1 * xu * yu - xd;
      const double fy = yu * c + t1 * (r2 + 2.0 * yu * yu) + 2.0 * t2 * xu * yu - yd;
      const double a00 = c + 2.0 * xu * xu * dc + 6.0 * t2 * xu + 2.0 * t1 * yu;
      const double a01 = 2.0 * xu * yu * dc + 2.0 * t2 * yu + 2.0 * t1 * xu;
      const double a11 = c + 2.0 * yu * yu * dc + 6.0 * t1 * yu + 2.0 * t2 * xu;
      const double dt = a00 * a11 - a01 * a01;
      if (dt == 0.0) break;
      const double dx = (a11 * fx - a01 * fy) / dt, dy = (a00 * fy - a01 * fx) / dt;
      xu = xu - dx;
      yu = yu - dy;
    }
  }
  *xo = f * xu + ppx;
  *yo = f * yu + ppy;
}

}  // namespace orc
