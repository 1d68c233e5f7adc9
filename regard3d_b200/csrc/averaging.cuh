// averaging.cuh -- pieces shared by the global-SfM averaging steps: rotations (rotavg.cu) and translations (transavg.cu).
#pragma once
#include "r3d_internal.cuh"
#include "lm_trust_region.cuh"

#include <vector>

namespace r3d {
namespace ra {

// The LM step over Nv variables, one CTA of kThreads (views or rotations first, then from index nb on the scales,
// bounded below by 1; nb = Nv: every variable unbounded): out[0] = 1/2 delta^T (D^2 delta - g) with the unclamped
// delta, out[1] = |x_new - x|^2 with x_new = Plus(x, scaled-back delta) (clamped), out[2] = |x|^2, out[3] =
// max |x - Plus(x, -g / scale)| (the projected unscaled gradient, from the current g).  A template, so that each
// translation unit that launches it has its own instance.
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_avg_step(const double* __restrict__ delta, const double* __restrict__ g,
                                                       const double* __restrict__ diag, const double* __restrict__ scale,
                                                       const double* __restrict__ x, uint32_t Nv, uint32_t nb, double inv_radius,
                                                       double* __restrict__ x_new, double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  double mcc = 0.0, dn = 0.0, xn = 0.0, gm = 0.0;
  for (uint32_t j = threadIdx.x; j < Nv; j += kThreads) {
    const double d2 = fmin(fmax(diag[j], 1e-6), 1e32) * inv_radius;
    mcc += delta[j] * (d2 * delta[j] - g[j]);
    const double d = delta[j] * scale[j];
    const double xj = x[j];
    const double gt = g[j] / scale[j];
    if (j < nb) {
      x_new[j] = xj + d;
      dn += d * d;
      gm = fmax(gm, fabs(gt));
    } else {
      const double xc = fmax(xj + d, 1.0);
      x_new[j] = xc;
      dn += (xc - xj) * (xc - xj);
      gm = fmax(gm, fabs(xj - fmax(xj - gt, 1.0)));
    }
    xn += xj * xj;
  }
  mcc = block_sum_fixed<kThreads>(mcc, red);
  dn = block_sum_fixed<kThreads>(dn, red);
  xn = block_sum_fixed<kThreads>(xn, red);
  gm = block_max_fixed<kThreads>(gm, red);
  if (threadIdx.x == 0) {
    out[0] = 0.5 * mcc;
    out[1] = dn;
    out[2] = xn;
    out[3] = gm;
  }
}

// 2-edge-connected components of an undirected multigraph on nodes 0..n-1 (edge k = (eu[k], ev[k]); parallel edges are
// not bridges, self-loops are ignored): bridges by Tarjan's low-link (iterative DFS), then connected components of the
// remaining edges.  Returns the component with the most nodes (>= 2; a tie keeps the one holding the smallest node), or
// -1; comp[v] = component of v, -1 for nodes without edges.  (rotavg.cu)
int largest_biedge_component(uint32_t n, const std::vector<uint32_t>& eu, const std::vector<uint32_t>& ev, std::vector<int>& comp);

}  // namespace ra
}  // namespace r3d
