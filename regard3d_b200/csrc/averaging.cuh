// averaging.cuh -- pieces shared by the global-SfM averaging steps: rotations (rotavg.cu) and translations (transavg.cu).
#pragma once
#include "r3d_internal.cuh"

#include <chrono>
#include <vector>

namespace r3d {
namespace ra {

// ---- fixed-order block reductions (every thread gets the result) --------------------------------------------------
template <int kThreads>
__device__ double block_sum_fixed(double v, double* red) {
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31u) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < kThreads / 32; ++w) s += red[w];
  return s;
}
template <int kThreads>
__device__ double block_max_fixed(double v, double* red) {
  for (int o = 16; o >= 1; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31u) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < kThreads / 32; ++w) s = fmax(s, red[w]);
  return s;
}

inline double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// 2-edge-connected components of an undirected multigraph on nodes 0..n-1 (edge k = (eu[k], ev[k]); parallel edges are
// not bridges, self-loops are ignored): bridges by Tarjan's low-link (iterative DFS), then connected components of the
// remaining edges.  Returns the component with the most nodes (>= 2; a tie keeps the one holding the smallest node), or
// -1; comp[v] = component of v, -1 for nodes without edges.  (rotavg.cu)
int largest_biedge_component(uint32_t n, const std::vector<uint32_t>& eu, const std::vector<uint32_t>& ev, std::vector<int>& comp);

template <typename T>
struct DevArr {  // device scratch out of the worker's pool (context.cu)
  DeviceWorker* w;
  T* p = nullptr;
  explicit DevArr(DeviceWorker& worker) : w(&worker) {}
  DevArr(const DevArr&) = delete;
  DevArr& operator=(const DevArr&) = delete;
  ~DevArr() { if (p) pool_release(*w, p); }
  bool alloc(size_t n) {
    p = (T*)pool_alloc(*w, std::max<size_t>(n, 1) * sizeof(T));
    return p != nullptr;
  }
};

}  // namespace ra
}  // namespace r3d
