// akaze.cu -- Fast-AKAZE and OpenCV's AKAZE keypoints on the device (SURVEY.md 3, the feature stage): R3DFParams'
// default detector and the compute-matches dialog's default, on one scale space (the AKAZE passes: DESIGN.md 2.3a).
// COMPILED WITH --fmad=false (regard3d_b200/build.py): every float operation below rounds like the CPU restatement
// (oracle/oracle_akaze.cpp), one operation at a time, in the same order, so levels and keypoints agree bit for bit.
//
// Replaces cv::AKAZE2::detect (src/thirdparty/fast-akaze, called from src/Regard3DFeatures.cpp:590-614):
//   levels      Allocate_Memory_Evolution (AKAZEFeatures.cpp:73-151)            host: level table, FED tau (libm)
//   base level  G(img, 1.6), Hessian, kcontrast from G(img, 1.0) -> Scharr     k_row / k_col, k_kmax, k_khist, k_kscan
//   level i     Lt (copy or INTER_AREA half), G(Lt, 1), Scharr, Hessian,       k_half, k_row / k_col, k_det, k_pmg2,
//               pm_g2, FED sweeps (:286-347)                                   k_fed_step, k_fed_update
//   extrema     threaded Find_Scale_Space_Extrema (:623-724)                   k_cand_rows, k_cand_write (raster-order
//                                                                              compaction), k_same_level (one warp per
//                                                                              image and level), k_lower, k_upper
//   refinement  Do_Subpixel_Refinement (:741-795)                              k_refine
//   orientation Compute_Main_Orientation (:1226-1298) up to getAngleV2         k_orient; atan2f and Regard3D's degree
//                                                                              conversion on the host
// One launch serves the same level of every image of a batch (grid.z = image).  The FED workspace Lstep is one flat
// buffer per image, zero at the start (see oracle_akaze.cpp: the four corners of each level replay whatever earlier
// sweeps left at those flat indices).
#include "r3d_internal.cuh"

#include <algorithm>
#include <cfloat>
#include <chrono>
#include <climits>
#include <cmath>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <memory>
#include <thread>
#include <vector>

struct r3d_features {
  std::vector<std::vector<r3d_akaze_keypoint>> kps;
  std::vector<std::vector<float>> desc;  // r3d_extract_features only: per image kps[i].size() x 144
};

namespace r3d {
namespace akaze {

constexpr int kMaxBatch = 16, kMaxTaps = 16, kNbins = 300;
constexpr float kSoffset = 1.6f, kDerivFactor = 1.5f, kPercentile = 0.7f;
constexpr double kPi = 3.14159265358979323846;

// ---- host: level table and FED steps (the same code as the oracle's, so the same floats) ----------------------------

int fround(float v) { return (int)(v + 0.5f); }

std::vector<r3d_akaze_level> level_table(int W, int H, int omax, int nsub) {
  const float smax = 10.0f * std::sqrt(2.0f);
  std::vector<r3d_akaze_level> ev;
  int lw = W, lh = H, power = 1;
  for (int i = 0; i < omax; ++i) {
    for (int j = 0; j < nsub; ++j) {
      r3d_akaze_level s{};
      s.esigma = kSoffset * std::pow(2.f, (float)j / nsub + i);
      s.sigma_size = fround(s.esigma * kDerivFactor / power);
      s.border = fround(smax * s.sigma_size) + 1;
      s.etime = 0.5f * (s.esigma * s.esigma);
      s.octave = i;
      s.sublevel = j;
      s.ratio = (float)power;
      s.width = lw;
      s.height = lh;
      if (s.border * 2 + 1 >= lw || s.border * 2 + 1 >= lh) return ev;
      ev.push_back(s);
    }
    power <<= 1;
    lh >>= 1;
    lw >>= 1;
    if (lw < 80 || lh < 40) break;
  }
  return ev;
}

bool fed_is_prime(int number) {
  if (number <= 1) return false;
  if (number == 2 || number == 3 || number == 5 || number == 7) return true;
  if (number % 2 == 0 || number % 3 == 0 || number % 5 == 0 || number % 7 == 0) return false;
  bool is_prime = true;
  const int upper = (int)std::sqrt(1.0f + number);
  for (int d = 11; d <= upper; d += 2)
    if (number % d == 0) is_prime = false;
  return is_prime;
}

// fed_tau_by_process_timeV2(T, 1, 0.25, reordering = true) (fed.cpp)
std::vector<float> fed_tau(float T, float tau_max) {
  const float t = T / (float)1;
  const int n = (int)(std::ceil(std::sqrt(3.0f * t / tau_max + 0.25f) - 0.5f - 1.0e-8f) + 0.5f);
  if (n <= 0) return {};
  const float scale = 3.0f * t / (tau_max * (float)(n * (n + 1)));
  std::vector<float> tauh(n), tau(n);
  const float c = 1.0f / (4.0f * n + 2.0f);
  const float d = scale * tau_max / 2.0f;
  for (int k = 0; k < n; ++k) {
    const float hk = std::cos((float)kPi * (2.0f * k + 1.0f) * c);
    tauh[k] = d / (hk * hk);
  }
  if (n == 1) return tauh;
  const int kappa = n / 2;
  int prime = n + 1;
  while (!fed_is_prime(prime)) prime++;
  for (int k = 0, l = 0; l < n; ++k, ++l) {
    int index = 0;
    while ((index = ((k + 1) * kappa) % prime - 1) >= n) k++;
    tau[l] = tauh[index];
  }
  return tau;
}

struct Taps {
  int n, replicate;
  float k[kMaxTaps];
};

Taps gaussian_taps(float sigma) {  // gaussian_2D_convolutionV2's kernel: cv::getGaussianKernel(ksize, sigma, CV_32F)
  Taps t{};
  int n = (int)std::ceil(2.0f * (1.0f + (sigma - 0.8f) / (0.3f)));
  if (n % 2 == 0) n += 1;
  t.n = n;
  t.replicate = 1;
  const double sd = (double)sigma, scale2x = -0.125 / (sd * sd);
  const int c = (n - 1) / 2;
  double e[kMaxTaps], sum = 0.0;
  for (int i = 0, x = 1 - n; i < c; ++i, x += 2) {
    e[i] = std::exp((double)(x * x) * scale2x);
    sum += e[i];
  }
  sum *= 2.0;
  sum += 1.0;
  const double mul = 1.0 / sum;
  for (int i = 0; i < c; ++i) t.k[i] = t.k[n - 1 - i] = (float)(e[i] * mul);
  t.k[c] = (float)mul;
  return t;
}

// compute_scharr_derivative_kernelsV2 (nldiffusion_functions.cpp): one axis' kernel of derivative order `order`
Taps deriv_taps(int order, int scale) {
  Taps t{};
  t.n = 3 + 2 * (scale - 1);
  const float w = 10.0f / 3.0f;
  const float norm = 1.0f / (2.0f * (w + 2.0f));
  if (scale == 1) {
    if (order == 0) t.k[0] = 3.0f / 32.0f, t.k[1] = 10.0f / 32.0f, t.k[2] = 3.0f / 32.0f;
    else t.k[0] = -1.0f, t.k[2] = 1.0f;
  } else if (order == 0) {
    t.k[0] = norm, t.k[t.n / 2] = w * norm, t.k[t.n - 1] = norm;
  } else {
    t.k[0] = -1.0f, t.k[t.n - 1] = 1.0f;
  }
  return t;
}

Taps scharr_taps(int order) {  // cv::Scharr's unnormalised kernels
  Taps t{};
  t.n = 3;
  if (order == 0) t.k[0] = 3.0f, t.k[1] = 10.0f, t.k[2] = 3.0f;
  else t.k[0] = -1.0f, t.k[2] = 1.0f;
  return t;
}

// ---- device ----------------------------------------------------------------------------------------------------------

struct Planes {  // one plane per image of the batch
  const float* src[kMaxBatch];
  float* dst[kMaxBatch];
  int w[kMaxBatch], h[kMaxBatch];
};

__device__ __forceinline__ int border_index(int p, int n, int replicate) {
  if (replicate) return p < 0 ? 0 : (p >= n ? n - 1 : p);
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

// separable filter, horizontal pass: dst = k[0] s[x - r] + k[1] s[x - r + 1] + ... in tap order
__global__ void k_row(Planes P, Taps t) {
  const int b = blockIdx.z, w = P.w[b], h = P.h[b];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const float* row = P.src[b] + (size_t)y * w;
  const int r = t.n / 2;
  float s = t.k[0] * row[border_index(x - r, w, t.replicate)];
  for (int i = 1; i < t.n; ++i) s = s + t.k[i] * row[border_index(x - r + i, w, t.replicate)];
  P.dst[b][(size_t)y * w + x] = s;
}

// separable filter, vertical pass
__global__ void k_col(Planes P, Taps t) {
  const int b = blockIdx.z, w = P.w[b], h = P.h[b];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const float* src = P.src[b];
  const int r = t.n / 2;
  float s = t.k[0] * src[(size_t)border_index(y - r, h, t.replicate) * w + x];
  for (int i = 1; i < t.n; ++i) s = s + t.k[i] * src[(size_t)border_index(y - r + i, h, t.replicate) * w + x];
  P.dst[b][(size_t)y * w + x] = s;
}

struct Det {
  const float *lxx[kMaxBatch], *lxy[kMaxBatch], *lyy[kMaxBatch];
  float* det[kMaxBatch];
  int n[kMaxBatch];
};
__global__ void k_det(Det D) {
  const int b = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D.n[b]; i += gridDim.x * blockDim.x)
    D.det[b][i] = D.lxx[b][i] * D.lyy[b][i] - D.lxy[b][i] * D.lxy[b][i];
}

// resize INTER_AREA to (w / 2, h / 2): the exact 2x2 mean, or OpenCV's fractional-area tables
struct Half {
  const float* src[kMaxBatch];
  float* dst[kMaxBatch];
  int w[kMaxBatch], h[kMaxBatch];
  const int* itab[kMaxBatch];    // xofs[dw + 1], xsi[nx], yofs[dh + 1], ysi[ny]; null: exact factor 2
  const float* ftab[kMaxBatch];  // xal[nx], yal[ny]
  int nx[kMaxBatch];
};
__global__ void k_half(Half H) {
  const int b = blockIdx.z, w = H.w[b], dw = w / 2, dh = H.h[b] / 2;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dw || y >= dh) return;
  const float* src = H.src[b];
  if (!H.itab[b]) {
    const float* s0 = src + (size_t)(2 * y) * w + 2 * x;
    const float* s1 = s0 + w;
    H.dst[b][(size_t)y * dw + x] = ((s0[0] + s0[1]) + (s1[0] + s1[1])) * 0.25f;
    return;
  }
  const int nx = H.nx[b];
  const int *xofs = H.itab[b], *xsi = xofs + dw + 1, *yofs = xsi + nx, *ysi = yofs + dh + 1;
  const float *xal = H.ftab[b], *yal = xal + nx;
  float v = 0.0f;
  for (int ty = yofs[y]; ty < yofs[y + 1]; ++ty) {
    const float* s = src + (size_t)ysi[ty] * w;
    float hsum = 0.0f;
    for (int tx = xofs[x]; tx < xofs[x + 1]; ++tx) hsum = hsum + s[xsi[tx]] * xal[tx];
    v = ty == yofs[y] ? yal[ty] * hsum : v + yal[ty] * hsum;
  }
  H.dst[b][(size_t)y * dw + x] = v;
}

// compute_k_percentileV2: exact maximum of the interior gradient norms, integer histogram, one-thread scan
struct KP {
  const float *lx[kMaxBatch], *ly[kMaxBatch];
  int w[kMaxBatch], h[kMaxBatch], id[kMaxBatch];  // id: the image's index in the batch (its kcontrast slot)
};
__device__ __forceinline__ float grad_norm(const KP& K, int b, int i) {
  const float a = K.lx[b][i], c = K.ly[b][i];
  return sqrtf(a * a + c * c);
}
__global__ void k_kmax(KP K, unsigned* hmax_bits) {
  const int b = blockIdx.y, w = K.w[b], n = (w - 2) * (K.h[b] - 2);
  unsigned m = 0;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
    m = max(m, __float_as_uint(grad_norm(K, b, (j / (w - 2) + 1) * w + j % (w - 2) + 1)));  // norms are >= 0
  for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&hmax_bits[b], m);
}
__global__ void k_khist(KP K, const unsigned* hmax_bits, int* hist) {
  const int b = blockIdx.y, w = K.w[b], n = (w - 2) * (K.h[b] - 2);
  const float hmax = __uint_as_float(hmax_bits[b]);
  if (hmax == 0.0f) return;
  const float mul = (kNbins - 1) / hmax;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
    atomicAdd(&hist[b * kNbins + (int)(grad_norm(K, b, (j / (w - 2) + 1) * w + j % (w - 2) + 1) * mul)], 1);
}
__global__ void k_kscan(KP K, const unsigned* hmax_bits, const int* hist, float* kc) {
  const int b = blockIdx.x;
  if (threadIdx.x) return;
  const float hmax = __uint_as_float(hmax_bits[b]);
  float k = 0.03f;
  if (hmax != 0.0f) {
    const int* hb = hist + b * kNbins;
    const int total = (K.w[b] - 2) * (K.h[b] - 2);
    const int nthreshold = (int)((total - hb[0]) * kPercentile);
    int nelements = 0;
    for (int i = 1; i < kNbins; ++i) {
      if (nelements >= nthreshold) {
        k = (float)hmax * i / kNbins;
        break;
      }
      nelements = nelements + hb[i];
    }
  }
  kc[K.id[b]] = k;
}
// kcontrast of level `l` of every image of the batch: the previous level's, times 0.75 on a new octave
__global__ void k_kstep(float* kc, int l, int scale) {
  const int b = threadIdx.x;
  if (b < kMaxBatch) kc[l * kMaxBatch + b] = scale ? kc[(l - 1) * kMaxBatch + b] * 0.75f : kc[(l - 1) * kMaxBatch + b];
}

// pm_g2V2
struct Flow {
  const float *lx[kMaxBatch], *ly[kMaxBatch];
  float* flow[kMaxBatch];
  int n[kMaxBatch], id[kMaxBatch];
};
__global__ void k_pmg2(Flow F, const float* kc) {
  const int b = blockIdx.y;
  const float k = kc[F.id[b]];
  const float inv_k2 = 1.0f / (k * k);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < F.n[b]; i += gridDim.x * blockDim.x) {
    const float a = F.lx[b][i], c = F.ly[b][i];
    F.flow[b][i] = 1.0f / (1.0f + ((a * a + c * c) * inv_k2));
  }
}

// nld_step_scalarV2 into the flat workspace; the corners of the first and the last row are not written
struct Fed {
  float* lt[kMaxBatch];
  const float* lf[kMaxBatch];
  float* lstep[kMaxBatch];
  int w[kMaxBatch], h[kMaxBatch];
};
__global__ void k_fed_step(Fed F) {
  const int b = blockIdx.z, w = F.w[b], h = F.h[b];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const bool top = y == 0, bottom = y == h - 1, left = x == 0, right = x == w - 1;
  if ((top || bottom) && (left || right)) return;
  const float* lt = F.lt[b];
  const float* lf = F.lf[b];
  auto at = [&](const float* a, int yy, int xx) { return a[(size_t)yy * w + xx]; };
  const float c = at(lt, y, x), fc = at(lf, y, x);
  float v;
  if (top || bottom) {
    const int yn = top ? 1 : h - 2;
    v = (fc + at(lf, y, x + 1)) * (at(lt, y, x + 1) - c) + (fc + at(lf, y, x - 1)) * (at(lt, y, x - 1) - c) +
        (fc + at(lf, yn, x)) * (at(lt, yn, x) - c);
  } else if (left) {
    v = (fc + at(lf, y, 1)) * (at(lt, y, 1) - c) + (fc + at(lf, y + 1, 0)) * (at(lt, y + 1, 0) - c) +
        (fc + at(lf, y - 1, 0)) * (at(lt, y - 1, 0) - c);
  } else if (right) {
    v = (fc + at(lf, y, x - 1)) * (at(lt, y, x - 1) - c) + (fc + at(lf, y + 1, x)) * (at(lt, y + 1, x) - c) +
        (fc + at(lf, y - 1, x)) * (at(lt, y - 1, x) - c);
  } else {
    v = (fc + at(lf, y, x + 1)) * (at(lt, y, x + 1) - c) + (fc + at(lf, y, x - 1)) * (at(lt, y, x - 1) - c) +
        (fc + at(lf, y + 1, x)) * (at(lt, y + 1, x) - c) + (fc + at(lf, y - 1, x)) * (at(lt, y - 1, x) - c);
  }
  F.lstep[b][(size_t)y * w + x] = v;
}
__global__ void k_fed_update(Fed F, float tau) {
  const int b = blockIdx.y, n = F.w[b] * F.h[b];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    F.lt[b][i] += F.lstep[b][i] * 0.5f * tau;
}

// ---- extrema ---------------------------------------------------------------------------------------------------------

struct Ext {  // one level of every image
  const float* det[kMaxBatch];
  int w[kMaxBatch], h[kMaxBatch];
  int* rows[kMaxBatch];        // per interior row: count, then (exclusive) output offset
  int2* out[kMaxBatch];        // (x, y) of the candidates, raster order
  int border;
};
__device__ __forceinline__ bool is_candidate(const float* L, int w, int x, int y, float thr) {
  const float* c = L + (size_t)y * w + x;
  const float v = *c;
  if (v <= thr) return false;
  if (v <= c[-1] || v <= c[1]) return false;
  if (v <= c[-w - 1] || v <= c[-w] || v <= c[-w + 1]) return false;
  if (v <= c[w - 1] || v <= c[w] || v <= c[w + 1]) return false;
  return true;
}
// one warp per interior row: count (write = 0) or write the row's candidates in raster order (write = 1)
__global__ void k_cand_rows(Ext E, float thr, int write) {
  const int b = blockIdx.z, w = E.w[b], h = E.h[b], bd = E.border;
  const int row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (row >= h - 2 * bd) return;
  const int y = row + bd;
  int base = write ? E.rows[b][row] : 0;
  for (int x0 = bd; x0 < w - bd; x0 += 32) {
    const int x = x0 + lane;
    const bool c = x < w - bd && is_candidate(E.det[b], w, x, y, thr);
    const unsigned m = __ballot_sync(0xffffffffu, c);
    if (write && c) E.out[b][base + __popc(m & ((1u << lane) - 1))] = make_int2(x, y);
    base += __popc(m);
  }
  if (!write && lane == 0) E.rows[b][row] = base;
}

struct KpDev {
  float x, y, size, angle, response;
  int octave, class_id;
};
static_assert(sizeof(KpDev) == sizeof(r3d_akaze_keypoint), "keypoint layout");

struct LevelRef {  // one (image, level): its Ldet, Lx, Ly, candidates and kept points
  const float *det, *lx, *ly;
  int w, h;
  const int2* cand;
  int n_cand;
  KpDev* kp;          // the same-level pass' output (capacity n_cand)
  int* n_kp;          // its length
  uint8_t* flags;     // bit 0: deleted by the lower-level pass, bit 1: deleted after the upper-level pass
  float ratio, size;  // octave ratio, esigma * derivative_factor
  int octave, level;
  // the same-level pass' cell grid: gx x gy cells of side `cell`, list heads, next links and each kept point's cell
  float cell;
  int gx, gy;
  int *head, *next, *cell_of;
};

// the same-level pass: candidates in raster order; the first kept point in vector order within the candidate's size
// is replaced in place by a stronger candidate, a weaker candidate is dropped, otherwise the candidate is appended.
// The pass is sequential by nature (each decision depends on the previous ones), so it runs one warp per (image,
// level).  The kept points are binned into a grid of square cells of side cell = 1.0625 size, one singly linked list
// per cell (head per cell, next per point): every kept point that can pass upstream's float test
// dx^2 + dy^2 <= size^2 lies within size (1 + 2^-22) of the candidate, well inside the 3x3 cells around it even after
// the rounding of x / cell.  Lanes 0-8 walk those nine lists and the warp takes the minimum index among the hits:
// that is upstream's first match in vector order.  A replacement moves its point, so it changes cells.
__device__ __forceinline__ int grid_cell(const LevelRef& L, float x, float y) {
  const int cx = min((int)(x / L.cell), L.gx - 1), cy = min((int)(y / L.cell), L.gy - 1);
  return cy * L.gx + cx;
}
__global__ void k_same_level(const LevelRef* refs, int n_refs) {
  const int r = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (r >= n_refs) return;
  const LevelRef L = refs[r];
  int n = 0;
  for (int c = 0; c < L.n_cand; ++c) {
    const int2 q = L.cand[c];
    KpDev p;
    p.x = (float)(q.x * L.ratio);
    p.y = (float)(q.y * L.ratio);
    p.size = L.size;
    p.angle = -1.0f;
    p.response = L.det[(size_t)q.y * L.w + q.x];
    p.octave = L.octave;
    p.class_id = L.level;
    const float r2 = p.size * p.size;
    const int home = grid_cell(L, p.x, p.y);
    int best = INT_MAX;
    if (lane < 9) {
      const int cx = home % L.gx + lane % 3 - 1, cy = home / L.gx + lane / 3 - 1;
      if (cx >= 0 && cx < L.gx && cy >= 0 && cy < L.gy)
        for (int i = L.head[cy * L.gx + cx]; i >= 0; i = L.next[i]) {
          const float dx = p.x - L.kp[i].x, dy = p.y - L.kp[i].y;
          if (dx * dx + dy * dy <= r2) best = min(best, i);
        }
    }
    best = __reduce_min_sync(0xffffffffu, best);
    if (lane == 0) {
      if (best != INT_MAX) {
        if (p.response > L.kp[best].response) {
          const int old = L.cell_of[best];
          L.kp[best] = p;
          if (old != home) {  // unlink from the old cell, push onto the new one
            int* link = &L.head[old];
            while (*link != best) link = &L.next[*link];
            *link = L.next[best];
            L.next[best] = L.head[home];
            L.head[home] = best;
            L.cell_of[best] = home;
          }
        }
      } else {
        L.kp[n] = p;
        L.cell_of[n] = home;
        L.next[n] = L.head[home];
        L.head[home] = n;
      }
    }
    if (best == INT_MAX) ++n;
    __syncwarp();
  }
  if (lane == 0) *L.n_kp = n;
}

// the lower-level pass (i ascending): a point of level i - 1 is deleted when a stronger point of level i lies within
// that point's size.  Order independent: pass i only writes level i - 1, whose own flags no later pass reads first.
__global__ void k_lower(const LevelRef* refs, int nl, int n_img) {
  const int b = blockIdx.z, i = blockIdx.y + 1;  // level i's points against level i - 1
  if (b >= n_img) return;
  const LevelRef lo = refs[b * nl + i - 1], up = refs[b * nl + i];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *lo.n_kp) return;
  const KpDev q = lo.kp[j];
  const int nu = *up.n_kp;
  bool del = false;
  for (int k = 0; k < nu && !del; ++k) {
    const KpDev& p = up.kp[k];
    const float dx = p.x - q.x, dy = p.y - q.y;
    if (dx * dx + dy * dy <= p.size * p.size && p.response > q.response) del = true;
  }
  lo.flags[j] = del ? 1 : 0;
}
// the upper-level pass (i descending): a point of level i + 1 is deleted when a stronger point of level i that the
// lower-level pass kept lies within the upper point's size
__global__ void k_upper(const LevelRef* refs, int nl, int n_img) {
  const int b = blockIdx.z, i = blockIdx.y;  // level i's points against level i + 1; level 0 keeps its flags
  if (b >= n_img) return;
  const LevelRef up = refs[b * nl + i];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *up.n_kp) return;
  uint8_t f = up.flags[j] & 1;
  bool del = f != 0;
  if (i > 0) {
    const LevelRef lo = refs[b * nl + i - 1];
    const KpDev q = up.kp[j];
    const int nlo = *lo.n_kp;
    for (int k = 0; k < nlo && !del; ++k) {
      if (lo.flags[k] & 1) continue;
      const KpDev& p = lo.kp[k];
      const float dx = p.x - q.x, dy = p.y - q.y;
      if (dx * dx + dy * dy <= q.size * q.size && p.response > q.response) del = true;
    }
  }
  up.flags[j] = f | (del ? 2 : 0);
}

// Do_Subpixel_Refinement: 3x3 differences, the 2x2 Cramer solve of cv::solve(Matx22f, Vec2f, DECOMP_LU) in double
// (0 when singular); out.class_id = -1 marks a point that is deleted or rejected (|d| > 1)
__global__ void k_refine(const LevelRef* refs, int nl, int n_img, KpDev* out, const int* out_ofs) {
  const int b = blockIdx.z, i = blockIdx.y;
  if (b >= n_img) return;
  const LevelRef L = refs[b * nl + i];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *L.n_kp) return;
  KpDev kp = L.kp[j];
  KpDev* o = out + out_ofs[b * nl + i] + j;
  if (L.flags[j] & 2) {
    o->class_id = -1;
    return;
  }
  const float* l = L.det;
  const int cols = L.w;
  const int x = (int)(kp.x / L.ratio), y = (int)(kp.y / L.ratio);
  const float Dx = 0.5f * (l[y * cols + x + 1] - l[y * cols + x - 1]);
  const float Dy = 0.5f * (l[(y + 1) * cols + x] - l[(y - 1) * cols + x]);
  const float Dxx = l[y * cols + x + 1] + l[y * cols + x - 1] - 2.0f * l[y * cols + x];
  const float Dyy = l[(y + 1) * cols + x] + l[(y - 1) * cols + x] - 2.0f * l[y * cols + x];
  const float Dxy = 0.25f * (l[(y + 1) * cols + x + 1] + l[(y - 1) * cols + x - 1] - l[(y - 1) * cols + x + 1] -
                             l[(y + 1) * cols + x - 1]);
  const float b0 = -Dx, b1 = -Dy;
  float dx = 0.0f, dy = 0.0f;
  double d = (double)Dxx * Dyy - (double)Dxy * Dxy;
  if (d != 0.0) {
    d = 1.0 / d;
    dx = (float)(((double)b0 * Dyy - (double)b1 * Dxy) * d);
    dy = (float)(((double)b1 * Dxx - (double)b0 * Dxy) * d);
  }
  if (fabsf(dx) > 1.0f || fabsf(dy) > 1.0f) {
    o->class_id = -1;
    return;
  }
  kp.x += dx * L.ratio;
  kp.y += dy * L.ratio;
  kp.angle = 0.0f;
  kp.size *= 2.0f;
  *o = kp;
}

// ---- AKAZE (cv::AKAZE of OpenCV 4): the same candidates, kept points as per-level masks --------------------------
// Each (image, level) has three uint8 masks of its pixels: m[0] after the same-level pass, m[1] after the lower-level
// passes, m[2] after the upper-level passes.  Pass i of either cross-level sweep reads its source level as the
// previous sweep left it (the next pass that changes that level runs later) and is the only pass that changes its
// target level, so every pass of a sweep runs at once, one warp per (image, level).
struct CvRef {
  const float* det;
  const int2* cand;  // raster order (k_cand_rows)
  int n_cand, w, h, r;  // r: sigma_size
  float ratio, size;
  int octave, level;
  uint8_t* m[3];
};

// find_neighbor_point: the first set pixel in row-major order of the window [y - R, y + R) x [x - R, x + R) with
// dx^2 + dy^2 <= R^2; lanes test 32 window cells at a time, the lowest set ballot bit is the first hit.  -1: none.
__device__ __forceinline__ int cv_find(const uint8_t* m, int w, int x, int y, int R, int lane) {
  const int side = 2 * R, n = side * side;
  for (int base = 0; base < n; base += 32) {
    const int k = base + lane, dy = k / side - R, dx = k % side - R;
    const bool hit = k < n && dx * dx + dy * dy <= R * R && m[(size_t)(y + dy) * w + x + dx] != 0;
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if (b) {
      const int f = base + __ffs(b) - 1;
      return (y + f / side - R) * w + x + f % side - R;
    }
  }
  return -1;
}

// the same-level pass: candidates in raster order; a candidate with a kept point in its window replaces that point
// when stronger and is dropped otherwise; without one it is kept
__global__ void k_cv_same(const CvRef* refs, int n_refs) {
  const int r = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (r >= n_refs) return;
  const CvRef L = refs[r];
  for (int c = 0; c < L.n_cand; ++c) {
    const int2 q = L.cand[c];
    const int p = q.y * L.w + q.x;
    const int hit = cv_find(L.m[0], L.w, q.x, q.y, L.r, lane);
    if (lane == 0) {
      if (hit < 0) {
        L.m[0][p] = 1;
      } else if (L.det[p] > L.det[hit]) {
        L.m[0][hit] = 0;
        L.m[0][p] = 1;
      }
    }
    __syncwarp();
  }
}

// the lower-level pass i (i >= 1): each point of level i, in raster order, looks at (x, y) * diff_ratio in level
// i - 1 within sigma_size_i * diff_ratio and clears the point found there when that one is weaker
__global__ void k_cv_lower(const CvRef* refs, int nl, int n_img, const int* n_levels) {
  const int t = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  const int b = t / nl, i = t % nl;
  if (b >= n_img || i < 1 || i >= n_levels[b]) return;
  const CvRef S = refs[b * nl + i], T = refs[b * nl + i - 1];
  const int dr = (int)(S.ratio / T.ratio), R = S.r * dr;
  for (int c = 0; c < S.n_cand; ++c) {
    const int2 q = S.cand[c];
    const int p = q.y * S.w + q.x;
    if (!S.m[0][p]) continue;
    const int hit = cv_find(T.m[1], T.w, q.x * dr, q.y * dr, R, lane);
    if (lane == 0 && hit >= 0 && S.det[p] > T.det[hit]) T.m[1][hit] = 0;
    __syncwarp();
  }
}

// the upper-level pass i (i <= levels - 2): each point of level i looks at (x, y) / diff_ratio in level i + 1 within
// sigma_size_(i+1) and clears the point found there when that one is weaker
__global__ void k_cv_upper(const CvRef* refs, int nl, int n_img, const int* n_levels) {
  const int t = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  const int b = t / nl, i = t % nl;
  if (b >= n_img || i + 1 >= n_levels[b]) return;
  const CvRef S = refs[b * nl + i], T = refs[b * nl + i + 1];
  const int dr = (int)(T.ratio / S.ratio);
  for (int c = 0; c < S.n_cand; ++c) {
    const int2 q = S.cand[c];
    const int p = q.y * S.w + q.x;
    if (!S.m[1][p]) continue;
    const int hit = cv_find(T.m[2], T.w, q.x / dr, q.y / dr, T.r, lane);
    if (lane == 0 && hit >= 0 && S.det[p] > T.det[hit]) T.m[2][hit] = 0;
    __syncwarp();
  }
}

// Do_Subpixel_Refinement of cv::AKAZE on every candidate still set in m[2]: the 2x2 solve of k_refine, then
// x = (x + dx) ratio + 0.5 (ratio - 1); out.class_id = -1 marks a cleared or rejected candidate
__global__ void k_cv_refine(const CvRef* refs, int nl, int n_img, KpDev* out, const int* out_ofs) {
  const int b = blockIdx.z, i = blockIdx.y;
  if (b >= n_img) return;
  const CvRef L = refs[b * nl + i];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= L.n_cand) return;
  KpDev* o = out + out_ofs[b * nl + i] + j;
  const int x = L.cand[j].x, y = L.cand[j].y, cols = L.w;
  const float* l = L.det;
  if (!L.m[2][y * cols + x]) {
    o->class_id = -1;
    return;
  }
  const float Dx = 0.5f * (l[y * cols + x + 1] - l[y * cols + x - 1]);
  const float Dy = 0.5f * (l[(y + 1) * cols + x] - l[(y - 1) * cols + x]);
  const float Dxx = l[y * cols + x + 1] + l[y * cols + x - 1] - 2.0f * l[y * cols + x];
  const float Dyy = l[(y + 1) * cols + x] + l[(y - 1) * cols + x] - 2.0f * l[y * cols + x];
  const float Dxy = 0.25f * (l[(y + 1) * cols + x + 1] + l[(y - 1) * cols + x - 1] - l[(y - 1) * cols + x + 1] -
                             l[(y + 1) * cols + x - 1]);
  const float b0 = -Dx, b1 = -Dy;
  float dx = 0.0f, dy = 0.0f;
  double d = (double)Dxx * Dyy - (double)Dxy * Dxy;
  if (d != 0.0) {
    d = 1.0 / d;
    dx = (float)(((double)b0 * Dyy - (double)b1 * Dxy) * d);
    dy = (float)(((double)b1 * Dxx - (double)b0 * Dxy) * d);
  }
  if (fabsf(dx) > 1.0f || fabsf(dy) > 1.0f) {
    o->class_id = -1;
    return;
  }
  KpDev kp;
  kp.x = ((float)x + dx) * L.ratio + 0.5f * (L.ratio - 1.0f);
  kp.y = ((float)y + dy) * L.ratio + 0.5f * (L.ratio - 1.0f);
  kp.size = L.size * 2.0f;
  kp.angle = 0.0f;
  kp.response = l[y * cols + x];
  kp.octave = L.octave;
  kp.class_id = L.level;
  *o = kp;
}

__host__ __device__ __forceinline__ float fast_atan2_deg(float y, float x) {  // hal::fastAtan2 (fastAtan32f), degrees
  const float r2d = (float)(180 / kPi);
  const float p1 = 0.9997878412794807f * r2d, p3 = -0.3258083974640975f * r2d, p5 = 0.1555786518463281f * r2d,
              p7 = -0.04432655554792128f * r2d;
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = ay / (ax + (float)DBL_EPSILON);
    c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    c = ax / (ay + (float)DBL_EPSILON);
    c2 = c * c;
    a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}

__device__ __forceinline__ float fast_atan2(float y, float x) {  // hal::fastAtan2 (OpenCV 4.x fastAtan32f), radians
  const float r2d = (float)(180 / kPi);
  const float p1 = 0.9997878412794807f * r2d, p3 = -0.3258083974640975f * r2d, p5 = 0.1555786518463281f * r2d,
              p7 = -0.04432655554792128f * r2d;
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = ay / (ax + (float)DBL_EPSILON);
    c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    c = ax / (ay + (float)DBL_EPSILON);
    c2 = c * c;
    a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a * (float)(kPi / 180);
}

struct Gauss25 {
  float g[49];
};

// Compute_Main_Orientation up to getAngleV2: 109 weighted derivative samples on radius 6 scale, their fastAtan2
// angles bucketed by the unstable counting sort into 42 slices, sliding 7-slice windows; (maxX, maxY) out
__global__ void k_orient(const KpDev* kps, int n, const LevelRef* refs, const int* ref_of, Gauss25 G, float2* out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const KpDev kp = kps[k];
  const LevelRef L = refs[ref_of[k]];
  const int scale = (int)(0.5f * kp.size / L.ratio + 0.5f);
  const int x0 = (int)(kp.x / L.ratio + 0.5f), y0 = (int)(kp.y / L.ratio + 0.5f);
  float resX[109], resY[109];
  uint8_t key[109];
  const int slices = 42, win = 7;
  const float quantum = (float)(2.0 * kPi / slices), amax = (float)(2.0 * kPi);
  const int nkeys = (int)(amax / quantum);
  uint8_t cum[64], idx[109];
  for (int i = 0; i <= nkeys; ++i) cum[i] = 0;
  int m = 0;
  for (int i = -6; i <= 6; ++i)
    for (int j = -6; j <= 6; ++j) {
      if (i * i + j * j >= 36) continue;
      const float wgt = G.g[abs(i) * 7 + abs(j)];
      const size_t p = (size_t)(y0 + i * scale) * L.w + (x0 + j * scale);
      resX[m] = wgt * L.lx[p];
      resY[m] = wgt * L.ly[p];
      key[m] = (uint8_t)(int)(fast_atan2(resY[m], resX[m]) / quantum);
      cum[key[m]]++;
      ++m;
    }
  for (int i = 1; i <= nkeys; ++i) cum[i] += cum[i - 1];
  for (int i = 0; i < 109; ++i) idx[--cum[key[i]]] = (uint8_t)i;
  float maxX = 0.0f, maxY = 0.0f;
  for (int i = cum[0]; i < cum[win]; ++i) maxX += resX[idx[i]], maxY += resY[idx[i]];
  float maxNorm = maxX * maxX + maxY * maxY;
  for (int sn = 1; sn <= slices - win; ++sn) {
    if (cum[sn] == cum[sn - 1] && cum[sn + win] == cum[sn + win - 1]) continue;
    float sx = 0.0f, sy = 0.0f;
    for (int i = cum[sn]; i < cum[sn + win]; ++i) sx += resX[idx[i]], sy += resY[idx[i]];
    const float nrm = sx * sx + sy * sy;
    if (nrm > maxNorm) maxNorm = nrm, maxX = sx, maxY = sy;
  }
  for (int sn = slices - win + 1; sn < slices; ++sn) {
    const int remain = sn + win - slices;
    if (cum[sn] == cum[sn - 1] && cum[remain] == cum[remain - 1]) continue;
    float sx = 0.0f, sy = 0.0f;
    for (int i = cum[sn]; i < cum[slices]; ++i) sx += resX[idx[i]], sy += resY[idx[i]];
    for (int i = cum[0]; i < cum[remain]; ++i) sx += resX[idx[i]], sy += resY[idx[i]];
    const float nrm = sx * sx + sy * sy;
    if (nrm > maxNorm) maxNorm = nrm, maxX = sx, maxY = sy;
  }
  out[k] = make_float2(maxX, maxY);
}

// ---- host driver -----------------------------------------------------------------------------------------------------

Gauss25 gauss25() {  // exp(-r^2 / 2 sigma^2) / (2 pi sigma^2), sigma 2.5, 8 decimals, pi = 3.14159 (as upstream's table)
  Gauss25 G;
  for (int i = 0; i < 7; ++i)
    for (int j = 0; j < 7; ++j)
      G.g[i * 7 + j] = (float)(std::round(std::exp(-(i * i + j * j) / 12.5) / (2.0 * 3.14159 * 6.25) * 1e8) / 1e8);
  return G;
}

// getAngleV2 (libm atan2f into [0, 2 pi)), then Regard3DFeatures::detectKeypoints' conversion to degrees
float regard3d_angle(float maxX, float maxY) {
  const float theta = atan2f(maxY, maxX);
  float a = theta >= 0 ? theta : theta + static_cast<float>(2.0f * kPi);
  a *= 180.0 / kPi;
  a += 90.0f;
  while (a < 0) a += 360.0f;
  while (a > 360.0f) a -= 360.0f;
  return a;
}

struct AreaTab {
  std::vector<int> si, ofs;
  std::vector<float> al;
};
AreaTab area_tab(int ssize, int dsize) {  // OpenCV's computeResizeAreaTab, grouped by destination index
  AreaTab t;
  const double scale = (double)ssize / dsize;
  for (int dx = 0; dx < dsize; ++dx) {
    t.ofs.push_back((int)t.si.size());
    const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    const double cell = std::min(scale, ssize - fsx1);
    int sx1 = (int)std::ceil(fsx1), sx2 = (int)std::floor(fsx2);
    sx2 = std::min(sx2, ssize - 1);
    sx1 = std::min(sx1, sx2);
    if (sx1 - fsx1 > 1e-3) t.si.push_back(sx1 - 1), t.al.push_back((float)((sx1 - fsx1) / cell));
    for (int sx = sx1; sx < sx2; ++sx) t.si.push_back(sx), t.al.push_back((float)(1.0 / cell));
    if (fsx2 - sx2 > 1e-3) t.si.push_back(sx2), t.al.push_back((float)(std::min(std::min(fsx2 - sx2, 1.0), cell) / cell));
  }
  t.ofs.push_back((int)t.si.size());
  return t;
}

struct Image {
  const float* host;
  int W, H;
  std::vector<r3d_akaze_level> lv;
};

// per image of a batch: everything in one pool block
struct ImgMem {
  std::vector<float*> Lt, Ls, Lx, Ly, Ldet;  // per level
  float *img, *ls, *sx, *sy, *flow, *lstep, *tmp, *lxx, *lxy, *lyy;
};

size_t image_bytes(const Image& im) {
  size_t px = 0;
  for (const r3d_akaze_level& l : im.lv) px += (size_t)l.width * l.height;
  return (5 * px + 10 * (size_t)im.W * im.H) * 4 + 4096;
}

struct Debug {  // r3d_debug_akaze_levels' / r3d_debug_akaze_masks' outputs (batch of one image)
  float *arrays, *kcontrast;
  r3d_akaze_keypoint* cands;  // Fast-AKAZE
  uint8_t* flags;
  uint32_t cap, *counts;
  uint8_t* masks;  // AKAZE: per level, the three masks
};

constexpr int kStages = 6;  // upload, scale space, candidates, same-level pass, cross-level passes, refine + orient
struct Timer {
  cudaEvent_t e[kStages + 1] = {};
  ~Timer() {
    for (cudaEvent_t x : e)
      if (x) cudaEventDestroy(x);
  }
};

dim3 grid2(int w, int h, int n) { return dim3((w + 31) / 32, (h + 7) / 8, n); }

// r3d_extract_features' state of one batch between its detection and its descriptors: run_batch leaves the original
// images resident (slot b = the batch's image b) and releases everything else; launch_describe runs k_liop on
// w.copy_stream, which the next batch's scale space overlaps; finish_describe downloads and releases.
struct Pending {
  uint32_t i0 = 0, i1 = 0;         // the batch's images, with or without levels
  std::vector<uint32_t> slot_img;  // image of each slot
  liop::Slots S{};
  std::vector<void*> held;         // image blocks, maps, descriptors
  float* d_desc = nullptr;
  uint32_t n = 0;                  // keypoints of the batch
};

// One batch of images on one device.  kps[b]: the image's keypoints on return.  keep: hand the original images to
// keep->held / keep->S instead of releasing them.
int run_batch(r3d_ctx* ctx, DeviceWorker& w, std::vector<Image*>& imgs, float threshold, int detector,
              std::vector<std::vector<r3d_akaze_keypoint>*>& kps_out, const Debug* dbg, double* stage_ms,
              uint32_t* launches, Pending* keep = nullptr) {
  const int B = (int)imgs.size();
  cudaStream_t st = w.stream;
  int nl = 0;
  for (Image* im : imgs) nl = std::max(nl, (int)im->lv.size());
  std::vector<void*> blocks;
  struct Guard {
    DeviceWorker* w;
    std::vector<void*>* p;
    ~Guard() {
      cudaStreamSynchronize(w->stream);
      for (void* q : *p) pool_release(*w, q);
    }
  } guard{&w, &blocks};
  auto alloc = [&](size_t bytes) -> void* {
    void* q = pool_alloc(w, std::max<size_t>(bytes, 4));
    if (q) blocks.push_back(q);
    return q;
  };
  Timer T;
  for (cudaEvent_t& e : T.e) R3D_CUDA_TRY(ctx, cudaEventCreate(&e));
  R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[0], st));
  uint32_t nlaunch = 0;

  std::vector<ImgMem> M(B);
  for (int b = 0; b < B; ++b) {
    Image& im = *imgs[b];
    const size_t P = (size_t)im.W * im.H;
    // the original image in a block of its own (no stage writes it): r3d_extract_features describes from it later
    float* base = (float*)alloc(image_bytes(im) - P * 4);
    float* img = (float*)pool_alloc(w, P * 4);
    if (img) (keep ? keep->held : blocks).push_back(img);
    if (!base || !img) return fail(ctx, R3D_ERR_NOMEM, "r3d_akaze_detect: device allocation failed");
    ImgMem& m = M[b];
    m.img = img;
    if (keep) keep->S.img[b] = img, keep->S.w[b] = im.W, keep->S.h[b] = im.H;
    float* p = base;
    for (float** q : {&m.ls, &m.sx, &m.sy, &m.flow, &m.lstep, &m.tmp, &m.lxx, &m.lxy, &m.lyy}) *q = p, p += P;
    for (const r3d_akaze_level& l : im.lv) {
      const size_t lp = (size_t)l.width * l.height;
      m.Lt.push_back(p), p += lp;
      m.Ls.push_back(p), p += lp;
      m.Lx.push_back(p), p += lp;
      m.Ly.push_back(p), p += lp;
      m.Ldet.push_back(p), p += lp;
    }
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(m.img, im.host, P * 4, cudaMemcpyHostToDevice, st));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(m.lstep, 0, P * 4, st));
  }
  R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[1], st));
  // the images that have level l
  auto members = [&](int l) {
    std::vector<int> v;
    for (int b = 0; b < B; ++b)
      if ((int)imgs[b]->lv.size() > l) v.push_back(b);
    return v;
  };
  // separable filter over one plane per listed image
  auto sep = [&](const std::vector<int>& who, const std::vector<const float*>& src, const std::vector<float*>& dst,
                 const std::vector<int>& ws, const std::vector<int>& hs, const Taps& tx, const Taps& ty) -> int {
    Planes a{}, c{};
    int mw = 0, mh = 0;
    for (size_t k = 0; k < who.size(); ++k) {
      const int b = who[k];
      a.src[k] = src[k], a.dst[k] = M[b].tmp, a.w[k] = ws[k], a.h[k] = hs[k];
      c.src[k] = M[b].tmp, c.dst[k] = dst[k], c.w[k] = ws[k], c.h[k] = hs[k];
      mw = std::max(mw, ws[k]), mh = std::max(mh, hs[k]);
    }
    k_row<<<grid2(mw, mh, (int)who.size()), dim3(32, 8), 0, st>>>(a, tx);
    k_col<<<grid2(mw, mh, (int)who.size()), dim3(32, 8), 0, st>>>(c, ty);
    nlaunch += 2;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return R3D_OK;
  };
  auto shape = [&](const std::vector<int>& who, int l, std::vector<int>& ws, std::vector<int>& hs) {
    ws.clear(), hs.clear();
    for (int b : who) {
      ws.push_back(l < 0 ? imgs[b]->W : imgs[b]->lv[l].width);
      hs.push_back(l < 0 ? imgs[b]->H : imgs[b]->lv[l].height);
    }
  };
  float* d_kc = (float*)alloc((size_t)kMaxBatch * std::max(nl, 1) * 4);
  unsigned* d_hmax = (unsigned*)alloc(kMaxBatch * 4);
  int* d_hist = (int*)alloc(kMaxBatch * kNbins * 4);
  if (!d_kc || !d_hmax || !d_hist) return fail(ctx, R3D_ERR_NOMEM, "r3d_akaze_detect: device allocation failed");
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_kc, 0, (size_t)kMaxBatch * std::max(nl, 1) * 4, st));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_hmax, 0, kMaxBatch * 4, st));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_hist, 0, kMaxBatch * kNbins * 4, st));
  const Taps g16 = gaussian_taps(kSoffset), g10 = gaussian_taps(1.0f), sd = scharr_taps(1), ss = scharr_taps(0);
  int rc;
  std::vector<int> ws, hs;

  // Compute_Determinant_Hessian_Response(l) for the listed images
  auto hessian = [&](const std::vector<int>& who, int l) -> int {
    const int sz = imgs[who[0]]->lv[l].sigma_size;
    const Taps d1 = deriv_taps(1, sz), d0 = deriv_taps(0, sz);
    std::vector<const float*> src;
    std::vector<float*> dst;
    shape(who, l, ws, hs);
    auto pass = [&](float* const ImgMem::*in_s, std::vector<float*> ImgMem::*in_v, float* ImgMem::*out_s,
                    std::vector<float*> ImgMem::*out_v, const Taps& tx, const Taps& ty) -> int {
      src.clear(), dst.clear();
      for (int b : who) {
        src.push_back(in_v ? (M[b].*in_v)[l] : M[b].*in_s);
        dst.push_back(out_v ? (M[b].*out_v)[l] : M[b].*out_s);
      }
      return sep(who, src, dst, ws, hs, tx, ty);
    };
    if ((rc = pass(nullptr, &ImgMem::Ls, nullptr, &ImgMem::Lx, d1, d0))) return rc;
    if ((rc = pass(nullptr, &ImgMem::Lx, &ImgMem::lxx, nullptr, d1, d0))) return rc;
    if ((rc = pass(nullptr, &ImgMem::Lx, &ImgMem::lxy, nullptr, d0, d1))) return rc;
    if ((rc = pass(nullptr, &ImgMem::Ls, nullptr, &ImgMem::Ly, d0, d1))) return rc;
    if ((rc = pass(nullptr, &ImgMem::Ly, &ImgMem::lyy, nullptr, d0, d1))) return rc;
    Det D{};
    int mx = 0;
    for (size_t k = 0; k < who.size(); ++k) {
      const int b = who[k];
      D.lxx[k] = M[b].lxx, D.lxy[k] = M[b].lxy, D.lyy[k] = M[b].lyy, D.det[k] = M[b].Ldet[l], D.n[k] = ws[k] * hs[k];
      mx = std::max(mx, D.n[k]);
    }
    k_det<<<dim3(std::min((mx + 255) / 256, 4096), (unsigned)who.size()), 256, 0, st>>>(D);
    ++nlaunch;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return R3D_OK;
  };

  // ---- base level ----
  std::vector<int> all = members(0);
  {
    std::vector<const float*> src;
    std::vector<float*> dst;
    shape(all, -1, ws, hs);
    for (int b : all) src.push_back(M[b].img), dst.push_back(M[b].Ls[0]);
    if ((rc = sep(all, src, dst, ws, hs, g16, g16))) return rc;
    if ((rc = hessian(all, 0))) return rc;
    shape(all, -1, ws, hs);
    for (int b : all)
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(M[b].Lt[0], M[b].Ls[0], (size_t)imgs[b]->W * imgs[b]->H * 4,
                                        cudaMemcpyDeviceToDevice, st));
    if (nl > 1) {
      std::vector<int> multi = members(1);
      shape(multi, -1, ws, hs);
      src.clear(), dst.clear();
      for (int b : multi) src.push_back(M[b].img), dst.push_back(M[b].ls);
      if ((rc = sep(multi, src, dst, ws, hs, g10, g10))) return rc;
      src.clear(), dst.clear();
      for (int b : multi) src.push_back(M[b].ls), dst.push_back(M[b].sx);
      if ((rc = sep(multi, src, dst, ws, hs, sd, ss))) return rc;
      dst.clear();
      for (int b : multi) dst.push_back(M[b].sy);
      if ((rc = sep(multi, src, dst, ws, hs, ss, sd))) return rc;
      KP K{};
      for (size_t k = 0; k < multi.size(); ++k) {
        const int b = multi[k];
        K.lx[k] = M[b].sx, K.ly[k] = M[b].sy, K.w[k] = ws[k], K.h[k] = hs[k], K.id[k] = b;
      }
      const dim3 g(512, (unsigned)multi.size());
      k_kmax<<<g, 256, 0, st>>>(K, d_hmax);
      k_khist<<<g, 256, 0, st>>>(K, d_hmax, d_hist);
      k_kscan<<<(unsigned)multi.size(), 32, 0, st>>>(K, d_hmax, d_hist, d_kc);
      nlaunch += 3;
      R3D_CUDA_TRY(ctx, cudaGetLastError());
    }
  }
  // ---- levels 1.. ----
  std::vector<std::vector<int>> half_i(B);
  std::vector<std::vector<float>> half_f(B);
  for (int l = 1; l < nl; ++l) {
    std::vector<int> who = members(l);
    const r3d_akaze_level& L0 = imgs[who[0]]->lv[l];
    const bool new_oct = L0.octave > imgs[who[0]]->lv[l - 1].octave;
    k_kstep<<<1, kMaxBatch, 0, st>>>(d_kc, l, new_oct ? 1 : 0);
    ++nlaunch;
    shape(who, l, ws, hs);
    if (new_oct) {
      Half Hh{};
      int mw = 0, mh = 0;
      for (size_t k = 0; k < who.size(); ++k) {
        const int b = who[k];
        const r3d_akaze_level& p = imgs[b]->lv[l - 1];
        Hh.src[k] = M[b].Lt[l - 1], Hh.dst[k] = M[b].Lt[l], Hh.w[k] = p.width, Hh.h[k] = p.height;
        mw = std::max(mw, ws[k]), mh = std::max(mh, hs[k]);
        if (p.width % 2 == 0 && p.height % 2 == 0) continue;
        const AreaTab tx = area_tab(p.width, p.width / 2), ty = area_tab(p.height, p.height / 2);
        std::vector<int>& I = half_i[b];
        std::vector<float>& F = half_f[b];
        I.clear(), F.clear();
        I.insert(I.end(), tx.ofs.begin(), tx.ofs.end());
        I.insert(I.end(), tx.si.begin(), tx.si.end());
        I.insert(I.end(), ty.ofs.begin(), ty.ofs.end());
        I.insert(I.end(), ty.si.begin(), ty.si.end());
        F.insert(F.end(), tx.al.begin(), tx.al.end());
        F.insert(F.end(), ty.al.begin(), ty.al.end());
        int* di = (int*)alloc(I.size() * 4);
        float* df = (float*)alloc(F.size() * 4);
        if (!di || !df) return fail(ctx, R3D_ERR_NOMEM, "r3d_akaze_detect: device allocation failed");
        R3D_CUDA_TRY(ctx, cudaMemcpyAsync(di, I.data(), I.size() * 4, cudaMemcpyHostToDevice, st));
        R3D_CUDA_TRY(ctx, cudaMemcpyAsync(df, F.data(), F.size() * 4, cudaMemcpyHostToDevice, st));
        Hh.itab[k] = di, Hh.ftab[k] = df, Hh.nx[k] = (int)tx.si.size();
      }
      k_half<<<grid2(mw, mh, (int)who.size()), dim3(32, 8), 0, st>>>(Hh);
      ++nlaunch;
      R3D_CUDA_TRY(ctx, cudaGetLastError());
    } else {
      for (size_t k = 0; k < who.size(); ++k)
        R3D_CUDA_TRY(ctx, cudaMemcpyAsync(M[who[k]].Lt[l], M[who[k]].Lt[l - 1], (size_t)ws[k] * hs[k] * 4,
                                          cudaMemcpyDeviceToDevice, st));
    }
    std::vector<const float*> src;
    std::vector<float*> dst;
    for (int b : who) src.push_back(M[b].Lt[l]), dst.push_back(M[b].Ls[l]);
    if ((rc = sep(who, src, dst, ws, hs, g10, g10))) return rc;
    src.clear(), dst.clear();
    for (int b : who) src.push_back(M[b].Ls[l]), dst.push_back(M[b].sx);
    if ((rc = sep(who, src, dst, ws, hs, sd, ss))) return rc;
    dst.clear();
    for (int b : who) dst.push_back(M[b].sy);
    if ((rc = sep(who, src, dst, ws, hs, ss, sd))) return rc;
    if ((rc = hessian(who, l))) return rc;
    shape(who, l, ws, hs);
    Flow F{};
    Fed E{};
    int mx = 0, mw = 0, mh = 0;
    for (size_t k = 0; k < who.size(); ++k) {
      const int b = who[k];
      F.lx[k] = M[b].sx, F.ly[k] = M[b].sy, F.flow[k] = M[b].flow, F.n[k] = ws[k] * hs[k], F.id[k] = b;
      E.lt[k] = M[b].Lt[l], E.lf[k] = M[b].flow, E.lstep[k] = M[b].lstep, E.w[k] = ws[k], E.h[k] = hs[k];
      mx = std::max(mx, F.n[k]), mw = std::max(mw, ws[k]), mh = std::max(mh, hs[k]);
    }
    const dim3 g1(std::min((mx + 255) / 256, 4096), (unsigned)who.size());
    k_pmg2<<<g1, 256, 0, st>>>(F, d_kc + l * kMaxBatch);
    ++nlaunch;
    for (float tau : fed_tau(L0.etime - imgs[who[0]]->lv[l - 1].etime, 0.25f)) {
      k_fed_step<<<grid2(mw, mh, (int)who.size()), dim3(32, 8), 0, st>>>(E);
      k_fed_update<<<g1, 256, 0, st>>>(E, tau);
      nlaunch += 2;
    }
    R3D_CUDA_TRY(ctx, cudaGetLastError());
  }
  R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[2], st));

  // ---- candidates: 3x3 maxima above the threshold inside the border, compacted in raster order ----
  std::vector<int> row_ofs(B * nl + 1, 0);  // offsets of each (image, level)'s interior rows
  for (int b = 0; b < B; ++b)
    for (int l = 0; l < nl; ++l) {
      int rows = 0;
      if (l < (int)imgs[b]->lv.size()) rows = std::max(0, imgs[b]->lv[l].height - 2 * imgs[b]->lv[l].border);
      row_ofs[b * nl + l + 1] = row_ofs[b * nl + l] + rows;
    }
  int* d_rows = (int*)alloc((size_t)row_ofs.back() * 4);
  if (!d_rows) return fail(ctx, R3D_ERR_NOMEM, "r3d_akaze_detect: device allocation failed");
  auto ext_of = [&](int l, const std::vector<int>& who, int2* const* outs) {
    Ext X{};
    X.border = imgs[who[0]]->lv[l].border;
    int mh = 0;
    for (size_t k = 0; k < who.size(); ++k) {
      const int b = who[k];
      X.det[k] = M[b].Ldet[l], X.w[k] = imgs[b]->lv[l].width, X.h[k] = imgs[b]->lv[l].height;
      X.rows[k] = d_rows + row_ofs[b * nl + l];
      X.out[k] = outs ? outs[k] : nullptr;
      mh = std::max(mh, X.h[k] - 2 * X.border);
    }
    return std::make_pair(X, mh);
  };
  for (int l = 0; l < nl; ++l) {
    std::vector<int> who = members(l);
    auto xm = ext_of(l, who, nullptr);
    if (xm.second <= 0) continue;
    k_cand_rows<<<dim3((xm.second + 7) / 8, 1, (unsigned)who.size()), 256, 0, st>>>(xm.first, threshold, 0);
    ++nlaunch;
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  std::vector<int> rows_h(row_ofs.back());
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(rows_h.data(), d_rows, rows_h.size() * 4, cudaMemcpyDeviceToHost, st));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  std::vector<int> cand_ofs(B * nl + 1, 0);
  for (int r = 0; r < B * nl; ++r) {
    int acc = 0;
    for (int k = row_ofs[r]; k < row_ofs[r + 1]; ++k) {
      const int c = rows_h[k];
      rows_h[k] = acc;
      acc += c;
    }
    cand_ofs[r + 1] = cand_ofs[r] + acc;
  }
  const int n_cand = cand_ofs.back();
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_rows, rows_h.data(), rows_h.size() * 4, cudaMemcpyHostToDevice, st));
  int2* d_cand = (int2*)alloc((size_t)n_cand * 8);
  KpDev* d_kp = (KpDev*)alloc((size_t)n_cand * sizeof(KpDev));
  KpDev* d_ref = (KpDev*)alloc((size_t)n_cand * sizeof(KpDev));
  uint8_t* d_flags = (uint8_t*)alloc((size_t)n_cand);
  int* d_nkp = (int*)alloc((size_t)B * nl * 4);
  int* d_cofs = (int*)alloc((size_t)(B * nl + 1) * 4);
  LevelRef* d_refs = (LevelRef*)alloc((size_t)B * nl * sizeof(LevelRef));
  int* d_link = (int*)alloc((size_t)n_cand * 2 * 4);  // next, cell_of
  // the cell grids: side 1.0625 size over the level's extent in image coordinates
  std::vector<size_t> grid_ofs(B * nl + 1, 0);
  std::vector<int2> grid_dim(B * nl, make_int2(1, 1));
  for (int b = 0; b < B; ++b)
    for (int l = 0; l < nl; ++l) {
      const int r = b * nl + l;
      if (l < (int)imgs[b]->lv.size()) {
        const r3d_akaze_level& L = imgs[b]->lv[l];
        const float cell = L.esigma * kDerivFactor * 1.0625f;
        grid_dim[r] = make_int2((int)((float)(L.width - 1) * L.ratio / cell) + 1,
                                (int)((float)(L.height - 1) * L.ratio / cell) + 1);
      }
      grid_ofs[r + 1] = grid_ofs[r] + (size_t)grid_dim[r].x * grid_dim[r].y;
    }
  int* d_heads = (int*)alloc(grid_ofs.back() * 4);
  if (!d_cand || !d_kp || !d_ref || !d_flags || !d_nkp || !d_cofs || !d_refs || !d_link || !d_heads)
    return fail(ctx, R3D_ERR_NOMEM, "r3d_akaze_detect: device allocation failed");
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_nkp, 0, (size_t)B * nl * 4, st));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_heads, 0xff, grid_ofs.back() * 4, st));  // empty lists (-1)
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_cofs, cand_ofs.data(), cand_ofs.size() * 4, cudaMemcpyHostToDevice, st));
  for (int l = 0; l < nl; ++l) {
    std::vector<int> who = members(l);
    std::vector<int2*> outs;
    for (int b : who) outs.push_back(d_cand + cand_ofs[b * nl + l]);
    auto xm = ext_of(l, who, outs.data());
    if (xm.second <= 0) continue;
    k_cand_rows<<<dim3((xm.second + 7) / 8, 1, (unsigned)who.size()), 256, 0, st>>>(xm.first, threshold, 1);
    ++nlaunch;
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  std::vector<LevelRef> refs(B * nl);
  for (int b = 0; b < B; ++b)
    for (int l = 0; l < nl; ++l) {
      LevelRef& R = refs[b * nl + l];
      const int r = b * nl + l;
      R.n_kp = d_nkp + r;
      R.kp = d_kp + cand_ofs[r];
      R.flags = d_flags + cand_ofs[r];
      R.cand = d_cand + cand_ofs[r];
      R.n_cand = cand_ofs[r + 1] - cand_ofs[r];
      R.head = d_heads + grid_ofs[r], R.gx = grid_dim[r].x, R.gy = grid_dim[r].y;
      R.next = d_link + cand_ofs[r], R.cell_of = d_link + n_cand + cand_ofs[r];
      if (l >= (int)imgs[b]->lv.size()) continue;
      const r3d_akaze_level& L = imgs[b]->lv[l];
      R.det = M[b].Ldet[l], R.lx = M[b].Lx[l], R.ly = M[b].Ly[l], R.w = L.width, R.h = L.height;
      R.ratio = L.ratio, R.size = L.esigma * kDerivFactor, R.octave = L.octave, R.level = l;
      R.cell = R.size * 1.0625f;
    }
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_refs, refs.data(), refs.size() * sizeof(LevelRef), cudaMemcpyHostToDevice, st));
  std::vector<int> nkp_h(B * nl);
  uint8_t* d_mask = nullptr;
  std::vector<size_t> mask_ofs(B * nl + 1, 0);  // AKAZE: each (image, level)'s pixels in one mask
  if (detector == R3D_DETECTOR_AKAZE) {
    for (int b = 0; b < B; ++b)
      for (int l = 0; l < nl; ++l) {
        const int r = b * nl + l;
        const bool has = l < (int)imgs[b]->lv.size();
        mask_ofs[r + 1] = mask_ofs[r] + (has ? (size_t)imgs[b]->lv[l].width * imgs[b]->lv[l].height : 0);
      }
    const size_t mp = std::max<size_t>(mask_ofs.back(), 1);
    d_mask = (uint8_t*)alloc(3 * mp);
    CvRef* d_cv = (CvRef*)alloc((size_t)B * nl * sizeof(CvRef));
    int* d_nlev = (int*)alloc((size_t)B * 4);
    if (!d_mask || !d_cv || !d_nlev) return fail(ctx, R3D_ERR_NOMEM, "r3d_detect_keypoints: device allocation failed");
    std::vector<CvRef> cv(B * nl);
    std::vector<int> nlev(B);
    for (int b = 0; b < B; ++b) {
      nlev[b] = (int)imgs[b]->lv.size();
      for (int l = 0; l < nl; ++l) {
        const int r = b * nl + l;
        CvRef& R = cv[r];
        R = CvRef{};
        for (int k = 0; k < 3; ++k) R.m[k] = d_mask + k * mp + mask_ofs[r];
        R.cand = d_cand + cand_ofs[r];
        R.n_cand = cand_ofs[r + 1] - cand_ofs[r];
        nkp_h[r] = R.n_cand;
        if (l >= nlev[b]) continue;
        const r3d_akaze_level& L = imgs[b]->lv[l];
        R.det = M[b].Ldet[l], R.w = L.width, R.h = L.height, R.r = L.sigma_size;
        R.ratio = L.ratio, R.size = L.esigma * kDerivFactor, R.octave = L.octave, R.level = l;
      }
    }
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_cv, cv.data(), cv.size() * sizeof(CvRef), cudaMemcpyHostToDevice, st));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_nlev, nlev.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_mask, 0, mp, st));
    R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[3], st));
    const unsigned warps = (unsigned)(B * nl + 3) / 4;
    k_cv_same<<<warps, 128, 0, st>>>(d_cv, B * nl);
    ++nlaunch;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[4], st));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_mask + mp, d_mask, mp, cudaMemcpyDeviceToDevice, st));
    k_cv_lower<<<warps, 128, 0, st>>>(d_cv, nl, B, d_nlev);
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_mask + 2 * mp, d_mask + mp, mp, cudaMemcpyDeviceToDevice, st));
    k_cv_upper<<<warps, 128, 0, st>>>(d_cv, nl, B, d_nlev);
    nlaunch += 2;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[5], st));
    int max_c = 1;
    for (int v : nkp_h) max_c = std::max(max_c, v);
    k_cv_refine<<<dim3((max_c + 127) / 128, nl, B), 128, 0, st>>>(d_cv, nl, B, d_ref, d_cofs);
    ++nlaunch;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
  } else {
    R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[3], st));
    k_same_level<<<(B * nl + 3) / 4, 128, 0, st>>>(d_refs, B * nl);
    ++nlaunch;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[4], st));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(nkp_h.data(), d_nkp, nkp_h.size() * 4, cudaMemcpyDeviceToHost, st));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(st));
    int max_kp = 1;
    for (int v : nkp_h) max_kp = std::max(max_kp, v);
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_flags, 0, (size_t)std::max(n_cand, 1), st));
    if (nl > 1) {
      k_lower<<<dim3((max_kp + 127) / 128, nl - 1, B), 128, 0, st>>>(d_refs, nl, B);
      ++nlaunch;
    }
    k_upper<<<dim3((max_kp + 127) / 128, nl, B), 128, 0, st>>>(d_refs, nl, B);
    ++nlaunch;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[5], st));

    // ---- refinement, orientation ----
    k_refine<<<dim3((max_kp + 127) / 128, nl, B), 128, 0, st>>>(d_refs, nl, B, d_ref, d_cofs);
    ++nlaunch;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
  }
  std::vector<KpDev> ref_h(n_cand);
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(ref_h.data(), d_ref, (size_t)n_cand * sizeof(KpDev), cudaMemcpyDeviceToHost, st));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  std::vector<KpDev> fin;
  std::vector<int> fin_ref, fin_img;
  for (int b = 0; b < B; ++b)
    for (int l = 0; l < nl; ++l) {
      const int r = b * nl + l;
      for (int j = 0; j < nkp_h[r]; ++j) {
        const KpDev& k = ref_h[cand_ofs[r] + j];
        if (k.class_id < 0) continue;
        fin.push_back(k), fin_ref.push_back(r), fin_img.push_back(b);
      }
    }
  const int nf = (int)fin.size();
  std::vector<float2> ori(nf);
  if (nf) {
    KpDev* d_fin = (KpDev*)alloc((size_t)nf * sizeof(KpDev));
    int* d_fref = (int*)alloc((size_t)nf * 4);
    float2* d_ori = (float2*)alloc((size_t)nf * 8);
    if (!d_fin || !d_fref || !d_ori) return fail(ctx, R3D_ERR_NOMEM, "r3d_akaze_detect: device allocation failed");
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_fin, fin.data(), (size_t)nf * sizeof(KpDev), cudaMemcpyHostToDevice, st));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_fref, fin_ref.data(), (size_t)nf * 4, cudaMemcpyHostToDevice, st));
    k_orient<<<(nf + 127) / 128, 128, 0, st>>>(d_fin, nf, d_refs, d_fref, gauss25(), d_ori);
    ++nlaunch;
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(ori.data(), d_ori, (size_t)nf * 8, cudaMemcpyDeviceToHost, st));
  }
  R3D_CUDA_TRY(ctx, cudaEventRecord(T.e[6], st));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  for (int k = 0; k < nf; ++k) {
    r3d_akaze_keypoint o;
    std::memcpy(&o, &fin[k], sizeof(o));
    // cv::AKAZE keeps fastAtan2's degrees; Regard3D converts only Fast-AKAZE's getAngleV2 radians
    o.angle = detector == R3D_DETECTOR_AKAZE ? fast_atan2_deg(ori[k].y, ori[k].x) : regard3d_angle(ori[k].x, ori[k].y);
    kps_out[fin_img[k]]->push_back(o);
  }
  for (int s = 0; s < kStages; ++s) {
    float ms = 0.0f;
    R3D_CUDA_TRY(ctx, cudaEventElapsedTime(&ms, T.e[s], T.e[s + 1]));
    stage_ms[s] += ms;
  }
  *launches += nlaunch;

  if (dbg) {  // batch of one image: every level's arrays, kcontrast, candidates and flags
    const Image& im = *imgs[0];
    float* a = dbg->arrays;
    for (int l = 0; l < nl; ++l) {
      const size_t lp = (size_t)im.lv[l].width * im.lv[l].height;
      for (float* src : {M[0].Lt[l], M[0].Ls[l], M[0].Lx[l], M[0].Ly[l], M[0].Ldet[l]}) {
        R3D_CUDA_TRY(ctx, cudaMemcpy(a, src, lp * 4, cudaMemcpyDeviceToHost));
        a += lp;
      }
    }
    std::vector<float> kc((size_t)kMaxBatch * nl);
    R3D_CUDA_TRY(ctx, cudaMemcpy(kc.data(), d_kc, kc.size() * 4, cudaMemcpyDeviceToHost));
    for (int l = 0; l < nl; ++l) dbg->kcontrast[l] = nl > 1 ? kc[l * kMaxBatch] : 0.0f;
    if (dbg->masks) {
      const size_t mp = std::max<size_t>(mask_ofs.back(), 1);
      uint8_t* m = dbg->masks;
      for (int l = 0; l < nl; ++l)
        for (int k = 0; k < 3; ++k) {
          const size_t lp = mask_ofs[l + 1] - mask_ofs[l];
          R3D_CUDA_TRY(ctx, cudaMemcpy(m, d_mask + k * mp + mask_ofs[l], lp, cudaMemcpyDeviceToHost));
          m += lp;
        }
      return R3D_OK;
    }
    size_t total = 0;
    for (int l = 0; l < nl; ++l) total += nkp_h[l];
    if (total > dbg->cap) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_akaze_levels: more candidates than cand_cap");
    size_t o = 0;
    for (int l = 0; l < nl; ++l) {
      dbg->counts[l] = nkp_h[l];
      R3D_CUDA_TRY(ctx, cudaMemcpy(dbg->cands + o, d_kp + cand_ofs[l], (size_t)nkp_h[l] * sizeof(KpDev),
                                   cudaMemcpyDeviceToHost));
      R3D_CUDA_TRY(ctx, cudaMemcpy(dbg->flags + o, d_flags + cand_ofs[l], (size_t)nkp_h[l], cudaMemcpyDeviceToHost));
      o += nkp_h[l];
    }
  }
  return R3D_OK;
}

bool known_detector(int detector) { return detector == R3D_DETECTOR_FAST_AKAZE || detector == R3D_DETECTOR_AKAZE; }

int check_options(const r3d_akaze_options* opt) {
  return opt && std::isfinite(opt->threshold) && opt->octaves >= 1 && opt->octaves <= 8 && opt->sublevels >= 1 &&
         opt->sublevels <= 8 && opt->diffusivity == R3D_AKAZE_DIFF_PM_G2;
}

int prepare(r3d_ctx* ctx, const float* const* images, const uint32_t* widths, const uint32_t* heights, uint32_t n,
            const r3d_akaze_options* opt, std::vector<Image>& out) {
  if (!ctx || (n && (!images || !widths || !heights)) || !check_options(opt))
    return fail(ctx, R3D_ERR_INVALID, "r3d_akaze_detect: bad arguments or options");
  out.resize(n);
  for (uint32_t i = 0; i < n; ++i) {
    if (!images[i] || widths[i] <= 2 || heights[i] <= 2 || widths[i] > 32767 || heights[i] > 32767)
      return fail(ctx, R3D_ERR_INVALID, "r3d_akaze_detect: image " + std::to_string(i) + " has a side <= 2 or > 32767");
    const size_t P = (size_t)widths[i] * heights[i];
    for (size_t k = 0; k < P; ++k)
      if (!std::isfinite(images[i][k]))
        return fail(ctx, R3D_ERR_INVALID, "r3d_akaze_detect: image " + std::to_string(i) + " has a non-finite pixel");
    out[i].host = images[i];
    out[i].W = (int)widths[i];
    out[i].H = (int)heights[i];
    out[i].lv = level_table(out[i].W, out[i].H, opt->octaves, opt->sublevels);
  }
  return R3D_OK;
}

// The maps on the host (libm cos / sin, as r3d_liop_describe computes them), 24 B per keypoint to the device, k_liop
// on w.copy_stream, timed by ev[0] / ev[1].  The stream is idle here: finish_describe waited for the previous batch.
int launch_describe(r3d_ctx* ctx, DeviceWorker& w, Pending& p, const std::vector<std::vector<r3d_akaze_keypoint>>& kps,
                    float factor, const liop::Tables* d_T, const cudaEvent_t* ev) {
  p.S.n = (int)p.slot_img.size();
  uint32_t n = 0;
  for (int s = 0; s < p.S.n; ++s) p.S.first[s] = n, n += (uint32_t)kps[p.slot_img[s]].size();
  p.S.first[p.S.n] = n;
  p.n = n;
  if (n == 0) return R3D_OK;
  std::vector<float> hM((size_t)n * 6);
  parallel_for(ctx->host_threads, (size_t)p.S.n, [&](size_t s) {
    const std::vector<r3d_akaze_keypoint>& k = kps[p.slot_img[s]];
    float* m = &hM[(size_t)p.S.first[s] * 6];
    for (size_t j = 0; j < k.size(); ++j) liop::affine_of(k[j].x, k[j].y, k[j].size, k[j].angle, factor, m + 6 * j);
  });
  float* d_M = (float*)pool_alloc(w, hM.size() * 4);
  if (d_M) p.held.push_back(d_M);
  p.d_desc = (float*)pool_alloc(w, (size_t)n * liop::kDim * 4);
  if (p.d_desc) p.held.push_back(p.d_desc);
  if (!d_M || !p.d_desc) return fail(ctx, R3D_ERR_NOMEM, "r3d_extract_features: device allocation failed");
  const cudaStream_t cs = w.copy_stream;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_M, hM.data(), hM.size() * 4, cudaMemcpyHostToDevice, cs));
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev[0], cs));
  if (int rc = liop::describe(ctx, cs, p.S, d_M, n, d_T, p.d_desc)) return rc;
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev[1], cs));
  return R3D_OK;
}

// waits for the batch's descriptors, downloads them per image and releases the batch's images
int finish_describe(r3d_ctx* ctx, DeviceWorker& w, Pending& p, std::vector<std::vector<float>>& desc,
                    const cudaEvent_t* ev, double* describe_ms, double* d2h_ms) {
  if (p.n) {
    R3D_CUDA_TRY(ctx, cudaEventSynchronize(ev[1]));
    float ms = 0.0f;
    R3D_CUDA_TRY(ctx, cudaEventElapsedTime(&ms, ev[0], ev[1]));
    *describe_ms += ms;
    const auto t0 = std::chrono::steady_clock::now();
    for (size_t s = 0; s < p.slot_img.size(); ++s) {
      const size_t k = p.S.first[s + 1] - p.S.first[s];
      std::vector<float>& d = desc[p.slot_img[s]];
      d.resize(k * liop::kDim);
      if (k)
        R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d.data(), p.d_desc + (size_t)p.S.first[s] * liop::kDim,
                                          k * liop::kDim * 4, cudaMemcpyDeviceToHost, w.copy_stream));
    }
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.copy_stream));
    *d2h_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }
  for (void* q : p.held) pool_release(w, q);
  p.held.clear();
  p.n = 0;
  return R3D_OK;
}

// r3d_extract_features' host side: describe the batches, then hand each finished image to the device's file writer or
// report it directly
struct Extract {
  float factor;
  const char* out_dir;
  const char* const* basenames;
  bool keep;                        // the caller wants the arrays (out != NULL); else the writer frees them
  std::function<void()> finished;   // one image done: progress
};

// one host thread per device: formats and writes the files of finished images while the device works on
struct Writer {
  std::mutex mu;
  std::condition_variable cv;
  std::deque<uint32_t> q;
  bool closed = false;
  std::atomic<bool> failed{false};
  std::string bad;  // the first path that could not be written
  double ms = 0.0;
  std::thread th;
  void push(uint32_t i) {
    {
      std::lock_guard<std::mutex> lk(mu);
      q.push_back(i);
    }
    cv.notify_one();
  }
  void close() {
    {
      std::lock_guard<std::mutex> lk(mu);
      closed = true;
    }
    cv.notify_one();
    if (th.joinable()) th.join();
  }
  void run(r3d_features& F, const Extract& X) {
    for (;;) {
      uint32_t i;
      {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return closed || !q.empty(); });
        if (q.empty()) return;
        i = q.front();
        q.pop_front();
      }
      if (failed) continue;
      const auto t0 = std::chrono::steady_clock::now();
      const std::vector<r3d_akaze_keypoint>& k = F.kps[i];
      std::vector<float> xyso(k.size() * 4);
      for (size_t j = 0; j < k.size(); ++j)  // SIOPointFeature: scale = size / 2 (Regard3DFeatures.cpp:846-849)
        xyso[4 * j] = k[j].x, xyso[4 * j + 1] = k[j].y, xyso[4 * j + 2] = k[j].size / 2.0f, xyso[4 * j + 3] = k[j].angle;
      const std::string base = std::string(X.out_dir) + "/" + X.basenames[i];
      const std::string feat = base + ".feat", desc = base + ".desc";
      if (const char* b = save_features(feat.c_str(), desc.c_str(), xyso.data(), F.desc[i].data(), k.size(), liop::kDim)) {
        bad = b;
        failed = true;
      } else {
        if (!X.keep) std::vector<r3d_akaze_keypoint>().swap(F.kps[i]), std::vector<float>().swap(F.desc[i]);
        X.finished();
      }
      ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
  }
};

struct Acc {  // one device's share of a call
  double ms[kStages] = {}, describe_ms = 0.0, d2h_ms = 0.0;
  uint32_t launches = 0, batches = 0, keypoints = 0;
  int rc = R3D_OK;
};

// r3d_akaze_detect (X == nullptr) and r3d_extract_features: the images are dealt to the context's devices in
// contiguous slices; each device runs its slice in batches of at most kMaxBatch images and half its free memory, on a
// host thread of its own.  With X, batch b's descriptors are computed on the second stream while batch b + 1 builds its
// scale space, and W[d] writes the files.
int run_devices(r3d_ctx* ctx, std::vector<Image>& ims, float threshold, int detector, r3d_features& F, const Extract* X,
                std::vector<std::unique_ptr<Writer>>* W, std::vector<Acc>& acc) {
  const uint32_t n_images = (uint32_t)ims.size();
  const int nd = (int)acc.size();
  auto run_device = [&](int d) {
    Acc& A = acc[d];
    DeviceWorker& w = ctx->workers[d];
    const uint32_t i0 = (uint32_t)((uint64_t)n_images * d / nd), i1 = (uint32_t)((uint64_t)n_images * (d + 1) / nd);
    auto cuda = [&](cudaError_t e, const char* what) {
      if (e != cudaSuccess) A.rc = fail(ctx, R3D_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
      return e == cudaSuccess;
    };
    if (!cuda(cudaSetDevice(w.device), "cudaSetDevice")) return;
    size_t free_b = 0, total_b = 0;
    if (!cuda(cudaMemGetInfo(&free_b, &total_b), "cudaMemGetInfo")) return;
    const size_t budget = std::max<size_t>(free_b / 2, (size_t)1 << 28);
    Pending prev, cur;
    liop::Tables* d_T = nullptr;
    Events<2> ev;
    struct Cleanup {  // on every exit: nothing on the second stream may still read a block that goes back to the pool
      DeviceWorker& w;
      Pending &a, &b;
      liop::Tables*& t;
      ~Cleanup() {
        cudaStreamSynchronize(w.copy_stream);
        for (Pending* p : {&a, &b})
          for (void* q : p->held) pool_release(w, q);
        pool_release(w, t);
      }
    } cleanup{w, prev, cur, d_T};
    if (X) {
      if (!cuda(ev.create(true), "cudaEventCreate")) return;
      if (!(d_T = liop::tables_to_device(w, w.stream)) || !cuda(cudaStreamSynchronize(w.stream), "tables")) {
        A.rc = fail(ctx, R3D_ERR_NOMEM, "r3d_extract_features: device allocation failed");
        return;
      }
    }
    // the images of a finished batch go to the writer, or are reported at once
    auto finish = [&](Pending& p) -> int {
      if (int rc = finish_describe(ctx, w, p, F.desc, ev.e, &A.describe_ms, &A.d2h_ms)) return rc;
      for (uint32_t i = p.i0; i < p.i1; ++i) {
        A.keypoints += (uint32_t)F.kps[i].size();
        if (W) (*W)[d]->push(i);
        else X->finished();
      }
      p.i0 = p.i1 = 0;
      return R3D_OK;
    };
    for (uint32_t i = i0; i < i1;) {
      if (W && (*W)[d]->failed) return;  // a file could not be written: the call fails, stop early
      std::vector<akaze::Image*> work;  // images too small for a single level have no keypoints and stay out
      std::vector<std::vector<r3d_akaze_keypoint>*> wout;
      size_t bytes = 0;
      int taken = 0;
      cur = Pending();
      cur.i0 = i;
      while (i < i1 && taken < akaze::kMaxBatch && (taken == 0 || bytes + akaze::image_bytes(ims[i]) <= budget)) {
        bytes += akaze::image_bytes(ims[i]);
        if (!ims[i].lv.empty()) work.push_back(&ims[i]), wout.push_back(&F.kps[i]), cur.slot_img.push_back(i);
        ++taken, ++i;
      }
      cur.i1 = i;
      if (!work.empty() &&
          (A.rc = run_batch(ctx, w, work, threshold, detector, wout, nullptr, A.ms, &A.launches, X ? &cur : nullptr)))
        return;
      ++A.batches;
      if (!X) continue;
      if ((A.rc = finish(prev))) return;
      if ((A.rc = launch_describe(ctx, w, cur, F.kps, X->factor, d_T, ev.e))) return;
      if (cur.n) ++A.launches;
      std::swap(prev, cur);
    }
    if (X) A.rc = finish(prev);
  };
  if (nd == 1) {
    run_device(0);
  } else {
    std::vector<std::thread> th;
    for (int d = 0; d < nd; ++d) th.emplace_back(run_device, d);
    for (std::thread& t : th) t.join();
  }
  for (const Acc& A : acc)
    if (A.rc) return A.rc;
  return R3D_OK;
}

}  // namespace akaze
}  // namespace r3d

using namespace r3d;

extern "C" void r3d_akaze_default_options(r3d_akaze_options* out) {
  if (out) *out = r3d_akaze_options{0.001f, 4, 4, R3D_AKAZE_DIFF_PM_G2};
}

extern "C" int r3d_akaze_levels(uint32_t width, uint32_t height, const r3d_akaze_options* opt, r3d_akaze_level* out,
                                int cap) {
  if (width <= 2 || height <= 2 || !akaze::check_options(opt) || (cap > 0 && !out))
    return fail(nullptr, R3D_ERR_INVALID, "r3d_akaze_levels: bad arguments");
  std::vector<r3d_akaze_level> lv = akaze::level_table((int)width, (int)height, opt->octaves, opt->sublevels);
  for (size_t i = 1; i < lv.size(); ++i)
    lv[i].n_tau = (uint32_t)akaze::fed_tau(lv[i].etime - lv[i - 1].etime, 0.25f).size();
  for (int i = 0; i < (int)lv.size() && i < cap; ++i) out[i] = lv[i];
  return (int)lv.size();
}

extern "C" int r3d_detect_keypoints(r3d_ctx* ctx, int detector, const float* const* images, const uint32_t* widths,
                                    const uint32_t* heights, uint32_t n_images, const r3d_akaze_options* opt,
                                    r3d_features** out) {
  if (!out) return fail(ctx, R3D_ERR_INVALID, "r3d_akaze_detect: out is NULL");
  *out = nullptr;
  if (!akaze::known_detector(detector)) return fail(ctx, R3D_ERR_INVALID, "r3d_detect_keypoints: unknown detector");
  std::vector<akaze::Image> ims;
  int rc = akaze::prepare(ctx, images, widths, heights, n_images, opt, ims);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  std::unique_ptr<r3d_features> F(new r3d_features());
  F->kps.resize(n_images);
  const int nd = (int)std::min<size_t>(ctx->workers.size(), std::max<uint32_t>(n_images, 1));
  std::vector<akaze::Acc> acc(nd);
  if ((rc = akaze::run_devices(ctx, ims, opt->threshold, detector, *F, nullptr, nullptr, acc))) return rc;
  r3d_akaze_timing T{};
  for (const akaze::Acc& A : acc) {
    T.upload_ms += A.ms[0], T.scale_space_ms += A.ms[1], T.candidates_ms += A.ms[2], T.same_level_ms += A.ms[3];
    T.cross_level_ms += A.ms[4], T.refine_orient_ms += A.ms[5];
    T.kernel_launches += A.launches, T.batches += A.batches;
  }
  T.total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  T.images = n_images;
  T.devices = (uint32_t)nd;
  for (auto& v : F->kps) T.keypoints += (uint32_t)v.size();
  ctx->akaze_timing = T;
  *out = F.release();
  return R3D_OK;
}

extern "C" int r3d_akaze_detect(r3d_ctx* ctx, const float* const* images, const uint32_t* widths,
                                const uint32_t* heights, uint32_t n_images, const r3d_akaze_options* opt,
                                r3d_features** out) {
  return r3d_detect_keypoints(ctx, R3D_DETECTOR_FAST_AKAZE, images, widths, heights, n_images, opt, out);
}

extern "C" uint32_t r3d_features_num_images(const r3d_features* f) { return f ? (uint32_t)f->kps.size() : 0; }
extern "C" uint32_t r3d_features_count(const r3d_features* f, uint32_t image) {
  return f && image < f->kps.size() ? (uint32_t)f->kps[image].size() : 0;
}
extern "C" const r3d_akaze_keypoint* r3d_features_get(const r3d_features* f, uint32_t image) {
  return f && image < f->kps.size() ? f->kps[image].data() : nullptr;
}
extern "C" void r3d_free_features(r3d_features* f) { delete f; }

extern "C" int r3d_get_akaze_timing(const r3d_ctx* ctx, r3d_akaze_timing* out) {
  if (!ctx || !out) return R3D_ERR_INVALID;
  *out = ctx->akaze_timing;
  return R3D_OK;
}

extern "C" void r3d_extract_default_options(r3d_extract_options* out) {
  if (!out) return;
  r3d_akaze_default_options(&out->akaze);
  out->kp_size_factor = 8.0f;
  out->out_dir = nullptr;
  out->basenames = nullptr;
}

extern "C" int r3d_extract_features_detector(r3d_ctx* ctx, int detector, const float* const* images,
                                             const uint32_t* widths, const uint32_t* heights, uint32_t n_images,
                                             const r3d_extract_options* opt, r3d_progress_cb cb, void* user,
                                             r3d_features** out) {
  if (out) *out = nullptr;
  if (!akaze::known_detector(detector))
    return fail(ctx, R3D_ERR_INVALID, "r3d_extract_features_detector: unknown detector");
  if (!opt || !std::isfinite(opt->kp_size_factor) || opt->kp_size_factor <= 0.0f)
    return fail(ctx, R3D_ERR_INVALID, "r3d_extract_features: bad options");
  const bool files = opt->out_dir != nullptr;
  if (files) {
    if (!*opt->out_dir || (n_images && !opt->basenames))
      return fail(ctx, R3D_ERR_INVALID, "r3d_extract_features: empty out_dir or no basenames");
    for (uint32_t i = 0; i < n_images; ++i)
      if (!opt->basenames[i] || !*opt->basenames[i])
        return fail(ctx, R3D_ERR_INVALID, "r3d_extract_features: basename " + std::to_string(i) + " is missing");
  } else if (!out) {
    return fail(ctx, R3D_ERR_INVALID, "r3d_extract_features: neither out nor out_dir");
  }
  std::vector<akaze::Image> ims;
  int rc = akaze::prepare(ctx, images, widths, heights, n_images, &opt->akaze, ims);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  std::unique_ptr<r3d_features> F(new r3d_features());
  F->kps.resize(n_images);
  F->desc.resize(n_images);
  const int nd = (int)std::min<size_t>(ctx->workers.size(), std::max<uint32_t>(n_images, 1));
  // R3DFeaturesThread::sendMsgToMainFrame (src/threads/R3DFeaturesThread.cpp:211-228), one call at a time
  std::mutex progress_mu;
  uint32_t done = 0;
  akaze::Extract X{opt->kp_size_factor, opt->out_dir, opt->basenames, out != nullptr, [&] {
                     std::lock_guard<std::mutex> lk(progress_mu);
                     ++done;
                     const float finished = static_cast<float>(done) / static_cast<int>(n_images);
                     if (cb) cb(finished * 0.4f + 0.2f, "", user);
                   }};
  std::vector<std::unique_ptr<akaze::Writer>> W;
  if (files)
    for (int d = 0; d < nd; ++d) {
      W.emplace_back(new akaze::Writer());
      akaze::Writer* wr = W.back().get();
      wr->th = std::thread([wr, &F, &X] { wr->run(*F, X); });
    }
  std::vector<akaze::Acc> acc(nd);
  rc = akaze::run_devices(ctx, ims, opt->akaze.threshold, detector, *F, &X, files ? &W : nullptr, acc);
  r3d_extract_timing T{};
  for (std::unique_ptr<akaze::Writer>& wr : W) {
    wr->close();
    T.write_ms += wr->ms;
    if (!rc && wr->failed) rc = fail(ctx, R3D_ERR_IO, "r3d_extract_features: cannot write " + wr->bad);
  }
  if (rc) return rc;
  for (const akaze::Acc& A : acc) {
    T.upload_ms += A.ms[0];
    for (int s = 1; s < akaze::kStages; ++s) T.detect_ms += A.ms[s];
    T.describe_ms += A.describe_ms, T.d2h_ms += A.d2h_ms;
    T.kernel_launches += A.launches, T.batches += A.batches, T.keypoints += A.keypoints;
  }
  T.total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  T.images = n_images;
  T.devices = (uint32_t)nd;
  ctx->extract_timing = T;
  if (out) *out = F.release();
  return R3D_OK;
}

extern "C" int r3d_extract_features(r3d_ctx* ctx, const float* const* images, const uint32_t* widths,
                                    const uint32_t* heights, uint32_t n_images, const r3d_extract_options* opt,
                                    r3d_progress_cb cb, void* user, r3d_features** out) {
  return r3d_extract_features_detector(ctx, R3D_DETECTOR_FAST_AKAZE, images, widths, heights, n_images, opt, cb, user,
                                       out);
}

extern "C" const float* r3d_features_descriptors(const r3d_features* f, uint32_t image) {
  return f && image < f->desc.size() && !f->desc[image].empty() ? f->desc[image].data() : nullptr;
}

extern "C" int r3d_get_extract_timing(const r3d_ctx* ctx, r3d_extract_timing* out) {
  if (!ctx || !out) return R3D_ERR_INVALID;
  *out = ctx->extract_timing;
  return R3D_OK;
}

extern "C" int r3d_debug_akaze_levels(r3d_ctx* ctx, const float* image, uint32_t width, uint32_t height,
                                      const r3d_akaze_options* opt, float* arrays, float* kcontrast,
                                      r3d_akaze_keypoint* cands, uint8_t* flags, uint32_t cand_cap,
                                      uint32_t* cand_counts) {
  std::vector<akaze::Image> ims;
  int rc = akaze::prepare(ctx, &image, &width, &height, 1, opt, ims);
  if (rc) return rc;
  if (!arrays || !kcontrast || !cand_counts || (cand_cap && (!cands || !flags)))
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_akaze_levels: bad arguments");
  if (ims[0].lv.empty()) return R3D_OK;
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::vector<akaze::Image*> batch{&ims[0]};
  std::vector<r3d_akaze_keypoint> kps;
  std::vector<std::vector<r3d_akaze_keypoint>*> outs{&kps};
  const akaze::Debug dbg{arrays, kcontrast, cands, flags, cand_cap, cand_counts, nullptr};
  double ms[akaze::kStages] = {};
  uint32_t launches = 0;
  return akaze::run_batch(ctx, w, batch, opt->threshold, R3D_DETECTOR_FAST_AKAZE, outs, &dbg, ms, &launches);
}

extern "C" int r3d_debug_akaze_masks(r3d_ctx* ctx, const float* image, uint32_t width, uint32_t height,
                                     const r3d_akaze_options* opt, float* arrays, float* kcontrast, uint8_t* masks) {
  std::vector<akaze::Image> ims;
  int rc = akaze::prepare(ctx, &image, &width, &height, 1, opt, ims);
  if (rc) return rc;
  if (!arrays || !kcontrast || !masks) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_akaze_masks: bad arguments");
  if (ims[0].lv.empty()) return R3D_OK;
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::vector<akaze::Image*> batch{&ims[0]};
  std::vector<r3d_akaze_keypoint> kps;
  std::vector<std::vector<r3d_akaze_keypoint>*> outs{&kps};
  uint32_t count = 0;
  const akaze::Debug dbg{arrays, kcontrast, nullptr, nullptr, 0, &count, masks};
  double ms[akaze::kStages] = {};
  uint32_t launches = 0;
  return akaze::run_batch(ctx, w, batch, opt->threshold, R3D_DETECTOR_AKAZE, outs, &dbg, ms, &launches);
}

extern "C" int r3d_debug_akaze_refine(r3d_ctx* ctx, const float* ldet, uint32_t width, uint32_t height, float ratio,
                                      const r3d_akaze_keypoint* in, uint32_t n, r3d_akaze_keypoint* out) {
  if (!ctx || !ldet || width < 3 || height < 3 || (n && (!in || !out)))
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_akaze_refine: bad arguments");
  for (uint32_t i = 0; i < n; ++i) {  // the 3x3 stencil must stay inside the plane
    const int x = (int)(in[i].x / ratio), y = (int)(in[i].y / ratio);
    if (!(x >= 1 && y >= 1 && x < (int)width - 1 && y < (int)height - 1))
      return fail(ctx, R3D_ERR_INVALID, "r3d_debug_akaze_refine: point outside the level's interior");
  }
  if (n == 0) return R3D_OK;
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  DevArr<float> d_det(w);
  DevArr<akaze::KpDev> d_in(w), d_out(w);
  DevArr<int> d_int(w);
  DevArr<uint8_t> d_flags(w);
  DevArr<akaze::LevelRef> d_ref(w);
  if (!d_det.alloc((size_t)width * height) || !d_in.alloc(n) || !d_out.alloc(n) || !d_int.alloc(2) ||
      !d_flags.alloc(n) || !d_ref.alloc(1))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_debug_akaze_refine: device allocation failed");
  const int ints[2] = {(int)n, 0};  // the point count, the output offset
  akaze::LevelRef R{};
  R.det = d_det.p, R.w = (int)width, R.h = (int)height, R.kp = d_in.p, R.n_kp = d_int.p, R.flags = d_flags.p;
  R.ratio = ratio;
  cudaStream_t st = w.stream;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_det.p, ldet, (size_t)width * height * 4, cudaMemcpyHostToDevice, st));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_in.p, in, (size_t)n * sizeof(akaze::KpDev), cudaMemcpyHostToDevice, st));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_out.p, in, (size_t)n * sizeof(akaze::KpDev), cudaMemcpyHostToDevice, st));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_int.p, ints, sizeof(ints), cudaMemcpyHostToDevice, st));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_flags.p, 0, n, st));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ref.p, &R, sizeof(R), cudaMemcpyHostToDevice, st));
  akaze::k_refine<<<dim3((n + 127) / 128, 1, 1), 128, 0, st>>>(d_ref.p, 1, 1, d_out.p, d_int.p + 1);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(out, d_out.p, (size_t)n * sizeof(akaze::KpDev), cudaMemcpyDeviceToHost, st));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return R3D_OK;
}
