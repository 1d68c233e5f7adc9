// oracle_akaze.cpp -- CPU ORACLE of Regard3D's default keypoint detector, Fast-AKAZE (test infrastructure).
//
// A restatement of the detection path of src/thirdparty/fast-akaze (AKAZEFeatures.cpp Allocate_Memory_Evolution,
// Create_Nonlinear_Scale_Space, Compute_Determinant_Hessian_Response, the threaded Find_Scale_Space_Extrema,
// Do_Subpixel_Refinement, Compute_Main_Orientation; nldiffusion_functions.cpp; fed.cpp) together with the OpenCV
// primitives it calls (GaussianBlur, Scharr, sepFilter2D, resize INTER_AREA, hal::fastAtan2, the 2x2 LU solve).
// Each primitive is written out with ONE fixed operation order; libr3dgpu's akaze.cu runs the same order, so the two
// agree bit for bit.  Against OpenCV's own primitives (SIMD / IPP orders) they agree to a few ulp of the image
// maximum; tests/test_oracle_akaze.py pins those bounds.
//
// Deviation kept on purpose: upstream's nld_step_scalar never writes the first and last column of the first and the
// last row, but the FED update adds its one flat Lstep workspace over the whole level.  The four corners of Lt thus
// pick up whatever that buffer held at those flat indices.  Here (and on the GPU) the buffer is zero at the start of
// each image; upstream's is uninitialised memory for the indices no earlier sweep wrote.
//
// Built with -ffp-contract=off and no -ffast-math (akaze.mk).
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

constexpr double kPi = 3.14159265358979323846;

struct Level {
  int32_t octave, sublevel, width, height, sigma_size, border;
  float esigma, etime, ratio;
  uint32_t n_tau;
};

struct Kp {  // the cv::KeyPoint fields the detector sets (r3d_akaze_keypoint layout)
  float x, y, size, angle, response;
  int32_t octave, class_id;
};

using Img = std::vector<float>;

int fround(float v) { return (int)(v + 0.5f); }

int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}
int replicate(int p, int n) { return p < 0 ? 0 : (p >= n ? n - 1 : p); }

// ---- kernels ------------------------------------------------------------------------------------------------------

// cv::getGaussianKernel(n, sigma, CV_32F) for sigma > 0 (OpenCV 4.x getGaussianKernelBitExact, rounded to float)
void gaussian_kernel(int n, double sigma, float* k) {
  const double scale2x = -0.125 / (sigma * sigma);
  const int c = (n - 1) / 2;
  std::vector<double> t(n);
  double sum = 0.0;
  for (int i = 0, x = 1 - n; i < c; ++i, x += 2) {
    t[i] = std::exp((double)(x * x) * scale2x);
    sum += t[i];
  }
  sum *= 2.0;
  sum += 1.0;
  const double mul = 1.0 / sum;
  for (int i = 0; i < c; ++i) k[i] = k[n - 1 - i] = (float)(t[i] * mul);
  k[c] = (float)mul;
}

int gaussian_ksize(float sigma) {  // gaussian_2D_convolutionV2
  int ks = (int)std::ceil(2.0f * (1.0f + (sigma - 0.8f) / (0.3f)));
  return (ks % 2 == 0) ? ks + 1 : ks;
}

// compute_scharr_derivative_kernelsV2: cv::getDerivKernels(dx, dy, SCHARR, normalize) at scale 1, else three taps
// spread over 2 scale + 1
int deriv_kernels(int dx, int dy, int scale, float* kx, float* ky) {
  const int n = 3 + 2 * (scale - 1);
  const float w = 10.0f / 3.0f;
  const float norm = 1.0f / (2.0f * (w + 2.0f));
  for (int pass = 0; pass < 2; ++pass) {
    float* k = pass == 0 ? kx : ky;
    const int order = pass == 0 ? dx : dy;
    for (int i = 0; i < n; ++i) k[i] = 0.0f;
    if (scale == 1) {
      if (order == 0) k[0] = 3.0f / 32.0f, k[1] = 10.0f / 32.0f, k[2] = 3.0f / 32.0f;
      else k[0] = -1.0f, k[1] = 0.0f, k[2] = 1.0f;
    } else if (order == 0) {
      k[0] = norm, k[n / 2] = w * norm, k[n - 1] = norm;
    } else {
      k[0] = -1.0f, k[n - 1] = 1.0f;
    }
  }
  return n;
}

// ---- filters ------------------------------------------------------------------------------------------------------

// separable filter: horizontal pass, then vertical pass; each output is k[0] * s[0] + k[1] * s[1] + ... in tap order
void sep_filter(const float* src, int w, int h, const float* kx, int nx, const float* ky, int ny, bool replicate_border,
                float* dst) {
  Img tmp((size_t)w * h);
  const int rx = nx / 2, ry = ny / 2;
  auto bx = [&](int p) { return replicate_border ? replicate(p, w) : reflect101(p, w); };
  auto by = [&](int p) { return replicate_border ? replicate(p, h) : reflect101(p, h); };
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      const float* row = src + (size_t)y * w;
      float s = kx[0] * row[bx(x - rx)];
      for (int t = 1; t < nx; ++t) s = s + kx[t] * row[bx(x - rx + t)];
      tmp[(size_t)y * w + x] = s;
    }
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float s = ky[0] * tmp[(size_t)by(y - ry) * w + x];
      for (int t = 1; t < ny; ++t) s = s + ky[t] * tmp[(size_t)by(y - ry + t) * w + x];
      dst[(size_t)y * w + x] = s;
    }
}

void gaussian_blur(const float* src, int w, int h, float sigma, float* dst) {
  const int n = gaussian_ksize(sigma);
  std::vector<float> k(n);
  gaussian_kernel(n, (double)sigma, k.data());
  sep_filter(src, w, h, k.data(), n, k.data(), n, true, dst);
}

void scharr(const float* src, int w, int h, int dx, int dy, float* dst) {  // cv::Scharr, scale 1, BORDER_REFLECT_101
  const float d[3] = {-1.0f, 0.0f, 1.0f}, s[3] = {3.0f, 10.0f, 3.0f};
  sep_filter(src, w, h, dx ? d : s, 3, dy ? d : s, 3, false, dst);
}

// cv::resize(src, dst, (w / 2, h / 2), INTER_AREA).  Exact factor 2 on both axes: the 2x2 mean ((a + b) + (c + d))
// * 0.25; otherwise OpenCV's fractional-area tables (computeResizeAreaTab), summed per row, then over rows.
struct AreaTap { int si, di; float alpha; };
std::vector<AreaTap> area_tab(int ssize, int dsize) {
  std::vector<AreaTap> tab;
  const double scale = (double)ssize / dsize;
  for (int dx = 0; dx < dsize; ++dx) {
    const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    const double cell = std::min(scale, ssize - fsx1);
    int sx1 = (int)std::ceil(fsx1), sx2 = (int)std::floor(fsx2);
    sx2 = std::min(sx2, ssize - 1);
    sx1 = std::min(sx1, sx2);
    if (sx1 - fsx1 > 1e-3) tab.push_back({sx1 - 1, dx, (float)((sx1 - fsx1) / cell)});
    for (int sx = sx1; sx < sx2; ++sx) tab.push_back({sx, dx, (float)(1.0 / cell)});
    if (fsx2 - sx2 > 1e-3) tab.push_back({sx2, dx, (float)(std::min(std::min(fsx2 - sx2, 1.0), cell) / cell)});
  }
  return tab;
}

void halfsample(const float* src, int w, int h, float* dst) {
  const int dw = w / 2, dh = h / 2;
  if (w == 2 * dw && h == 2 * dh) {
    for (int y = 0; y < dh; ++y)
      for (int x = 0; x < dw; ++x) {
        const float* s0 = src + (size_t)(2 * y) * w + 2 * x;
        const float* s1 = s0 + w;
        dst[(size_t)y * dw + x] = ((s0[0] + s0[1]) + (s1[0] + s1[1])) * 0.25f;
      }
    return;
  }
  const std::vector<AreaTap> xt = area_tab(w, dw), yt = area_tab(h, dh);
  Img buf(dw);
  for (int dy = 0; dy < dh; ++dy) {
    float* d = dst + (size_t)dy * dw;
    bool first = true;
    for (const AreaTap& ty : yt) {
      if (ty.di != dy) continue;
      const float* s = src + (size_t)ty.si * w;
      std::fill(buf.begin(), buf.end(), 0.0f);
      for (const AreaTap& tx : xt) buf[tx.di] = buf[tx.di] + s[tx.si] * tx.alpha;
      for (int x = 0; x < dw; ++x) d[x] = first ? ty.alpha * buf[x] : d[x] + ty.alpha * buf[x];
      first = false;
    }
  }
}

// hal::fastAtan2 (OpenCV 4.x fastAtan32f), radians
float fast_atan2(float y, float x) {
  static const float p1 = 0.9997878412794807f * (float)(180 / kPi), p3 = -0.3258083974640975f * (float)(180 / kPi),
                     p5 = 0.1555786518463281f * (float)(180 / kPi), p7 = -0.04432655554792128f * (float)(180 / kPi);
  const float ax = std::fabs(x), ay = std::fabs(y);
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

// cv::solve(Matx22f, Vec2f, Vec2f, DECOMP_LU): the 2x2 Cramer branch of lapack.cpp, in double; 0 when singular
void solve2(float a00, float a01, float a10, float a11, float b0, float b1, float* x) {
  double d = (double)a00 * a11 - (double)a01 * a10;
  if (d == 0.0) {
    x[0] = x[1] = 0.0f;
    return;
  }
  d = 1.0 / d;
  const double t = (float)(((double)b0 * a11 - (double)b1 * a01) * d);
  x[1] = (float)(((double)b1 * a00 - (double)b0 * a10) * d);
  x[0] = (float)t;
}

// compute_k_percentileV2 (nbins bins, interior pixels, bin 0 excluded)
float k_percentile(const float* lx, const float* ly, int w, int h, float perc, int nbins) {
  Img modg;
  modg.reserve((size_t)(w - 2) * (h - 2));
  for (int y = 1; y < h - 1; ++y)
    for (int x = 1; x < w - 1; ++x) {
      const size_t i = (size_t)y * w + x;
      modg.push_back(std::sqrt(lx[i] * lx[i] + ly[i] * ly[i]));
    }
  float hmax = 0.0f;
  for (float v : modg)
    if (hmax < v) hmax = v;
  if (hmax == 0.0f) return 0.03f;
  const float mul = (nbins - 1) / hmax;
  std::vector<int32_t> hist(nbins, 0);
  for (float v : modg) hist[(int)(v * mul)]++;
  const int total = (int)modg.size();
  const int nthreshold = (int)((total - hist[0]) * perc);
  int nelements = 0;
  for (int k = 1; k < nbins; ++k) {
    if (nelements >= nthreshold) return (float)hmax * k / nbins;
    nelements = nelements + hist[k];
  }
  return 0.03f;
}

// ---- FED ----------------------------------------------------------------------------------------------------------

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

// fed_tau_by_process_timeV2(T, 1, tau_max, reordering = true)
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

// ---- level table --------------------------------------------------------------------------------------------------

constexpr float kSoffset = 1.6f, kDerivFactor = 1.5f, kPercentile = 0.7f;
constexpr int kNbins = 300;

std::vector<Level> level_table(int W, int H, int omax, int nsub) {
  const float smax = 10.0f * std::sqrt(2.0f);
  std::vector<Level> ev;
  int lw = W, lh = H, power = 1;
  for (int i = 0; i < omax; ++i) {
    for (int j = 0; j < nsub; ++j) {
      Level s{};
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

// ---- the detector -------------------------------------------------------------------------------------------------

struct LevelData {
  Img Lt, Lsmooth, Lx, Ly, Ldet;
  float kcontrast = 0.0f;
  std::vector<float> tau;                 // FED steps from the previous level to this one
  std::vector<Kp> cand;                   // after the same-level pass
  std::vector<uint8_t> del_lower, del_upper;  // deletion flags after the lower- and the upper-level pass
};

struct State {
  int W, H;
  std::vector<Level> lv;
  std::vector<LevelData> ld;
  std::vector<Kp> kps;
  std::vector<float> ori;  // per keypoint (maxX, maxY)
  // how often the rarer branches ran: same-level replacements, singular 2x2 systems, |d| > 1 rejections
  int n_replaced = 0, n_singular = 0, n_rejected = 0;
};

void hessian(const Level& s, LevelData& d) {
  const int w = s.width, h = s.height;
  float dxkx[64], dxky[64], dykx[64], dyky[64];
  const int n = deriv_kernels(1, 0, s.sigma_size, dxkx, dxky);
  deriv_kernels(0, 1, s.sigma_size, dykx, dyky);
  Img lxx((size_t)w * h), lxy((size_t)w * h), lyy((size_t)w * h);
  d.Lx.resize((size_t)w * h);
  d.Ly.resize((size_t)w * h);
  d.Ldet.resize((size_t)w * h);
  sep_filter(d.Lsmooth.data(), w, h, dxkx, n, dxky, n, false, d.Lx.data());
  sep_filter(d.Lx.data(), w, h, dxkx, n, dxky, n, false, lxx.data());
  sep_filter(d.Lx.data(), w, h, dykx, n, dyky, n, false, lxy.data());
  sep_filter(d.Lsmooth.data(), w, h, dykx, n, dyky, n, false, d.Ly.data());
  sep_filter(d.Ly.data(), w, h, dykx, n, dyky, n, false, lyy.data());
  for (size_t j = 0; j < (size_t)w * h; ++j) d.Ldet[j] = lxx[j] * lyy[j] - lxy[j] * lxy[j];
}

// nld_step_scalarV2 into the flat workspace (corners of the first and last row untouched), then Lt += Lstep 0.5 tau
void fed_sweep(float* lt, const float* lf, float* lstep, int w, int h, float tau) {
  auto at = [&](const float* a, int y, int x) { return a[(size_t)y * w + x]; };
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      const bool top = y == 0, bottom = y == h - 1, left = x == 0, right = x == w - 1;
      if ((top || bottom) && (left || right)) continue;
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
      lstep[(size_t)y * w + x] = v;
    }
  for (size_t k = 0; k < (size_t)w * h; ++k) lt[k] += lstep[k] * 0.5f * tau;
}

void scale_space(State& S, const float* img, int omax, int nsub) {
  const int W = S.W, H = S.H;
  S.lv = level_table(W, H, omax, nsub);
  const size_t nl = S.lv.size();
  S.ld.assign(nl, LevelData());
  if (nl == 0) return;
  LevelData& d0 = S.ld[0];
  d0.Lsmooth.resize((size_t)W * H);
  gaussian_blur(img, W, H, kSoffset, d0.Lsmooth.data());
  hessian(S.lv[0], d0);
  d0.Lt = d0.Lsmooth;
  if (nl == 1) return;
  Img ls((size_t)W * H), lx((size_t)W * H), ly((size_t)W * H), lflow((size_t)W * H), lstep((size_t)W * H, 0.0f);
  gaussian_blur(img, W, H, 1.0f, ls.data());
  scharr(ls.data(), W, H, 1, 0, lx.data());
  scharr(ls.data(), W, H, 0, 1, ly.data());
  float kcontrast = k_percentile(lx.data(), ly.data(), W, H, kPercentile, kNbins);
  d0.kcontrast = kcontrast;
  for (size_t i = 1; i < nl; ++i) {
    const Level& s = S.lv[i];
    LevelData& d = S.ld[i];
    const int w = s.width, h = s.height;
    d.Lt.resize((size_t)w * h);
    if (s.octave > S.lv[i - 1].octave) {
      halfsample(S.ld[i - 1].Lt.data(), S.lv[i - 1].width, S.lv[i - 1].height, d.Lt.data());
      kcontrast = kcontrast * 0.75f;
    } else {
      d.Lt = S.ld[i - 1].Lt;
    }
    d.kcontrast = kcontrast;
    d.Lsmooth.resize((size_t)w * h);
    gaussian_blur(d.Lt.data(), w, h, 1.0f, d.Lsmooth.data());
    scharr(d.Lsmooth.data(), w, h, 1, 0, lx.data());
    scharr(d.Lsmooth.data(), w, h, 0, 1, ly.data());
    hessian(s, d);
    const float inv_k2 = 1.0f / (kcontrast * kcontrast);
    for (size_t k = 0; k < (size_t)w * h; ++k) lflow[k] = 1.0f / (1.0f + ((lx[k] * lx[k] + ly[k] * ly[k]) * inv_k2));
    d.tau = fed_tau(s.etime - S.lv[i - 1].etime, 0.25f);
    for (float tau : d.tau) fed_sweep(d.Lt.data(), lflow.data(), lstep.data(), w, h, tau);
  }
}

bool find_neighbor(const Kp& p, const std::vector<Kp>& v, const uint8_t* del, size_t from, size_t& idx, bool inv) {
  for (size_t i = from; i < v.size(); ++i) {
    if (del && del[i]) continue;
    const float dx = p.x - v[i].x, dy = p.y - v[i].y;
    const float r = inv ? v[i].size : p.size;
    if (dx * dx + dy * dy <= r * r) {
      idx = i;
      return true;
    }
  }
  return false;
}

void extrema(State& S, float threshold) {
  const size_t nl = S.lv.size();
  for (size_t i = 0; i < nl; ++i) {  // 1. same level, raster order
    const Level& s = S.lv[i];
    LevelData& d = S.ld[i];
    const int w = s.width;
    const float* L = d.Ldet.data();
    for (int y = s.border; y < s.height - s.border; ++y)
      for (int x = s.border; x < w - s.border; ++x) {
        const float v = L[(size_t)y * w + x];
        if (v <= threshold) continue;
        const float* c = L + (size_t)y * w + x;
        if (v <= c[-1] || v <= c[1]) continue;
        if (v <= c[-w - 1] || v <= c[-w] || v <= c[-w + 1]) continue;
        if (v <= c[w - 1] || v <= c[w] || v <= c[w + 1]) continue;
        const Kp p{(float)(x * s.ratio), (float)(y * s.ratio), s.esigma * kDerivFactor, -1.0f, v, s.octave, (int32_t)i};
        size_t idx = 0;
        if (find_neighbor(p, d.cand, nullptr, 0, idx, false)) {
          if (p.response > d.cand[idx].response) d.cand[idx] = p, S.n_replaced++;
          continue;
        }
        d.cand.push_back(p);
      }
    d.del_lower.assign(d.cand.size(), 0);
  }
  for (size_t i = 1; i < nl; ++i) {  // 2. lower level, i ascending
    std::vector<Kp>& lo = S.ld[i - 1].cand;
    uint8_t* del = S.ld[i - 1].del_lower.data();
    for (const Kp& pt : S.ld[i].cand) {
      size_t idx = 0;
      while (find_neighbor(pt, lo, del, idx, idx, false)) {
        if (pt.response > lo[idx].response) del[idx] = 1;
        ++idx;
      }
    }
  }
  for (size_t i = 0; i < nl; ++i) S.ld[i].del_upper = S.ld[i].del_lower;
  for (int i = (int)nl - 2; i >= 0; --i) {  // 3. upper level, i descending
    const std::vector<Kp>& cur = S.ld[i].cand;
    std::vector<Kp>& up = S.ld[i + 1].cand;
    uint8_t* del = S.ld[i + 1].del_upper.data();
    for (size_t j = 0; j < cur.size(); ++j) {
      if (S.ld[i].del_upper[j]) continue;
      size_t idx = 0;
      while (find_neighbor(cur[j], up, del, idx, idx, true)) {
        if (cur[j].response > up[idx].response) del[idx] = 1;
        ++idx;
      }
    }
  }
}

// Do_Subpixel_Refinement for one point of a level: false when rejected (|d| > 1); *singular: the 2x2 was singular
bool refine_point(const float* L, int cols, float ratio, Kp& kp, bool* singular) {
  const int x = (int)(kp.x / ratio), y = (int)(kp.y / ratio);
  const float Dx = 0.5f * (L[y * cols + x + 1] - L[y * cols + x - 1]);
  const float Dy = 0.5f * (L[(y + 1) * cols + x] - L[(y - 1) * cols + x]);
  const float Dxx = L[y * cols + x + 1] + L[y * cols + x - 1] - 2.0f * L[y * cols + x];
  const float Dyy = L[(y + 1) * cols + x] + L[(y - 1) * cols + x] - 2.0f * L[y * cols + x];
  const float Dxy = 0.25f * (L[(y + 1) * cols + x + 1] + L[(y - 1) * cols + x - 1] - L[(y - 1) * cols + x + 1] -
                             L[(y + 1) * cols + x - 1]);
  float dst[2];
  solve2(Dxx, Dxy, Dxy, Dyy, -Dx, -Dy, dst);
  *singular = (double)Dxx * Dyy - (double)Dxy * Dxy == 0.0;
  if (std::fabs(dst[0]) > 1.0f || std::fabs(dst[1]) > 1.0f) return false;
  kp.x += dst[0] * ratio;
  kp.y += dst[1] * ratio;
  kp.angle = 0.0f;
  kp.size *= 2.0f;
  return true;
}

void refine(State& S) {
  for (size_t i = 0; i < S.lv.size(); ++i) {
    for (size_t j = 0; j < S.ld[i].cand.size(); ++j) {
      if (S.ld[i].del_upper[j]) continue;
      Kp kp = S.ld[i].cand[j];
      bool singular = false;
      const bool ok = refine_point(S.ld[i].Ldet.data(), S.lv[i].width, S.lv[i].ratio, kp, &singular);
      S.n_singular += singular;
      if (!ok) {
        S.n_rejected++;
        continue;
      }
      S.kps.push_back(kp);
    }
  }
}

// the orientation weights: the normalised 2-D Gaussian exp(-r^2 / 2 sigma^2) / (2 pi sigma^2), sigma = 2.5, at integer
// offsets (0..6, 0..6), rounded to 8 decimals as upstream prints them; upstream evaluated it with pi = 3.14159
void gauss25(float* g) {
  for (int i = 0; i < 7; ++i)
    for (int j = 0; j < 7; ++j)
      g[i * 7 + j] = (float)(std::round(std::exp(-(i * i + j * j) / 12.5) / (2.0 * 3.14159 * 6.25) * 1e8) / 1e8);
}

// Compute_Main_Orientation up to getAngleV2: the winning window's (maxX, maxY)
void orientation_sums(const Kp& kp, const Level& s, const LevelData& d, float* out) {
  float g25[49];
  gauss25(g25);
  const int scale = fround(0.5f * kp.size / s.ratio);
  const int x0 = fround(kp.x / s.ratio), y0 = fround(kp.y / s.ratio);
  const int cols = s.width;
  float resX[109], resY[109], ang[109];
  int k = 0;
  for (int i = -6; i <= 6; ++i)
    for (int j = -6; j <= 6; ++j) {
      if (i * i + j * j >= 36) continue;
      const float wgt = g25[std::abs(i) * 7 + std::abs(j)];
      const size_t p = (size_t)(y0 + i * scale) * cols + (x0 + j * scale);
      resX[k] = wgt * d.Lx[p];
      resY[k] = wgt * d.Ly[p];
      ++k;
    }
  for (int i = 0; i < 109; ++i) ang[i] = fast_atan2(resY[i], resX[i]);
  const int slices = 42, win = 7;
  const float quantum = (float)(2.0 * kPi / slices), amax = (float)(2.0 * kPi);
  const int nkeys = (int)(amax / quantum);
  uint8_t cum[64], idx[109];
  std::memset(cum, 0, nkeys + 1);
  for (int i = 0; i < 109; ++i) cum[(int)(ang[i] / quantum)]++;
  for (int i = 1; i <= nkeys; ++i) cum[i] += cum[i - 1];
  for (int i = 0; i < 109; ++i) idx[--cum[(int)(ang[i] / quantum)]] = (uint8_t)i;
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
  out[0] = maxX;
  out[1] = maxY;
}

// getAngleV2 (libm atan2f into [0, 2 pi)), then Regard3DFeatures::detectKeypoints' conversion to degrees
float regard3d_angle(float maxX, float maxY) {
  float theta = atan2f(maxY, maxX);
  float a = theta >= 0 ? theta : theta + static_cast<float>(2.0f * kPi);
  a *= 180.0 / kPi;
  a += 90.0f;
  while (a < 0) a += 360.0f;
  while (a > 360.0f) a -= 360.0f;
  return a;
}

}  // namespace

extern "C" {

typedef Level orc_akaze_level;
typedef Kp orc_akaze_keypoint;

int orc_akaze_level_table(int w, int h, int omax, int nsub, orc_akaze_level* out, int cap) {
  std::vector<Level> lv = level_table(w, h, omax, nsub);
  for (size_t i = 1; i < lv.size(); ++i) lv[i].n_tau = (uint32_t)fed_tau(lv[i].etime - lv[i - 1].etime, 0.25f).size();
  for (int i = 0; i < (int)lv.size() && i < cap; ++i) out[i] = lv[i];
  return (int)lv.size();
}
int orc_akaze_fed_tau(float T, float tau_max, float* out, int cap) {
  const std::vector<float> t = fed_tau(T, tau_max);
  for (int i = 0; i < (int)t.size() && i < cap; ++i) out[i] = t[i];
  return (int)t.size();
}
void orc_akaze_gaussian_kernel(int n, double sigma, float* k) { gaussian_kernel(n, sigma, k); }
int orc_akaze_deriv_kernels(int dx, int dy, int scale, float* kx, float* ky) { return deriv_kernels(dx, dy, scale, kx, ky); }
void orc_akaze_gaussian_blur(const float* src, int w, int h, float sigma, float* dst) { gaussian_blur(src, w, h, sigma, dst); }
void orc_akaze_scharr(const float* src, int w, int h, int dx, int dy, float* dst) { scharr(src, w, h, dx, dy, dst); }
void orc_akaze_sep_filter(const float* src, int w, int h, const float* kx, int nx, const float* ky, int ny, float* dst) {
  sep_filter(src, w, h, kx, nx, ky, ny, false, dst);
}
void orc_akaze_halfsample(const float* src, int w, int h, float* dst) { halfsample(src, w, h, dst); }
void orc_akaze_fast_atan2(const float* y, const float* x, int n, float* out) {
  for (int i = 0; i < n; ++i) out[i] = fast_atan2(y[i], x[i]);
}
void orc_akaze_solve2(const float* A, const float* b, float* x) { solve2(A[0], A[1], A[2], A[3], b[0], b[1], x); }
float orc_akaze_k_percentile(const float* lx, const float* ly, int w, int h, float perc, int nbins) {
  return k_percentile(lx, ly, w, h, perc, nbins);
}
void orc_akaze_gauss25(float* out) { gauss25(out); }
float orc_akaze_angle(float maxX, float maxY) { return regard3d_angle(maxX, maxY); }

// The whole detector on one float image in [0, 1]: returns an opaque state the getters below read.
void* orc_akaze_detect(const float* img, int w, int h, float threshold, int omax, int nsub) {
  State* S = new State();
  S->W = w;
  S->H = h;
  scale_space(*S, img, omax, nsub);
  extrema(*S, threshold);
  refine(*S);
  S->ori.resize(S->kps.size() * 2);
  for (size_t k = 0; k < S->kps.size(); ++k) {
    Kp& kp = S->kps[k];
    orientation_sums(kp, S->lv[kp.class_id], S->ld[kp.class_id], &S->ori[2 * k]);
    kp.angle = regard3d_angle(S->ori[2 * k], S->ori[2 * k + 1]);
  }
  return S;
}
void orc_akaze_free(void* s) { delete (State*)s; }
int orc_akaze_num_levels(void* s) { return (int)((State*)s)->lv.size(); }
void orc_akaze_get_level(void* s, int i, orc_akaze_level* out) {
  State* S = (State*)s;
  *out = S->lv[i];
  out->n_tau = (uint32_t)S->ld[i].tau.size();
}
float orc_akaze_get_kcontrast(void* s, int i) { return ((State*)s)->ld[i].kcontrast; }
// which: 0 Lt, 1 Lsmooth, 2 Lx, 3 Ly, 4 Ldet
void orc_akaze_get_array(void* s, int i, int which, float* out) {
  const LevelData& d = ((State*)s)->ld[i];
  const Img* a[5] = {&d.Lt, &d.Lsmooth, &d.Lx, &d.Ly, &d.Ldet};
  std::memcpy(out, a[which]->data(), a[which]->size() * 4);
}
int orc_akaze_num_candidates(void* s, int i) { return (int)((State*)s)->ld[i].cand.size(); }
void orc_akaze_get_candidates(void* s, int i, orc_akaze_keypoint* out, uint8_t* del_lower, uint8_t* del_upper) {
  const LevelData& d = ((State*)s)->ld[i];
  std::memcpy(out, d.cand.data(), d.cand.size() * sizeof(Kp));
  std::memcpy(del_lower, d.del_lower.data(), d.cand.size());
  std::memcpy(del_upper, d.del_upper.data(), d.cand.size());
}
// refinement alone on given points of one level's Ldet (w columns); a rejected point gets class_id -1
void orc_akaze_refine(const float* ldet, int w, float ratio, const orc_akaze_keypoint* in, int n, orc_akaze_keypoint* out) {
  for (int i = 0; i < n; ++i) {
    Kp kp = in[i];
    bool singular = false;
    if (!refine_point(ldet, w, ratio, kp, &singular)) kp = in[i], kp.class_id = -1;
    out[i] = kp;
  }
}
void orc_akaze_get_stats(void* s, int* out) {
  const State* S = (const State*)s;
  out[0] = S->n_replaced, out[1] = S->n_singular, out[2] = S->n_rejected;
}
int orc_akaze_num_keypoints(void* s) { return (int)((State*)s)->kps.size(); }
void orc_akaze_get_keypoints(void* s, orc_akaze_keypoint* out, float* ori) {
  State* S = (State*)s;
  std::memcpy(out, S->kps.data(), S->kps.size() * sizeof(Kp));
  if (ori) std::memcpy(ori, S->ori.data(), S->ori.size() * 4);
}

}  // extern "C"
