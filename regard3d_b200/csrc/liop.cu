// liop.cu -- LIOP-144 descriptors of a view's keypoints on the device (SURVEY.md 8f-1).
// COMPILED WITH --fmad=false (regard3d_b200/build.py): the float / double arithmetic below must round like the
// reference's host code (bilinear samples, Gaussian taps, neighbour interpolation), one operation at a time.
//
// Replaces Regard3DFeatures::extractLIOPFeatures (src/Regard3DFeatures.cpp:719-861), per keypoint:
//   M      2x3 inverse affine map from (x, y, size, angle)                       :766-800   (host: libm cos/sin)
//   warp   cv::warpAffine(img, patch 41x41, M, INTER_LINEAR | WARP_INVERSE_MAP)  :803       k_liop: stage 1
//   blur   cv::GaussianBlur(patch, sigma 1.2)  (11 taps, BORDER_REFLECT_101)     :807       k_liop: stage 2
//   desc   r3d_vl_liopdesc_process (src/thirdparty/liop/vl_liop.c:434-575)       :828       k_liop: stages 3-5
// One CTA per keypoint of a whole batch of images: a by-value table (Slots) holds each image's pointer and shape and
// the range of keypoints that sample it; r3d_liop_describe launches it with one slot.  The descriptor is order based: 673 disc pixels ranked by intensity with the reference's own
// quick sort (vl_qsort-def.h:123-162 -- the order of EQUAL intensities is a property of that exact procedure, and
// equal intensities are common in flat image regions), six rank bins, per pixel the order pattern of 4 neighbours
// sampled on a radius-6 circle, weighted by the number of neighbour pairs that differ by more than 5/255 of the
// patch's intensity range.  The sort is therefore replayed sequentially by one thread (on packed key|index words in
// shared memory); everything around it is data parallel.
#include "r3d_internal.cuh"

#include <cmath>

namespace r3d {
namespace liop {

constexpr int kSide = 41, kPix = kSide * kSide;
constexpr int kNeigh = 4, kSpatialBins = 6;
constexpr int kMaxDisc = 704;          // >= number of disc pixels (673 for a 41x41 patch, radius 6)
constexpr int kThreads = 128;

struct Tables {                        // r3d_vl_liopdesc_new (vl_liop.c:318-394), built once on the host (libm)
  uint32_t n_disc;
  uint16_t pixels[kMaxDisc];
  double sx[kMaxDisc * kNeigh], sy[kMaxDisc * kNeigh];
};

// cv::getGaussianKernel(11, 1.2, CV_32F) of OpenCV 4.x (bit-exact kernel, rounded to float)
__constant__ float c_gauss[11] = {0x1.d9b2eep-15f, 0x1.50eab6p-10f, 0x1.dea402p-7f, 0x1.538cacp-4f, 0x1.e1217cp-3f, 0x1.546e7ep-2f,
                                  0x1.e1217cp-3f,  0x1.538cacp-4f,  0x1.dea402p-7f, 0x1.50eab6p-10f, 0x1.d9b2eep-15f};

__device__ __forceinline__ int reflect101(int p, int len) {
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}
__device__ __forceinline__ long long floor_d(double x) {  // vl_floor_d
  const long long xi = (long long)x;
  return (x >= 0 || (double)xi == x) ? xi : xi - 1;
}

__global__ void __launch_bounds__(kThreads) k_liop(Slots S, const float* __restrict__ Ms, uint32_t n,
                                                   const Tables* __restrict__ T, float* __restrict__ desc_out) {
  __shared__ float s_a[kPix], s_b[kPix];
  __shared__ unsigned long long s_sort[kMaxDisc];  // (intensity bits << 32) | disc index: swapped as one word
  __shared__ uint16_t s_rank_of[kMaxDisc];         // sorted position -> disc index
  __shared__ float s_desc[kDim];
  __shared__ int2 s_stack[64];
  __shared__ float s_thr, s_norm;
  const uint32_t kp = blockIdx.x;
  if (kp >= n) return;
  int slot = 0;
  while (slot + 1 < S.n && kp >= S.first[slot + 1]) ++slot;
  const float* __restrict__ img = S.img[slot];
  const int w = S.w[slot], h = S.h[slot];
  const int tid = threadIdx.x;
  const bool raw_patches = Ms == nullptr;  // diagnostics: img holds n ready 41x41 patches (stages 1-2 skipped)
  if (raw_patches) {
    for (int p = tid; p < kPix; p += kThreads) s_a[p] = img[(size_t)kp * kPix + p];
  }
  if (!raw_patches)
  // ---- 1. warpAffine: 1/32-pixel fixed-point source coordinates, float bilinear weights (imgwarp.cpp) ----
  {
    double M[6];
    for (int i = 0; i < 6; ++i) M[i] = (double)Ms[6 * (size_t)kp + i];
    const int AB_BITS = 10, AB_SCALE = 1 << AB_BITS, INTER_BITS = 5, INTER_TAB_SIZE = 1 << INTER_BITS;
    const int round_delta = AB_SCALE / INTER_TAB_SIZE / 2;
    for (int p = tid; p < kPix; p += kThreads) {
      const int dy = p / kSide, dx = p % kSide;
      const int X0 = __double2int_rn((M[1] * dy + M[2]) * AB_SCALE) + round_delta;  // saturate_cast<int> = cvRound
      const int Y0 = __double2int_rn((M[4] * dy + M[5]) * AB_SCALE) + round_delta;
      const int adelta = __double2int_rn(M[0] * dx * AB_SCALE), bdelta = __double2int_rn(M[3] * dx * AB_SCALE);
      const int X = (X0 + adelta) >> (AB_BITS - INTER_BITS), Y = (Y0 + bdelta) >> (AB_BITS - INTER_BITS);
      int sx = X >> INTER_BITS, sy = Y >> INTER_BITS;
      sx = max(-32768, min(32767, sx));
      sy = max(-32768, min(32767, sy));
      const float fx = (float)(X & (INTER_TAB_SIZE - 1)) * (1.f / INTER_TAB_SIZE);
      const float fy = (float)(Y & (INTER_TAB_SIZE - 1)) * (1.f / INTER_TAB_SIZE);
      const float vx0 = 1.f - fx, vy0 = 1.f - fy;
      const float w0 = vy0 * vx0, w1 = vy0 * fx, w2 = fy * vx0, w3 = fy * fx;
      float v = 0.f;
      if (!(sx >= w || sx + 1 < 0 || sy >= h || sy + 1 < 0)) {
        const bool x0 = sx >= 0 && sx < w, x1 = sx + 1 >= 0 && sx + 1 < w, y0 = sy >= 0 && sy < h, y1 = sy + 1 >= 0 && sy + 1 < h;
        const float v0 = (x0 && y0) ? img[(size_t)sy * w + sx] : 0.f;
        const float v1 = (x1 && y0) ? img[(size_t)sy * w + sx + 1] : 0.f;
        const float v2 = (x0 && y1) ? img[(size_t)(sy + 1) * w + sx] : 0.f;
        const float v3 = (x1 && y1) ? img[(size_t)(sy + 1) * w + sx + 1] : 0.f;
        v = v0 * w0 + v1 * w1 + v2 * w2 + v3 * w3;
      }
      s_a[p] = v;
    }
  }
  __syncthreads();
  // ---- 2. GaussianBlur sigma 1.2: rows tap by tap, columns in the symmetric form (filter.cpp) ----
  if (!raw_patches)
  for (int p = tid; p < kPix; p += kThreads) {
    const int y = p / kSide, x = p % kSide;
    float s = s_a[y * kSide + reflect101(x - 5, kSide)] * c_gauss[0];
    for (int k = 1; k < 11; ++k) s = s + s_a[y * kSide + reflect101(x - 5 + k, kSide)] * c_gauss[k];
    s_b[p] = s;
  }
  __syncthreads();
  if (!raw_patches)
  for (int p = tid; p < kPix; p += kThreads) {
    const int y = p / kSide, x = p % kSide;
    float s = c_gauss[5] * s_b[p];
    for (int k = 1; k <= 5; ++k) s = s + c_gauss[5 + k] * (s_b[reflect101(y + k, kSide) * kSide + x] + s_b[reflect101(y - k, kSide) * kSide + x]);
    s_a[p] = s;  // the patch
  }
  for (int i = tid; i < kDim; i += kThreads) s_desc[i] = 0.f;
  __syncthreads();
  // ---- 3. rank the disc pixels by intensity: the reference's quick sort, replayed by one thread ----
  const int nd = (int)T->n_disc;
  for (int i = tid; i < nd; i += kThreads)
    s_sort[i] = ((unsigned long long)__float_as_uint(s_a[T->pixels[i]]) << 32) | (unsigned)i;
  __syncthreads();
  if (tid == 0) {
    int sp = 0;
    s_stack[sp++] = make_int2(0, nd - 1);
    while (sp > 0) {
      const int2 seg = s_stack[--sp];
      int begin = seg.x, end = seg.y;
      // the two sub-ranges of a partition are independent: the larger one is pushed, the smaller one processed next
      // (stack depth <= log2 n); the result does not depend on the processing order
      for (;;) {
        int pivot = (end + begin) / 2;
        { const unsigned long long t = s_sort[pivot]; s_sort[pivot] = s_sort[end]; s_sort[end] = t; }
        const float pk = __uint_as_float((unsigned)(s_sort[end] >> 32));
        int low = begin;
        for (int i = begin; i < end; ++i) {
          const unsigned long long e = s_sort[i];
          if (__uint_as_float((unsigned)(e >> 32)) - pk <= 0) {  // patch_cmp(...) <= 0
            s_sort[i] = s_sort[low];
            s_sort[low] = e;
            ++low;
          }
        }
        { const unsigned long long t = s_sort[low]; s_sort[low] = s_sort[end]; s_sort[end] = t; }
        pivot = low;
        const bool hasL = pivot > begin, hasR = pivot < end;
        const int lb = begin, le = pivot - 1, rb = pivot + 1, re = end;
        if (hasL && hasR) {
          if (le - lb > re - rb) { s_stack[sp++] = make_int2(lb, le); begin = rb; end = re; }
          else { s_stack[sp++] = make_int2(rb, re); begin = lb; end = le; }
        } else if (hasL) { begin = lb; end = le; }
        else if (hasR) { begin = rb; end = re; }
        else break;
        if (begin >= end) break;  // a one-element range: its partition is the identity
      }
    }
    const float lo = __uint_as_float((unsigned)(s_sort[0] >> 32)), hi = __uint_as_float((unsigned)(s_sort[nd - 1] >> 32));
    s_thr = (float)(5.0 / 255) * (hi - lo);  // threshold = -intensityThreshold * (max - min), intensityThreshold = -(5.0/255)
  }
  __syncthreads();
  for (int i = tid; i < nd; i += kThreads) s_rank_of[i] = (uint16_t)(s_sort[i] & 0xffffu);
  __syncthreads();
  // ---- 4. per ranked pixel: 4 neighbours (double bilinear), their order pattern, the weight ----
  const float threshold = s_thr;
  const int binArea = nd / kSpatialBins;
  for (int i = tid; i < nd; i += kThreads) {
    int bin = i / binArea;
    if (bin > kSpatialBins - 1) bin = kSpatialBins - 1;
    const int disc = s_rank_of[i];
    float nI[kNeigh];
    int nP[kNeigh];
    for (int t = 0; t < kNeigh; ++t) {
      const double x = T->sx[kNeigh * disc + t], y = T->sy[kNeigh * disc + t];
      const long long ix = floor_d(x), iy = floor_d(y);
      const double wx = x - (double)ix, wy = y - (double)iy;
      double a = 0, b = 0, c = 0, d = 0;
      const int L = kSide;
      if (ix >= 0 && iy >= 0) a = (double)s_a[ix + iy * L];
      if (ix < L - 1 && iy >= 0) b = (double)s_a[ix + 1 + iy * L];
      if (ix >= 0 && iy < L - 1) c = (double)s_a[ix + (iy + 1) * L];
      if (ix < L - 1 && iy < L - 1) d = (double)s_a[ix + 1 + (iy + 1) * L];
      nP[t] = t;
      nI[t] = (float)((1.0 - wy) * (a + (b - a) * wx) + wy * (c + (d - c) * wx));
    }
    // neigh_sort: the same quick sort on 4 elements (explicit little stack)
    {
      int stb[4], ste[4], sp = 0;
      stb[0] = 0; ste[0] = kNeigh - 1; sp = 1;
      while (sp > 0) {
        --sp;
        const int begin = stb[sp], end = ste[sp];
        int pivot = (end + begin) / 2;
        { const int t = nP[pivot]; nP[pivot] = nP[end]; nP[end] = t; }
        const float pk = nI[nP[end]];
        int low = begin;
        for (int q = begin; q < end; ++q)
          if (nI[nP[q]] - pk <= 0) { const int t = nP[low]; nP[low] = nP[q]; nP[q] = t; ++low; }
        { const int t = nP[low]; nP[low] = nP[end]; nP[end] = t; }
        pivot = low;
        if (pivot > begin) { stb[sp] = begin; ste[sp] = pivot - 1; ++sp; }
        if (pivot < end) { stb[sp] = pivot + 1; ste[sp] = end; ++sp; }
      }
    }
    int permIndex = 0;  // get_permutation_index
    for (int a = 0; a < kNeigh; ++a) {
      permIndex = permIndex * (kNeigh - a) + nP[a];
      for (int b = a + 1; b < kNeigh; ++b)
        if (nP[b] > nP[a]) nP[b]--;
    }
    float weight = 0.f;
    for (int k = 0; k < kNeigh; ++k)
      for (int t = k + 1; t < kNeigh; ++t) {
        const float a = nI[k], b = nI[t];
        weight += (a > b + threshold || b > a + threshold) ? 1.f : 0.f;
      }
    if (weight != 0.f) atomicAdd(&s_desc[permIndex + 24 * bin], weight);  // small integers: exact in any order
  }
  __syncthreads();
  // ---- 5. L2 normalisation: float accumulation in index order, double sqrt stored back to float ----
  if (tid == 0) {
    float norm = 0.f;
    for (int i = 0; i < kDim; ++i) norm += s_desc[i] * s_desc[i];
    const double r = sqrt((double)norm);
    s_norm = (float)(r > 1e-12 ? r : 1e-12);
  }
  __syncthreads();
  for (int i = tid; i < kDim; i += kThreads) desc_out[(size_t)kp * kDim + i] = s_desc[i] / s_norm;
}

static const Tables& host_tables() {
  static Tables* T = [] {
    Tables* t = new Tables();
    const long center = (kSide - 1) / 2;
    const float radius = 6.0f;                       // DEFAULT_RADIUS
    const double tt = center - radius + 0.6;
    const long t2 = (long)(tt * tt);
    uint32_t n = 0;
    for (long y = 0; y < kSide; ++y)
      for (long x = 0; x < kSide; ++x) {
        const long dx = x - center, dy = y - center;
        if (x == 0 && y == 0) continue;
        if (dx * dx + dy * dy <= t2 && n < (uint32_t)kMaxDisc) t->pixels[n++] = (uint16_t)(x + y * kSide);
      }
    t->n_disc = n;
    for (uint32_t i = 0; i < n; ++i) {
      const double dangle = 2 * M_PI / (double)kNeigh;
      const long pixel = t->pixels[i];
      const double x = (double)((pixel % kSide) - center), y = (double)((pixel / kSide) - center);
      const double angle0 = atan2(y, x);
      for (int k = 0; k < kNeigh; ++k) {
        t->sx[k + kNeigh * i] = x + radius * cos(angle0 + dangle * k) + center;
        t->sy[k + kNeigh * i] = y + radius * sin(angle0 + dangle * k) + center;
      }
    }
    return t;
  }();
  return *T;
}

// The 2x3 inverse map of src/Regard3DFeatures.cpp:766-800 (float arithmetic; cos / sin in double by the host's libm,
// exactly what the reference's host code evaluates)
void affine_of(float x, float y, float kp_size, float kp_angle, float factor, float* M) {
  const float angle = -90.0f - kp_angle;
  const float scale = kp_size / (float)kSide * factor;
  const float alpha = (float)(scale * std::cos(angle * M_PI / 180.0f));
  const float beta = (float)(scale * std::sin(angle * M_PI / 180.0f));
  const float trans_x = x - 20.0f, trans_y = y - 20.0f;
  M[0] = alpha;
  M[1] = beta;
  M[2] = beta * trans_y + alpha * trans_x - beta * y + (1.0f - alpha) * x;
  M[3] = -beta;
  M[4] = alpha;
  M[5] = alpha * trans_y - beta * trans_x + beta * x + (1.0f - alpha) * y;
}

Tables* tables_to_device(DeviceWorker& w, cudaStream_t st) {
  Tables* d = (Tables*)pool_alloc(w, sizeof(Tables));
  if (d && cudaMemcpyAsync(d, &host_tables(), sizeof(Tables), cudaMemcpyHostToDevice, st) != cudaSuccess) {
    pool_release(w, d);
    return nullptr;
  }
  return d;
}

int describe(r3d_ctx* ctx, cudaStream_t st, const Slots& S, const float* d_M, uint32_t n, const Tables* d_T,
             float* d_desc) {
  if (n == 0) return R3D_OK;
  k_liop<<<n, kThreads, 0, st>>>(S, d_M, n, d_T, d_desc);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

}  // namespace liop
}  // namespace r3d

using namespace r3d;

extern "C" int r3d_liop_describe(r3d_ctx* ctx, const float* image, uint32_t width, uint32_t height, const r3d_keypoint* kps,
                                 uint32_t n, float kp_size_factor, float* desc_out) {
  if (!ctx || (n && (!image || !kps || !desc_out)) || width == 0 || height == 0 || width > 32767 || height > 32767)
    return fail(ctx, R3D_ERR_INVALID, "r3d_liop_describe: bad arguments");
  if (n == 0) return R3D_OK;
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  const liop::Tables& T = liop::host_tables();
  std::vector<float> hM((size_t)n * 6);
  parallel_for(ctx->host_threads, (n + 1023) / 1024, [&](size_t blk) {
    const uint32_t i1 = (uint32_t)std::min<size_t>((blk + 1) * 1024, n);
    for (uint32_t i = (uint32_t)(blk * 1024); i < i1; ++i)
      liop::affine_of(kps[i].x, kps[i].y, kps[i].size, kps[i].angle, kp_size_factor, &hM[(size_t)i * 6]);
  });
  struct Guard {
    DeviceWorker* w;
    std::vector<void*> p;
    ~Guard() { cudaStreamSynchronize(w->stream); for (void* q : p) pool_release(*w, q); }
  } g{&w, {}};
  auto alloc = [&](size_t bytes) -> void* { void* q = pool_alloc(w, bytes); if (q) g.p.push_back(q); return q; };
  float* d_img = (float*)alloc((size_t)width * height * 4);
  float* d_M = (float*)alloc((size_t)n * 6 * 4);
  float* d_desc = (float*)alloc((size_t)n * liop::kDim * 4);
  liop::Tables* d_T = (liop::Tables*)alloc(sizeof(liop::Tables));
  if (!d_img || !d_M || !d_desc || !d_T) return fail(ctx, R3D_ERR_NOMEM, "r3d_liop_describe: device allocation failed");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_img, image, (size_t)width * height * 4, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_M, hM.data(), hM.size() * 4, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_T, &T, sizeof(liop::Tables), cudaMemcpyHostToDevice, w.stream));
  liop::Slots S{};
  S.img[0] = d_img, S.w[0] = (int)width, S.h[0] = (int)height, S.first[1] = n, S.n = 1;
  int rc = liop::describe(ctx, w.stream, S, d_M, n, d_T, d_desc);
  if (rc) return rc;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(desc_out, d_desc, (size_t)n * liop::kDim * 4, cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  return R3D_OK;
}

// Diagnostics: r3d_vl_liopdesc_process alone on n ready 41x41 float patches (the unit the compiled reference pins)
extern "C" int r3d_debug_liop_process(r3d_ctx* ctx, const float* patches, uint32_t n, float* desc_out) {
  if (!ctx || (n && (!patches || !desc_out))) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_liop_process: bad arguments");
  if (n == 0) return R3D_OK;
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  const liop::Tables& T = liop::host_tables();
  struct Guard {
    DeviceWorker* w;
    std::vector<void*> p;
    ~Guard() { cudaStreamSynchronize(w->stream); for (void* q : p) pool_release(*w, q); }
  } g{&w, {}};
  auto alloc = [&](size_t bytes) -> void* { void* q = pool_alloc(w, bytes); if (q) g.p.push_back(q); return q; };
  float* d_p = (float*)alloc((size_t)n * liop::kPix * 4);
  float* d_desc = (float*)alloc((size_t)n * liop::kDim * 4);
  liop::Tables* d_T = (liop::Tables*)alloc(sizeof(liop::Tables));
  if (!d_p || !d_desc || !d_T) return fail(ctx, R3D_ERR_NOMEM, "r3d_debug_liop_process: device allocation failed");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_p, patches, (size_t)n * liop::kPix * 4, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_T, &T, sizeof(liop::Tables), cudaMemcpyHostToDevice, w.stream));
  liop::Slots S{};
  S.img[0] = d_p, S.w[0] = liop::kSide, S.h[0] = liop::kSide, S.first[1] = n, S.n = 1;
  int rc = liop::describe(ctx, w.stream, S, nullptr, n, d_T, d_desc);
  if (rc) return rc;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(desc_out, d_desc, (size_t)n * liop::kDim * 4, cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  return R3D_OK;
}
