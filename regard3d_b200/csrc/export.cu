// export.cu -- what follows the SfM engine (DESIGN.md 4.5i):
//   r3d_sfm_colorize_plan        OpenMVGHelper::ColorizeTracks' greedy loop as one cooperative kernel: per round a
//                                per-view count of the remaining landmarks' observations, a first-max argmax, then the
//                                chosen view's landmarks are marked and compacted out
//   r3d_sfm_write_colorized_ply  plyHelper::exportToPly with colours (host)
//   r3d_undistort_images         OpenMVG 1.4 UndistortImage with black fill, the first step of every densification export
// Built without FMA contraction and with detmath's atan: every output byte is a pure function of the inputs, and the
// CPU restatement (oracle/oracle_export.cpp) reproduces it.
#include "r3d_internal.cuh"
#include "r3d_sfm.h"
#include "detmath.cuh"

#include <cooperative_groups.h>

#include <cstdio>
#include <cstring>

namespace cg = cooperative_groups;

namespace r3d {
namespace exk {

constexpr int kPlanThreads = 256;
constexpr uint32_t kSmemViews = 11776;  // per-CTA histogram in shared memory up to this many views (46 KB + 2 KB static)

struct PlanState {
  uint32_t next_m;   // landmarks left after the current round
  uint32_t chosen;   // view index of the current round
  uint32_t rounds;
};

// One persistent cooperative grid runs every round; three grid barriers per round, no host round trip.
// obs_vi / obs_pix: view index and truncated (x, y) per observation, landmark l's observations in
// [obs_ofs[l], obs_ofs[l + 1]) in view order.  remA / remB: the remaining landmarks, compacted each round (their order
// does not matter: counts are sums and every landmark is decided on its own).
__global__ void __launch_bounds__(kPlanThreads) k_colorize_plan(
    uint32_t n_lm, uint32_t n_views, const uint64_t* __restrict__ obs_ofs, const uint32_t* __restrict__ obs_vi,
    const int2* __restrict__ obs_pix, uint32_t* remA, uint32_t* remB, uint32_t* counts, PlanState* st,
    uint32_t* __restrict__ round_view, uint32_t* __restrict__ lm_round, int2* __restrict__ lm_pixel) {
  extern __shared__ uint32_t hist[];
  __shared__ uint32_t red_c[kPlanThreads], red_v[kPlanThreads];
  cg::grid_group grid = cg::this_grid();
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  const bool smem_hist = n_views <= kSmemViews;
  for (uint32_t l = gtid; l < n_lm; l += gsz) remA[l] = l;
  for (uint32_t v = gtid; v < n_views; v += gsz) counts[v] = 0u;
  grid.sync();
  uint32_t m = n_lm, r = 0;
  uint32_t *rem = remA, *nxt = remB;
  while (m > 0) {
    // a. observations per view of the remaining landmarks
    if (smem_hist) {
      for (uint32_t v = threadIdx.x; v < n_views; v += blockDim.x) hist[v] = 0u;
      __syncthreads();
    }
    for (uint32_t i = gtid; i < m; i += gsz) {
      const uint32_t l = rem[i];
      for (uint64_t o = obs_ofs[l]; o < obs_ofs[l + 1]; ++o) atomicAdd(smem_hist ? &hist[obs_vi[o]] : &counts[obs_vi[o]], 1u);
    }
    if (smem_hist) {
      __syncthreads();
      for (uint32_t v = threadIdx.x; v < n_views; v += blockDim.x)
        if (hist[v]) atomicAdd(&counts[v], hist[v]);
    }
    grid.sync();
    // b. the first view in index (= id) order with the largest count
    if (blockIdx.x == 0) {
      uint32_t bc = 0u, bv = 0xffffffffu;
      for (uint32_t v = threadIdx.x; v < n_views; v += blockDim.x) {
        const uint32_t c = counts[v];
        if (c > bc) { bc = c; bv = v; }  // v ascends per thread: a tie keeps the earlier view
      }
      red_c[threadIdx.x] = bc;
      red_v[threadIdx.x] = bv;
      __syncthreads();
      for (int s = kPlanThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
          const uint32_t c = red_c[threadIdx.x + s], v = red_v[threadIdx.x + s];
          if (c > red_c[threadIdx.x] || (c == red_c[threadIdx.x] && v < red_v[threadIdx.x])) {
            red_c[threadIdx.x] = c;
            red_v[threadIdx.x] = v;
          }
        }
        __syncthreads();
      }
      if (threadIdx.x == 0) {
        st->chosen = red_v[0];
        st->next_m = 0u;
        round_view[r] = red_v[0];
      }
    }
    grid.sync();
    // c. colour the chosen view's landmarks, keep the others for the next round
    const uint32_t chosen = *(volatile uint32_t*)&st->chosen;
    for (uint32_t v = gtid; v < n_views; v += gsz) counts[v] = 0u;
    for (uint32_t i = gtid; i < m; i += gsz) {
      const uint32_t l = rem[i];
      bool hit = false;
      for (uint64_t o = obs_ofs[l]; o < obs_ofs[l + 1]; ++o) {
        if (obs_vi[o] == chosen) {
          lm_round[l] = r;
          lm_pixel[l] = obs_pix[o];
          hit = true;
          break;
        }
      }
      if (!hit) nxt[atomicAdd(&st->next_m, 1u)] = l;
    }
    grid.sync();
    m = *(volatile uint32_t*)&st->next_m;
    uint32_t* t = rem;
    rem = nxt;
    nxt = t;
    ++r;
  }
  if (gtid == 0) st->rounds = r;
}

// ---- undistortion -------------------------------------------------------------------------------------------------
constexpr int kRun = 4;             // output pixels per thread, consecutive in raster order
constexpr int kUndistThreads = 256;

struct Cam {
  int model;
  double f, ppx, ppy, d[5];
};

// cam->get_d_pixel((i, j)) = cam2ima(add_disto(ima2cam(p))), OpenMVG 1.4's operation order per model
__device__ __forceinline__ void d_pixel(const Cam& c, double i, double j, double* dx, double* dy) {
  const double x = (i - c.ppx) / c.f, y = (j - c.ppy) / c.f;
  double xd, yd;
  if (c.model == R3D_CAM_PINHOLE_FISHEYE) {
    const double r = sqrt(x * x + y * y);
    const double th = dm::atan_pos(r);
    const double th2 = th * th, th3 = th2 * th, th4 = th2 * th2, th5 = th4 * th, th7 = th3 * th3 * th, th8 = th4 * th4,
                 th9 = th8 * th;
    const double thd = th + c.d[0] * th3 + c.d[1] * th5 + c.d[2] * th7 + c.d[3] * th9;
    const double inv_r = r > 1e-8 ? 1.0 / r : 1.0;
    const double cd = r > 1e-8 ? thd * inv_r : 1.0;
    xd = x * cd;
    yd = y * cd;
  } else if (c.model == R3D_CAM_PINHOLE_BROWN) {
    const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
    const double kd = c.d[0] * r2 + c.d[1] * r4 + c.d[2] * r6;
    const double tx = c.d[4] * (r2 + 2.0 * x * x) + 2.0 * c.d[3] * x * y;
    const double ty = c.d[3] * (r2 + 2.0 * y * y) + 2.0 * c.d[4] * x * y;
    xd = x + (x * kd + tx);
    yd = y + (y * kd + ty);
  } else if (c.model == R3D_CAM_PINHOLE_RADIAL3) {
    const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
    const double rc = 1.0 + c.d[0] * r2 + c.d[1] * r4 + c.d[2] * r6;
    xd = x * rc;
    yd = y * rc;
  } else {  // radial K1
    const double rc = 1.0 + c.d[0] * (x * x + y * y);
    xd = x * rc;
    yd = y * rc;
  }
  *dx = c.f * xd + c.ppx;
  *dy = c.f * yd + c.ppy;
}

// one output pixel: black unless Contains((int)dy, (int)dx), then the bilinear sample at ((float)dy, (float)dx)
__device__ __forceinline__ uint32_t undistort_px(const Cam& c, const uint8_t* __restrict__ in, int w, int h, int i, int j) {
  double dx, dy;
  d_pixel(c, (double)i, (double)j, &dx, &dy);
  // (int)d in [0, w) <=> -1 < d < w; NaN fails both
  if (!(dx > -1.0 && dx < (double)w && dy > -1.0 && dy < (double)h)) return 0u;
  const float fx = (float)dx, fy = (float)dy;
  const float flx = floorf(fx), fly = floorf(fy);
  const float ax = fx - flx, ay = fy - fly;
  const float cx[2] = {1.0f - ax, ax}, cy[2] = {1.0f - ay, ay};
  const int gx = (int)flx, gy = (int)fly;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, tw = 0.0;
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const int yy = gy + a;
    if (yy < 0 || yy >= h) continue;
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int xx = gx + b;
      if (xx < 0 || xx >= w) continue;
      const float wt = cx[b] * cy[a];
      const uint8_t* p = in + 3 * ((size_t)yy * (size_t)w + (size_t)xx);
      const double wd = (double)wt;
      s0 = s0 + (double)p[0] * wd;
      s1 = s1 + (double)p[1] * wd;
      s2 = s2 + (double)p[2] * wd;
      tw = tw + wd;
    }
  }
  if (tw <= 0.2) return 0u;
  if (tw != 1.0) {
    s0 = s0 / tw;
    s1 = s1 / tw;
    s2 = s2 / tw;
  }
  const uint32_t r0 = (uint32_t)fmin(fmax(s0, 0.0), 255.0), r1 = (uint32_t)fmin(fmax(s1, 0.0), 255.0),
                 r2 = (uint32_t)fmin(fmax(s2, 0.0), 255.0);
  return r0 | (r1 << 8) | (r2 << 16);
}

// kRun consecutive output pixels per thread (raster order across rows), written as three 32-bit words when whole
__global__ void __launch_bounds__(kUndistThreads) k_undistort(Cam c, const uint8_t* __restrict__ in, int w, int h,
                                                              uint8_t* __restrict__ out) {
  const uint64_t npx = (uint64_t)w * (uint64_t)h;
  const uint64_t p0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * kRun;
  if (p0 >= npx) return;
  int j = (int)(p0 / (uint64_t)w), i = (int)(p0 - (uint64_t)j * (uint64_t)w);
  uint32_t px[kRun];
#pragma unroll
  for (int k = 0; k < kRun; ++k) {
    px[k] = (p0 + k < npx) ? undistort_px(c, in, w, h, i, j) : 0u;
    if (++i == w) { i = 0; ++j; }
  }
  uint8_t* o = out + 3 * p0;
  if (p0 + kRun <= npx) {  // 12 bytes at a multiple of 12 from a 256-byte aligned base: 4-byte aligned
    uint32_t* o4 = (uint32_t*)o;
    o4[0] = px[0] | (px[1] << 24);
    o4[1] = (px[1] >> 8) | (px[2] << 16);
    o4[2] = (px[2] >> 16) | (px[3] << 8);
  } else {
    for (uint64_t k = 0; p0 + k < npx; ++k) {
      o[3 * k] = (uint8_t)px[k];
      o[3 * k + 1] = (uint8_t)(px[k] >> 8);
      o[3 * k + 2] = (uint8_t)(px[k] >> 16);
    }
  }
}

}  // namespace exk
}  // namespace r3d

using namespace r3d;

extern "C" int r3d_sfm_colorize_plan(r3d_ctx* ctx, const r3d_sfm_data* sd, uint32_t* round_view, uint32_t* n_rounds,
                                     uint32_t* lm_round, int32_t* lm_pixel) try {
  if (!ctx || !sd || !round_view || !n_rounds || (!sd->structure.empty() && (!lm_round || !lm_pixel)))
    return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_colorize_plan: bad arguments");
  *n_rounds = 0;
  r3d_sfm::Flat F;
  int rc = r3d_sfm::flatten(*sd, /*skip_undefined=*/false, F);
  if (rc == R3D_ERR_INVALID) return fail(ctx, rc, "r3d_sfm_colorize_plan: an observation of a view without a pose or intrinsic");
  if (rc) return fail(ctx, rc, "r3d_sfm_colorize_plan: a pose is shared by views with different intrinsics");
  const uint32_t n_lm = (uint32_t)F.lm_ids.size(), n_views = (uint32_t)sd->views.size();
  const size_t n_obs = F.obs_view.size();
  if (n_obs > 0xffffffffull) return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_sfm_colorize_plan: more than 2^32 observations");
  // view index and truncated pixel per observation; the inputs upstream leaves undefined are refused here
  std::map<uint32_t, uint32_t> vidx;
  std::vector<uint32_t> vw, vh;
  for (const auto& kv : sd->views) {
    vidx.emplace(kv.first, (uint32_t)vidx.size());
    vw.push_back(kv.second.width);
    vh.push_back(kv.second.height);
  }
  std::vector<uint32_t> obs_vi(n_obs);
  std::vector<int2> obs_pix(n_obs);
  for (uint32_t l = 0; l < n_lm; ++l) {
    if (F.obs_ofs[l + 1] == F.obs_ofs[l])
      return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_colorize_plan: landmark " + std::to_string(F.lm_ids[l]) + " has no observation");
    for (uint64_t o = F.obs_ofs[l]; o < F.obs_ofs[l + 1]; ++o) {
      const uint32_t vi = vidx.at(F.obs_view[o]);
      const double x = F.obs_xy[2 * o], y = F.obs_xy[2 * o + 1];
      if (!(x > -1.0 && x < (double)vw[vi] && y > -1.0 && y < (double)vh[vi]))
        return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_colorize_plan: landmark " + std::to_string(F.lm_ids[l]) +
                                              " is observed outside view " + std::to_string(F.obs_view[o]));
      obs_vi[o] = vi;
      obs_pix[o] = make_int2((int)x, (int)y);
    }
  }
  if (n_lm == 0) return R3D_OK;
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  DevArr<uint64_t> d_ofs(w);
  DevArr<uint32_t> d_vi(w), d_remA(w), d_remB(w), d_counts(w), d_round_view(w), d_lm_round(w);
  DevArr<int2> d_pix(w), d_lm_pixel(w);
  DevArr<exk::PlanState> d_st(w);
  if (!d_ofs.alloc(n_lm + 1) || !d_vi.alloc(n_obs) || !d_pix.alloc(n_obs) || !d_remA.alloc(n_lm) || !d_remB.alloc(n_lm) ||
      !d_counts.alloc(n_views) || !d_round_view.alloc(n_views) || !d_lm_round.alloc(n_lm) || !d_lm_pixel.alloc(n_lm) ||
      !d_st.alloc(1))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_sfm_colorize_plan: device allocation failed");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ofs.p, F.obs_ofs.data(), (n_lm + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_vi.p, obs_vi.data(), n_obs * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_pix.p, obs_pix.data(), n_obs * sizeof(int2), cudaMemcpyHostToDevice, w.stream));
  const size_t smem = n_views <= exk::kSmemViews ? n_views * sizeof(uint32_t) : 0;
  int per_sm = 0;
  R3D_CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, exk::k_colorize_plan, exk::kPlanThreads, smem));
  if (per_sm < 1) return fail(ctx, R3D_ERR_CUDA, "r3d_sfm_colorize_plan: the plan kernel cannot be resident");
  const uint32_t need = (n_lm + exk::kPlanThreads - 1) / exk::kPlanThreads;
  int grid = (int)std::min<uint64_t>((uint64_t)per_sm * (uint64_t)w.sm_count, std::max<uint32_t>(need, 1u));
  uint32_t a_n_lm = n_lm, a_n_views = n_views;
  const uint64_t* a_ofs = d_ofs.p;
  const uint32_t* a_vi = d_vi.p;
  const int2* a_pix = d_pix.p;
  void* args[] = {&a_n_lm, &a_n_views, &a_ofs, &a_vi, &a_pix, &d_remA.p, &d_remB.p, &d_counts.p, &d_st.p, &d_round_view.p,
                  &d_lm_round.p, &d_lm_pixel.p};
  R3D_CUDA_TRY(ctx, cudaLaunchCooperativeKernel((void*)exk::k_colorize_plan, dim3(grid), dim3(exk::kPlanThreads), args, smem,
                                                w.stream));
  exk::PlanState hs{};
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(&hs, d_st.p, sizeof(hs), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(round_view, d_round_view.p, n_views * sizeof(uint32_t), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(lm_round, d_lm_round.p, n_lm * sizeof(uint32_t), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(lm_pixel, d_lm_pixel.p, n_lm * sizeof(int2), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  // view index -> view id
  std::vector<uint32_t> ids;
  ids.reserve(n_views);
  for (const auto& kv : sd->views) ids.push_back(kv.first);
  for (uint32_t r = 0; r < hs.rounds; ++r) round_view[r] = ids[round_view[r]];
  *n_rounds = hs.rounds;
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; }

extern "C" int r3d_sfm_write_colorized_ply(const r3d_sfm_data* sd, const uint8_t* colors, const char* path) try {
  if (!sd || !path || !*path) {
    set_global_error("r3d_sfm_write_colorized_ply: bad arguments");
    return R3D_ERR_INVALID;
  }
  FILE* f = std::fopen(path, "wb");
  if (!f) {
    set_global_error(std::string("r3d_sfm_write_colorized_ply: cannot write ") + path);
    return R3D_ERR_IO;
  }
  std::vector<char> buf(1 << 20);
  std::setvbuf(f, buf.data(), _IOFBF, buf.size());
  std::fprintf(f, "ply\nformat ascii 1.0\nelement vertex %zu\nproperty double x\nproperty double y\nproperty double z\n"
                  "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n",
               sd->structure.size() + sd->poses.size());
  size_t k = 0;
  for (const auto& kv : sd->structure) {  // std::fixed << std::setprecision(16) formats as %.16f
    const double* X = kv.second.X;
    if (colors)
      std::fprintf(f, "%.16f %.16f %.16f %d %d %d\n", X[0], X[1], X[2], (int)colors[3 * k], (int)colors[3 * k + 1],
                   (int)colors[3 * k + 2]);
    else
      std::fprintf(f, "%.16f %.16f %.16f 255 255 255\n", X[0], X[1], X[2]);
    ++k;
  }
  for (const auto& kv : sd->poses)
    std::fprintf(f, "%.16f %.16f %.16f 0 255 0\n", kv.second.C[0], kv.second.C[1], kv.second.C[2]);
  const bool ok = std::fflush(f) == 0 && !std::ferror(f);
  if (std::fclose(f) != 0 || !ok) {
    set_global_error(std::string("r3d_sfm_write_colorized_ply: cannot write ") + path);
    return R3D_ERR_IO;
  }
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; }

namespace {

// dst <- src on the host pool: the pinned staging copies run at memory bandwidth, not one core's
void par_copy(r3d_ctx* ctx, void* dst, const void* src, size_t bytes) {
  constexpr size_t kPiece = 4u << 20;
  const size_t n = (bytes + kPiece - 1) / kPiece;
  parallel_for(std::max(ctx->host_threads, 1), n, [&](size_t i) {
    const size_t a = i * kPiece, b = std::min(bytes, a + kPiece);
    std::memcpy((uint8_t*)dst + a, (const uint8_t*)src + a, b - a);
  });
}

struct UndistortStage {  // per device: the pinned host buffers of two images in flight
  DeviceWorker* w;
  void* h_in[2] = {nullptr, nullptr};
  void* h_out[2] = {nullptr, nullptr};
  explicit UndistortStage(DeviceWorker& worker) : w(&worker) {}
  ~UndistortStage() {  // an early return may leave copies in flight: nothing is released under them
    cudaStreamSynchronize(w->copy_stream);
    cudaStreamSynchronize(w->stream);
    for (int s = 0; s < 2; ++s) {
      if (h_in[s]) cudaFreeHost(h_in[s]);
      if (h_out[s]) cudaFreeHost(h_out[s]);
    }
  }
};

struct WorkerTiming { double up = 0, kern = 0, down = 0, stage = 0; uint32_t launches = 0; };

// the images todo (non-pinhole) on one device, two in flight
int undistort_run(r3d_ctx* ctx, DeviceWorker& w, const std::vector<uint32_t>& todo, const r3d_sfm_intrinsic* intr,
                  const uint8_t* const* rgb, const uint32_t* widths, const uint32_t* heights, uint8_t* const* out,
                  WorkerTiming& t) {
  if (todo.empty()) return R3D_OK;
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  size_t cap = 0;
  for (uint32_t k : todo) cap = std::max(cap, (size_t)widths[k] * heights[k] * 3);
  DevArr<uint8_t> d_in0(w), d_in1(w), d_out0(w), d_out1(w);
  UndistortStage S(w);  // declared after the device blocks: its destructor waits before they go back to the pool
  if (!d_in0.alloc(cap) || !d_in1.alloc(cap) || !d_out0.alloc(cap + 16) || !d_out1.alloc(cap + 16))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_undistort_images: device allocation failed");
  uint8_t* d_in[2] = {d_in0.p, d_in1.p};
  uint8_t* d_out[2] = {d_out0.p, d_out1.p};
  const size_t n_slots = std::min<size_t>(2, todo.size());
  for (size_t s = 0; s < n_slots; ++s) {
    R3D_CUDA_TRY(ctx, cudaHostAlloc(&S.h_in[s], cap, cudaHostAllocDefault));
    R3D_CUDA_TRY(ctx, cudaHostAlloc(&S.h_out[s], cap, cudaHostAllocDefault));
  }
  // per slot: 0/1 around the upload, 2/3 around the kernel, 4/5 around the download
  Events<6> ev[2];
  for (size_t s = 0; s < n_slots; ++s) R3D_CUDA_TRY(ctx, ev[s].create());
  std::vector<uint8_t> used(2, 0);
  auto collect = [&](size_t q) -> int {  // image todo[q] done: read the slot's times, copy its result out
    const int s = (int)(q & 1);
    R3D_CUDA_TRY(ctx, cudaEventSynchronize(ev[s].e[5]));
    t.up += ev[s].ms(0, 1);
    t.kern += ev[s].ms(2, 3);
    t.down += ev[s].ms(4, 5);
    const uint32_t k = todo[q];
    const double t0 = now_ms();
    par_copy(ctx, out[k], S.h_out[s], (size_t)widths[k] * heights[k] * 3);
    t.stage += now_ms() - t0;
    return R3D_OK;
  };
  for (size_t q = 0; q < todo.size(); ++q) {
    const int s = (int)(q & 1);
    const uint32_t k = todo[q];
    const size_t bytes = (size_t)widths[k] * heights[k] * 3;
    if (used[s]) R3D_CUDA_TRY(ctx, cudaEventSynchronize(ev[s].e[1]));  // the slot's previous upload has left h_in
    double t0 = now_ms();
    par_copy(ctx, S.h_in[s], rgb[k], bytes);
    t.stage += now_ms() - t0;
    // the upload overwrites d_in[s]: the slot's previous kernel (ordered before ev 3) must be done with it
    if (used[s]) R3D_CUDA_TRY(ctx, cudaStreamWaitEvent(w.copy_stream, ev[s].e[3], 0));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev[s].e[0], w.copy_stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_in[s], S.h_in[s], bytes, cudaMemcpyHostToDevice, w.copy_stream));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev[s].e[1], w.copy_stream));
    // kernel and download on the compute stream, behind the previous image's download
    R3D_CUDA_TRY(ctx, cudaStreamWaitEvent(w.stream, ev[s].e[1], 0));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev[s].e[2], w.stream));
    exk::Cam c;
    c.model = intr[k].model;
    c.f = intr[k].focal;
    c.ppx = intr[k].ppx;
    c.ppy = intr[k].ppy;
    for (int i = 0; i < 5; ++i) c.d[i] = intr[k].disto[i];
    const uint64_t threads = ((uint64_t)widths[k] * heights[k] + exk::kRun - 1) / exk::kRun;
    exk::k_undistort<<<(unsigned)((threads + exk::kUndistThreads - 1) / exk::kUndistThreads), exk::kUndistThreads, 0, w.stream>>>(
        c, d_in[s], (int)widths[k], (int)heights[k], d_out[s]);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    ++t.launches;
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev[s].e[3], w.stream));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev[s].e[4], w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(S.h_out[s], d_out[s], bytes, cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev[s].e[5], w.stream));
    used[s] = 1;
    // while image q is in flight, hand the previous one back (its slot's h_out is free for image q + 1 afterwards)
    if (q >= 1) {
      const int rc = collect(q - 1);
      if (rc) return rc;
    }
  }
  return collect(todo.size() - 1);
}

}  // namespace

extern "C" int r3d_undistort_images(r3d_ctx* ctx, uint32_t n, const r3d_sfm_intrinsic* intr, const uint8_t* const* rgb,
                                    const uint32_t* widths, const uint32_t* heights, uint8_t* const* out,
                                    r3d_undistort_timing* timing) try {
  const double t_start = now_ms();
  if (!ctx) return fail(ctx, R3D_ERR_INVALID, "r3d_undistort_images: bad arguments");
  if (n > 0 && (!intr || !rgb || !widths || !heights || !out))
    return fail(ctx, R3D_ERR_INVALID, "r3d_undistort_images: bad arguments");
  for (uint32_t k = 0; k < n; ++k) {
    if (!rgb[k] || !out[k] || widths[k] == 0 || heights[k] == 0 || widths[k] > 0x7fffffffu || heights[k] > 0x7fffffffu)
      return fail(ctx, R3D_ERR_INVALID, "r3d_undistort_images: image " + std::to_string(k) + ": NULL buffer or zero size");
    if (intr[k].model < R3D_CAM_PINHOLE || intr[k].model > R3D_CAM_PINHOLE_FISHEYE)
      return fail(ctx, R3D_ERR_INVALID, "r3d_undistort_images: image " + std::to_string(k) + ": unknown camera model");
  }
  r3d_undistort_timing tm{};
  tm.images = n;
  // pinhole (have_disto() false): the image itself
  std::vector<uint32_t> todo;
  for (uint32_t k = 0; k < n; ++k) {
    if (intr[k].model == R3D_CAM_PINHOLE) {
      const double t0 = now_ms();
      par_copy(ctx, out[k], rgb[k], (size_t)widths[k] * heights[k] * 3);
      tm.stage_ms += now_ms() - t0;
      ++tm.copied;
    } else {
      todo.push_back(k);
    }
  }
  const size_t nw = ctx->workers.size();
  const std::vector<uint64_t> cut = balanced_cuts(todo.size(), nw, [&](uint64_t q) {
    return (double)widths[todo[q]] * (double)heights[todo[q]] / 65536.0;
  });
  std::vector<WorkerTiming> wt(nw);
  const int rc = fan_out(ctx, [&](size_t k, DeviceWorker& w) {
    const std::vector<uint32_t> mine(todo.begin() + cut[k], todo.begin() + cut[k + 1]);
    return undistort_run(ctx, w, mine, intr, rgb, widths, heights, out, wt[k]);
  });
  if (rc) return rc;
  for (const WorkerTiming& x : wt) {
    tm.upload_ms += x.up;
    tm.kernel_ms += x.kern;
    tm.download_ms += x.down;
    tm.stage_ms += x.stage;
    tm.kernel_launches += x.launches;
  }
  tm.devices = (uint32_t)nw;
  tm.total_ms = now_ms() - t_start;
  if (timing) *timing = tm;
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; }
