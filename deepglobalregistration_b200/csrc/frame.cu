// The normalised frame and the distance transform (frame.cuh), restated in oracle/fgr.py (normalise) and
// oracle/goicp.py (DistanceTransform):
//   cloud_stats_kernel   one CTA per cloud: fp64 mean (dgr_block_sum) and max |x - mean|
//   normalise_kernel     both clouds centred on their means and divided by the frame scale
//   dt_fill / dt_occupy  G^3 grid over [-e, e]^3: 0 in every cell a target point falls in (clamped), "far" elsewhere
//   dt_line_x_kernel     exact 1-D squared distance to the nearest occupied cell along x, one line per thread
//   dt_fh_kernel         the Felzenszwalb-Huttenlocher lower envelope along y, then z, in integer arithmetic
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"
#include "frame.cuh"

namespace {

constexpr int kStatThreads = 1024;
constexpr int kDtFar = 0x3fffffff;

__global__ void __launch_bounds__(kStatThreads)
cloud_stats_kernel(const float* __restrict__ src, int64_t n_src, const float* __restrict__ tgt, int64_t n_tgt,
                   double* __restrict__ stat) {
  __shared__ double s_part[kStatThreads / 32][3];
  __shared__ double s_mean[3];
  const float* x = blockIdx.x ? tgt : src;
  const int64_t n = blockIdx.x ? n_tgt : n_src;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double a[3] = {0.0, 0.0, 0.0};
  for (int64_t i = threadIdx.x; i < n; i += kStatThreads)
    for (int c = 0; c < 3; ++c) a[c] += (double)x[3 * i + c];
  const double s = dgr_block_sum<kStatThreads>(a, s_part);
  if (threadIdx.x < 3) s_mean[threadIdx.x] = s / (double)n;
  __syncthreads();
  const double m[3] = {s_mean[0], s_mean[1], s_mean[2]};
  double mx = 0.0;                                      // a maximum does not depend on the order
  for (int64_t i = threadIdx.x; i < n; i += kStatThreads) {
    double p[3];
    dgr_frame_point(x, i, m, 1.0, p);
    const double o[3] = {0.0, 0.0, 0.0};
    mx = fmax(mx, dgr_dist3(p, o));
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, d));
  __syncthreads();
  if (lane == 0) s_part[warp][0] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kStatThreads / 32; ++w) mx = fmax(mx, s_part[w][0]);
    for (int c = 0; c < 3; ++c) stat[4 * blockIdx.x + c] = m[c];
    stat[4 * blockIdx.x + 3] = mx;
  }
}

__global__ void normalise_kernel(const float* __restrict__ src, int64_t n_s, const float* __restrict__ tgt,
                                 int64_t n_t, const double* __restrict__ stat, double* __restrict__ xn,
                                 float* __restrict__ y32) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const double s = dgr_frame_scale(stat);
  if (xn != nullptr && i < n_s)
    for (int a = 0; a < 3; ++a) xn[3 * i + a] = __ddiv_rn(__dsub_rn((double)src[3 * i + a], stat[a]), s);
  if (i < n_t)
    for (int a = 0; a < 3; ++a)
      y32[3 * i + a] = __double2float_rn(__ddiv_rn(__dsub_rn((double)tgt[3 * i + a], stat[4 + a]), s));
}

__global__ void dt_fill_kernel(int32_t* __restrict__ dt, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dt[i] = kDtFar;
}

__global__ void dt_occupy_kernel(const float* __restrict__ y32, int64_t n_t, int G, float e32, float h32,
                                 int32_t* __restrict__ dt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_t) return;
  const int ix = dt_axis(y32[3 * i], e32, h32, G), iy = dt_axis(y32[3 * i + 1], e32, h32, G),
            iz = dt_axis(y32[3 * i + 2], e32, h32, G);
  dt[((int64_t)iz * G + iy) * G + ix] = 0;                 // idempotent
}

// along x: squared distance to the nearest occupied cell of the line (far when there is none)
__global__ void dt_line_x_kernel(int32_t* __restrict__ dt, int G) {
  const int64_t line = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (line >= (int64_t)G * G) return;
  int32_t* r = dt + line * G;
  int last = -1;
  for (int x = 0; x < G; ++x) {                           // forward: distance to the last occupied cell
    if (r[x] == 0) last = x;
    r[x] = last >= 0 ? x - last : kDtFar;
  }
  int next = -1;
  for (int x = G - 1; x >= 0; --x) {
    int d = r[x];
    if (d == 0) next = x;
    if (next >= 0 && next - x < d) d = next - x;
    r[x] = d < kDtFar ? d * d : kDtFar;
  }
}

// lines along y (pass_z = 0) or z (pass_z = 1): d[q] = min_p (q - p)^2 + f[p] by the lower envelope of the
// parabolas of the finite f[p]; intersections compared by cross-multiplication in int64
__global__ void __launch_bounds__(128) dt_fh_kernel(int32_t* __restrict__ dt, int G, int pass_z) {
  const int64_t line = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (line >= (int64_t)G * G) return;
  const int64_t GG = (int64_t)G * G;
  const int64_t base = pass_z ? line : (line / G) * GG + line % G, stride = pass_z ? GG : G;
  int16_t v[kDtMaxG];
  int32_t fv[kDtMaxG];
  int m = 0;
  for (int q = 0; q < G; ++q) {
    const int32_t f = dt[base + q * stride];
    if (f >= kDtFar) continue;
    while (m >= 2) {
      const int64_t a = v[m - 2], b = v[m - 1];
      const int64_t hb = (int64_t)fv[m - 1] + b * b;
      const int64_t n1 = ((int64_t)f + (int64_t)q * q) - hb, d1 = 2 * (q - b);
      const int64_t n2 = hb - ((int64_t)fv[m - 2] + a * a), d2 = 2 * (b - a);
      if (n1 * d2 <= n2 * d1) --m; else break;
    }
    v[m] = (int16_t)q;
    fv[m] = f;
    ++m;
  }
  if (m == 0) return;
  int k = 0;
  for (int q = 0; q < G; ++q) {
    while (k + 1 < m) {
      const int dn = (q - v[k + 1]) * (q - v[k + 1]) + fv[k + 1], dc = (q - v[k]) * (q - v[k]) + fv[k];
      if (dn <= dc) ++k; else break;
    }
    dt[base + q * stride] = (q - v[k]) * (q - v[k]) + fv[k];
  }
}

}  // namespace

void dgr_cloud_stats(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, double* stat,
                     cudaStream_t st) {
  cloud_stats_kernel<<<2, kStatThreads, 0, st>>>(src, n_src, tgt, n_tgt, stat);
}

int32_t dgr_goicp_dt_check(int64_t n_src, int64_t n_tgt, int32_t G, double e) {
  DGR_ARG_CHECK(n_src >= 1 && n_src <= kGoicpMaxSrc, "n_src must lie in [1, 1024]");
  DGR_ARG_CHECK(n_tgt >= 1 && n_tgt < (1ll << 31), "n_tgt must lie in [1, 2^31)");
  DGR_ARG_CHECK(G >= 16 && G <= kDtMaxG, "dt_size must lie in [16, 512]");
  DGR_ARG_CHECK(e > 0.0 && isfinite(e), "dt_expand must be positive");
  return DGR_OK;
}

int dgr_normalise_dt(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, int G, double e, double* stat,
                     double* xn, float* y32, int32_t* dt, cudaStream_t st) {
  const float e32 = (float)e, h32 = (float)(2.0 * e / G);
  const int64_t cells = (int64_t)G * G * G, lines = (int64_t)G * G;
  dgr_cloud_stats(src, n_src, tgt, n_tgt, stat, st);
  normalise_kernel<<<dgr_blocks(n_src > n_tgt ? n_src : n_tgt, 256), 256, 0, st>>>(src, n_src, tgt, n_tgt, stat, xn,
                                                                                    y32);
  dt_fill_kernel<<<dgr_blocks(cells, 256), 256, 0, st>>>(dt, cells);
  dt_occupy_kernel<<<dgr_blocks(n_tgt, 256), 256, 0, st>>>(y32, n_tgt, G, e32, h32, dt);
  dt_line_x_kernel<<<dgr_blocks(lines, 128), 128, 0, st>>>(dt, G);
  dt_fh_kernel<<<dgr_blocks(lines, 128), 128, 0, st>>>(dt, G, 0);
  dt_fh_kernel<<<dgr_blocks(lines, 128), 128, 0, st>>>(dt, G, 1);
  return 7;
}

extern "C" {

int32_t dgr_goicp_dt_build(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, int32_t dt_size,
                           double dt_expand, double* stat, float* tgt_norm, int32_t* dt, void* stream) {
  DGR_ARG_CHECK(src != nullptr && tgt != nullptr && stat != nullptr && tgt_norm != nullptr && dt != nullptr,
                "null pointer");
  const int32_t r = dgr_goicp_dt_check(n_src, n_tgt, dt_size, dt_expand);
  if (r != DGR_OK) return r;
  dgr_note_launches(dgr_normalise_dt(src, n_src, tgt, n_tgt, dt_size, dt_expand, stat, nullptr, tgt_norm, dt,
                                     (cudaStream_t)stream));
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
