// RGB-D odometry: open3d's legacy ComputeRGBDOdometry (RGBDOdometry.cpp, RGBDOdometryJacobian.cpp) with the hybrid and
// the colour Jacobian, restated in oracle/rgbd_odometry.py (which states every reading and departure).  The images are
// bit for bit the oracle's: every float op is an explicit __fmul_rn / __fadd_rn / __fsub_rn and every fp64 op of the
// filters and of the projection an explicit __d*_rn, so nothing contracts into an FMA.
//   odo_filter_kernel      one pass of a separable 3-tap filter (replicated border) over up to 4 images: float
//                          products summed in fp64 from +0, rounded once; the depth range test on read
//   odo_project_kernel     a thread per source pixel: its point (float, open3d's XYZ image) moved by the pose in fp64,
//                          projected and rounded; a match within max_depth_diff writes the target pixel's z-buffer
//                          with one 64-bit atomicMin of (float bits of the transformed depth, source pixel)
//   odo_norm_rows_kernel   a warp per target row: the intensity sums of the matches (lane-strided, then a butterfly)
//   odo_scale_kernel       the row sums in row order; 0.5 / mean, or the call's failure without a match
//   odo_scale_apply_kernel / odo_down_kernel   intensity scaling; the 2x2-average pyramid
//   odo_accum_kernel<H>    8 lanes per target pixel: read and reset its z-buffer slot, the hybrid (H) or colour rows
//                          into the 29 fixed-order sums (add_row, icp.cu's lane layout), per-CTA partials
//   odo_update_kernel      the partials in CTA order, cholesky6_step, zyx_update_left; a failed solve sets `done`,
//                          and every later launch of the call is a no-op
//   odo_info_kernel        the ten target-point sums of the final full-resolution matches; dgr_info_final
//   odo_finish_kernel      the result block
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>

#include "common.cuh"
#include "kabsch.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 2368;
constexpr int kStride = 32;                             // doubles per CTA partial
constexpr int kNv = 29;                                 // J^T J (21), J^T r (6), count, sum r^2
constexpr int kUpdateThreads = 256;
constexpr int kInfoNv = 10;
constexpr int kStateWords = 32;
constexpr int kHead = DGR_ODOMETRY_RESULT_HEAD;
constexpr uint64_t kEmpty = ~0ull;                      // z-buffer sentinel: above every (positive float, pixel) key
constexpr double kSobelScale = 0.125;
constexpr double kLambdaDepth = 0.968;                  // open3d's LAMBDA_HYBRID_DEPTH

struct OdoState {
  double T[12];                                         // current pose, row-major [R | t]
  double scale_s, scale_t;                              // intensity normalisation
  int iteration, done;
};

// One pyramid level: the images and the camera K / 2^l
struct Level {
  const float *Is, *Ds, *It, *Dt, *gIx, *gIy, *gDx, *gDy;
  int W, H;
  double fx, fy, cx, cy, inv_fx, inv_fy;
};

struct FilterImg {
  const float* src;
  float* dst;
  float k[3];
  int depth_range;                                      // values outside [min_depth, max_depth] or <= 0 read as NaN
};

struct FilterJob {
  FilterImg img[4];
  int W, H, vertical;
  double min_depth, max_depth;
  uint64_t* zfill;                                      // when set, image 0's threads write the z-buffer sentinel
};

__global__ void odo_init_kernel(const OdoState init, OdoState* st, double* result) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *st = init;
  for (int k = threadIdx.x; k < DGR_ODOMETRY_RESULT; k += blockDim.x) result[k] = 0.0;
}

__global__ void __launch_bounds__(kThreads) odo_filter_kernel(const FilterJob job) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = job.W, H = job.H;
  if (i >= (int64_t)W * H) return;
  if (job.zfill != nullptr && blockIdx.y == 0) job.zfill[i] = kEmpty;
  const FilterImg f = job.img[blockIdx.y];
  const int x = (int)(i % W), y = (int)(i / W);
  double acc = 0.0;
#pragma unroll
  for (int q = -1; q <= 1; ++q) {
    const int xs = job.vertical ? x : min(max(x + q, 0), W - 1);
    const int ys = job.vertical ? min(max(y + q, 0), H - 1) : y;
    float v = f.src[(int64_t)ys * W + xs];
    if (f.depth_range) {
      const double d = v;
      if (d < job.min_depth || d > job.max_depth || d <= 0.0) v = __int_as_float(0x7fc00000);
    }
    acc = __dadd_rn(acc, (double)__fmul_rn(v, f.k[q + 1]));
  }
  f.dst[i] = __double2float_rn(acc);
}

// open3d's ConvertDepthImageToXYZImage at pixel i: ((u - cx) d) / fx rounded to float (d the float depth)
__device__ __forceinline__ void pixel_point(const Level& lv, const float* __restrict__ depth, int64_t i, double p[3]) {
  const int u = (int)(i % lv.W), v = (int)(i / lv.W);
  const double d = depth[i];
  p[0] = (double)__double2float_rn(__dmul_rn(__dmul_rn(__dsub_rn((double)u, lv.cx), d), lv.inv_fx));
  p[1] = (double)__double2float_rn(__dmul_rn(__dmul_rn(__dsub_rn((double)v, lv.cy), d), lv.inv_fy));
  p[2] = d;
}

// q = R p + t, row a: ((R[a][0] p0 + R[a][1] p1) + R[a][2] p2) + t[a]
__device__ __forceinline__ void move_point(const double* T, const double p[3], double q[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a)
    q[a] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * a], p[0]), __dmul_rn(T[4 * a + 1], p[1])),
                               __dmul_rn(T[4 * a + 2], p[2])), T[4 * a + 3]);
}

__global__ void __launch_bounds__(kThreads)
odo_project_kernel(const Level lv, const OdoState* __restrict__ st, double max_diff, uint64_t* __restrict__ zbuf) {
  if (st->done) return;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)lv.W * lv.H) return;
  if (isnan(lv.Ds[i])) return;
  double p[3], q[3];
  pixel_point(lv, lv.Ds, i, p);
  move_point(st->T, p, q);
  if (!(q[2] > 0.0)) return;
  const double uf = __dadd_rn(__ddiv_rn(__dadd_rn(__dmul_rn(lv.fx, q[0]), __dmul_rn(lv.cx, q[2])), q[2]), 0.5);
  const double vf = __dadd_rn(__ddiv_rn(__dadd_rn(__dmul_rn(lv.fy, q[1]), __dmul_rn(lv.cy, q[2])), q[2]), 0.5);
  if (!(uf > -1.0 && uf < (double)lv.W && vf > -1.0 && vf < (double)lv.H)) return;
  const int64_t t = (int64_t)(int)vf * lv.W + (int)uf;   // (int) truncates, as open3d's cast
  const float dt = lv.Dt[t];
  if (isnan(dt)) return;
  if (!(fabs(__dsub_rn(q[2], (double)dt)) <= max_diff)) return;
  const uint64_t key = ((uint64_t)__float_as_uint(__double2float_rn(q[2])) << 32) | (uint64_t)(uint32_t)i;
  atomicMin(reinterpret_cast<unsigned long long*>(zbuf + t), (unsigned long long)key);
}

// Warp per target row: lane l adds the matches of columns l, l + 32, ... in order (count, source and target filtered
// intensity, fp64), then a butterfly 16, 8, 4, 2, 1; the slots are reset for the next pass
__global__ void __launch_bounds__(kThreads)
odo_norm_rows_kernel(const float* __restrict__ Gs, const float* __restrict__ Gt, int W, int H,
                     uint64_t* __restrict__ zbuf, double* __restrict__ rows) {
  const int row = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (row >= H) return;                                 // whole warps
  double n = 0.0, ss = 0.0, tt = 0.0;
  for (int x = lane; x < W; x += 32) {
    const int64_t t = (int64_t)row * W + x;
    const uint64_t key = zbuf[t];
    if (key == kEmpty) continue;
    zbuf[t] = kEmpty;
    n += 1.0;
    ss += (double)Gs[(uint32_t)key];
    tt += (double)Gt[t];
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    n += __shfl_xor_sync(0xffffffffu, n, d);
    ss += __shfl_xor_sync(0xffffffffu, ss, d);
    tt += __shfl_xor_sync(0xffffffffu, tt, d);
  }
  if (lane == 0) {
    rows[3 * (int64_t)row] = n;
    rows[3 * (int64_t)row + 1] = ss;
    rows[3 * (int64_t)row + 2] = tt;
  }
}

// open3d's NormalizeIntensity: the row sums in row order; scale = 0.5 / (sum / n); no match ends the call
__global__ void odo_scale_kernel(const double* __restrict__ rows, int H, OdoState* st) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  double n = 0.0, ss = 0.0, tt = 0.0;
  for (int y = 0; y < H; ++y) {
    n += rows[3 * y];
    ss += rows[3 * y + 1];
    tt += rows[3 * y + 2];
  }
  if (n > 0.0) {
    st->scale_s = 0.5 / (ss / n);
    st->scale_t = 0.5 / (tt / n);
  } else {
    st->scale_s = st->scale_t = 0.0;
    st->done = 1;
  }
}

// open3d's LinearTransformImage(scale, 0): (float)(scale * v + 0.0)
__global__ void __launch_bounds__(kThreads)
odo_scale_apply_kernel(const float* __restrict__ Gs, const float* __restrict__ Gt, int64_t n,
                       const OdoState* __restrict__ st, float* __restrict__ Is, float* __restrict__ It) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Is[i] = __double2float_rn(__dadd_rn(__dmul_rn(st->scale_s, (double)Gs[i]), 0.0));
  It[i] = __double2float_rn(__dadd_rn(__dmul_rn(st->scale_t, (double)Gt[i]), 0.0));
}

struct DownJob {
  const float* src[4];
  float* dst[4];
  int Wp, W, H;
};

// open3d's Image::Downsample: (((p00 + p10) + p01) + p11) / 4 in float
__global__ void __launch_bounds__(kThreads) odo_down_kernel(const DownJob job) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)job.W * job.H) return;
  const int x = (int)(i % job.W), y = (int)(i / job.W);
  const float* s = job.src[blockIdx.y];
  const int64_t a = (int64_t)(2 * y) * job.Wp + 2 * x, b = a + job.Wp;
  const float v = __fadd_rn(__fadd_rn(__fadd_rn(s[a], s[a + 1]), s[b]), s[b + 1]);
  job.dst[blockIdx.y][i] = __fmul_rn(v, 0.25f);
}

// open3d's RGBDOdometryJacobianFromHybridTerm (kHybrid) / FromColorTerm at a match: source point p moved to q, target
// pixel t, source pixel s
template <bool kHybrid>
__device__ __forceinline__ void odo_rows(const Level& lv, const double q[3], int64_t s, int64_t t, int sub,
                                         double* acc) {
  const double invz = 1.0 / q[2];
  const double dIdx = kSobelScale * (double)lv.gIx[t], dIdy = kSobelScale * (double)lv.gIy[t];
  const double c0 = dIdx * lv.fx * invz, c1 = dIdy * lv.fy * invz;
  const double c2 = -(c0 * q[0] + c1 * q[1]) * invz;
  const double photo = (double)__fsub_rn(lv.It[t], lv.Is[s]);
  const double si = kHybrid ? sqrt(1.0 - kLambdaDepth) : 1.0;
  const double J0[6] = {si * (-q[2] * c1 + q[1] * c2), si * (q[2] * c0 - q[0] * c2), si * (-q[1] * c0 + q[0] * c1),
                        si * c0, si * c1, si * c2};
  const double r0 = si * photo;
  add_row<false>(acc, sub, J0, r0, 1.0);
  double r2 = r0 * r0;
  if (kHybrid) {
    const double sd = sqrt(kLambdaDepth);
    double dDdx = kSobelScale * (double)lv.gDx[t], dDdy = kSobelScale * (double)lv.gDy[t];
    if (isnan(dDdx)) dDdx = 0.0;
    if (isnan(dDdy)) dDdy = 0.0;
    const double d0 = dDdx * lv.fx * invz, d1 = dDdy * lv.fy * invz;
    const double d2 = -(d0 * q[0] + d1 * q[1]) * invz;
    const double J1[6] = {sd * ((-q[2] * d1 + q[1] * d2) - q[1]), sd * ((q[2] * d0 - q[0] * d2) + q[0]),
                          sd * (-q[1] * d0 + q[0] * d1), sd * d0, sd * d1, sd * (d2 - 1.0)};
    const double r1 = sd * ((double)lv.Dt[t] - q[2]);
    add_row<false>(acc, sub, J1, r1, 1.0);
    r2 += r1 * r1;
  }
  add_sum(acc, sub, 27, 1.0);
  add_sum(acc, sub, 28, r2);
}

template <bool kHybrid>
__global__ void __launch_bounds__(kThreads)
odo_accum_kernel(const Level lv, const OdoState* __restrict__ st, uint64_t* __restrict__ zbuf,
                 double* __restrict__ part) {
  constexpr int kSlots = (kNv + 7) / 8;
  if (st->done) return;
  double T[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) T[k] = st->T[k];
  double acc[kSlots];
#pragma unroll
  for (int a = 0; a < kSlots; ++a) acc[a] = 0.0;
  const int lane = threadIdx.x & 31, sub = lane & 7;
  const int64_t n = (int64_t)lv.W * lv.H;
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) >> 3;
  for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3; i0 < ((n + groups - 1) / groups) * groups;
       i0 += groups) {
    uint64_t key = kEmpty;                              // lane 0 of the group reads and resets the slot
    if (sub == 0 && i0 < n) {
      key = zbuf[i0];
      if (key != kEmpty) zbuf[i0] = kEmpty;
    }
    key = __shfl_sync(0xffffffffu, key, lane & ~7);
    if (key == kEmpty) continue;
    const int64_t s = (int64_t)(uint32_t)key;
    double p[3], q[3];
    pixel_point(lv, lv.Ds, s, p);
    move_point(T, p, q);
    odo_rows<kHybrid>(lv, q, s, i0, sub, acc);
  }
  __shared__ double red[kThreads / 32][kStride];
  const int warp = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < kSlots; ++a) {
    double v = acc[a];
    v += __shfl_xor_sync(0xffffffffu, v, 8);            // the 4 groups of the warp, same sub
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    if (lane < 8) red[warp][8 * a + lane] = v;
  }
  __syncthreads();
  if (threadIdx.x < kNv) {
    double v = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) v += red[w][threadIdx.x];
    part[(int64_t)blockIdx.x * kStride + threadIdx.x] = v;
  }
}

// one CTA of 8 warps: warp w sums partials k = w, w + 8, ... over the CTAs (each lane-strided, then a butterfly; a
// 29-warp CTA would cap the solve at 64 registers and spill); thread 0 records the step's correspondence count and
// solves J^T J x = -J^T r
__global__ void __launch_bounds__(kUpdateThreads)
odo_update_kernel(OdoState* st, const double* __restrict__ part, int n_blocks, double* __restrict__ result) {
  __shared__ double tot[kStride];
  if (st->done) return;                                 // uniform per launch
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < kNv; k += kUpdateThreads / 32) {
    double v = 0.0;
    for (int b = lane; b < n_blocks; b += 32) v += part[(int64_t)b * kStride + k];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if (lane == 0) tot[k] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int k = st->iteration;
  result[kHead + k] = tot[27];
  st->iteration = k + 1;
  double x[6], T0[12];
  if (!cholesky6_step(tot, tot + 21, x)) {
    st->done = 1;
    return;
  }
  for (int q = 0; q < 12; ++q) T0[q] = st->T[q];
  zyx_update_left(x, T0, st->T);
}

// open3d's CreateInformationMatrix: the ten sums of the target points (float XYZ image) of the full-resolution
// matches, per CTA (dgr_block_sum); zero partials once the call has failed, so dgr_info_final reads written words
__global__ void __launch_bounds__(kThreads)
odo_info_kernel(const Level lv, const OdoState* __restrict__ st, const uint64_t* __restrict__ zbuf,
                double* __restrict__ part) {
  double v[kInfoNv];
#pragma unroll
  for (int k = 0; k < kInfoNv; ++k) v[k] = 0.0;
  const int64_t n = (int64_t)lv.W * lv.H;
  if (!st->done) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
      if (zbuf[t] == kEmpty) continue;
      double q[3];
      pixel_point(lv, lv.Dt, t, q);
      v[0] += 1.0;
      v[1] += q[0]; v[2] += q[1]; v[3] += q[2];
      v[4] += q[0] * q[0]; v[5] += q[0] * q[1]; v[6] += q[0] * q[2];
      v[7] += q[1] * q[1]; v[8] += q[1] * q[2]; v[9] += q[2] * q[2];
    }
  }
  __shared__ double red[kThreads / 32][kInfoNv];
  const double tot = dgr_block_sum<kThreads>(v, red);
  if (threadIdx.x < kInfoNv) part[(int64_t)blockIdx.x * kInfoNv + threadIdx.x] = tot;
}

__global__ void odo_finish_kernel(const OdoState* __restrict__ st, double* __restrict__ result) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const bool ok = !st->done;
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) result[4 * r + c] = r == 3 ? (c == 3 ? 1.0 : 0.0) : (ok ? st->T[4 * r + c] : r == c);
  result[16] = ok ? 1.0 : 0.0;
  result[17] = (double)st->iteration;
  if (!ok) {
    for (int k = 0; k < 36; ++k) result[18 + k] = (k % 7 == 0) ? 1.0 : 0.0;
    result[54] = 0.0;
  }
}

inline int accum_blocks(int64_t n_pix) {
  const unsigned b = dgr_blocks(n_pix * 8, kThreads);   // 8 lanes per target pixel
  return b > (unsigned)kMaxBlocks ? kMaxBlocks : (int)b;
}

inline int info_blocks(int64_t n_pix) {
  const unsigned b = dgr_blocks(n_pix, kThreads);
  return b > (unsigned)kMaxBlocks ? kMaxBlocks : (int)b;
}

struct OdoWs {
  OdoState* state;
  float* img[DGR_ODOMETRY_MAX_LEVELS][8];               // Is, Ds, It, Dt, dI/dx, dI/dy, dD/dx, dD/dy
  float *Gs, *Gt;
  float* tmp[4];
  uint64_t* zbuf;
  double* rows;
  double* part;
};

// workspace size in 8-byte words; carves `base` when it is not null (offsets: the word offsets of the images)
int64_t odo_layout(int W, int H, int L, void* base, OdoWs* w, int64_t* offsets) {
  static_assert(sizeof(OdoState) <= kStateWords * sizeof(double), "state workspace too small");
  DgrCarver c(base);
  OdoWs r;
  r.state = reinterpret_cast<OdoState*>(c.take<double>(kStateWords));
  for (int l = 0; l < L; ++l) {
    const int64_t n = (int64_t)(W >> l) * (H >> l);
    for (int k = 0; k < 8; ++k) {
      if (offsets != nullptr) offsets[8 * l + k] = c.words;
      r.img[l][k] = c.take<float>(n);
    }
  }
  const int64_t n0 = (int64_t)W * H;
  if (offsets != nullptr) offsets[8 * L] = c.words;
  r.Gs = c.take<float>(n0);
  if (offsets != nullptr) offsets[8 * L + 1] = c.words;
  r.Gt = c.take<float>(n0);
  for (int k = 0; k < 4; ++k) r.tmp[k] = c.take<float>(n0);
  if (offsets != nullptr) offsets[8 * L + 2] = c.words;
  r.zbuf = c.take<uint64_t>(n0);
  r.rows = c.take<double>(3 * (int64_t)H);
  const int64_t pb = (int64_t)accum_blocks(n0) * kStride, ib = (int64_t)info_blocks(n0) * kInfoNv;
  r.part = c.take<double>(pb > ib ? pb : ib);
  if (w != nullptr) *w = r;
  return c.words;
}

int32_t check_size(int32_t width, int32_t height, int32_t levels) {
  DGR_ARG_CHECK(levels >= 1 && levels <= DGR_ODOMETRY_MAX_LEVELS, "levels must lie in [1, DGR_ODOMETRY_MAX_LEVELS]");
  DGR_ARG_CHECK(width >= 1 && height >= 1 && (int64_t)width * height < (1ll << 31), "image size out of range");
  DGR_ARG_CHECK((width >> (levels - 1)) >= 1 && (height >> (levels - 1)) >= 1,
                "the coarsest pyramid level has no pixel");
  return DGR_OK;
}

Level make_level(const OdoWs& w, int W, int H, const double* intr, int l) {
  Level lv;
  lv.Is = w.img[l][0]; lv.Ds = w.img[l][1]; lv.It = w.img[l][2]; lv.Dt = w.img[l][3];
  lv.gIx = w.img[l][4]; lv.gIy = w.img[l][5]; lv.gDx = w.img[l][6]; lv.gDy = w.img[l][7];
  lv.W = W >> l;
  lv.H = H >> l;
  double s = 1.0;                                       // open3d's CreatePyramidCameraMatrix: 0.5 K per level
  for (int k = 0; k < l; ++k) s *= 0.5;
  lv.fx = intr[0] * s; lv.fy = intr[1] * s; lv.cx = intr[2] * s; lv.cy = intr[3] * s;
  lv.inv_fx = 1.0 / lv.fx;
  lv.inv_fy = 1.0 / lv.fy;
  return lv;
}

FilterImg filter_img(const float* src, float* dst, float k0, float k1, float k2, int depth_range) {
  FilterImg f;
  f.src = src; f.dst = dst; f.k[0] = k0; f.k[1] = k1; f.k[2] = k2; f.depth_range = depth_range;
  return f;
}

void filter4(const FilterImg (&img)[4], int W, int H, int vertical, double min_depth, double max_depth,
             uint64_t* zfill, cudaStream_t st) {
  FilterJob job;
  for (int k = 0; k < 4; ++k) job.img[k] = img[k];
  job.W = W; job.H = H; job.vertical = vertical; job.min_depth = min_depth; job.max_depth = max_depth;
  job.zfill = zfill;
  odo_filter_kernel<<<dim3(dgr_blocks((int64_t)W * H, kThreads), 4), kThreads, 0, st>>>(job);
}

}  // namespace

extern "C" {

int32_t dgr_rgbd_odometry_ws_elems(int32_t width, int32_t height, int32_t levels, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr, "null pointer");
  DGR_TRY(check_size(width, height, levels));
  *n_elems = odo_layout(width, height, levels, nullptr, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_rgbd_odometry_ws_layout(int32_t width, int32_t height, int32_t levels, int64_t* offsets) {
  DGR_ARG_CHECK(offsets != nullptr, "null pointer");
  DGR_TRY(check_size(width, height, levels));
  odo_layout(width, height, levels, nullptr, nullptr, offsets);
  return DGR_OK;
}

int32_t dgr_rgbd_odometry(const float* src_intensity, const float* src_depth, const float* tgt_intensity,
                          const float* tgt_depth, int32_t width, int32_t height, const double* intrinsic,
                          const double* odo_init, int32_t jacobian, const int32_t* iterations, int32_t levels,
                          double max_depth_diff, double min_depth, double max_depth, uint64_t* ws, double* result,
                          void* stream) {
  DGR_ARG_CHECK(src_intensity != nullptr && src_depth != nullptr && tgt_intensity != nullptr &&
                tgt_depth != nullptr && intrinsic != nullptr && odo_init != nullptr && iterations != nullptr &&
                ws != nullptr && result != nullptr, "null pointer");
  DGR_TRY(check_size(width, height, levels));
  DGR_ARG_CHECK(jacobian == DGR_ODOMETRY_JACOBIAN_HYBRID || jacobian == DGR_ODOMETRY_JACOBIAN_COLOR,
                "unknown jacobian");
  for (int l = 0; l < levels; ++l)
    DGR_ARG_CHECK(iterations[l] >= 0 && iterations[l] <= DGR_ODOMETRY_MAX_ITERATIONS,
                  "iterations per level must lie in [0, DGR_ODOMETRY_MAX_ITERATIONS]");
  DGR_ARG_CHECK(intrinsic[0] > 0.0 && intrinsic[1] > 0.0 && std::isfinite(intrinsic[0]) &&
                std::isfinite(intrinsic[1]) && std::isfinite(intrinsic[2]) && std::isfinite(intrinsic[3]),
                "focal lengths must be finite and positive, the principal point finite");
  bool zero = true;
  for (int k = 0; k < 16; ++k) {
    DGR_ARG_CHECK(std::isfinite(odo_init[k]), "odo_init must be finite");
    zero = zero && odo_init[k] == 0.0;
  }
  DGR_ARG_CHECK(min_depth >= 0.0 && min_depth < max_depth && std::isfinite(max_depth),
                "depth range must satisfy 0 <= min_depth < max_depth < inf");
  DGR_ARG_CHECK(max_depth_diff > 0.0 && std::isfinite(max_depth_diff), "max_depth_diff must be finite and positive");
  cudaStream_t st = (cudaStream_t)stream;
  const int W = width, H = height, L = levels;
  const int64_t n0 = (int64_t)W * H;
  OdoWs w;
  odo_layout(W, H, L, ws, &w, nullptr);
  OdoState init;
  for (int k = 0; k < 12; ++k) init.T[k] = zero ? (k % 5 == 0 ? 1.0 : 0.0) : odo_init[k];   // open3d: zero -> I
  init.scale_s = init.scale_t = 0.0;
  init.iteration = 0;
  init.done = 0;
  int launches = 0;
  odo_init_kernel<<<1, 256, 0, st>>>(init, w.state, result);
  ++launches;
  // range test and Gaussian3 of both frames; the z-buffer sentinel
  filter4({filter_img(src_intensity, w.tmp[0], 0.25f, 0.5f, 0.25f, 0), filter_img(src_depth, w.tmp[1], 0.25f, 0.5f, 0.25f, 1),
           filter_img(tgt_intensity, w.tmp[2], 0.25f, 0.5f, 0.25f, 0), filter_img(tgt_depth, w.tmp[3], 0.25f, 0.5f, 0.25f, 1)},
          W, H, 0, min_depth, max_depth, w.zbuf, st);
  filter4({filter_img(w.tmp[0], w.Gs, 0.25f, 0.5f, 0.25f, 0), filter_img(w.tmp[1], w.img[0][1], 0.25f, 0.5f, 0.25f, 0),
           filter_img(w.tmp[2], w.Gt, 0.25f, 0.5f, 0.25f, 0), filter_img(w.tmp[3], w.img[0][3], 0.25f, 0.5f, 0.25f, 0)},
          W, H, 1, min_depth, max_depth, nullptr, st);
  launches += 2;
  // intensity normalisation over the full-resolution matches at odo_init
  const Level l0 = make_level(w, W, H, intrinsic, 0);
  odo_project_kernel<<<dgr_blocks(n0, kThreads), kThreads, 0, st>>>(l0, w.state, max_depth_diff, w.zbuf);
  odo_norm_rows_kernel<<<dgr_blocks((int64_t)H * 32, kThreads), kThreads, 0, st>>>(w.Gs, w.Gt, W, H, w.zbuf, w.rows);
  odo_scale_kernel<<<1, 32, 0, st>>>(w.rows, H, w.state);
  odo_scale_apply_kernel<<<dgr_blocks(n0, kThreads), kThreads, 0, st>>>(w.Gs, w.Gt, n0, w.state, w.img[0][0],
                                                                        w.img[0][2]);
  launches += 4;
  // pyramid, then the target gradients of every level
  for (int l = 1; l < L; ++l) {
    DownJob job;
    for (int k = 0; k < 4; ++k) { job.src[k] = w.img[l - 1][k]; job.dst[k] = w.img[l][k]; }
    job.Wp = W >> (l - 1);
    job.W = W >> l;
    job.H = H >> l;
    odo_down_kernel<<<dim3(dgr_blocks((int64_t)job.W * job.H, kThreads), 4), kThreads, 0, st>>>(job);
    ++launches;
  }
  for (int l = 0; l < L; ++l) {
    const int Wl = W >> l, Hl = H >> l;
    filter4({filter_img(w.img[l][2], w.tmp[0], -1.0f, 0.0f, 1.0f, 0), filter_img(w.img[l][2], w.tmp[1], 1.0f, 2.0f, 1.0f, 0),
             filter_img(w.img[l][3], w.tmp[2], -1.0f, 0.0f, 1.0f, 0), filter_img(w.img[l][3], w.tmp[3], 1.0f, 2.0f, 1.0f, 0)},
            Wl, Hl, 0, min_depth, max_depth, nullptr, st);
    filter4({filter_img(w.tmp[0], w.img[l][4], 1.0f, 2.0f, 1.0f, 0), filter_img(w.tmp[1], w.img[l][5], -1.0f, 0.0f, 1.0f, 0),
             filter_img(w.tmp[2], w.img[l][6], 1.0f, 2.0f, 1.0f, 0), filter_img(w.tmp[3], w.img[l][7], -1.0f, 0.0f, 1.0f, 0)},
            Wl, Hl, 1, min_depth, max_depth, nullptr, st);
    launches += 2;
  }
  // coarse to fine: (project, accumulate, update) per step, all enqueued
  for (int l = L - 1; l >= 0; --l) {
    const Level lv = make_level(w, W, H, intrinsic, l);
    const int64_t n = (int64_t)lv.W * lv.H;
    const int blocks = accum_blocks(n);
    for (int k = 0; k < iterations[L - 1 - l]; ++k) {
      odo_project_kernel<<<dgr_blocks(n, kThreads), kThreads, 0, st>>>(lv, w.state, max_depth_diff, w.zbuf);
      if (jacobian == DGR_ODOMETRY_JACOBIAN_HYBRID)
        odo_accum_kernel<true><<<blocks, kThreads, 0, st>>>(lv, w.state, w.zbuf, w.part);
      else
        odo_accum_kernel<false><<<blocks, kThreads, 0, st>>>(lv, w.state, w.zbuf, w.part);
      odo_update_kernel<<<1, kUpdateThreads, 0, st>>>(w.state, w.part, blocks, result);
      launches += 3;
    }
  }
  // information matrix at the final pose; the matches stay in the z-buffer (reset at the start of the next call)
  odo_project_kernel<<<dgr_blocks(n0, kThreads), kThreads, 0, st>>>(l0, w.state, max_depth_diff, w.zbuf);
  const int ib = info_blocks(n0);
  odo_info_kernel<<<ib, kThreads, 0, st>>>(l0, w.state, w.zbuf, w.part);
  dgr_info_final(w.part, ib, result + 18, st);
  odo_finish_kernel<<<1, 32, 0, st>>>(w.state, result);
  launches += 4;
  dgr_note_launches(launches);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
