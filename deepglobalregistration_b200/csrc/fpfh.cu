// FPFH features: open3d 0.10's ComputeFPFHFeature(KDTreeSearchParamHybrid(radius, max_nn)) on a cloud with normals,
// restated in oracle/fpfh.py (which pins every convention).  The cloud is searched through its own voxel hash (a
// dgr_unique_first table with at most one point per cell), reach = ceil(radius / cell) <= 6.  No atomics: every
// sum has a fixed order, so a call gives the same bits on every run.
//   fpfh_neighbour_kernel  a warp per point: the in-radius keys (dgr_gather_in_radius); the first max_nn without the
//                          point itself, with their fp64 d^2, into the workspace in rank order
//   fpfh_spfh_kernel       a warp per point: the fp64 pair features of its list, the 33 bin counts by ballot, each
//                          bin = 100 / m added count times
//   fpfh_kernel            4 threads per point: threads 0..2 the weighted sums of one 11-bin group over the
//                          neighbours' SPFH rows in list order, the scaling and the point's own SPFH (explicit
//                          round-to-nearest fp64, no contraction), rounded to float once; thread 3 the zero columns
//                          33 .. ld - 1
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace {

constexpr int kWarps = 4;                               // neighbour / SPFH kernels: warps (points) per block
constexpr int kBins = 11;
constexpr int kDim = 3 * kBins;
constexpr int kMaxReach = 6;
constexpr int kMaxNN = 128;
constexpr int kFpfhThreads = 128;                       // fpfh_kernel: 32 points x 4 threads

struct FpfhWs {
  double* d2;          // [n, max_nn] d^2 of the kept neighbours, rank order
  double* spfh;        // [n, 33]
  int32_t* nb;         // [n, max_nn] rows of the kept neighbours
  int32_t* m;          // [n] kept neighbours (without the point itself)
};

// workspace size in 8-byte words; carves `base` when it is not null
int64_t fpfh_layout(int64_t n, int max_nn, void* base, FpfhWs* ws) {
  const int64_t K = max_nn;
  DgrCarver c(base);
  FpfhWs w;
  w.d2 = c.take<double>(n * K);
  w.spfh = c.take<double>(n * kDim);
  w.nb = c.take<int32_t>(n * K);
  w.m = c.take<int32_t>(n);
  if (ws != nullptr) *ws = w;
  return c.words;
}

__global__ void __launch_bounds__(kWarps * 32)
fpfh_neighbour_kernel(const float* __restrict__ xyz, int64_t n, const dgr_keyspec_t* __restrict__ spec_p,
                      const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask,
                      int32_t batch, double cell, int reach, double r2, double gap_limit, int slots, int max_nn,
                      FpfhWs ws, int32_t* __restrict__ counts) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarps + warp;
  if (i >= n) return;                                   // uniform per warp
  double* kd = reinterpret_cast<double*>(smem_raw) + (size_t)warp * slots;
  int32_t* kj = reinterpret_cast<int32_t*>(reinterpret_cast<double*>(smem_raw) + (size_t)kWarps * slots) +
                (size_t)warp * slots;
  const dgr_keyspec_t s = *spec_p;
  const double p[3] = {(double)xyz[3 * i], (double)xyz[3 * i + 1], (double)xyz[3 * i + 2]};
  const int cnt = dgr_gather_in_radius(xyz, p, cell, reach, r2, gap_limit, batch, s, keys, vals, mask, kd, kj);
  // the point itself (d^2 = 0: rank 0 when present, rows being distinct points) is dropped; the others keep
  // their rank among the first max_nn, shifted down by one
  bool self = false;
  for (int k = lane; k < cnt; k += 32) self = self || kj[k] == (int32_t)i;
  const int has_self = __any_sync(0xffffffffu, self) ? 1 : 0;
  const int K = max_nn;
  for (int k = lane; k < cnt; k += 32) {
    const double dk = kd[k];
    const int32_t jk = kj[k];
    if (jk == (int32_t)i) continue;
    const int rank = dgr_key_rank(kd, kj, cnt, dk, jk);
    if (rank < max_nn) {
      const int pos = rank - has_self;
      ws.nb[i * K + pos] = jk;
      ws.d2[i * K + pos] = dk;
    }
  }
  if (lane == 0) {
    counts[i] = cnt;
    ws.m[i] = min(cnt, max_nn) - has_self;
  }
}

__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2];
}

__device__ __forceinline__ void cross3(const double a[3], const double b[3], double out[3]) {
  out[0] = a[1] * b[2] - a[2] * b[1];
  out[1] = a[2] * b[0] - a[0] * b[2];
  out[2] = a[0] * b[1] - a[1] * b[0];
}

__device__ __forceinline__ int clamp_bin(double scaled) {
  const int b = (int)floor(scaled);
  return b < 0 ? 0 : (b >= kBins ? kBins - 1 : b);
}

// open3d's ComputePairFeatures of (p1, n1) -> (p2, n2), binned: the three bins (0 .. 32) of (alpha, phi, theta);
// a degenerate pair (|d| = 0 or |v| = 0) gives the zero feature, bins 5, 16, 27
__device__ void pair_bins(const double p1[3], const double n1[3], const double p2[3], const double n2[3],
                          int out[3]) {
  double alpha = 0.0, phi = 0.0, theta = 0.0;
  double d[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const double dn = sqrt(dot3(d, d));
  if (dn != 0.0) {
    const double a1 = dot3(n1, d) / dn, a2 = dot3(n2, d) / dn;
    const bool swap = acos(fabs(a1)) > acos(fabs(a2));
    const double* m1 = swap ? n2 : n1;
    const double* m2 = swap ? n1 : n2;
    if (swap)
      for (int a = 0; a < 3; ++a) d[a] = -d[a];
    double v[3], w[3];
    cross3(d, m1, v);
    const double vn = sqrt(dot3(v, v));
    if (vn != 0.0) {
      for (int a = 0; a < 3; ++a) v[a] /= vn;
      cross3(m1, v, w);
      theta = swap ? -a2 : a1;
      phi = dot3(v, m2);
      alpha = atan2(dot3(w, m2), dot3(m1, m2));
    }
  }
  out[0] = clamp_bin(11.0 * (alpha + M_PI) / (2.0 * M_PI));
  out[1] = kBins + clamp_bin(11.0 * (phi + 1.0) * 0.5);
  out[2] = 2 * kBins + clamp_bin(11.0 * (theta + 1.0) * 0.5);
}

__global__ void __launch_bounds__(kWarps * 32)
fpfh_spfh_kernel(const float* __restrict__ xyz, const float* __restrict__ normals, int64_t n, int max_nn,
                 FpfhWs ws) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarps + warp;
  if (i >= n) return;                                   // uniform per warp
  const int K = max_nn;
  const int m = ws.m[i];
  const double p1[3] = {(double)xyz[3 * i], (double)xyz[3 * i + 1], (double)xyz[3 * i + 2]};
  const double n1[3] = {(double)normals[3 * i], (double)normals[3 * i + 1], (double)normals[3 * i + 2]};
  // lane l counts bin l, and lane 0 also bin 32
  int own = 0, own32 = 0;
  for (int k0 = 0; k0 < m; k0 += 32) {
    const int k = k0 + lane;
    int b[3] = {-1, -1, -1};
    if (k < m) {
      const int64_t j = ws.nb[i * K + k];
      const double p2[3] = {(double)xyz[3 * j], (double)xyz[3 * j + 1], (double)xyz[3 * j + 2]};
      const double n2[3] = {(double)normals[3 * j], (double)normals[3 * j + 1], (double)normals[3 * j + 2]};
      pair_bins(p1, n1, p2, n2, b);
    }
#pragma unroll
    for (int g = 0; g < 3; ++g)
      for (int q = 0; q < kBins; ++q) {
        const int bin = g * kBins + q;
        const int c = __popc(__ballot_sync(0xffffffffu, b[g] == bin));
        if (bin == lane) own += c;
        if (bin == 32 && lane == 0) own32 += c;
      }
  }
  // every addend is 100 / m: repeated addition, the same sum in any pair order
  const double incr = m > 0 ? __ddiv_rn(100.0, (double)m) : 0.0;
  double v = 0.0, v32 = 0.0;
  for (int t = 0; t < own; ++t) v = __dadd_rn(v, incr);
  for (int t = 0; t < own32; ++t) v32 = __dadd_rn(v32, incr);
  ws.spfh[i * kDim + lane] = v;
  if (lane == 0) ws.spfh[i * kDim + 32] = v32;
}

__global__ void __launch_bounds__(kFpfhThreads)
fpfh_kernel(int64_t n, int max_nn, FpfhWs ws, int ld, float* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * kFpfhThreads + threadIdx.x;
  const int64_t i = t >> 2;
  const int g = (int)(t & 3);
  if (i >= n) return;
  float* row = out + i * ld;
  if (g == 3) {
    for (int q = kDim; q < ld; ++q) row[q] = 0.0f;
    return;
  }
  const int K = max_nn;
  const int m = ws.m[i];
  double f[kBins];
#pragma unroll
  for (int q = 0; q < kBins; ++q) f[q] = 0.0;
  if (m > 0) {
    double sum = 0.0;
    for (int k = 0; k < m; ++k) {
      const double dist = ws.d2[i * K + k];
      if (dist == 0.0) continue;
      const double* nbr = ws.spfh + (int64_t)ws.nb[i * K + k] * kDim + g * kBins;
#pragma unroll
      for (int q = 0; q < kBins; ++q) {
        const double val = __ddiv_rn(nbr[q], dist);
        f[q] = __dadd_rn(f[q], val);
        sum = __dadd_rn(sum, val);
      }
    }
    const double* own = ws.spfh + i * kDim + g * kBins;
    if (sum != 0.0) {
      const double scale = __ddiv_rn(100.0, sum);
#pragma unroll
      for (int q = 0; q < kBins; ++q) f[q] = __dadd_rn(__dmul_rn(f[q], scale), own[q]);
    } else {
#pragma unroll
      for (int q = 0; q < kBins; ++q) f[q] = __dadd_rn(f[q], own[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < kBins; ++q) row[g * kBins + q] = __double2float_rn(f[q]);
}

}  // namespace

extern "C" {

int32_t dgr_fpfh_ws_elems(int64_t n, int32_t max_nn, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n >= 0, "bad arguments");
  DGR_ARG_CHECK(max_nn >= 1 && max_nn <= kMaxNN, "max_nn must lie in [1, 128]");
  *n_elems = fpfh_layout(n, max_nn, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_compute_fpfh(const float* xyz, const float* normals, int64_t n, const dgr_keyspec_t* spec,
                         const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t batch, double cell,
                         double radius, int32_t max_nn, int32_t ld, void* ws, float* out, int32_t* counts,
                         void* stream) {
  DGR_ARG_CHECK(n >= 0 && n < (1ll << 31), "point count out of range");
  DGR_ARG_CHECK(normals != nullptr, "normals are required");
  DGR_ARG_CHECK(n == 0 || (xyz != nullptr && spec != nullptr && keys != nullptr && vals != nullptr && ws != nullptr &&
                           out != nullptr && counts != nullptr), "null pointer");
  DGR_TRY(dgr_check_hash_search(cap, cell, radius, kMaxReach));
  DGR_ARG_CHECK(max_nn >= 1 && max_nn <= kMaxNN, "max_nn must lie in [1, 128]");
  DGR_ARG_CHECK(ld >= kDim, "row stride ld must be at least 33");
  if (n == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  FpfhWs w;
  fpfh_layout(n, max_nn, ws, &w);
  const int reach = (int)ceil(radius / cell);
  const double gap_limit = dgr_gap_limit(radius, cell);
  const int slots = dgr_live_cells(reach, gap_limit);
  const size_t smem = (size_t)kWarps * slots * (sizeof(double) + sizeof(int32_t));     // < 103 KB (reach 6)
  DGR_ENSURE_SMEM(fpfh_neighbour_kernel, smem);
  fpfh_neighbour_kernel<<<dgr_blocks(n, kWarps), kWarps * 32, smem, st>>>(
      xyz, n, spec, keys, vals, (uint64_t)cap - 1, batch, cell, reach, radius * radius, gap_limit, slots, max_nn, w,
      counts);
  fpfh_spfh_kernel<<<dgr_blocks(n, kWarps), kWarps * 32, 0, st>>>(xyz, normals, n, max_nn, w);
  fpfh_kernel<<<dgr_blocks(n * 4, kFpfhThreads), kFpfhThreads, 0, st>>>(n, max_nn, w, ld, out);
  dgr_note_launches(3);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
