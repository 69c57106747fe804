// The normalised frame and the distance transform of the target (frame.cu), shared by FGR, Go-ICP, Super4PCS and
// PointNetLK.  Cloud c (source 0, target 1) has fp64 statistics stat[4 c .. 4 c + 3] = mean xyz and largest centred
// norm; the normalised frame is x -> (x - mean) / s with s = frame scale.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// Go-ICP's source bound (its shared-memory arrays hold the source) and the largest grid side (dt_fh_kernel's envelope)
constexpr int kGoicpMaxSrc = 1024;
constexpr int kDtMaxG = 512;

// one launch of 2 CTAs: stat of the source and of the target, each in a fixed order
void dgr_cloud_stats(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, double* stat, cudaStream_t st);
// Go-ICP's argument bounds on the clouds and the grid (dgr_goicp_dt_build, dgr_goicp)
int32_t dgr_goicp_dt_check(int64_t n_src, int64_t n_tgt, int32_t G, double e);
// dgr_cloud_stats, the normalised clouds (xn fp64 source, may be null; y32 fp32 target) and the G^3 distance transform
// of y32 over [-e, e]^3 (dgr_goicp_dt_build's grid).  Returns the number of launches.
int dgr_normalise_dt(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, int G, double e, double* stat,
                     double* xn, float* y32, int32_t* dt, cudaStream_t st);

// s = the larger cloud's largest centred norm, 1 when both clouds are a single point
__device__ __forceinline__ double dgr_frame_scale(const double* __restrict__ stat) {
  const double s = fmax(stat[3], stat[7]);
  return s > 0.0 ? s : 1.0;
}

// p = (x[i] - m) / scale in fp64, as oracle/fgr.py::normalise rounds it
__device__ __forceinline__ void dgr_frame_point(const float* __restrict__ x, int64_t i, const double m[3], double scale,
                                                double p[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = __ddiv_rn(__dsub_rn((double)__ldg(x + 3 * i + c), m[c]), scale);
}

// |a - b| as numpy evaluates it: sqrt((dx dx + dy dy) + dz dz), no contraction
__device__ __forceinline__ double dgr_dist3(const double a[3], const double b[3]) {
  const double dx = __dsub_rn(a[0], b[0]), dy = __dsub_rn(a[1], b[1]), dz = __dsub_rn(a[2], b[2]);
  return sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

// The 4x4 row-major pose in the input frame of the normalised pose y = R x + t (R row-major):
// x = (X - m_s) / s, y = (Y - m_t) / s  =>  Y = R X + (m_t + s t - R m_s)
__device__ __forceinline__ void dgr_frame_pose(const double R[9], const double t[3], const double* __restrict__ stat,
                                               double s, double* __restrict__ result) {
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) result[4 * a + b] = R[3 * a + b];
    result[4 * a + 3] = stat[4 + a] + s * t[a] - (R[3 * a] * stat[0] + R[3 * a + 1] * stat[1] + R[3 * a + 2] * stat[2]);
  }
  result[12] = 0.0; result[13] = 0.0; result[14] = 0.0; result[15] = 1.0;
}

// Distance-transform lookup: cell floor((q + e) / h) clamped to the grid, h sqrt(stored), plus the distance from q to
// the box [-e, e]^3; every step an IEEE fp32 operation (oracle/goicp.py, DistanceTransform.lookup).
__device__ __forceinline__ int dt_axis(float q, float e32, float h32, int G) {
  float u = floorf(__fdiv_rn(__fadd_rn(q, e32), h32));
  u = fminf(fmaxf(u, 0.f), (float)(G - 1));
  return (int)u;
}

__device__ __forceinline__ float dt_lookup(const int32_t* __restrict__ dt, int G, float e32, float h32, float qx,
                                           float qy, float qz) {
  const int ix = dt_axis(qx, e32, h32, G), iy = dt_axis(qy, e32, h32, G), iz = dt_axis(qz, e32, h32, G);
  const int v = __ldg(dt + ((int64_t)iz * G + iy) * G + ix);
  const float D = __fmul_rn(h32, __fsqrt_rn((float)v));
  const float ox = fmaxf(__fsub_rn(fabsf(qx), e32), 0.f), oy = fmaxf(__fsub_rn(fabsf(qy), e32), 0.f),
              oz = fmaxf(__fsub_rn(fabsf(qz), e32), 0.f);
  const float o2 = __fadd_rn(__fadd_rn(__fmul_rn(ox, ox), __fmul_rn(oy, oy)), __fmul_rn(oz, oz));
  return __fadd_rn(D, __fsqrt_rn(o2));
}
