// Go-ICP's distance-transform lookup (goicp.cu builds the grid), shared with super4pcs.cu: cell
// floor((q + e) / h) clamped to the grid, h sqrt(stored), plus the distance from q to the box [-e, e]^3; every step
// an IEEE fp32 operation (oracle/goicp.py, DistanceTransform.lookup).
#pragma once
#include <stdint.h>

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
