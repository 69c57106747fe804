// Correspondence post-processing and pose estimation:
//   dgr_inlier_coords      6-D coordinate assembly   (core/deep_global_registration.py:261-262)
//   dgr_sigmoid_clip_sum   inlier weights + gate sum (core/deep_global_registration.py:269-272)
//   dgr_se3_register       weighted Procrustes (core/registration.py:91-113) followed by the
//                          robust SE(3) refinement (core/registration.py:135-194) with the loss
//                          of core/loss.py:42-61.
//
// The reference runs the refinement as <=1000 PyTorch iterations of ~15 tiny kernels and
// three .item() host syncs each.  Here the whole optimisation is ONE launch: a thread-block
// cluster of 8 CTAs keeps the active (non-zero weight) correspondences resident in its
// 8 x ~200 KB of shared memory, every iteration reduces the 13 loss/gradient moments with
// warp shuffles, exchanges the per-CTA partials through distributed shared memory, and
// each CTA redundantly applies the (deterministic) Gram-Schmidt backward pass, the Adam
// update and the reference's stopping rule - no host round trip, no global memory traffic
// after the prologue.  The 3x3 SVD is a one-sided Jacobi iteration in fp64 on one thread.
#include <cooperative_groups.h>

#include "common.cuh"
#include "kabsch.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kClusterSize = 8;
constexpr int kRegThreads = 512;
constexpr int kMaxVals = 16;
constexpr int kSmemPoints = 7168;   // per CTA: 7 floats * 7168 = 196 KB

__global__ void inlier_coords_kernel(const int32_t* __restrict__ c0, const int32_t* __restrict__ c1,
                                     const int32_t* __restrict__ idx1, int64_t n0,
                                     int32_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n0) return;
  int4 a = reinterpret_cast<const int4*>(c0)[i];
  int4 b = reinterpret_cast<const int4*>(c1)[idx1[i]];
  int32_t* o = out + i * 7;
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
  o[4] = b.y; o[5] = b.z; o[6] = b.w;
}

// One CTA: thread k sums rows k, k + 1024, ... in fp64, then dgr_block_sum, so the gate sum that picks Procrustes or
// the safeguard has the same bits on every run.
constexpr int kGateThreads = 1024;

__global__ void __launch_bounds__(kGateThreads)
sigmoid_clip_sum_kernel(const float* __restrict__ logit, int64_t n, float clip, float* __restrict__ w,
                        double* wsum) {
  __shared__ double part[kGateThreads / 32][1];
  double acc[1] = {0.0};
  for (int64_t i = threadIdx.x; i < n; i += kGateThreads) {
    float s = 1.f / (1.f + expf(-logit[i]));
    if (clip > 0.f && s < clip) s = 0.f;
    w[i] = s;
    acc[0] += (double)s;
  }
  const double t = dgr_block_sum<kGateThreads>(acc, part);
  if (threadIdx.x == 0) *wsum = t;
}

// gather the correspondences into structure-of-arrays form: 7 arrays of length n
__global__ void pack_corr_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                 const int32_t* __restrict__ idx1, const float* __restrict__ w,
                                 int64_t n, float* __restrict__ pack) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t j = idx1 != nullptr ? (int64_t)idx1[i] : i;
  pack[0 * n + i] = x[3 * i + 0];
  pack[1 * n + i] = x[3 * i + 1];
  pack[2 * n + i] = x[3 * i + 2];
  pack[3 * n + i] = y[3 * j + 0];
  pack[4 * n + i] = y[3 * j + 1];
  pack[5 * n + i] = y[3 * j + 2];
  pack[6 * n + i] = w[i];
}

// ---------------------------------------------------------------------------------------
// rot6d -> R (ortho2rotation, core/registration.py:16-64) and its backward pass
// ---------------------------------------------------------------------------------------
struct Rot6dCache {
  float x[3], y[3], yr[3], nx, nu, ip, n2, f;
  bool clamp_x, clamp_n2, clamp_u;
};

__device__ void rot6d_forward(const float p[6], float R[9], Rot6dCache& c) {
  float n = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
  c.clamp_x = n < 1e-8f;
  c.nx = fmaxf(n, 1e-8f);
  for (int k = 0; k < 3; ++k) { c.x[k] = p[k] / c.nx; c.yr[k] = p[3 + k]; }
  c.ip = c.x[0] * c.yr[0] + c.x[1] * c.yr[1] + c.x[2] * c.yr[2];
  float n2 = c.x[0] * c.x[0] + c.x[1] * c.x[1] + c.x[2] * c.x[2];
  c.clamp_n2 = n2 < 1e-8f;
  c.n2 = fmaxf(n2, 1e-8f);
  c.f = c.ip / c.n2;
  float u[3];
  for (int k = 0; k < 3; ++k) u[k] = c.yr[k] - c.f * c.x[k];
  float nu = sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
  c.clamp_u = nu < 1e-8f;
  c.nu = fmaxf(nu, 1e-8f);
  for (int k = 0; k < 3; ++k) c.y[k] = u[k] / c.nu;
  float z[3] = {c.x[1] * c.y[2] - c.x[2] * c.y[1], c.x[2] * c.y[0] - c.x[0] * c.y[2],
                c.x[0] * c.y[1] - c.x[1] * c.y[0]};
  for (int k = 0; k < 3; ++k) { R[3 * k + 0] = c.x[k]; R[3 * k + 1] = c.y[k]; R[3 * k + 2] = z[k]; }
}

// G = dL/dR row-major; out g[6] = dL/d rot6d
__device__ void rot6d_backward(const Rot6dCache& c, const float G[9], float g[6]) {
  float gx[3], gy[3], gz[3];
  for (int k = 0; k < 3; ++k) { gx[k] = G[3 * k + 0]; gy[k] = G[3 * k + 1]; gz[k] = G[3 * k + 2]; }
  // z = x cross y
  float gxt[3] = {gx[0] + (c.y[1] * gz[2] - c.y[2] * gz[1]), gx[1] + (c.y[2] * gz[0] - c.y[0] * gz[2]),
                  gx[2] + (c.y[0] * gz[1] - c.y[1] * gz[0])};
  float gyt[3] = {gy[0] + (gz[1] * c.x[2] - gz[2] * c.x[1]), gy[1] + (gz[2] * c.x[0] - gz[0] * c.x[2]),
                  gy[2] + (gz[0] * c.x[1] - gz[1] * c.x[0])};
  // y = u / max(|u|, 1e-8)
  float gu[3];
  if (c.clamp_u) {
    for (int k = 0; k < 3; ++k) gu[k] = gyt[k] / c.nu;
  } else {
    float d = c.y[0] * gyt[0] + c.y[1] * gyt[1] + c.y[2] * gyt[2];
    for (int k = 0; k < 3; ++k) gu[k] = (gyt[k] - c.y[k] * d) / c.nu;
  }
  // u = y_raw - f x
  float gyr[3] = {gu[0], gu[1], gu[2]};
  float gf = -(gu[0] * c.x[0] + gu[1] * c.x[1] + gu[2] * c.x[2]);
  for (int k = 0; k < 3; ++k) gxt[k] -= c.f * gu[k];
  // f = ip / max(n2, 1e-8)
  float gip = gf / c.n2;
  float gn2 = c.clamp_n2 ? 0.f : -gf * c.ip / (c.n2 * c.n2);
  for (int k = 0; k < 3; ++k) {
    gxt[k] += gip * c.yr[k] + 2.f * gn2 * c.x[k];
    gyr[k] += gip * c.x[k];
  }
  // x = x_raw / max(|x_raw|, 1e-8)
  if (c.clamp_x) {
    for (int k = 0; k < 3; ++k) g[k] = gxt[k] / c.nx;
  } else {
    float d = c.x[0] * gxt[0] + c.x[1] * gxt[1] + c.x[2] * gxt[2];
    for (int k = 0; k < 3; ++k) g[k] = (gxt[k] - c.x[k] * d) / c.nx;
  }
  for (int k = 0; k < 3; ++k) g[3 + k] = gyr[k];
}

// ---------------------------------------------------------------------------------------
// the cluster kernel
// ---------------------------------------------------------------------------------------
struct RegShared {
  DgrReduceShared<kMaxVals, kRegThreads, kClusterSize> red;   // the per-iteration sums over the cluster
  float params[16];   // R (9) + t (3)
  int counts[kClusterSize];
  int flags[4];
};

__global__ void __cluster_dims__(kClusterSize, 1, 1) __launch_bounds__(kRegThreads, 1)
se3_register_kernel(const float* __restrict__ pack, int64_t n, float q, int max_iter,
                    int max_break_count, float break_ratio, float lr0, float gamma, float eps,
                    float* __restrict__ result) {
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  RegShared& sh = *reinterpret_cast<RegShared*>(smem_raw);
  float* pts = reinterpret_cast<float*>(smem_raw + ((sizeof(RegShared) + 15) / 16) * 16);
  const int tid = threadIdx.x;
  const unsigned rank = cluster.block_rank();
  int parity = 0;

  // ---- prologue: this CTA's slice, active correspondences compacted into shared memory ----
  const int64_t per = (n + kClusterSize - 1) / kClusterSize;
  const int64_t lo = min(n, (int64_t)rank * per), hi = min(n, lo + per);
  __shared__ int s_count;
  if (tid == 0) s_count = 0;
  __syncthreads();
  // ordered compaction, 512 candidates per round
  for (int64_t base = lo; base < hi; base += kRegThreads) {
    int64_t i = base + tid;
    float wv = (i < hi) ? pack[6 * n + i] : 0.f;
    int act = (wv != 0.f) ? 1 : 0;
    int tot;
    const int excl = dgr_block_exclusive_scan<kRegThreads>(act, &tot);
    const int pos = s_count + excl;
    if (act && pos < kSmemPoints) {
#pragma unroll
      for (int a = 0; a < 7; ++a) pts[a * kSmemPoints + pos] = pack[a * n + i];
    }
    __syncthreads();
    if (tid == 0) s_count += tot;
    __syncthreads();
  }
  const int m_local = s_count;
  // agree on the mode: resident (all slices fit) or streaming from global memory
  if (tid == 0) {
    for (unsigned r = 0; r < kClusterSize; ++r) cluster.map_shared_rank(&sh, r)->counts[rank] = m_local;
  }
  cluster.sync();
  bool resident = true;
  int m_total = 0;
  for (int r = 0; r < kClusterSize; ++r) {
    resident = resident && (sh.counts[r] <= kSmemPoints);
    m_total += sh.counts[r];
  }
  const int64_t cnt = resident ? (int64_t)m_local : (hi - lo);
  auto load_pt = [&](int64_t k, float (&x)[3], float (&y)[3], float& w) {
    if (resident) {
      x[0] = pts[0 * kSmemPoints + k]; x[1] = pts[1 * kSmemPoints + k]; x[2] = pts[2 * kSmemPoints + k];
      y[0] = pts[3 * kSmemPoints + k]; y[1] = pts[4 * kSmemPoints + k]; y[2] = pts[5 * kSmemPoints + k];
      w = pts[6 * kSmemPoints + k];
    } else {
      const int64_t i = lo + k;
      x[0] = pack[0 * n + i]; x[1] = pack[1 * n + i]; x[2] = pack[2 * n + i];
      y[0] = pack[3 * n + i]; y[1] = pack[4 * n + i]; y[2] = pack[5 * n + i];
      w = pack[6 * n + i];
    }
  };

  // ---- weighted Procrustes: first moments -------------------------------------------------
  // Procrustes normalises by sum |w| (core/registration.py:96), the loss by sum w (core/loss.py:61)
  {
    double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t k = tid; k < cnt; k += kRegThreads) {
      float x[3], y[3], w;
      load_pt(k, x, y, w);
      a[0] += fabsf(w);
      a[1] += w * x[0]; a[2] += w * x[1]; a[3] += w * x[2];
      a[4] += w * y[0]; a[5] += w * y[1]; a[6] += w * y[2];
      a[7] += w;
    }
    for (int k = 0; k < 8; ++k) v[k] = (double)a[k];
    dgr_allreduce<kClusterSize>(sh.red, v, parity);
  }
  const double W1 = sh.red.tot[0], Wsum = sh.red.tot[7];
  const float wden = (float)W1 + eps;
  float mux[3], muy[3];
  for (int k = 0; k < 3; ++k) {
    mux[k] = (float)(sh.red.tot[1 + k] / (double)wden);
    muy[k] = (float)(sh.red.tot[4 + k] / (double)wden);
  }
  __syncthreads();
  // ---- second moments Sxy = sum wn (y - muy)(x - mux)^T -------------------------------------
  {
    float a[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t k = tid; k < cnt; k += kRegThreads) {
      float x[3], y[3], w;
      load_pt(k, x, y, w);
      const float wn = w / wden;
      const float dx[3] = {wn * (x[0] - mux[0]), wn * (x[1] - mux[1]), wn * (x[2] - mux[2])};
      const float dy[3] = {y[0] - muy[0], y[1] - muy[1], y[2] - muy[2]};
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) a[3 * r + c] += dy[r] * dx[c];
    }
    double v[9];
    for (int k = 0; k < 9; ++k) v[k] = (double)a[k];
    dgr_allreduce<kClusterSize>(sh.red, v, parity);
  }
  if (tid == 0) {
    double S[3][3], R[3][3];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) S[r][c] = (double)(float)sh.red.tot[3 * r + c];   // fp32 Sxy, as the reference
    if (m_total > 0) {
      kabsch_rotation(S, R);
    } else {
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[r][c] = (r == c);
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) sh.params[3 * r + c] = (float)R[r][c];
    for (int r = 0; r < 3; ++r) {
      float rm = sh.params[3 * r + 0] * mux[0] + sh.params[3 * r + 1] * mux[1] + sh.params[3 * r + 2] * mux[2];
      sh.params[9 + r] = muy[r] - rm;
    }
  }
  __syncthreads();

  // ---- refinement state (replicated in thread 0 of every CTA) --------------------------------
  float p6[6], tr[3], m1[9], m2[9];
  double lr = lr0, b1t = 1.0, b2t = 1.0;
  float loss_prev = 0.f, loss = 0.f;
  int breaks = 0, iters = 0;
  Rot6dCache cache;
  if (tid == 0) {
    for (int k = 0; k < 3; ++k) { p6[k] = sh.params[3 * k + 0]; p6[3 + k] = sh.params[3 * k + 1]; tr[k] = sh.params[9 + k]; }
    for (int k = 0; k < 9; ++k) m1[k] = m2[k] = 0.f;
  }
  const float invq = 1.f / q;
  for (int it = 0; it < max_iter; ++it) {
    iters = it;
    if (tid == 0) {
      float R[9];
      rot6d_forward(p6, R, cache);
      for (int k = 0; k < 9; ++k) sh.params[k] = R[k];
      for (int k = 0; k < 3; ++k) sh.params[9 + k] = tr[k];
    }
    __syncthreads();
    float R[9], t[3];
    for (int k = 0; k < 9; ++k) R[k] = sh.params[k];
    for (int k = 0; k < 3; ++k) t[k] = sh.params[9 + k];
    float a[13];
#pragma unroll
    for (int k = 0; k < 13; ++k) a[k] = 0.f;
    for (int64_t k = tid; k < cnt; k += kRegThreads) {
      float x[3], y[3], w;
      load_pt(k, x, y, w);
      float r[3];
#pragma unroll
      for (int c = 0; c < 3; ++c)
        r[c] = ((R[3 * c + 0] * x[0] + R[3 * c + 1] * x[1] + R[3 * c + 2] * x[2] + t[c]) - y[c]) / q;
      const float s = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
      float rho, drho;   // rho(s), d rho / d s
      if (s < 1.f) {
        rho = 0.5f * s;
        drho = 0.5f;
      } else {
        const float rt = sqrtf(s + eps);
        rho = 0.5f * (rt - 0.5f);
        drho = 0.25f / rt;
      }
      a[0] += w * rho;
      const float gs = w * drho * 2.f * invq;
      const float g[3] = {gs * r[0], gs * r[1], gs * r[2]};
      a[1] += g[0]; a[2] += g[1]; a[3] += g[2];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        a[4 + 3 * c + 0] += g[c] * x[0];
        a[4 + 3 * c + 1] += g[c] * x[1];
        a[4 + 3 * c + 2] += g[c] * x[2];
      }
    }
    double v[13];
#pragma unroll
    for (int k = 0; k < 13; ++k) v[k] = (double)a[k];
    dgr_allreduce<kClusterSize>(sh.red, v, parity);
    // every thread evaluates the stop rule on identical data so the cluster stays in lock step
    const double w1 = Wsum;
    loss = (float)(sh.red.tot[0] / w1);
    if (it == 0) loss_prev = loss;   // the reference evaluates loss_prev on the initial pose
    if (loss < 1e-7f) break;
    if (tid == 0) {
      float G[9], grad[9];
      for (int k = 0; k < 9; ++k) G[k] = (float)(sh.red.tot[4 + k] / w1);
      rot6d_backward(cache, G, grad);
      for (int k = 0; k < 3; ++k) grad[6 + k] = (float)(sh.red.tot[1 + k] / w1);
      b1t *= 0.9;
      b2t *= 0.999;
      const float step_size = (float)(lr / (1.0 - b1t));
      const float bc2_sqrt = (float)sqrt(1.0 - b2t);
      for (int k = 0; k < 9; ++k) {
        m1[k] = m1[k] + (grad[k] - m1[k]) * 0.1f;
        m2[k] = m2[k] * 0.999f + grad[k] * grad[k] * 0.001f;
        const float denom = sqrtf(m2[k]) / bc2_sqrt + 1e-8f;
        const float upd = step_size * (m1[k] / denom);
        if (k < 6) p6[k] -= upd; else tr[k - 6] -= upd;
      }
      lr *= (double)gamma;
    }
    bool stop = false;
    if (fabsf(loss_prev - loss) < loss_prev * break_ratio) {
      ++breaks;
      if (breaks >= max_break_count) stop = true;
    }
    loss_prev = loss;
    if (stop) break;
  }
  if (rank == 0 && tid == 0) {
    float R[9];
    if (max_iter > 0) {
      rot6d_forward(p6, R, cache);
    } else {
      for (int k = 0; k < 9; ++k) R[k] = sh.params[k];
      for (int k = 0; k < 3; ++k) tr[k] = sh.params[9 + k];
    }
    for (int k = 0; k < 9; ++k) result[k] = R[k];
    for (int k = 0; k < 3; ++k) result[9 + k] = tr[k];
    result[12] = (float)iters;
    result[13] = loss;
    result[14] = (float)breaks;
    result[15] = (float)m_total;
  }
  cluster.sync();   // nobody exits while peers may still write into its shared memory
}

}  // namespace

extern "C" {

int32_t dgr_inlier_coords(const int32_t* coords0, const int32_t* coords1, const int32_t* idx1,
                          int64_t n0, int32_t* out, void* stream) {
  if (n0 == 0) return DGR_OK;
  inlier_coords_kernel<<<dgr_blocks(n0, 256), 256, 0, (cudaStream_t)stream>>>(coords0, coords1, idx1, n0,
                                                                           out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_sigmoid_clip_sum(const float* logit, int64_t n, float clip, float* w, double* wsum,
                             void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  sigmoid_clip_sum_kernel<<<1, kGateThreads, 0, st>>>(logit, n, clip, w, wsum);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_se3_register(const float* x, const float* y, const int32_t* idx1, const float* w,
                         int64_t n, float quantization_size, int32_t max_iter,
                         int32_t max_break_count, float break_threshold_ratio, float lr, float gamma,
                         float* pack_ws, int32_t* cnt_ws, float* result, void* stream) {
  (void)cnt_ws;
  DGR_ARG_CHECK(n >= 1, "need at least one correspondence");
  DGR_ARG_CHECK(quantization_size > 0, "quantization_size must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  pack_corr_kernel<<<dgr_blocks(n, 256), 256, 0, st>>>(x, y, idx1, w, n, pack_ws);
  const size_t smem = ((sizeof(RegShared) + 15) / 16) * 16 + (size_t)7 * kSmemPoints * sizeof(float);
  DGR_ENSURE_SMEM(se3_register_kernel, smem);
  const float eps = 1.1920928955078125e-07f;   // np.finfo(np.float32).eps, core/loss.py:44
  se3_register_kernel<<<kClusterSize, kRegThreads, smem, st>>>(pack_ws, n, quantization_size, max_iter,
                                                              max_break_count, break_threshold_ratio,
                                                              lr, gamma, eps, result);
  dgr_note_launches(2);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
