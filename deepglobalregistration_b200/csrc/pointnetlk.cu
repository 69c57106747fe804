// PointNetLK (Aoki, Goforth, Srivatsan & Lucey, CVPR 2019): a PointNet feature phi(P) in R^1024 under an
// inverse-compositional Lucas-Kanade loop.  oracle/pointnetlk.py is the specification.
//
//   pnet_pack_kernel     once per checkpoint: eval-mode BatchNorm folded into each 1x1 layer in fp64, rounded to
//                        fp32 once; layers 2-5 split into TF32 hi / lo tiles in the K-major SWIZZLE_128B image the
//                        wgmma operands need (tc_common.cuh), one slab per (layer, 128 output rows, 32 inputs)
//   pnet_forward_kernel  one CTA = 128 points of one pose: pose applied in fp64 and rounded to fp32 once, layer 1
//                        (K = 3) in FFMA, layers 2-5 as 3xTF32 wgmma with every activation in shared memory; the
//                        weight slabs stream through two bulk-copy stages; layer 5's epilogue reduces the max over
//                        the tile's rows and only the 1024 maxima per pose reach global memory (integer atomicMax:
//                        the features are >= +0, so they order like their bit patterns and every run gives the
//                        same bits; a NaN's bits order above +inf, so a NaN input point makes its features NaN)
//   lk_init_kernel       the 7 Jacobian poses (I, exp(-delta e_i)), g = I
//   lk_jacobian_kernel   J = (f0 - f_i) / delta, H = J^T J (fixed-order block reductions), the Cholesky check
//   lk_step_kernel       r = phi(g S) - f0, dx = -H^-1 J^T r, |dx| < xtol test, g <- exp(dx) g
//   lk_final_kernel      pose = translate(mean_T) g translate(-mean_S)
// All max_iter (forward, step) pairs are enqueued up front; every kernel returns at once after the device `done`
// flag is set, so a call makes no host read.  No floating-point atomics.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"
#include "kabsch.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int kF = 1024;                                  // feature width
constexpr int kTileM = 128;                               // points per CTA (two warpgroups of 64 rows)
constexpr int kThreads = 256;
__host__ __device__ constexpr int cin_of(int l) { return l == 0 ? 3 : l < 4 ? 64 : 128; }
__host__ __device__ constexpr int cout_of(int l) { return l < 3 ? 64 : l == 3 ? 128 : 1024; }
constexpr int kNSlabs = 38;                               // 2 + 2 + 2 (layers 2-4) + 8 x 4 (layer 5)
constexpr int kHdrBytes = 6144;                           // W1 [64][3], b1 [64] (1 KB), b2..b5 (1280 floats)
constexpr int kStageBytes = 32768;                        // largest slab: 128 rows x 128 B, hi and lo
constexpr int kActChunkBytes = 2 * kTileM * 128;          // hi | lo of 32 TF32 channels for 128 rows
constexpr int kActBytes = 4 * kActChunkBytes;             // 128 channels
constexpr double kBnEps = 1e-5;

// slab k of the packed image: layers 2 and 3 hold 64-row slabs (16 KB), layers 4 and 5 128-row slabs (32 KB)
__host__ __device__ constexpr int slab_bytes(int k) { return k < 4 ? 16384 : 32768; }
__host__ __device__ constexpr int slab_offset(int k) { return kHdrBytes + (k < 4 ? k * 16384 : 65536 + (k - 4) * 32768); }
constexpr int kPackedBytes = slab_offset(kNSlabs);        // 1 185 792
static_assert(kPackedBytes == DGR_POINTNET_PACKED_BYTES, "packed size");

__host__ __device__ constexpr int param_offset(int l) {   // fp64 words before layer l in the parameter vector
  int o = 0;
  for (int i = 0; i < l; ++i) o += cout_of(i) * cin_of(i) + 5 * cout_of(i);
  return o;
}
static_assert(param_offset(5) == DGR_POINTNET_PARAMS, "parameter count");

__device__ __forceinline__ int bias_offset(int l) {       // float index in the header: b1 at 192, b2.. at 256
  return l == 0 ? 192 : 256 + (l >= 2 ? 64 : 0) + (l >= 3 ? 64 : 0) + (l >= 4 ? 128 : 0);
}

// ---------------------------------------------------------------------------------------
// packing: one thread per folded weight or bias of every layer
// ---------------------------------------------------------------------------------------
__global__ void pnet_pack_kernel(const double* __restrict__ params, unsigned char* __restrict__ packed) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int l = 0;
  int64_t rel = e;
  while (l < 5 && rel >= (int64_t)cout_of(l) * (cin_of(l) + 1)) { rel -= (int64_t)cout_of(l) * (cin_of(l) + 1); ++l; }
  if (l == 5) return;
  const int cin = cin_of(l), cout = cout_of(l);
  const double* p = params + param_offset(l);
  const double* W = p;                       // [cout][cin]
  const double* b = W + cout * cin;
  const double* gamma = b + cout;
  const double* beta = gamma + cout;
  const double* mean = beta + cout;
  const double* var = mean + cout;
  const bool is_bias = rel >= (int64_t)cout * cin;
  const int n = is_bias ? (int)(rel - (int64_t)cout * cin) : (int)(rel / cin);
  const int k = is_bias ? 0 : (int)(rel % cin);
  const double s = __ddiv_rn(gamma[n], __dsqrt_rn(__dadd_rn(var[n], kBnEps)));
  float* hdr = reinterpret_cast<float*>(packed);
  if (is_bias) {
    hdr[bias_offset(l) + n] = (float)__dadd_rn(__dmul_rn(__dsub_rn(b[n], mean[n]), s), beta[n]);
    return;
  }
  const float w = (float)__dmul_rn(W[n * cin + k], s);
  if (l == 0) { hdr[n * 3 + k] = w; return; }
  // slab of (layer, row block, 32-input chunk) and the element's place in its swizzled hi / lo tiles
  int slab, row;
  if (l < 4) { slab = 2 * (l - 1) + k / 32; row = n; }
  else { slab = 6 + (n / 128) * 4 + k / 32; row = n % 128; }
  const int rows = slab_bytes(slab) / 256;
  const int q = (k % 32) / 4;
  float* hi = reinterpret_cast<float*>(packed + slab_offset(slab));
  const int off = row * 32 + ((q ^ (row & 7)) << 2) + (k % 4);
  const float h = tf32_round(w);
  hi[off] = h;
  hi[rows * 32 + off] = w - h;
}

// ---------------------------------------------------------------------------------------
// fused forward
// ---------------------------------------------------------------------------------------
struct FwdShared {
  unsigned long long full[2];
  float hdr[kHdrBytes / 4];
  unsigned cmax[kF];
};

constexpr size_t fwd_smem_bytes() { return 1024 + kActBytes + 2 * kStageBytes + sizeof(FwdShared); }

__device__ __forceinline__ void issue_slab(const unsigned char* packed, int k, unsigned char* stage, uint32_t bar) {
  mbar_arrive_expect_tx(bar, slab_bytes(k));
  bulk_g2s(smem_u32(stage), packed + slab_offset(k), slab_bytes(k), bar);
}

// ReLU that writes +0 (never -0, whose bits would order above every feature) and keeps NaN, as torch's ReLU does
__device__ __forceinline__ float relu_nan(float x) { return (x > 0.f || x != x) ? x : 0.f; }
// max that keeps NaN (fmaxf drops it): a NaN input point makes its features NaN, as the oracle's np.max does
__device__ __forceinline__ float max_nan(float a, float b) { return (a > b || a != a) ? a : b; }

// byte offset of channel `col` (pair col, col + 1) of tile row r in the activation image (chunk col / 32)
__device__ __forceinline__ uint32_t act_off(int r, int col) {
  return (uint32_t)((col >> 5) * kActChunkBytes + r * 128 + ((((col & 31) >> 2) ^ (r & 7)) << 4) + (col & 3) * 4);
}

// relu(acc + bias) of a [64 x N] warpgroup accumulator, split hi / lo into the activation image (own rows only)
template <int N>
__device__ __forceinline__ void store_act(const float (&acc)[N / 2], const float* bias, unsigned char* act, int r0) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    const int col = 8 * i + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float x0 = acc[4 * i + 2 * h] + bias[col], x1 = acc[4 * i + 2 * h + 1] + bias[col + 1];
      const float v0 = relu_nan(x0), v1 = relu_nan(x1);
      const float h0 = tf32_round(v0), h1 = tf32_round(v1);
      const uint32_t off = act_off(r0 + 8 * h, col);
      *reinterpret_cast<float2*>(act + off) = make_float2(h0, h1);
      *reinterpret_cast<float2*>(act + kTileM * 128 + off) = make_float2(v0 - h0, v1 - h1);
    }
  }
}

// feats (uint32 bits of float [B][1024], zeroed by the caller) = max over points of phi(R (p - centre) + t)
__global__ void __launch_bounds__(kThreads, 1)
pnet_forward_kernel(const float* __restrict__ pts, int n, const double* __restrict__ centre,
                    const double* __restrict__ poses, const unsigned char* __restrict__ packed,
                    unsigned* __restrict__ feats, const int32_t* __restrict__ done) {
  if (done != nullptr && *done) return;
  extern __shared__ __align__(16) unsigned char smem_dyn[];
  unsigned char* act = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
  unsigned char* stage = act + kActBytes;
  FwdShared& sh = *reinterpret_cast<FwdShared*>(stage + 2 * kStageBytes);
  const int t = threadIdx.x, wg = t >> 7, lane = t & 31;
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * kTileM;
  const int rows = min(kTileM, n - p0);

  if (t == 0) {
    for (int s = 0; s < 2; ++s) mbar_init(smem_u32(&sh.full[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (t == 0) {
    issue_slab(packed, 0, stage, smem_u32(&sh.full[0]));
    issue_slab(packed, 1, stage + kStageBytes, smem_u32(&sh.full[1]));
  }
  for (int i = t; i < kHdrBytes / 4; i += kThreads) sh.hdr[i] = __ldg(reinterpret_cast<const float*>(packed) + i);
  for (int i = t; i < kF; i += kThreads) sh.cmax[i] = 0u;
  __syncthreads();

  // layer 1: thread pair (2 r, 2 r + 1) owns row r, 32 output channels each; padding rows repeat row 0 of the tile
  // (a duplicate point leaves the max unchanged)
  {
    const int r = t >> 1, half = t & 1;
    const int64_t src = (int64_t)p0 + (r < rows ? r : 0);
    const double* g = poses + 12 * b;
    const double c[3] = {centre ? centre[0] : 0.0, centre ? centre[1] : 0.0, centre ? centre[2] : 0.0};
    const double d[3] = {__dsub_rn((double)pts[3 * src], c[0]), __dsub_rn((double)pts[3 * src + 1], c[1]),
                         __dsub_rn((double)pts[3 * src + 2], c[2])};
    float q[3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
      q[a] = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(g[4 * a], d[0]), __dmul_rn(g[4 * a + 1], d[1])),
                                        __dmul_rn(g[4 * a + 2], d[2])),
                              g[4 * a + 3]);
#pragma unroll
    for (int pc = 0; pc < 8; ++pc) {
      float v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int o = 32 * half + 4 * pc + u;
        const float x = fmaf(sh.hdr[3 * o + 2], q[2], fmaf(sh.hdr[3 * o + 1], q[1], fmaf(sh.hdr[3 * o], q[0], sh.hdr[192 + o])));
        v[u] = relu_nan(x);
      }
      split_store(make_float4(v[0], v[1], v[2], v[3]), act + half * kActChunkBytes,
                  act + half * kActChunkBytes + kTileM * 128, (uint32_t)(r * 128 + ((pc ^ (r & 7)) << 4)));
    }
  }
  fence_proxy_async();
  __syncthreads();

  const int r0 = wg * 64 + ((t >> 5) & 3) * 16 + (lane >> 2);   // accumulator rows r0 and r0 + 8
  const uint32_t a_base = smem_u32(act) + wg * 64 * 128;
  int s = 0;
  // one 32-input slab of the current layer: D[64, N] += A[chunk c] . slab^T, then hand the stage to slab s + 2
  auto slab_step = [&](auto& acc, auto n_tag, int c) {
    constexpr int N = decltype(n_tag)::value;
    const int st = s & 1;
    mbar_wait(smem_u32(&sh.full[st]), (s >> 1) & 1);
    wgmma_fence();
    const uint32_t a = a_base + c * kActChunkBytes;
    const uint32_t bh = smem_u32(stage + st * kStageBytes);
    mma_chunk<N, false, 3>(acc, a, a + kTileM * 128, bh, bh + slab_bytes(s) / 2);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(acc);
    __syncthreads();
    if (t == 0 && s + 2 < kNSlabs) issue_slab(packed, s + 2, stage + st * kStageBytes, smem_u32(&sh.full[st]));
    ++s;
  };
  using N64 = std::integral_constant<int, 64>;
  using N128 = std::integral_constant<int, 128>;
  // layers 2 and 3 (64 -> 64), layer 4 (64 -> 128): outputs overwrite the warpgroup's own rows in place
#pragma unroll 1
  for (int l = 1; l <= 2; ++l) {
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    slab_step(acc, N64{}, 0);
    slab_step(acc, N64{}, 1);
    store_act<64>(acc, sh.hdr + bias_offset(l), act, r0);
    fence_proxy_async();
    __syncthreads();
  }
  {
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    slab_step(acc, N128{}, 0);
    slab_step(acc, N128{}, 1);
    store_act<128>(acc, sh.hdr + bias_offset(3), act, r0);
    fence_proxy_async();
    __syncthreads();
  }
  // layer 5 (128 -> 1024) in 8 blocks of 128 outputs; epilogue: relu, max over the tile's rows
  const float* b5 = sh.hdr + bias_offset(4);
#pragma unroll 1
  for (int nb = 0; nb < 8; ++nb) {
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll 1
    for (int c = 0; c < 4; ++c) slab_step(acc, N128{}, c);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int col = nb * 128 + 8 * i + 2 * (lane & 3);
      float m[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float x0 = acc[4 * i + e] + b5[col + e], x1 = acc[4 * i + 2 + e] + b5[col + e];
        m[e] = max_nan(relu_nan(x0), relu_nan(x1));
      }
#pragma unroll
      for (int d = 4; d < 32; d <<= 1) {
        m[0] = max_nan(m[0], __shfl_xor_sync(0xffffffffu, m[0], d));
        m[1] = max_nan(m[1], __shfl_xor_sync(0xffffffffu, m[1], d));
      }
      if (lane < 4) {
        atomicMax(&sh.cmax[col], __float_as_uint(m[0]));
        atomicMax(&sh.cmax[col + 1], __float_as_uint(m[1]));
      }
    }
  }
  __syncthreads();
  for (int i = t; i < kF; i += kThreads)
    if (sh.cmax[i] != 0u) atomicMax(feats + (size_t)b * kF + i, sh.cmax[i]);
}

// ---------------------------------------------------------------------------------------
// Lucas-Kanade
// ---------------------------------------------------------------------------------------
struct LkState {         // g first: the forward reads it as its pose
  double g[12];          // current pose (row-major [R | t]) in the centred frames
  double H[21];          // J^T J, upper triangle row-major
  double last_dx, last_r;
  int32_t iterations, status, done, pad;
};

struct LkWs {
  double* stat;          // [8] dgr_cloud_stats
  double* jposes;        // [7][12]
  LkState* st;
  unsigned* fj;          // [7][1024] Jacobian features (f0 first)
  unsigned* f;           // [1024] features of the current iterate
  double* J;             // [1024][6]
};

int64_t lk_layout(uint64_t* base, LkWs* w) {
  const int64_t sizes[6] = {8, 84, (int64_t)(sizeof(LkState) + 7) / 8, 7 * kF / 2, kF / 2, 6 * kF};
  int64_t ofs[6], total = 0;
  for (int k = 0; k < 6; ++k) { ofs[k] = total; total += sizes[k]; }
  if (base != nullptr) {
    w->stat = reinterpret_cast<double*>(base + ofs[0]);
    w->jposes = reinterpret_cast<double*>(base + ofs[1]);
    w->st = reinterpret_cast<LkState*>(base + ofs[2]);
    w->fj = reinterpret_cast<unsigned*>(base + ofs[3]);
    w->f = reinterpret_cast<unsigned*>(base + ofs[4]);
    w->J = reinterpret_cast<double*>(base + ofs[5]);
  }
  return total;
}

// SE(3) exponential of xi = (omega, v): [R | t] row-major, R = I + A W + B W^2, t = (I + B W + C W^2) v
__device__ void se3_exp(const double xi[6], double E[12]) {
  const double w0 = xi[0], w1 = xi[1], w2 = xi[2];
  const double th2 = w0 * w0 + w1 * w1 + w2 * w2, th = sqrt(th2);
  double A, B, C;
  if (th < 1e-2) {         // Taylor series: the closed forms lose digits to cancellation here
    A = 1.0 - th2 / 6.0 * (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0 * (1.0 - th2 / 72.0)));
    B = 0.5 * (1.0 - th2 / 12.0 * (1.0 - th2 / 30.0 * (1.0 - th2 / 56.0 * (1.0 - th2 / 90.0))));
    C = (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0 * (1.0 - th2 / 72.0 * (1.0 - th2 / 110.0)))) / 6.0;
  } else {
    A = sin(th) / th;
    B = (1.0 - cos(th)) / th2;
    C = (th - sin(th)) / (th2 * th);
  }
  const double W[3][3] = {{0.0, -w2, w1}, {w2, 0.0, -w0}, {-w1, w0, 0.0}};
  double W2[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) W2[r][c] = W[r][0] * W[0][c] + W[r][1] * W[1][c] + W[r][2] * W[2][c];
  for (int r = 0; r < 3; ++r) {
    double t = 0.0;
    for (int c = 0; c < 3; ++c) {
      const double id = r == c ? 1.0 : 0.0;
      E[4 * r + c] = id + A * W[r][c] + B * W2[r][c];
      t += (id + B * W[r][c] + C * W2[r][c]) * xi[3 + c];
    }
    E[4 * r + 3] = t;
  }
}

// fixed-order sum of one double per thread over a 1024-thread block; valid in every thread
__device__ double block_sum_1024(double v, double* red) {
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int k = 0; k < 32; ++k) s += red[k];
  return s;
}

__global__ void lk_init_kernel(double delta, LkWs w) {
  const int i = threadIdx.x;
  if (i < 7) {
    double xi[6] = {0, 0, 0, 0, 0, 0};
    if (i > 0) xi[i - 1] = -delta;
    se3_exp(xi, w.jposes + 12 * i);          // exp(0) = I exactly (Taylor branch)
  }
  if (i < 12) w.st->g[i] = i % 5 == 0 ? 1.0 : 0.0;
  if (i == 0) {
    w.st->last_dx = 0.0;
    w.st->last_r = 0.0;
    w.st->iterations = 0;
    w.st->status = 0;
    w.st->done = 0;
  }
}

__global__ void __launch_bounds__(kF) lk_jacobian_kernel(double delta, LkWs w, double* jac_out) {
  __shared__ double red[32];
  const int k = threadIdx.x;
  const double f0 = (double)__uint_as_float(w.fj[k]);
  double J[6];
  for (int i = 0; i < 6; ++i) {
    J[i] = (f0 - (double)__uint_as_float(w.fj[(i + 1) * kF + k])) / delta;
    w.J[6 * k + i] = J[i];
    if (jac_out != nullptr) jac_out[6 * k + i] = J[i];
  }
  int m = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = a; b < 6; ++b) {
      const double h = block_sum_1024(J[a] * J[b], red);
      if (k == 0) w.st->H[m] = h;
      ++m;
    }
  if (k == 0) {
    const double zero[6] = {0, 0, 0, 0, 0, 0};
    double x[6];
    if (!cholesky6_step(w.st->H, zero, x)) {
      w.st->status = 1;
      w.st->done = 1;
    }
  }
}

__global__ void __launch_bounds__(kF) lk_step_kernel(int it, double xtol, LkWs w, double* log) {
  __shared__ double red[32];
  if (w.st->done) return;
  const int k = threadIdx.x;
  const double r = (double)__uint_as_float(w.f[k]) - (double)__uint_as_float(w.fj[k]);
  double jr[6];
  for (int i = 0; i < 6; ++i) jr[i] = block_sum_1024(w.J[6 * k + i] * r, red);
  const double rr = block_sum_1024(r * r, red);
  if (k != 0) return;
  LkState& st = *w.st;
  double dx[6];
  if (!cholesky6_step(st.H, jr, dx))
    for (int i = 0; i < 6; ++i) dx[i] = 0.0;
  const double ndx = sqrt(dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2] + dx[3] * dx[3] + dx[4] * dx[4] + dx[5] * dx[5]);
  if (log != nullptr) {
    double* row = log + 16 * it;
    for (int i = 0; i < 12; ++i) row[i] = st.g[i];
    row[12] = ndx;
    row[13] = sqrt(rr);
    row[14] = 0.0;
    row[15] = 0.0;
  }
  st.iterations = it + 1;
  st.last_dx = ndx;
  st.last_r = sqrt(rr);
  if (ndx < xtol) {
    st.done = 1;
    return;
  }
  double E[12], g[12];
  se3_exp(dx, E);
  for (int i = 0; i < 12; ++i) g[i] = st.g[i];
  for (int r2 = 0; r2 < 3; ++r2)
    for (int c = 0; c < 4; ++c)
      st.g[4 * r2 + c] = E[4 * r2] * g[c] + E[4 * r2 + 1] * g[4 + c] + E[4 * r2 + 2] * g[8 + c] + (c == 3 ? E[4 * r2 + 3] : 0.0);
}

__global__ void lk_final_kernel(LkWs w, int64_t n_src, int64_t n_tgt, double* result) {
  if (threadIdx.x != 0) return;
  const LkState& st = *w.st;
  const double* ms = w.stat;
  const double* mt = w.stat + 4;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) result[4 * r + c] = st.g[4 * r + c];
    result[4 * r + 3] = st.g[4 * r + 3] - (st.g[4 * r] * ms[0] + st.g[4 * r + 1] * ms[1] + st.g[4 * r + 2] * ms[2]) + mt[r];
  }
  result[12] = 0; result[13] = 0; result[14] = 0; result[15] = 1;
  result[16] = st.iterations;
  result[17] = st.last_dx;
  result[18] = st.last_r;
  result[19] = st.status;
  result[20] = (double)n_src;
  result[21] = (double)n_tgt;
  result[22] = 0;                         // host reads
  for (int i = 23; i < 32; ++i) result[i] = 0;
}

int32_t launch_forward(const float* pts, int64_t n, const double* centre, const double* poses, int B,
                       const void* packed, unsigned* feats, const int32_t* done, cudaStream_t st) {
  const size_t smem = fwd_smem_bytes();
  DGR_ENSURE_SMEM(pnet_forward_kernel, smem);
  pnet_forward_kernel<<<dim3((unsigned)((n + kTileM - 1) / kTileM), B), kThreads, smem, st>>>(
      pts, (int)n, centre, poses, (const unsigned char*)packed, feats, done);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // namespace

extern "C" {

int32_t dgr_pointnet_pack(const double* params, void* packed, void* stream) {
  DGR_ARG_CHECK(params != nullptr && packed != nullptr, "null pointer");
  pnet_pack_kernel<<<dgr_blocks(DGR_POINTNET_PARAMS, 256), 256, 0, (cudaStream_t)stream>>>(params,
                                                                                           (unsigned char*)packed);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_pointnet_forward(const float* points, int64_t n, const double* centre, const double* poses, int32_t n_poses,
                             const void* packed, float* features, void* stream) {
  DGR_ARG_CHECK(points != nullptr && poses != nullptr && packed != nullptr && features != nullptr, "null pointer");
  DGR_ARG_CHECK(n >= 1 && n < (1ll << 31) - kTileM, "n must lie in [1, 2^31 - 128]");
  DGR_ARG_CHECK(n_poses >= 1 && n_poses <= 65535, "n_poses must lie in [1, 65535]");
  cudaStream_t st = (cudaStream_t)stream;
  DGR_CUDA_CHECK(cudaMemsetAsync(features, 0, sizeof(float) * kF * n_poses, st));
  const int32_t rc = launch_forward(points, n, centre, poses, n_poses, packed, reinterpret_cast<unsigned*>(features),
                                    nullptr, st);
  dgr_note_launches(1);
  return rc;
}

int32_t dgr_pointnetlk_ws_elems(int64_t n_src, int64_t n_tgt, int32_t max_iter, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_src >= 0 && n_tgt >= 0 && max_iter >= 0, "bad arguments");
  *n_elems = lk_layout(nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_pointnetlk(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, const void* packed,
                       double delta, int32_t max_iter, double xtol, uint64_t* ws, double* jac_out, double* log,
                       double* result, void* stream) {
  DGR_ARG_CHECK(src != nullptr && tgt != nullptr && packed != nullptr && ws != nullptr && result != nullptr,
                "null pointer");
  DGR_ARG_CHECK(n_src >= 1 && n_src < (1ll << 31) - kTileM && n_tgt >= 1 && n_tgt < (1ll << 31) - kTileM,
                "point counts must lie in [1, 2^31 - 128]");
  DGR_ARG_CHECK(delta > 0.0 && isfinite(delta), "delta must be positive");
  DGR_ARG_CHECK(max_iter >= 1 && max_iter <= 1000, "max_iter must lie in [1, 1000]");
  DGR_ARG_CHECK(xtol >= 0.0 && isfinite(xtol), "xtol must be >= 0");
  cudaStream_t st = (cudaStream_t)stream;
  LkWs w;
  lk_layout(ws, &w);
  int launches = 0;
  dgr_cloud_stats(src, n_src, tgt, n_tgt, w.stat, st);
  lk_init_kernel<<<1, 32, 0, st>>>(delta, w);
  DGR_CUDA_CHECK(cudaMemsetAsync(w.fj, 0, sizeof(unsigned) * 7 * kF, st));
  int32_t rc = launch_forward(tgt, n_tgt, w.stat + 4, w.jposes, 7, packed, w.fj, nullptr, st);
  if (rc != DGR_OK) return rc;
  lk_jacobian_kernel<<<1, kF, 0, st>>>(delta, w, jac_out);
  launches += 4;
  for (int it = 0; it < max_iter; ++it) {
    DGR_CUDA_CHECK(cudaMemsetAsync(w.f, 0, sizeof(unsigned) * kF, st));
    rc = launch_forward(src, n_src, w.stat, reinterpret_cast<const double*>(w.st), 1, packed, w.f,
                        reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(w.st) + offsetof(LkState, done)),
                        st);
    if (rc != DGR_OK) return rc;
    lk_step_kernel<<<1, kF, 0, st>>>(it, xtol, w, log);
    launches += 2;
  }
  lk_final_kernel<<<1, 32, 0, st>>>(w, n_src, n_tgt, result);
  dgr_note_launches(launches + 1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
