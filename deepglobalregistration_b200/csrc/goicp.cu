// Go-ICP (Yang, Li, Campbell & Jia, "Go-ICP: A Globally Optimal Solution to 3D ICP Point-Set Registration", TPAMI
// 2016): nested branch and bound over angle-axis rotation cubes and translation cubes, bounded through a distance
// transform of the target, with trimmed ICP proposing incumbents.  oracle/goicp.py restates every step (the
// specification); every bound is an fp32 lookup summed in fp64 over a fixed pairwise tree, so a bound has the same
// bits here and in numpy.
//   dgr_normalise_dt        both clouds centred on their fp64 means and divided by s, and the target's G^3 distance
//                           transform over [-e, e]^3 (frame.cu)
//   per round (one pinned host read before it):
//     goicp_round_kernel     one CTA per rotation child of the B smallest pool cubes: rotated source and gamma_r in
//                            shared memory; the upper-bound and the lower-bound inner search over translation cubes,
//                            8 warps evaluating the 8 children of a popped cube, the cube pool in shared memory
//     goicp_incumbent_kernel the (UB, key)-smallest child; when it beats E*, ICP starts from its pose (device flag)
//     30 x (dgr_knn_top1_packed, goicp_icp_step_kernel)   trimmed ICP, every launch predicated on the flag
//     goicp_eval_kernel      the objective at the ICP pose; the incumbent becomes the better pose
//     goicp_children_kernel  children with LB < E*: flags, dgr_block_scan_inplace, bitonic sort by (LB, key)
//     goicp_merge_kernel     the rest of the sorted pool (LB < E*) merged with the sorted children: the next pool
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"
#include "frame.cuh"
#include "kabsch.cuh"

namespace {

constexpr int kMaxSrc = kGoicpMaxSrc;
constexpr int kRoundThreads = 256;                       // 8 warps: one per translation child
constexpr int kInnerCap = 1536;                          // translation cubes in a CTA's shared-memory pool
constexpr int kMaxLevel = 19;                            // 3 x 19-bit cube coordinates + the level in a 64-bit key
constexpr int kMaxB = 512;                               // cubes per round: 8 B children sort in one CTA
constexpr int kIcpIters = 30;
constexpr int kIcpThreads = 1024;
constexpr int kSkew = kMaxSrc + kMaxSrc / 32;            // a term buffer, skewed so lane l reading [32 l, 32 l + 32) is
                                                         // conflict-free
constexpr double kSqrt3 = 1.7320508075688772;            // the double nearest sqrt(3)
constexpr double kPi = 3.141592653589793;
constexpr double kHalfPi = 1.5707963267948966;
constexpr double kPi2 = kPi * kPi;

struct GoHost {          // what the host reads once per round
  double E, lb_min;
  int32_t pool_n, stop;
};

struct GoState {
  GoHost h;
  double T[12];          // incumbent pose, normalised frame, row-major [R | t]
  double icpT[12];       // ICP pose
  double candT[12];      // the round's best child pose
  double candE, mse_prev;
  double children, tcubes, icp_runs, overflows, hw;
  int32_t n_child, run_icp, icp_live, icp_updates;
};
constexpr int kStateWords = 64;
static_assert(sizeof(GoState) <= kStateWords * 8, "state workspace too small");

struct ChildRec {        // 8 words
  double ub, lb, t[3];
  uint64_t key;
  int64_t tcubes;
  int32_t status;        // 0 searched, 1 outside the pi-ball, 2 parent at the finest level
  int32_t ovf;           // inner searches that overflowed their pool
};

struct GoParams {
  const double* xn;      // [n_s][3] normalised source
  const float* y32;      // [n_t][3] normalised target
  const int32_t* dt;     // [G][G][G], x fastest
  int n_s, n_t, K, Pn, trim, G;
  float e32, h32;
  double eps;
  double rmin[3], rw, tmin[3], tw;
};

struct GoWs {
  GoState* st;
  double* stat;          // [8]
  double* xn;
  float* p32;            // [n_s][3] ICP: the source at the current ICP pose
  float* y32;
  uint64_t* packed;      // [n_s]
  int32_t* dt;
  double* pool_lb[2];
  uint64_t* pool_key[2];
  ChildRec* child;       // [8 B]
  double* clb;           // [8 B] sorted children kept
  uint64_t* ckey;
};

int64_t goicp_layout(int64_t n_s, int64_t n_t, int64_t G, int64_t cap, int64_t B, uint64_t* base, GoWs* w) {
  DgrCarver c(base);
  GoWs r;
  r.st = reinterpret_cast<GoState*>(c.take<uint64_t>(kStateWords));
  r.stat = c.take<double>(8);
  r.xn = c.take<double>(3 * n_s);
  r.p32 = c.take<float>(3 * n_s);
  r.y32 = c.take<float>(3 * n_t);
  r.packed = c.take<uint64_t>(n_s);
  r.dt = c.take<int32_t>(G * G * G);
  for (int k = 0; k < 2; ++k) {
    r.pool_lb[k] = c.take<double>(cap);
    r.pool_key[k] = c.take<uint64_t>(cap);
  }
  r.child = c.take<ChildRec>(8 * B);
  r.clb = c.take<double>(8 * B);
  r.ckey = c.take<uint64_t>(8 * B);
  if (w != nullptr) *w = r;
  return c.words;
}

// ---------------------------------------------------------------------------------------
// cubes: key = level << 57 | kx << 38 | ky << 19 | kz; child o of a cube takes bits (o >> 2, o >> 1, o) & 1 in
// (x, y, z), so children ascend in key order with o
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int key_level(uint64_t k) { return (int)(k >> 57); }

__device__ __forceinline__ uint64_t key_child(uint64_t k, int o) {
  const uint64_t m = 0x7ffffull;
  const uint64_t kx = 2 * ((k >> 38) & m) + ((o >> 2) & 1), ky = 2 * ((k >> 19) & m) + ((o >> 1) & 1),
                 kz = 2 * (k & m) + (o & 1);
  return ((uint64_t)(key_level(k) + 1) << 57) | (kx << 38) | (ky << 19) | kz;
}

// centre and half-width sigma = width / 2^(L+1) of a cube of the domain (mn, width)
__device__ __forceinline__ void cube_geom(uint64_t k, const double mn[3], double width, double c[3], double& sigma) {
  const uint64_t m = 0x7ffffull;
  sigma = scalbn(width, -(key_level(k) + 1));
  const uint64_t kk[3] = {(k >> 38) & m, (k >> 19) & m, k & m};
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = __dadd_rn(mn[a], __dmul_rn(sigma, (double)(2 * kk[a] + 1)));
}

__device__ __forceinline__ bool key_less(double a, uint64_t ka, double b, uint64_t kb) {
  return a < b || (a == b && ka < kb);
}

// angle-axis r -> R (row-major), every operation rounded as numpy rounds it
__device__ void rodrigues(const double r[3], double R[9]) {
  const double th = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(r[0], r[0]), __dmul_rn(r[1], r[1])), __dmul_rn(r[2], r[2])));
  if (th == 0.0) {
    for (int q = 0; q < 9; ++q) R[q] = (q % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  const double kx = __ddiv_rn(r[0], th), ky = __ddiv_rn(r[1], th), kz = __ddiv_rn(r[2], th);
  const double c = cos(th), s = sin(th), C = __dsub_rn(1.0, c);
  R[0] = __dadd_rn(c, __dmul_rn(__dmul_rn(kx, kx), C));
  R[1] = __dsub_rn(__dmul_rn(__dmul_rn(kx, ky), C), __dmul_rn(kz, s));
  R[2] = __dadd_rn(__dmul_rn(__dmul_rn(kx, kz), C), __dmul_rn(ky, s));
  R[3] = __dadd_rn(__dmul_rn(__dmul_rn(kx, ky), C), __dmul_rn(kz, s));
  R[4] = __dadd_rn(c, __dmul_rn(__dmul_rn(ky, ky), C));
  R[5] = __dsub_rn(__dmul_rn(__dmul_rn(ky, kz), C), __dmul_rn(kx, s));
  R[6] = __dsub_rn(__dmul_rn(__dmul_rn(kx, kz), C), __dmul_rn(ky, s));
  R[7] = __dadd_rn(__dmul_rn(__dmul_rn(ky, kz), C), __dmul_rn(kx, s));
  R[8] = __dadd_rn(c, __dmul_rn(__dmul_rn(kz, kz), C));
}

// one row of R times x: (R0 x0 + R1 x1) + R2 x2, no contraction
__device__ __forceinline__ double rot_row(const double* R, const double x[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(R[0], x[0]), __dmul_rn(R[1], x[1])), __dmul_rn(R[2], x[2]));
}

__device__ __forceinline__ int sk(int i) { return i + (i >> 5); }

// Sum of leaves t[0 .. K) (fp32, widened) over the pairwise tree of 1024 leaves (zero-padding a power-of-two tree
// leaves its sum unchanged): lane l adds leaves [32 l, 32 l + 32) as a tree, the lanes combine by shfl_down.
// The sum is valid in lane 0.
__device__ __forceinline__ double warp_tree_sum(const float* t, int K, int lane) {
  double v = 0.0;
  const int base = lane * 32;
  if (base < K) {
    double a[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int i0 = base + 2 * j;
      const double x0 = i0 < K ? (double)t[sk(i0)] : 0.0, x1 = i0 + 1 < K ? (double)t[sk(i0 + 1)] : 0.0;
      a[j] = x0 + x1;
    }
#pragma unroll
    for (int w = 8; w >= 1; w >>= 1)
#pragma unroll
      for (int j = 0; j < w; ++j) a[j] = a[2 * j] + a[2 * j + 1];
    v = a[0];
  }
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) v += __shfl_down_sync(0xffffffffu, v, d);
  return v;
}

// ascending bitonic sort of t[0 .. Pn) (skewed) by one warp
__device__ __forceinline__ void warp_sort(float* t, int Pn, int lane) {
  for (int k = 2; k <= Pn; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int p = lane; p < Pn / 2; p += 32) {
        const int i = 2 * p - (p & (j - 1)), q = i + j;
        const float a = t[sk(i)], b = t[sk(q)];
        if ((a > b) == ((i & k) == 0)) { t[sk(i)] = b; t[sk(q)] = a; }
      }
      __syncwarp();
    }
}

// The two bounds of one translation cube (centre t32, gamma_t gt) for the rotated source (xs, ys, zs) with
// per-point rotation uncertainty gam (nullptr: 0): u = sum of the K smallest max(e_i - gamma_ri, 0)^2 and
// l = the same with gamma_ri + gamma_t.  One warp; valid in lane 0.
__device__ void warp_bounds(const GoParams& P, const float* xs, const float* ys, const float* zs, const float* gam,
                            const float t32[3], float gt, float* tu, float* tl, int lane, double& u, double& l) {
  for (int i = lane; i < P.n_s; i += 32) {
    const float e = dt_lookup(P.dt, P.G, P.e32, P.h32, __fadd_rn(xs[i], t32[0]), __fadd_rn(ys[i], t32[1]),
                              __fadd_rn(zs[i], t32[2]));
    const float g = gam != nullptr ? gam[i] : 0.f;
    const float du = fmaxf(__fsub_rn(e, g), 0.f), dl = fmaxf(__fsub_rn(e, __fadd_rn(g, gt)), 0.f);
    tu[sk(i)] = __fmul_rn(du, du);
    tl[sk(i)] = __fmul_rn(dl, dl);
  }
  if (P.trim) {
    for (int i = P.n_s + lane; i < P.Pn; i += 32) {
      tu[sk(i)] = __int_as_float(0x7f800000);
      tl[sk(i)] = __int_as_float(0x7f800000);
    }
    __syncwarp();
    warp_sort(tu, P.Pn, lane);
    warp_sort(tl, P.Pn, lane);
  }
  __syncwarp();
  u = warp_tree_sum(tu, P.K, lane);
  l = warp_tree_sum(tl, P.K, lane);
  __syncwarp();
}

struct RoundSmem {
  float xs[kMaxSrc], ys[kMaxSrc], zs[kMaxSrc], gam[kMaxSrc];
  float tu[kRoundThreads / 32][kSkew], tl[kRoundThreads / 32][kSkew];
  double plb[kInnerCap];
  uint64_t pkey[kInnerCap];
};

// Best-first search over translation cubes (whole CTA).  use_gam: the lower-bound pass.  -> E-bar (and the
// translation centre that set it, in t_best), tcubes += cubes evaluated, ovf = 1 when the pool overflowed.
__device__ double inner_search(const GoParams& P, RoundSmem& S, bool use_gam, double E0, double t_best[3],
                               int64_t& tcubes, int& ovf) {
  __shared__ double s_E, s_t[3], s_u[8], s_l[8], s_extra, s_left;
  __shared__ uint64_t s_cur;
  __shared__ int s_n, s_stop, s_ovf;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    S.plb[0] = 0.0;
    S.pkey[0] = 0;
    s_n = 1;
    s_E = E0;
    double sg;
    cube_geom(0, P.tmin, P.tw, s_t, sg);
    s_ovf = 0;
    s_extra = __longlong_as_double(0x7ff0000000000000ll);
    s_left = s_extra;
  }
  __syncthreads();
  int64_t evals = 0;
  while (true) {
    if (warp == 0) {
      const int n = s_n;
      double b = __longlong_as_double(0x7ff0000000000000ll);
      uint64_t bk = ~0ull;
      int bi = -1;
      for (int i = lane; i < n; i += 32)
        if (key_less(S.plb[i], S.pkey[i], b, bk)) { b = S.plb[i]; bk = S.pkey[i]; bi = i; }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, b, d);
        const uint64_t ok = __shfl_xor_sync(0xffffffffu, bk, d);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, d);
        if (oi >= 0 && (bi < 0 || key_less(ob, ok, b, bk))) { b = ob; bk = ok; bi = oi; }
      }
      if (lane == 0) {
        int stop = 0;
        if (s_ovf || bi < 0) {                          // overflow: only the smallest LB left was wanted
          stop = 1;
          s_left = fmin(bi >= 0 ? b : s_left, s_extra);
        } else {
          S.plb[bi] = S.plb[n - 1];
          S.pkey[bi] = S.pkey[n - 1];
          s_n = n - 1;
          if (s_E - b < P.eps) {
            stop = 1;
          } else if (key_level(bk) >= kMaxLevel) {      // cannot split: as an overflow, this LB is the smallest left
            stop = 1;
            s_ovf = 1;
            s_left = b;
          } else {
            s_cur = bk;
          }
        }
        s_stop = stop;
      }
    }
    __syncthreads();
    if (s_stop) break;
    {
      const uint64_t ck = key_child(s_cur, warp);
      double c[3], sg;
      cube_geom(ck, P.tmin, P.tw, c, sg);
      const float t32[3] = {__double2float_rn(c[0]), __double2float_rn(c[1]), __double2float_rn(c[2])};
      const float gt = __double2float_rn(__dmul_rn(kSqrt3, sg));
      double u, l;
      warp_bounds(P, S.xs, S.ys, S.zs, use_gam ? S.gam : nullptr, t32, gt, S.tu[warp], S.tl[warp], lane, u, l);
      if (lane == 0) { s_u[warp] = u; s_l[warp] = l; }
    }
    __syncthreads();
    evals += 8;
    if (tid == 0) {
      int best = -1;
      for (int o = 0; o < 8; ++o)                       // keys ascend with o: the first smallest u wins a tie
        if (s_u[o] < s_E && (best < 0 || s_u[o] < s_u[best])) best = o;
      if (best >= 0) {
        s_E = s_u[best];
        double sg;
        cube_geom(key_child(s_cur, best), P.tmin, P.tw, s_t, sg);
      }
      int cnt = 0;
      double mn = __longlong_as_double(0x7ff0000000000000ll);
      for (int o = 0; o < 8; ++o)
        if (s_l[o] < s_E) { ++cnt; mn = fmin(mn, s_l[o]); }
      if (s_n + cnt > kInnerCap) {
        s_ovf = 1;
        s_extra = mn;
      } else {
        for (int o = 0; o < 8; ++o)
          if (s_l[o] < s_E) {
            S.plb[s_n] = s_l[o];
            S.pkey[s_n] = key_child(s_cur, o);
            ++s_n;
          }
      }
    }
    __syncthreads();
  }
  tcubes += evals;
  ovf = s_ovf;
  for (int a = 0; a < 3; ++a) t_best[a] = s_t[a];
  double E = s_E;
  if (use_gam && s_ovf) E = fmin(E, s_left);
  __syncthreads();                                      // the shared state is reused by the next search
  return E;
}

__global__ void __launch_bounds__(kRoundThreads, 2)
goicp_round_kernel(GoParams P, const uint64_t* __restrict__ pool_key, const GoState* __restrict__ st,
                   ChildRec* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  RoundSmem& S = *reinterpret_cast<RoundSmem*>(smem_raw);
  const int c = blockIdx.x, tid = threadIdx.x;
  ChildRec& rec = out[c];
  const uint64_t pkey = pool_key[c >> 3];
  if (key_level(pkey) >= kMaxLevel) {
    if (tid == 0) { rec.status = 2; rec.ovf = 0; rec.tcubes = 0; rec.key = pkey; }
    return;
  }
  const uint64_t ck = key_child(pkey, c & 7);
  double r0[3], sr;
  cube_geom(ck, P.rmin, P.rw, r0, sr);
  double n2 = 0.0;
  {
    double d[3];
    for (int a = 0; a < 3; ++a) d[a] = fmax(__dsub_rn(fabs(r0[a]), sr), 0.0);
    n2 = __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
  }
  if (n2 > kPi2) {
    if (tid == 0) { rec.status = 1; rec.ovf = 0; rec.tcubes = 0; rec.key = ck; }
    return;
  }
  double R[9];
  rodrigues(r0, R);
  const double gr = 2.0 * sin(fmin(__dmul_rn(kSqrt3, sr) / 2.0, kHalfPi));
  for (int i = tid; i < P.n_s; i += kRoundThreads) {
    const double x[3] = {P.xn[3 * i], P.xn[3 * i + 1], P.xn[3 * i + 2]};
    S.xs[i] = __double2float_rn(rot_row(R, x));
    S.ys[i] = __double2float_rn(rot_row(R + 3, x));
    S.zs[i] = __double2float_rn(rot_row(R + 6, x));
    const double nx = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(x[0], x[0]), __dmul_rn(x[1], x[1])), __dmul_rn(x[2], x[2])));
    S.gam[i] = __double2float_rn(__dmul_rn(gr, nx));
  }
  __syncthreads();
  const double E0 = st->h.E;
  int64_t tc = 0;
  int o1 = 0, o2 = 0;
  double tb[3], tl[3];
  const double ub = inner_search(P, S, false, E0, tb, tc, o1);
  const double lb = inner_search(P, S, true, E0, tl, tc, o2);
  if (tid == 0) {
    rec.ub = ub;
    rec.lb = lb;
    for (int a = 0; a < 3; ++a) rec.t[a] = tb[a];
    rec.key = ck;
    rec.tcubes = tc;
    rec.status = 0;
    rec.ovf = o1 + o2;
  }
}

// p32 = fp32(T x) for the ICP correspondences (all threads of the block)
__device__ void icp_points(const double* __restrict__ xn, int n_s, const double* T, float* __restrict__ p32) {
  for (int i = threadIdx.x; i < n_s; i += blockDim.x)
    for (int a = 0; a < 3; ++a)
      p32[3 * i + a] = (float)(T[4 * a] * xn[3 * i] + T[4 * a + 1] * xn[3 * i + 1] + T[4 * a + 2] * xn[3 * i + 2] +
                               T[4 * a + 3]);
}

__global__ void __launch_bounds__(kIcpThreads)
goicp_init_kernel(const double* __restrict__ xn, int n_s, GoState* st, double* pool_lb, uint64_t* pool_key,
                  float* __restrict__ p32) {
  __shared__ double sT[12];
  if (threadIdx.x == 0) {
    st->h.E = __longlong_as_double(0x7ff0000000000000ll);
    st->h.lb_min = 0.0;
    st->h.pool_n = 1;
    st->h.stop = 0;
    for (int q = 0; q < 12; ++q) {
      const double v = (q % 5 == 0) ? 1.0 : 0.0;
      st->T[q] = v; st->icpT[q] = v; st->candT[q] = v; sT[q] = v;
    }
    st->candE = st->h.E;
    st->mse_prev = st->h.E;
    st->children = st->tcubes = st->overflows = 0.0;
    st->icp_runs = 1.0;
    st->hw = 1.0;
    st->n_child = 0;
    st->run_icp = 1;
    st->icp_live = 1;
    st->icp_updates = 0;
    pool_lb[0] = 0.0;
    pool_key[0] = 0;
  }
  __syncthreads();
  icp_points(xn, n_s, sT, p32);
}

// the (UB, key)-smallest searched child; ICP starts from its pose when it beats E*.  Also the round's counters.
__global__ void __launch_bounds__(kIcpThreads)
goicp_incumbent_kernel(GoParams P, const ChildRec* __restrict__ rec, int nc, GoState* st, float* __restrict__ p32) {
  __shared__ double sT[12];
  __shared__ int s_run;
  if (threadIdx.x == 0) {
    int best = -1;
    double ch = 0.0, tcub = 0.0, ov = 0.0;
    for (int c = 0; c < nc; ++c) {
      if (rec[c].status == 2) st->h.stop = 1;
      if (rec[c].status != 0) continue;
      ch += 1.0;
      tcub += (double)rec[c].tcubes;
      ov += (double)rec[c].ovf;
      if (best < 0 || key_less(rec[c].ub, rec[c].key, rec[best].ub, rec[best].key)) best = c;
    }
    st->children += ch;
    st->tcubes += tcub;
    st->overflows += ov;
    const int run = best >= 0 && rec[best].ub < st->h.E;
    if (run) {
      double r0[3], sr, R[9];
      cube_geom(rec[best].key, P.rmin, P.rw, r0, sr);
      rodrigues(r0, R);
      for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) st->candT[4 * a + b] = R[3 * a + b];
        st->candT[4 * a + 3] = rec[best].t[a];
      }
      for (int q = 0; q < 12; ++q) { st->icpT[q] = st->candT[q]; sT[q] = st->candT[q]; }
      st->candE = rec[best].ub;
      st->mse_prev = __longlong_as_double(0x7ff0000000000000ll);
      st->icp_updates = 0;
      st->icp_runs += 1.0;
    }
    st->run_icp = run;
    st->icp_live = run;
    s_run = run;
  }
  __syncthreads();
  if (s_run) icp_points(P.xn, P.n_s, sT, p32);
}

// One trimmed-ICP update: the K nearest (d^2, row) pairs of the current correspondences; stop when the trimmed MSE
// fell by less than 1e-6 of its previous value, otherwise T <- the Kabsch pose of those pairs (fp64 sums, lanes by
// butterfly, warps in order).  Stops after kIcpIters updates.
__global__ void __launch_bounds__(kIcpThreads)
goicp_icp_step_kernel(GoParams P, const uint64_t* __restrict__ packed, GoState* st, float* __restrict__ p32) {
  if (!st->icp_live) return;                            // uniform per launch
  __shared__ double sd[kMaxSrc];
  __shared__ int si[kMaxSrc];
  __shared__ double red[kIcpThreads / 32][1];
  __shared__ double tot[16];
  __shared__ double sT[12];
  __shared__ int s_live;
  const int tid = threadIdx.x;
  double T[12];
  for (int q = 0; q < 12; ++q) T[q] = st->icpT[q];
  if (tid < P.n_s) {
    const int j = (int)(packed[tid] & 0xffffffffull);
    double d2 = 0.0;
    for (int a = 0; a < 3; ++a) {
      const double p = T[4 * a] * P.xn[3 * tid] + T[4 * a + 1] * P.xn[3 * tid + 1] + T[4 * a + 2] * P.xn[3 * tid + 2] +
                       T[4 * a + 3];
      const double e = p - (double)P.y32[3 * j + a];
      d2 += e * e;
    }
    sd[tid] = d2;
    si[tid] = tid;
  } else if (tid < P.Pn) {
    sd[tid] = __longlong_as_double(0x7ff0000000000000ll);
    si[tid] = 0x7fffffff;
  }
  __syncthreads();
  for (int k = 2; k <= P.Pn; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (tid < P.Pn / 2) {
        const int i = 2 * tid - (tid & (j - 1)), q = i + j;
        const double a = sd[i], b = sd[q];
        const int ia = si[i], ib = si[q];
        const bool gt = a > b || (a == b && ia > ib);
        if (gt == ((i & k) == 0)) { sd[i] = b; sd[q] = a; si[i] = ib; si[q] = ia; }
      }
      __syncthreads();
    }
  // sums over the kept pairs: d^2, x (3), y (3), y x^T (9)
  double x[3] = {0, 0, 0}, y[3] = {0, 0, 0}, d2 = 0.0;
  if (tid < P.K) {
    const int i = si[tid];
    const int j = (int)(packed[i] & 0xffffffffull);
    for (int a = 0; a < 3; ++a) { x[a] = P.xn[3 * i + a]; y[a] = (double)P.y32[3 * j + a]; }
    d2 = sd[tid];
  }
  for (int k = 0; k < 16; ++k) {
    const double v[1] = {k == 0 ? d2 : k < 4 ? x[k - 1] : k < 7 ? y[k - 4] : y[(k - 7) / 3] * x[(k - 7) % 3]};
    const double s = dgr_block_sum<kIcpThreads>(v, red);
    if (tid == 0) tot[k] = s;
    __syncthreads();
  }
  if (tid == 0) {
    const double K = (double)P.K, mse = tot[0] / K;
    int live = 1;
    if (st->mse_prev - mse < 1e-6 * st->mse_prev) {
      live = 0;
    } else {
      double mx[3], my[3], S[3][3], R[3][3];
      for (int a = 0; a < 3; ++a) { mx[a] = tot[1 + a] / K; my[a] = tot[4 + a] / K; }
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) S[a][b] = tot[7 + 3 * a + b] / K - my[a] * mx[b];
      kabsch_rotation(S, R);
      for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) st->icpT[4 * a + b] = R[a][b];
        st->icpT[4 * a + 3] = my[a] - (R[a][0] * mx[0] + R[a][1] * mx[1] + R[a][2] * mx[2]);
      }
      st->mse_prev = mse;
      st->icp_updates += 1;
      if (st->icp_updates >= kIcpIters) live = 0;
    }
    st->icp_live = live;
    for (int q = 0; q < 12; ++q) sT[q] = st->icpT[q];
    s_live = live;
  }
  __syncthreads();
  if (s_live) icp_points(P.xn, P.n_s, sT, p32);
}

// E at the ICP pose; init: it becomes the incumbent, otherwise the better of it and the candidate child (the child
// on a tie)
__global__ void __launch_bounds__(kRoundThreads)
goicp_eval_kernel(GoParams P, GoState* st, int init) {
  __shared__ float xs[kMaxSrc], ys[kMaxSrc], zs[kMaxSrc];
  __shared__ float tu[kSkew], tl[kSkew];
  if (!init && !st->run_icp) return;                    // uniform per launch
  double T[12];
  for (int q = 0; q < 12; ++q) T[q] = st->icpT[q];
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  for (int i = threadIdx.x; i < P.n_s; i += blockDim.x) {
    const double x[3] = {P.xn[3 * i], P.xn[3 * i + 1], P.xn[3 * i + 2]};
    xs[i] = __double2float_rn(rot_row(R, x));
    ys[i] = __double2float_rn(rot_row(R + 3, x));
    zs[i] = __double2float_rn(rot_row(R + 6, x));
  }
  __syncthreads();
  if (threadIdx.x >= 32) return;
  const float t32[3] = {__double2float_rn(T[3]), __double2float_rn(T[7]), __double2float_rn(T[11])};
  double u, l;
  warp_bounds(P, xs, ys, zs, nullptr, t32, 0.f, tu, tl, threadIdx.x, u, l);
  if (threadIdx.x != 0) return;
  const bool icp_wins = init || u < st->candE;
  st->h.E = icp_wins ? u : st->candE;
  for (int q = 0; q < 12; ++q) st->T[q] = icp_wins ? T[q] : st->candT[q];
}

// children with LB < E* (E* after this round's incumbent update), compacted in child order, sorted by (LB, key)
__global__ void __launch_bounds__(1024)
goicp_children_kernel(const ChildRec* __restrict__ rec, int nc, GoState* st, double* __restrict__ clb,
                      uint64_t* __restrict__ ckey) {
  __shared__ int32_t flag[8 * kMaxB];
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* lb = reinterpret_cast<double*>(smem_raw);
  uint64_t* key = reinterpret_cast<uint64_t*>(lb + 8 * kMaxB);
  const double E = st->h.E;
  for (int c = threadIdx.x; c < nc; c += blockDim.x) flag[c] = rec[c].status == 0 && rec[c].lb < E;
  __syncthreads();
  const int n = dgr_block_scan_inplace(flag, nc);
  int Pn = 1;
  while (Pn < n) Pn <<= 1;
  for (int c = threadIdx.x; c < nc; c += blockDim.x) {
    const bool keep = rec[c].status == 0 && rec[c].lb < E;
    if (keep) { lb[flag[c]] = rec[c].lb; key[flag[c]] = rec[c].key; }
  }
  for (int i = n + threadIdx.x; i < Pn; i += blockDim.x) {
    lb[i] = __longlong_as_double(0x7ff0000000000000ll);
    key[i] = ~0ull;
  }
  __syncthreads();
  for (int k = 2; k <= Pn; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int p = threadIdx.x; p < Pn / 2; p += blockDim.x) {
        const int i = 2 * p - (p & (j - 1)), q = i + j;
        const double a = lb[i], b = lb[q];
        const uint64_t ka = key[i], kb = key[q];
        if (key_less(b, kb, a, ka) == ((i & k) == 0)) { lb[i] = b; lb[q] = a; key[i] = kb; key[q] = ka; }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < n; i += blockDim.x) { clb[i] = lb[i]; ckey[i] = key[i]; }
  if (threadIdx.x == 0) st->n_child = n;
}

// first index of a sorted list whose (lb, key) is not below (v, kv)
__device__ __forceinline__ int rank_below(const double* lb, const uint64_t* key, int n, double v, uint64_t kv) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (key_less(lb[mid], key[mid], v, kv)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// next pool = (cur[Bp .. n) with LB < E*) merged with the sorted children; both sorted by (LB, key), keys unique
__global__ void goicp_merge_kernel(const double* __restrict__ alb, const uint64_t* __restrict__ akey, int n, int Bp,
                                   const double* __restrict__ clb, const uint64_t* __restrict__ ckey, GoState* st,
                                   int64_t cap, double* __restrict__ olb, uint64_t* __restrict__ okey) {
  const double E = st->h.E;
  const double* A = alb + Bp;
  const uint64_t* Ak = akey + Bp;
  int nA;
  {
    int lo = 0, hi = n - Bp;                             // first entry with LB >= E*
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (A[mid] < E) lo = mid + 1; else hi = mid;
    }
    nA = lo;
  }
  const int nB = st->n_child;
  const int64_t total = (int64_t)nA + nB;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g == 0) {
    const double inf = __longlong_as_double(0x7ff0000000000000ll);
    const double m = fmin(nA > 0 ? A[0] : inf, nB > 0 ? clb[0] : inf);
    st->h.lb_min = total > 0 ? m : E;
    if (total > cap) {
      st->h.stop = 1;
    } else {
      st->h.pool_n = (int32_t)total;
      st->hw = fmax(st->hw, (double)total);
    }
  }
  if (total > cap) return;
  if (g < nA) {
    const int64_t pos = g + rank_below(clb, ckey, nB, A[g], Ak[g]);
    olb[pos] = A[g];
    okey[pos] = Ak[g];
  } else if (g < total) {
    const int j = (int)(g - nA);
    const int pos = j + rank_below(A, Ak, nA, clb[j], ckey[j]);
    olb[pos] = clb[j];
    okey[pos] = ckey[j];
  }
}

__global__ void goicp_result_kernel(const GoState* __restrict__ st, const double* __restrict__ stat, int K, double eps,
                                    int converged, int rounds, int host_reads, double* __restrict__ result) {
  if (threadIdx.x != 0) return;
  const double s = dgr_frame_scale(stat);
  const double* T = st->T;
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}, t[3] = {T[3], T[7], T[11]};
  dgr_frame_pose(R, t, stat, s, result);
  result[16] = st->h.E;
  result[17] = st->h.pool_n == 0 ? st->h.E : st->h.lb_min;
  result[18] = eps;
  result[19] = (double)K;
  result[20] = converged;
  result[21] = rounds;
  result[22] = st->children;
  result[23] = st->tcubes;
  result[24] = st->icp_runs;
  result[25] = st->overflows;
  result[26] = st->hw;
  result[27] = s;
  result[28] = host_reads;
  result[29] = 0.0; result[30] = 0.0; result[31] = 0.0;
}

// the per-round host read: pinned, one per host thread
GoHost* pinned_host() {
  static thread_local GoHost* p = nullptr;
  if (p == nullptr && cudaHostAlloc(reinterpret_cast<void**>(&p), sizeof(GoHost), cudaHostAllocDefault) != cudaSuccess)
    p = nullptr;
  return p;
}

}  // namespace

extern "C" {

int32_t dgr_goicp_ws_elems(int64_t n_src, int64_t n_tgt, int32_t dt_size, int64_t max_rotation_cubes,
                           int32_t cubes_per_round, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_src >= 0 && n_tgt >= 0 && dt_size >= 0 && max_rotation_cubes >= 0 &&
                cubes_per_round >= 0, "bad arguments");
  *n_elems = goicp_layout(n_src, n_tgt, dt_size, max_rotation_cubes, cubes_per_round, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_goicp(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, double mse_thresh,
                  double trim_fraction, int32_t dt_size, double dt_expand, const double* rot_min, double rot_width,
                  const double* trans_min, double trans_width, int32_t cubes_per_round, int32_t max_rounds,
                  int64_t max_rotation_cubes, uint64_t* ws, double* result, void* stream) {
  DGR_ARG_CHECK(src != nullptr && tgt != nullptr && rot_min != nullptr && trans_min != nullptr && ws != nullptr &&
                result != nullptr, "null pointer");
  const int32_t r = dgr_goicp_dt_check(n_src, n_tgt, dt_size, dt_expand);
  if (r != DGR_OK) return r;
  DGR_ARG_CHECK(trim_fraction >= 0.0 && trim_fraction < 1.0, "trim_fraction must lie in [0, 1)");
  DGR_ARG_CHECK(mse_thresh > 0.0 && isfinite(mse_thresh), "mse_thresh must be positive");
  DGR_ARG_CHECK(rot_width > 0.0 && trans_width > 0.0 && isfinite(rot_width) && isfinite(trans_width),
                "domain widths must be positive");
  for (int a = 0; a < 3; ++a)
    DGR_ARG_CHECK(isfinite(rot_min[a]) && isfinite(trans_min[a]), "domain corners must be finite");
  DGR_ARG_CHECK(cubes_per_round >= 1 && cubes_per_round <= kMaxB, "cubes_per_round must lie in [1, 512]");
  DGR_ARG_CHECK(max_rounds >= 0, "max_rounds must be >= 0");
  DGR_ARG_CHECK(max_rotation_cubes >= 8ll * cubes_per_round && max_rotation_cubes < (1ll << 31),
                "max_rotation_cubes must hold one round's children (8 cubes_per_round)");
  GoHost* host = pinned_host();
  DGR_ARG_CHECK(host != nullptr, "pinned host buffer unavailable");
  cudaStream_t st = (cudaStream_t)stream;
  GoWs w;
  goicp_layout(n_src, n_tgt, dt_size, max_rotation_cubes, cubes_per_round, ws, &w);
  GoParams P;
  P.xn = w.xn; P.y32 = w.y32; P.dt = w.dt;
  P.n_s = (int)n_src; P.n_t = (int)n_tgt; P.G = dt_size;
  const int64_t K = (int64_t)floor((double)n_src * (1.0 - trim_fraction));
  P.K = K < 1 ? 1 : (int)K;
  P.trim = P.K < P.n_s;
  P.Pn = 1;
  while (P.Pn < P.n_s) P.Pn <<= 1;
  P.e32 = (float)dt_expand;
  P.h32 = (float)(2.0 * dt_expand / dt_size);
  P.eps = mse_thresh * P.K;
  for (int a = 0; a < 3; ++a) { P.rmin[a] = rot_min[a]; P.tmin[a] = trans_min[a]; }
  P.rw = rot_width;
  P.tw = trans_width;

  int launches = dgr_normalise_dt(src, n_src, tgt, n_tgt, dt_size, dt_expand, w.stat, w.xn, w.y32, w.dt, st);
  GoState* S = w.st;
  const auto icp = [&]() {
    for (int k = 0; k < kIcpIters; ++k) {
      dgr_knn_top1_packed(w.p32, P.n_s, w.y32, P.n_t, 3, w.packed, &S->icp_live, st);
      goicp_icp_step_kernel<<<1, kIcpThreads, 0, st>>>(P, w.packed, S, w.p32);
    }
    launches += 2 * kIcpIters;
  };
  goicp_init_kernel<<<1, kIcpThreads, 0, st>>>(w.xn, P.n_s, S, w.pool_lb[0], w.pool_key[0], w.p32);
  icp();
  goicp_eval_kernel<<<1, kRoundThreads, 0, st>>>(P, S, 1);
  launches += 2;
  DGR_LAUNCH_CHECK();

  const size_t round_smem = sizeof(RoundSmem);
  DGR_ENSURE_SMEM(goicp_round_kernel, round_smem);
  const size_t child_smem = (size_t)8 * kMaxB * 16;
  DGR_ENSURE_SMEM(goicp_children_kernel, child_smem);
  int cur = 0, rounds = 0, reads = 0, converged = 0;
  while (true) {
    DGR_CUDA_CHECK(cudaMemcpyAsync(host, &S->h, sizeof(GoHost), cudaMemcpyDeviceToHost, st));
    DGR_CUDA_CHECK(cudaStreamSynchronize(st));
    ++reads;
    const GoHost h = *host;
    if (h.stop) break;
    if (h.pool_n == 0 || h.E - h.lb_min < P.eps) { converged = 1; break; }
    if (rounds >= max_rounds) break;
    const int Bp = h.pool_n < cubes_per_round ? h.pool_n : cubes_per_round, nc = 8 * Bp;
    goicp_round_kernel<<<nc, kRoundThreads, round_smem, st>>>(P, w.pool_key[cur], S, w.child);
    goicp_incumbent_kernel<<<1, kIcpThreads, 0, st>>>(P, w.child, nc, S, w.p32);
    icp();
    goicp_eval_kernel<<<1, kRoundThreads, 0, st>>>(P, S, 0);
    goicp_children_kernel<<<1, 1024, child_smem, st>>>(w.child, nc, S, w.clb, w.ckey);
    const int64_t span = (int64_t)h.pool_n - Bp + nc;
    goicp_merge_kernel<<<dgr_blocks(span, 256), 256, 0, st>>>(w.pool_lb[cur], w.pool_key[cur], h.pool_n, Bp, w.clb,
                                                              w.ckey, S, max_rotation_cubes, w.pool_lb[cur ^ 1],
                                                              w.pool_key[cur ^ 1]);
    launches += 5;
    DGR_LAUNCH_CHECK();
    ++rounds;
    cur ^= 1;                                           // an overflowing merge writes nothing, but sets the stop flag
  }
  goicp_result_kernel<<<1, 32, 0, st>>>(S, w.stat, P.K, P.eps, converged, rounds, reads, result);
  dgr_note_launches(launches + 1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
