// Super4PCS (Mellado, Aiger & Mitra, "Super 4PCS: Fast Global Pointcloud Registration via Smart Indexing", SGP 2014;
// after 4PCS, Aiger, Mitra & Cohen-Or, SIGGRAPH 2008): 4-point congruent sets between a coplanar source base and
// pairs of the target, each congruent set fitted by Kabsch and scored by its largest common pointset (LCP) through
// Go-ICP's distance transform of the target.  oracle/super4pcs.py restates every step (the specification); the
// geometry is fp64 in the oracle's operation order with no contraction, so the counts have the same bits here and
// in numpy.  Every round of B bases is enqueued up front; each kernel returns at once when the device `done` flag
// is set, so the only host read is the caller's read of the result.
//   dgr_normalise_dt         the normalised frame and the target's distance transform, as Go-ICP's (frame.cu)
//   s4_init_kernel           state, the target sample Q (fp64), r = max |p|, D, delta; base log cleared
//   per round:
//     s4_base_kernel         a warp per base: 32 counter-hash triplets (a lane each), the fourth point (lanes over rows)
//     s4_pair_count_kernel   a (base, tile of kTileRows rows of Q x Q) per CTA: |S1|, |S2| of the tile
//     s4_pair_scan_kernel    the tile counts of each base scanned (dgr_block_scan_inplace); the join's hash cleared
//     s4_pair_scatter_kernel the pairs of a tile in row-major order (dgr_block_exclusive_scan), capped
//     s4_hash_*_kernel       e2 of every S2 pair bucketed by its delta-grid cell: counts, scan, placement
//     s4_join_count_kernel   a thread per S1 pair: the S2 pairs in the 27 cells around e1 meeting every predicate
//     s4_join_scan_kernel    per-pair counts scanned in int64: candidate offsets in (i, j) order, saturated at the cap
//     s4_join_write_kernel   each pair's matches written in ascending j, one visit per slot, until the cap is reached
//                            (the slot order inside a bucket never reaches the output)
//     s4_fit_kernel          a warp per candidate: Kabsch + residual test, the 64-row prefilter (DT gathers)
//     s4_select_kernel       a CTA per base: histogram of the 0..64 prefilter counts, the first V in order
//     s4_lcp_kernel          a CTA per verified candidate: the LCP over all of P
//     s4_best_kernel         base and round bests, counters, the base log; sets `done`
//   s4_result_kernel         the de-normalised pose and the counters
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"
#include "frame.cuh"
#include "kabsch.cuh"

namespace {

constexpr int kMaxSrc = 1024;
constexpr int kMaxQ = 4096;
constexpr int kTriplets = 32;                            // one lane each
constexpr int kPrefilter = 64;
constexpr int kTileRows = 8;                             // rows u of Q per pair tile
constexpr int kLogWidth = 16;
constexpr double kPi = 3.141592653589793;

struct S4State {
  double s, delta, r, D;
  double bases, valid, cands, pairs_dropped, cands_dropped;
  double R[9], t[3];
  float d32;
  int32_t done, best_lcp, best_base, best_cand, rounds;
};
constexpr int kStateWords = 64;
static_assert(sizeof(S4State) <= kStateWords * 8, "state workspace too small");

struct BaseRec {
  double P4[4][3];                                       // b1, b2 | b3, b4 (normalised source)
  double r1, r2, lo1sq, hi1sq, lo2sq, hi2sq, lo_c, hi_c;
  int32_t rows[4];
  int64_t ncand_raw;
  int32_t valid, n1, n2, m1, m2, ncand, nver;
};

struct S4Params {
  const double* xn;      // [n_s][3]
  const double* q;       // [n_q][3]
  const int32_t* dt;
  int n_s, n_q, G;
  float e32, h32;
  int cap, maxc, V, tiles;
  int64_t H;             // hash buckets per base (a power of two)
  double overlap, delta_m, angle_tol, tf;
  uint64_t seed;
  S4State* st;
  BaseRec* rec;          // [B]
  int32_t* cnt;          // [B][2][tiles]
  int2* pairs;           // [B][2][cap]
  int32_t* hcnt;         // [B][H + 1]
  int32_t* hcur;         // [B][H]
  int32_t* ent;          // [B][cap]
  int32_t* jc;           // [B][cap]
  int2* cand;            // [B][maxc]
  int32_t* pcnt;         // [B][maxc]
  int32_t* sel;          // [B][V]
  int32_t* lcp;          // [B][V]
  int32_t* log;          // [max_bases][16] or null
};

// ---------------------------------------------------------------------------------------
// fp64 vector arithmetic in the oracle's order, no contraction
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}
__device__ __forceinline__ void sub3(const double a[3], const double b[3], double o[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = __dsub_rn(a[k], b[k]);
}
__device__ __forceinline__ void cross3(const double a[3], const double b[3], double o[3]) {
  o[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  o[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  o[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}
__device__ __forceinline__ double dist2(const double* a, const double* b) {
  double d[3];
  sub3(a, b, d);
  return dot3(d, d);
}
// ((R0 x0 + R1 x1) + R2 x2) + t
__device__ __forceinline__ double xform_row(const double* R, double t, const double* x) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[0], x[0]), __dmul_rn(R[1], x[1])), __dmul_rn(R[2], x[2])), t);
}
// e = q_u + r (q_v - q_u)
__device__ __forceinline__ void epoint(const double* qu, const double* qv, double r, double e[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) e[k] = __dadd_rn(qu[k], __dmul_rn(r, __dsub_rn(qv[k], qu[k])));
}

// closest-point parameters of the lines x1 -> x2 and x3 -> x4; true when both lie in [0, 1]
__device__ bool seg_params(const double* x1, const double* x2, const double* x3, const double* x4, double& s,
                           double& t) {
  double d1[3], d2[3], r[3];
  sub3(x2, x1, d1);
  sub3(x4, x3, d2);
  sub3(x1, x3, r);
  const double a11 = dot3(d1, d1), a12 = dot3(d1, d2), a22 = dot3(d2, d2), e1 = dot3(d1, r), e2 = dot3(d2, r);
  const double den = __dsub_rn(__dmul_rn(a11, a22), __dmul_rn(a12, a12));
  if (!(den > 0.0)) return false;
  s = __ddiv_rn(__dsub_rn(__dmul_rn(a12, e2), __dmul_rn(a22, e1)), den);
  t = __ddiv_rn(__dsub_rn(__dmul_rn(a11, e2), __dmul_rn(a12, e1)), den);
  return s >= 0.0 && s <= 1.0 && t >= 0.0 && t <= 1.0;
}

__device__ __constant__ int kPairing[3][4] = {{0, 1, 2, 3}, {0, 2, 1, 3}, {0, 3, 1, 2}};

// the first pairing of (p1, p2, p3, p4) whose two closest-point parameters lie in [0, 1], or -1
__device__ int first_pairing(const double* const p[4], double& s, double& t) {
  for (int k = 0; k < 3; ++k)
    if (seg_params(p[kPairing[k][0]], p[kPairing[k][1]], p[kPairing[k][2]], p[kPairing[k][3]], s, t)) return k;
  return -1;
}

// Kabsch of the base onto Qd; false when a residual exceeds delta
__device__ bool fit4(const double P4[4][3], const double Qd[4][3], double delta2, double R[9], double t[3]) {
  double mp[3], mq[3], S[3][3], Rm[3][3];
  for (int a = 0; a < 3; ++a) {
    mp[a] = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(P4[0][a], P4[1][a]), P4[2][a]), P4[3][a]), 0.25);
    mq[a] = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(Qd[0][a], Qd[1][a]), Qd[2][a]), Qd[3][a]), 0.25);
  }
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c) {
      double v = 0.0;
      for (int k = 0; k < 4; ++k) v = __dadd_rn(v, __dmul_rn(__dsub_rn(Qd[k][a], mq[a]), __dsub_rn(P4[k][c], mp[c])));
      S[a][c] = __dmul_rn(v, 0.25);
    }
  kabsch_rotation(S, Rm);
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c) R[3 * a + c] = Rm[a][c];
  for (int a = 0; a < 3; ++a) t[a] = __dsub_rn(mq[a], xform_row(R + 3 * a, 0.0, mp));
  bool ok = true;
  for (int k = 0; k < 4; ++k) {
    double y[3];
    for (int a = 0; a < 3; ++a) y[a] = xform_row(R + 3 * a, t[a], P4[k]);
    ok = ok && dist2(y, Qd[k]) <= delta2;
  }
  return ok;
}

__device__ __forceinline__ bool lcp_hit(const S4Params& P, const double R[9], const double t[3], const double* x,
                                        float d32) {
  const float y0 = __double2float_rn(xform_row(R, t[0], x)), y1 = __double2float_rn(xform_row(R + 3, t[1], x)),
              y2 = __double2float_rn(xform_row(R + 6, t[2], x));
  return dt_lookup(P.dt, P.G, P.e32, P.h32, y0, y1, y2) <= d32;
}

__device__ __forceinline__ void cand_quad(const S4Params& P, int b, int k, double Qd[4][3]) {
  const int2 c = P.cand[(int64_t)b * P.maxc + k];
  const int2 p1 = P.pairs[((int64_t)b * 2) * P.cap + c.x], p2 = P.pairs[((int64_t)b * 2 + 1) * P.cap + c.y];
  const int rows[4] = {p1.x, p1.y, p2.x, p2.y};
  for (int m = 0; m < 4; ++m)
    for (int a = 0; a < 3; ++a) Qd[m][a] = P.q[3 * rows[m] + a];
}

// ---------------------------------------------------------------------------------------
// setup
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
s4_init_kernel(S4Params P, const double* __restrict__ stat, const float* __restrict__ y32, int64_t n_t,
               int max_bases) {
  __shared__ double red[32];
  S4State* st = P.st;
  for (int k = threadIdx.x; k < P.n_q; k += blockDim.x) {
    const int64_t row = (int64_t)k * n_t / P.n_q;
    for (int a = 0; a < 3; ++a) const_cast<double*>(P.q)[3 * k + a] = (double)y32[3 * row + a];
  }
  if (P.log != nullptr)
    for (int64_t k = threadIdx.x; k < (int64_t)max_bases * kLogWidth; k += blockDim.x) P.log[k] = -1;
  double m = 0.0;                                        // max is order-independent
  for (int i = threadIdx.x; i < P.n_s; i += blockDim.x) m = fmax(m, sqrt(dot3(P.xn + 3 * i, P.xn + 3 * i)));
  for (int d = 16; d > 0; d >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, d));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, red[w]);
    const double s = dgr_frame_scale(stat);
    st->s = s;
    st->delta = __ddiv_rn(P.delta_m, s);
    st->d32 = __double2float_rn(st->delta);
    st->r = m;
    st->D = __dmul_rn(P.overlap, __dmul_rn(2.0, m));
    st->bases = st->valid = st->cands = st->pairs_dropped = st->cands_dropped = 0.0;
    for (int q = 0; q < 9; ++q) st->R[q] = (q % 4 == 0) ? 1.0 : 0.0;
    st->t[0] = st->t[1] = st->t[2] = 0.0;
    st->done = 0;
    st->best_lcp = -1;
    st->best_base = -1;
    st->best_cand = -1;
    st->rounds = 0;
  }
}

// ---------------------------------------------------------------------------------------
// base selection: a warp per base
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) s4_base_kernel(S4Params P, int base0) {
  const S4State* st = P.st;
  if (st->done) return;
  const int b = blockIdx.x, lane = threadIdx.x;
  const uint64_t gb = (uint64_t)(base0 + b);
  BaseRec& R = P.rec[b];
  const double D = st->D, delta = st->delta;
  const double lo = __dmul_rn(D, 0.25), lo2 = __dmul_rn(lo, lo), hi2 = __dmul_rn(D, D);
  int idx[3];
  for (int k = 0; k < 3; ++k)
    idx[k] = (int)dgr_counter_pick(P.seed, 3 * ((uint64_t)kTriplets * gb + lane) + k, (uint32_t)P.n_s);
  const double *a = P.xn + 3 * idx[0], *bb = P.xn + 3 * idx[1], *c = P.xn + 3 * idx[2];
  double ab[3], ac[3], cr[3];
  sub3(bb, a, ab);
  sub3(c, a, ac);
  cross3(ab, ac, cr);
  const double area = dot3(cr, cr), e0 = dist2(bb, a), e1 = dist2(c, bb), e2 = dist2(a, c);
  bool ok = idx[0] != idx[1] && idx[1] != idx[2] && idx[0] != idx[2] && area > 0.0;
  ok = ok && e0 >= lo2 && e0 <= hi2 && e1 >= lo2 && e1 <= hi2 && e2 >= lo2 && e2 <= hi2;
  double best = ok ? area : -1.0;
  int bl = lane;
  for (int d = 16; d > 0; d >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, d);
    const int ol = __shfl_xor_sync(0xffffffffu, bl, d);
    if (ob > best || (ob == best && ol < bl)) { best = ob; bl = ol; }
  }
  int tri[3];
  for (int k = 0; k < 3; ++k) tri[k] = __shfl_sync(0xffffffffu, idx[k], bl);
  double crt[3];
  for (int k = 0; k < 3; ++k) crt[k] = __shfl_sync(0xffffffffu, cr[k], bl);
  int l_best = -1;
  double k_best = 0.0;
  if (best > 0.0) {
    const double *ta = P.xn + 3 * tri[0], *tb = P.xn + 3 * tri[1], *tc = P.xn + 3 * tri[2];
    for (int l = lane; l < P.n_s; l += 32) {
      if (l == tri[0] || l == tri[1] || l == tri[2]) continue;
      const double* x = P.xn + 3 * l;
      if (!(dist2(x, ta) <= hi2 && dist2(x, tb) <= hi2 && dist2(x, tc) <= hi2)) continue;
      double d[3];
      sub3(x, ta, d);
      const double key = fabs(dot3(crt, d));
      if (l_best >= 0 && !(key < k_best)) continue;     // rows ascend per lane: the first smallest stays
      const double* p4[4] = {ta, tb, tc, x};
      double s, t;
      if (first_pairing(p4, s, t) < 0) continue;
      l_best = l;
      k_best = key;
    }
  }
  for (int d = 16; d > 0; d >>= 1) {
    const double ok2 = __shfl_xor_sync(0xffffffffu, k_best, d);
    const int ol = __shfl_xor_sync(0xffffffffu, l_best, d);
    if (ol >= 0 && (l_best < 0 || ok2 < k_best || (ok2 == k_best && ol < l_best))) { k_best = ok2; l_best = ol; }
  }
  if (lane != 0) return;
  const bool valid = best > 0.0 && l_best >= 0 && __ddiv_rn(k_best, sqrt(best)) <= delta;
  R.valid = valid;
  R.n1 = R.n2 = R.m1 = R.m2 = R.ncand_raw = R.ncand = R.nver = 0;
  for (int k = 0; k < 4; ++k) R.rows[k] = -1;
  if (!valid) return;
  const int rows4[4] = {tri[0], tri[1], tri[2], l_best};
  const double* p4[4] = {P.xn + 3 * rows4[0], P.xn + 3 * rows4[1], P.xn + 3 * rows4[2], P.xn + 3 * rows4[3]};
  double s, t;
  const int w = first_pairing(p4, s, t);
  for (int k = 0; k < 4; ++k) {
    R.rows[k] = rows4[kPairing[w][k]];
    for (int q = 0; q < 3; ++q) R.P4[k][q] = p4[kPairing[w][k]][q];
  }
  R.r1 = s;
  R.r2 = t;
  double v1[3], v2[3];
  sub3(R.P4[1], R.P4[0], v1);
  sub3(R.P4[3], R.P4[2], v2);
  const double d1 = sqrt(dot3(v1, v1)), d2 = sqrt(dot3(v2, v2));
  const double cs = __ddiv_rn(dot3(v1, v2), __dmul_rn(d1, d2));
  const double tol = P.angle_tol > 0.0 ? P.angle_tol : __ddiv_rn(__dmul_rn(2.0, delta), fmin(d1, d2));
  const double th = acos(fmin(fmax(cs, -1.0), 1.0));
  R.lo_c = cos(fmin(__dadd_rn(th, tol), kPi));
  R.hi_c = cos(fmax(__dsub_rn(th, tol), 0.0));
  const double l1 = fmax(__dsub_rn(d1, delta), 0.0), h1 = __dadd_rn(d1, delta);
  const double l2 = fmax(__dsub_rn(d2, delta), 0.0), h2 = __dadd_rn(d2, delta);
  R.lo1sq = __dmul_rn(l1, l1);
  R.hi1sq = __dmul_rn(h1, h1);
  R.lo2sq = __dmul_rn(l2, l2);
  R.hi2sq = __dmul_rn(h2, h2);
}

// ---------------------------------------------------------------------------------------
// S1 / S2: tiles of kTileRows rows of Q x Q
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void pair_flags(const S4Params& P, const BaseRec& R, int64_t e, int64_t nelem, int u0,
                                           int& u, int& v, bool& f1, bool& f2) {
  f1 = f2 = false;
  if (e >= nelem) return;
  u = u0 + (int)(e / P.n_q);
  v = (int)(e % P.n_q);
  if (u == v) return;
  const double dd = dist2(P.q + 3 * v, P.q + 3 * u);
  f1 = dd >= R.lo1sq && dd <= R.hi1sq;
  f2 = dd >= R.lo2sq && dd <= R.hi2sq;
}

__global__ void __launch_bounds__(256) s4_pair_count_kernel(S4Params P) {
  __shared__ int s_c[2];
  if (P.st->done) return;
  const int b = blockIdx.y, tile = blockIdx.x;
  const BaseRec& R = P.rec[b];
  int32_t* cnt = P.cnt + (int64_t)b * 2 * P.tiles;
  if (!R.valid) {
    if (threadIdx.x == 0) { cnt[tile] = 0; cnt[P.tiles + tile] = 0; }
    return;
  }
  if (threadIdx.x == 0) { s_c[0] = 0; s_c[1] = 0; }
  __syncthreads();
  const int u0 = tile * kTileRows;
  const int64_t nelem = (int64_t)min(kTileRows, P.n_q - u0) * P.n_q;
  int c1 = 0, c2 = 0;
  for (int64_t e = threadIdx.x; e < nelem; e += blockDim.x) {
    int u, v;
    bool f1, f2;
    pair_flags(P, R, e, nelem, u0, u, v, f1, f2);
    c1 += f1;
    c2 += f2;
  }
  c1 = __reduce_add_sync(0xffffffffu, c1);
  c2 = __reduce_add_sync(0xffffffffu, c2);
  if ((threadIdx.x & 31) == 0) { atomicAdd(&s_c[0], c1); atomicAdd(&s_c[1], c2); }   // integer: order-free
  __syncthreads();
  if (threadIdx.x == 0) { cnt[tile] = s_c[0]; cnt[P.tiles + tile] = s_c[1]; }
}

__global__ void __launch_bounds__(1024) s4_pair_scan_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.x;
  BaseRec& R = P.rec[b];
  if (!R.valid) return;
  int32_t* cnt = P.cnt + (int64_t)b * 2 * P.tiles;
  const int n1 = dgr_block_scan_inplace(cnt, P.tiles);
  __syncthreads();
  const int n2 = dgr_block_scan_inplace(cnt + P.tiles, P.tiles);
  int32_t* h = P.hcnt + (int64_t)b * (P.H + 1);
  for (int64_t k = threadIdx.x; k <= P.H; k += blockDim.x) h[k] = 0;
  if (threadIdx.x == 0) {
    R.n1 = n1;
    R.n2 = n2;
    R.m1 = min(n1, P.cap);
    R.m2 = min(n2, P.cap);
  }
}

__global__ void __launch_bounds__(256) s4_pair_scatter_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.y, tile = blockIdx.x;
  const BaseRec& R = P.rec[b];
  if (!R.valid) return;
  const int32_t* cnt = P.cnt + (int64_t)b * 2 * P.tiles;
  int o1 = cnt[tile], o2 = cnt[P.tiles + tile];
  if (o1 >= P.cap && o2 >= P.cap) return;
  int2* S1 = P.pairs + (int64_t)b * 2 * P.cap;
  int2* S2 = S1 + P.cap;
  const int u0 = tile * kTileRows;
  const int64_t nelem = (int64_t)min(kTileRows, P.n_q - u0) * P.n_q;
  for (int64_t e0 = 0; e0 < nelem; e0 += 256) {
    int u = 0, v = 0, t1, t2;
    bool f1, f2;
    pair_flags(P, R, e0 + threadIdx.x, nelem, u0, u, v, f1, f2);
    const int p1 = o1 + dgr_block_exclusive_scan<256>(f1, &t1);
    __syncthreads();
    const int p2 = o2 + dgr_block_exclusive_scan<256>(f2, &t2);
    __syncthreads();
    if (f1 && p1 < P.cap) S1[p1] = make_int2(u, v);
    if (f2 && p2 < P.cap) S2[p2] = make_int2(u, v);
    o1 += t1;
    o2 += t2;
  }
}

// ---------------------------------------------------------------------------------------
// the invariant-point join: e2 of every kept S2 pair hashed by its delta-grid cell
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t cell_bucket(const long long c[3], int64_t H) {
  const uint64_t m = 0x1fffffull;
  const uint64_t k = (((uint64_t)c[0] & m) << 42) | (((uint64_t)c[1] & m) << 21) | ((uint64_t)c[2] & m);
  return dgr_mix64(k) & (uint64_t)(H - 1);
}

// The hash cell is delta (1 + 2^-20) wide: two points within delta then lie in neighbouring cells whatever the
// rounding of the division (its error is ~2^-53 |e / delta|, far below the 2^-20 margin), so the 27 cells around
// e1 hold every S2 pair the exact predicate can accept.
__device__ __forceinline__ void cell_of(const double e[3], double delta, long long c[3]) {
  const double w = __dmul_rn(delta, 1.0 + 0x1p-20);
  for (int a = 0; a < 3; ++a) c[a] = (long long)floor(__ddiv_rn(e[a], w));
}

__device__ __forceinline__ void e2_of(const S4Params& P, const BaseRec& R, int b, int j, double e[3]) {
  const int2 p = P.pairs[((int64_t)b * 2 + 1) * P.cap + j];
  epoint(P.q + 3 * p.x, P.q + 3 * p.y, R.r2, e);
}

__global__ void __launch_bounds__(256) s4_hash_count_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  const BaseRec& R = P.rec[b];
  if (!R.valid || j >= R.m2) return;
  double e[3];
  long long c[3];
  e2_of(P, R, b, j, e);
  cell_of(e, P.st->delta, c);
  atomicAdd(P.hcnt + (int64_t)b * (P.H + 1) + cell_bucket(c, P.H), 1);   // counts: order-free
}

__global__ void __launch_bounds__(1024) s4_hash_scan_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.x;
  if (!P.rec[b].valid) return;
  int32_t* h = P.hcnt + (int64_t)b * (P.H + 1);
  const int tot = dgr_block_scan_inplace(h, P.H);
  if (threadIdx.x == 0) h[P.H] = tot;
  int32_t* cur = P.hcur + (int64_t)b * P.H;
  for (int64_t k = threadIdx.x; k < P.H; k += blockDim.x) cur[k] = h[k];
}

__global__ void __launch_bounds__(256) s4_hash_place_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  const BaseRec& R = P.rec[b];
  if (!R.valid || j >= R.m2) return;
  double e[3];
  long long c[3];
  e2_of(P, R, b, j, e);
  cell_of(e, P.st->delta, c);
  // the slot within a bucket depends on scheduling; the candidates' order never does (s4_join_write_kernel)
  const int slot = atomicAdd(P.hcur + (int64_t)b * P.H + cell_bucket(c, P.H), 1);
  P.ent[(int64_t)b * P.cap + slot] = j;
}

// every S2 pair j congruent with S1 pair i, in bucket order (each bucket of the 27 cells around e1 visited once)
template <class F>
__device__ void join_visit(const S4Params& P, const BaseRec& R, int b, int i, double delta, F&& f) {
  const int2 p1 = P.pairs[((int64_t)b * 2) * P.cap + i];
  const double *qu = P.q + 3 * p1.x, *qv = P.q + 3 * p1.y;
  double e1[3], va[3];
  epoint(qu, qv, R.r1, e1);
  sub3(qv, qu, va);
  const double na = sqrt(dot3(va, va)), d2 = __dmul_rn(delta, delta);
  long long c0[3];
  cell_of(e1, delta, c0);
  const int32_t* h = P.hcnt + (int64_t)b * (P.H + 1);
  const int32_t* ent = P.ent + (int64_t)b * P.cap;
  uint64_t seen[27];
  int ns = 0;
  for (int o = 0; o < 27; ++o) {
    const long long c[3] = {c0[0] + o % 3 - 1, c0[1] + (o / 3) % 3 - 1, c0[2] + o / 9 - 1};
    const uint64_t bk = cell_bucket(c, P.H);
    bool dup = false;
    for (int k = 0; k < ns; ++k) dup = dup || seen[k] == bk;
    if (dup) continue;
    seen[ns++] = bk;
    for (int s = h[bk], e = h[bk + 1]; s < e; ++s) {
      const int j = ent[s];
      const int2 p2 = P.pairs[((int64_t)b * 2 + 1) * P.cap + j];
      if (p1.x == p2.x || p1.x == p2.y || p1.y == p2.x || p1.y == p2.y) continue;
      const double *qw = P.q + 3 * p2.x, *qx = P.q + 3 * p2.y;
      double e2[3], vb[3];
      epoint(qw, qx, R.r2, e2);
      if (!(dist2(e1, e2) <= d2)) continue;
      sub3(qx, qw, vb);
      const double cs = __ddiv_rn(dot3(va, vb), __dmul_rn(na, sqrt(dot3(vb, vb))));
      if (cs >= R.lo_c && cs <= R.hi_c) f(j);
    }
  }
}

__global__ void __launch_bounds__(256) s4_join_count_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const BaseRec& R = P.rec[b];
  if (!R.valid || i >= R.m1) return;
  int n = 0;
  join_visit(P, R, b, i, P.st->delta, [&](int) { ++n; });
  P.jc[(int64_t)b * P.cap + i] = n;
}

// offsets in int64 (|S1| |S2| can exceed 2^31), stored saturated at max_candidates: a pair at or past the cap
// writes nothing
__global__ void __launch_bounds__(1024) s4_join_scan_kernel(S4Params P) {
  __shared__ long long part[1024];
  if (P.st->done) return;
  const int b = blockIdx.x;
  BaseRec& R = P.rec[b];
  if (!R.valid) return;
  int32_t* jc = P.jc + (int64_t)b * P.cap;
  const int m = R.m1, per = (m + 1023) / 1024, lo = min((int)threadIdx.x * per, m), hi = min(lo + per, m);
  long long sum = 0;
  for (int i = lo; i < hi; ++i) sum += jc[i];
  part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long acc = 0;
    for (int k = 0; k < 1024; ++k) { const long long v = part[k]; part[k] = acc; acc += v; }
    R.ncand_raw = acc;
    R.ncand = (int)(acc < P.maxc ? acc : P.maxc);
  }
  __syncthreads();
  long long off = part[threadIdx.x];
  for (int i = lo; i < hi; ++i) {
    const int c = jc[i];
    jc[i] = (int)(off < P.maxc ? off : P.maxc);
    off += c;
  }
}

__global__ void __launch_bounds__(256) s4_join_write_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const BaseRec& R = P.rec[b];
  if (!R.valid || i >= R.m1) return;
  const int off = P.jc[(int64_t)b * P.cap + i];
  const double delta = P.st->delta;
  int2* out = P.cand + (int64_t)b * P.maxc;
  int last = -1;
  for (int pos = off; pos < P.maxc; ++pos) {           // the next-larger j per visit: at most maxc - off + 1 visits
    int nxt = 0x7fffffff;
    join_visit(P, R, b, i, delta, [&](int j) { if (j > last && j < nxt) nxt = j; });
    if (nxt == 0x7fffffff) break;
    out[pos] = make_int2(i, nxt);
    last = nxt;
  }
}

// ---------------------------------------------------------------------------------------
// fit + prefilter (a warp per candidate), selection, full LCP, best of round
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) s4_fit_kernel(S4Params P) {
  if (P.st->done) return;
  const int b = blockIdx.y, lane = threadIdx.x & 31, k = blockIdx.x * 8 + (threadIdx.x >> 5);
  const BaseRec& R = P.rec[b];
  if (!R.valid || k >= R.ncand) return;                 // uniform per warp
  double Qd[4][3], Rm[9], t[3];
  cand_quad(P, b, k, Qd);
  const double delta = P.st->delta;
  const bool ok = fit4(R.P4, Qd, __dmul_rn(delta, delta), Rm, t);
  int n = -1;
  if (ok) {
    n = 0;
    const float d32 = P.st->d32;
    for (int m = lane; m < kPrefilter; m += 32) {
      const int row = (int)((int64_t)m * P.n_s / kPrefilter);
      n += __popc(__ballot_sync(0xffffffffu, lcp_hit(P, Rm, t, P.xn + 3 * row, d32)));
    }
  }
  if (lane == 0) P.pcnt[(int64_t)b * P.maxc + k] = n;
}

__global__ void __launch_bounds__(256) s4_select_kernel(S4Params P) {
  __shared__ int hist[kPrefilter + 1];
  __shared__ int s_cut, s_need;
  if (P.st->done) return;
  const int b = blockIdx.x;
  BaseRec& R = P.rec[b];
  if (!R.valid) return;
  const int32_t* pc = P.pcnt + (int64_t)b * P.maxc;
  for (int c = threadIdx.x; c <= kPrefilter; c += blockDim.x) hist[c] = 0;
  __syncthreads();
  for (int k = threadIdx.x; k < R.ncand; k += blockDim.x)
    if (pc[k] >= 0) atomicAdd(&hist[pc[k]], 1);          // counts: order-free
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0, cut = 0, need = hist[0];
    for (int c = kPrefilter; c >= 0; --c) {
      if (acc + hist[c] >= P.V) { cut = c; need = P.V - acc; break; }
      acc += hist[c];
    }
    s_cut = cut;
    s_need = need;
  }
  __syncthreads();
  const int cut = s_cut, need = s_need;
  int carry_eq = 0, carry_sel = 0;
  int32_t* sel = P.sel + (int64_t)b * P.V;
  for (int k0 = 0; k0 < R.ncand; k0 += 256) {
    const int k = k0 + threadIdx.x;
    const int c = k < R.ncand ? pc[k] : -1;
    const int eq = c == cut, gt = c > cut;
    int teq, tsel;
    const int req = carry_eq + dgr_block_exclusive_scan<256>(eq, &teq);
    __syncthreads();
    const int take = gt || (eq && req < need);
    const int pos = carry_sel + dgr_block_exclusive_scan<256>(take, &tsel);
    __syncthreads();
    if (take) sel[pos] = k;
    carry_eq += teq;
    carry_sel += tsel;
  }
  if (threadIdx.x == 0) R.nver = carry_sel;
}

__global__ void __launch_bounds__(256) s4_lcp_kernel(S4Params P) {
  __shared__ double sR[9], st_[3];
  __shared__ int s_n;
  if (P.st->done) return;
  const int b = blockIdx.y, slot = blockIdx.x;
  const BaseRec& R = P.rec[b];
  if (!R.valid || slot >= R.nver) return;
  const int k = P.sel[(int64_t)b * P.V + slot];
  if (threadIdx.x == 0) {
    double Qd[4][3], Rm[9], t[3];
    cand_quad(P, b, k, Qd);
    fit4(R.P4, Qd, 0.0, Rm, t);
    for (int q = 0; q < 9; ++q) sR[q] = Rm[q];
    for (int a = 0; a < 3; ++a) st_[a] = t[a];
    s_n = 0;
  }
  __syncthreads();
  double Rm[9], t[3];
  for (int q = 0; q < 9; ++q) Rm[q] = sR[q];
  for (int a = 0; a < 3; ++a) t[a] = st_[a];
  const float d32 = P.st->d32;
  int n = 0;
  for (int i = threadIdx.x; i < P.n_s; i += blockDim.x) n += lcp_hit(P, Rm, t, P.xn + 3 * i, d32);
  n = __reduce_add_sync(0xffffffffu, n);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_n, n);      // integer: order-free
  __syncthreads();
  if (threadIdx.x == 0) P.lcp[(int64_t)b * P.V + slot] = s_n;
}

__global__ void s4_best_kernel(S4Params P, int base0, int nb) {
  S4State* st = P.st;
  if (st->done || threadIdx.x != 0) return;
  for (int b = 0; b < nb; ++b) {
    const BaseRec& R = P.rec[b];
    int bl = -1, bk = -1;
    for (int s = 0; s < R.nver; ++s) {
      const int v = P.lcp[(int64_t)b * P.V + s];
      if (v > bl) { bl = v; bk = P.sel[(int64_t)b * P.V + s]; }
    }
    st->bases += 1.0;
    st->valid += R.valid;
    st->cands += R.ncand;
    st->pairs_dropped += (double)(max(R.n1 - P.cap, 0) + max(R.n2 - P.cap, 0));
    st->cands_dropped += (double)(R.ncand_raw - R.ncand);
    if (P.log != nullptr) {
      int32_t* L = P.log + (int64_t)(base0 + b) * kLogWidth;
      const int32_t v[kLogWidth] = {R.rows[0], R.rows[1], R.rows[2], R.rows[3], R.valid, R.n1, R.n2, R.ncand,
                                    (int32_t)min(R.ncand_raw - R.ncand, (int64_t)0x7fffffff), R.nver, bl, bk,
                                    0, 0, 0, 0};
      for (int q = 0; q < kLogWidth; ++q) L[q] = v[q];
    }
    if (bl > st->best_lcp) {
      st->best_lcp = bl;
      st->best_base = base0 + b;
      st->best_cand = bk;
      double Qd[4][3], t[3];
      cand_quad(P, b, bk, Qd);
      fit4(R.P4, Qd, 0.0, st->R, t);
      for (int a = 0; a < 3; ++a) st->t[a] = t[a];
    }
  }
  st->rounds += 1;
  if ((double)max(st->best_lcp, 0) >= P.tf * P.n_s) st->done = 1;
}

__global__ void s4_result_kernel(const S4State* __restrict__ st, const double* __restrict__ stat, int n_s,
                                 double* __restrict__ result) {
  if (threadIdx.x != 0) return;
  const double s = st->s;
  dgr_frame_pose(st->R, st->t, stat, s, result);
  const int lcp = max(st->best_lcp, 0);
  result[16] = (double)lcp / n_s;
  result[17] = lcp;
  result[18] = st->bases;
  result[19] = st->valid;
  result[20] = st->cands;
  result[21] = st->pairs_dropped;
  result[22] = st->cands_dropped;
  result[23] = st->best_base;
  result[24] = st->best_cand;
  result[25] = st->rounds;
  result[26] = s;
  result[27] = 0.0;                                      // host reads inside the call
  for (int k = 28; k < 32; ++k) result[k] = 0.0;
}

// ---------------------------------------------------------------------------------------
// workspace
// ---------------------------------------------------------------------------------------
int64_t hash_buckets(int64_t cap) {
  int64_t H = 1;
  while (H < 2 * cap) H <<= 1;
  return H;
}

struct S4Ws {
  double* stat;
  double* xn;
  float* y32;
  int32_t* dt;
};

int64_t s4_layout(int64_t n_s, int64_t n_t, int64_t n_q, int64_t G, int64_t B, int64_t cap, int64_t maxc, int64_t V,
                  uint64_t* base, S4Ws* w, S4Params* P) {
  const int64_t tiles = (n_q + kTileRows - 1) / kTileRows, H = hash_buckets(cap);
  DgrCarver c(base);
  S4Ws ws;
  S4Params p;
  p.st = reinterpret_cast<S4State*>(c.take<uint64_t>(kStateWords));
  ws.stat = c.take<double>(8);
  ws.xn = c.take<double>(3 * n_s);
  ws.y32 = c.take<float>(3 * n_t);
  ws.dt = c.take<int32_t>(G * G * G);
  p.xn = ws.xn;
  p.dt = ws.dt;
  p.q = c.take<double>(3 * n_q);
  p.rec = c.take<BaseRec>(B);
  p.cnt = c.take<int32_t>(2 * B * tiles);
  p.pairs = c.take<int2>(2 * B * cap);
  p.hcnt = c.take<int32_t>(B * (H + 1));
  p.hcur = c.take<int32_t>(B * H);
  p.ent = c.take<int32_t>(B * cap);
  p.jc = c.take<int32_t>(B * cap);
  p.cand = c.take<int2>(B * maxc);
  p.pcnt = c.take<int32_t>(B * maxc);
  p.sel = c.take<int32_t>(B * V);
  p.lcp = c.take<int32_t>(B * V);
  p.tiles = (int)tiles;
  p.H = H;
  if (w != nullptr) { *w = ws; *P = p; }
  return c.words;
}

int32_t s4_check(int64_t n_src, int64_t n_tgt, int64_t n_q, double overlap, double delta, double angle_tol,
                 int32_t G, double e, int32_t max_bases, int32_t B, int64_t cap, int64_t maxc, int32_t V, double tf) {
  DGR_ARG_CHECK(n_src >= 4 && n_src <= kMaxSrc, "n_src must lie in [4, 1024]");
  DGR_ARG_CHECK(n_q >= 4 && n_q <= kMaxQ, "n_sample_tgt must lie in [4, 4096]");
  DGR_ARG_CHECK(n_tgt >= n_q && n_tgt < (1ll << 31), "n_tgt must lie in [n_sample_tgt, 2^31)");
  DGR_ARG_CHECK(overlap > 0.0 && overlap <= 1.0, "overlap must lie in (0, 1]");
  DGR_ARG_CHECK(delta > 0.0 && isfinite(delta), "delta must be positive");
  DGR_ARG_CHECK(angle_tol >= 0.0 && isfinite(angle_tol), "angle_tol must be >= 0 (0: 2 delta / min(d1, d2))");
  DGR_ARG_CHECK(G >= 16 && G <= 512, "dt_size must lie in [16, 512]");
  DGR_ARG_CHECK(e > 0.0 && isfinite(e), "dt_expand must be positive");
  DGR_ARG_CHECK(max_bases >= 1, "max_bases must be >= 1");
  DGR_ARG_CHECK(B >= 1 && B <= 65535, "bases_per_round must lie in [1, 65535]");
  DGR_ARG_CHECK(cap >= 1 && cap <= (1 << 24), "max_pairs must lie in [1, 2^24]");
  DGR_ARG_CHECK(maxc >= 1 && maxc <= (1 << 24), "max_candidates must lie in [1, 2^24]");
  DGR_ARG_CHECK(V >= 1 && V <= maxc && V <= 65535, "verify_per_base must lie in [1, max_candidates]");
  DGR_ARG_CHECK(tf >= 0.0 && tf <= 1.0, "terminate_fraction must lie in [0, 1]");
  return DGR_OK;
}

}  // namespace

extern "C" {

int32_t dgr_super4pcs_ws_elems(int64_t n_src, int64_t n_tgt, int64_t n_sample_tgt, int32_t dt_size,
                               int32_t bases_per_round, int64_t max_pairs, int64_t max_candidates,
                               int32_t verify_per_base, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_src >= 0 && n_tgt >= 0 && n_sample_tgt >= 0 && dt_size >= 0 &&
                bases_per_round >= 0 && max_pairs >= 0 && max_candidates >= 0 && verify_per_base >= 0,
                "bad arguments");
  *n_elems = s4_layout(n_src, n_tgt, n_sample_tgt, dt_size, bases_per_round, max_pairs, max_candidates,
                       verify_per_base, nullptr, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_super4pcs(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, int64_t n_sample_tgt,
                      double overlap, double delta, double angle_tol, int32_t dt_size, double dt_expand,
                      int32_t max_bases, int32_t bases_per_round, int64_t max_pairs, int64_t max_candidates,
                      int32_t verify_per_base, double terminate_fraction, uint64_t seed, uint64_t* ws,
                      int32_t* base_log, double* result, void* stream) {
  DGR_ARG_CHECK(src != nullptr && tgt != nullptr && ws != nullptr && result != nullptr, "null pointer");
  const int32_t r = s4_check(n_src, n_tgt, n_sample_tgt, overlap, delta, angle_tol, dt_size, dt_expand, max_bases,
                             bases_per_round, max_pairs, max_candidates, verify_per_base, terminate_fraction);
  if (r != DGR_OK) return r;
  cudaStream_t st = (cudaStream_t)stream;
  const int B = bases_per_round;
  S4Ws w;
  S4Params P;
  s4_layout(n_src, n_tgt, n_sample_tgt, dt_size, B, max_pairs, max_candidates, verify_per_base, ws, &w, &P);
  P.n_s = (int)n_src;
  P.n_q = (int)n_sample_tgt;
  P.G = dt_size;
  P.e32 = (float)dt_expand;
  P.h32 = (float)(2.0 * dt_expand / dt_size);
  P.cap = (int)max_pairs;
  P.maxc = (int)max_candidates;
  P.V = verify_per_base;
  P.overlap = overlap;
  P.delta_m = delta;
  P.angle_tol = angle_tol;
  P.tf = terminate_fraction;
  P.seed = seed;
  P.log = base_log;

  int launches = dgr_normalise_dt(src, n_src, tgt, n_tgt, dt_size, dt_expand, w.stat, w.xn, w.y32, w.dt, st);
  s4_init_kernel<<<1, 1024, 0, st>>>(P, w.stat, w.y32, n_tgt, max_bases);
  ++launches;
  DGR_LAUNCH_CHECK();
  const unsigned pair_blocks = dgr_blocks(max_pairs, 256), cand_blocks = dgr_blocks(max_candidates, 8);
  for (int base0 = 0; base0 < max_bases; base0 += B) {
    const int nb = max_bases - base0 < B ? max_bases - base0 : B;
    const dim3 tiles(P.tiles, nb), pg(pair_blocks, nb);
    s4_base_kernel<<<nb, 32, 0, st>>>(P, base0);
    s4_pair_count_kernel<<<tiles, 256, 0, st>>>(P);
    s4_pair_scan_kernel<<<nb, 1024, 0, st>>>(P);
    s4_pair_scatter_kernel<<<tiles, 256, 0, st>>>(P);
    s4_hash_count_kernel<<<pg, 256, 0, st>>>(P);
    s4_hash_scan_kernel<<<nb, 1024, 0, st>>>(P);
    s4_hash_place_kernel<<<pg, 256, 0, st>>>(P);
    s4_join_count_kernel<<<pg, 256, 0, st>>>(P);
    s4_join_scan_kernel<<<nb, 1024, 0, st>>>(P);
    s4_join_write_kernel<<<pg, 256, 0, st>>>(P);
    s4_fit_kernel<<<dim3(cand_blocks, nb), 256, 0, st>>>(P);
    s4_select_kernel<<<nb, 256, 0, st>>>(P);
    s4_lcp_kernel<<<dim3(verify_per_base, nb), 256, 0, st>>>(P);
    s4_best_kernel<<<1, 32, 0, st>>>(P, base0, nb);
    launches += 14;
    DGR_LAUNCH_CHECK();
  }
  s4_result_kernel<<<1, 32, 0, st>>>(P.st, w.stat, P.n_s, result);
  dgr_note_launches(launches + 1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
