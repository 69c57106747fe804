// Native executor: one C call per network forward and one per scan pair.
//
// Round 1 drove the path from Python: ~275 kernel launches and 7 blocking device-to-host
// reads per pair, every buffer a torch allocation.  Here the same kernels are sequenced by
// C++ on the context's own stream over a grow-only device arena:
//
//   dgr_net_create      a ResUNet2-family network (model/resunet.py:419-665) as a table of
//                       layers: ME-layout kernels, eval-BatchNorm folded to scale / shift, TF32
//                       hi|lo weight slabs packed once;
//   dgr_net_forward     coordinate phase (coarse maps, Bloom filters, kernel-map probes: no host
//                       round trip, device-side row counts - coordplan.cu) -> ONE read of the
//                       meta block (rows per level, pairs / tiles per map) -> pair lists, work
//                       lists and the launch-only convolution phase;
//   dgr_pair_register   DeepGlobalRegistration.register() (core/deep_global_registration.py:
//                       238-324) for the default configuration: voxelise both scans into one
//                       batched sparse tensor, FCGF forward, feature kNN, 6-D coordinates,
//                       inlier network, weights + gate sum, weighted Procrustes + SE(3)
//                       refinement, optional ICP - three host reads in total (FCGF meta, inlier
//                       meta, result).  The safeguard decision stays with the caller
//                       (dgr_pair_safeguard runs RANSAC on the buffers the context still holds).
//
// Contexts are independent (own stream, arena, pinned staging): two host threads with one
// context each keep two pairs in flight on one GPU, so the latency-bound stages of one pair
// (kernel-map probes, the 8-CTA refinement cluster, host reads) overlap the convolutions of
// the other (SURVEY 8e allows two pairs in flight explicitly).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <tuple>
#include <vector>

#include <nvtx3/nvToolsExt.h>      // header-only: ranges show up in Nsight Systems / ncu --nvtx, no-ops otherwise

#include "common.cuh"

namespace {

constexpr int kTileRows = 128;
constexpr int kMetaInts = 256;
constexpr int kMetaNetBase = 8;       // meta[0..8): pair counts (N, N0, N1, key overflow)
constexpr int kMetaPerMap = 5;
constexpr int kKeyMargin = 32;        // spare cells around the bounding box (7^3 kernels, stride-8 flooring); _abi.KEY_MARGIN

bool tc_f16_enabled();
int tc_f16_min_cout();

__global__ void fill_f32_kernel(float* p, int64_t n, float v) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// [R (9) | t (3)] float -> row-major 3x4 double [R | t]
__global__ void pose_to_T12_kernel(const float* __restrict__ res, double* __restrict__ T12) {
  const int k = threadIdx.x;
  if (k < 12) {
    const int r = k / 4, c = k % 4;
    T12[k] = c < 3 ? (double)res[3 * r + c] : (double)res[9 + r];
  }
}

__global__ void pack_result_kernel(const float* __restrict__ se3, const double* __restrict__ wsum,
                                   const double* __restrict__ icp, double* __restrict__ out) {
  const int k = threadIdx.x;
  if (k < 16) out[k] = (double)se3[k];
  if (k == 16) out[16] = *wsum;
  if (k >= 17 && k < 37) out[k] = icp != nullptr ? icp[k - 17] : 0.0;
}

static inline int64_t next_pow2(int64_t n) {
  int64_t p = 1;
  while (p < n) p <<= 1;
  return p;
}

// ---------------------------------------------------------------------------------------
// device arena: bump allocation, reset per call, grows to the high-water mark
// ---------------------------------------------------------------------------------------
struct Arena {
  struct Chunk {
    char* p;
    size_t cap;
  };
  std::vector<Chunk> chunks;
  size_t cur = 0, off = 0, used = 0, high = 0;
  int64_t n_malloc = 0;

  int32_t alloc_raw(size_t bytes, void** out) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (bytes == 0) bytes = 256;
    while (cur < chunks.size() && off + bytes > chunks[cur].cap) {
      ++cur;
      off = 0;
    }
    if (cur >= chunks.size()) {
      size_t cap = bytes > ((size_t)256 << 20) ? bytes : ((size_t)256 << 20);
      void* p = nullptr;
      DGR_CUDA_CHECK(cudaMalloc(&p, cap));
      ++n_malloc;
      chunks.push_back({(char*)p, cap});
      cur = chunks.size() - 1;
      off = 0;
    }
    *out = chunks[cur].p + off;
    off += bytes;
    used += bytes;
    if (used > high) high = used;
    return DGR_OK;
  }
  // Called when nothing enqueued on the context's stream still uses the arena.
  int32_t reset() {
    if (chunks.size() > 1) {      // consolidate: one block a quarter above the high-water mark
      for (auto& c : chunks) DGR_CUDA_CHECK(cudaFree(c.p));
      chunks.clear();
      size_t cap = high + high / 4 + ((size_t)64 << 20);
      void* p = nullptr;
      DGR_CUDA_CHECK(cudaMalloc(&p, cap));
      ++n_malloc;
      chunks.push_back({(char*)p, cap});
    }
    cur = 0;
    off = 0;
    used = 0;
    return DGR_OK;
  }
  void release() {
    for (auto& c : chunks) cudaFree(c.p);
    chunks.clear();
  }
};

struct ProfileRec {
  cudaEvent_t e0, e1;
  double flops, bytes;
  int kind;   // 0 = tensor-core conv, 1 = fp32 conv, 2 = table conv
};

}  // namespace

struct dgr_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  Arena arena;
  int32_t* meta_dev = nullptr;
  int32_t* meta_host = nullptr;      // pinned
  double* res_dev = nullptr;
  double* res_host = nullptr;        // pinned
  void* stage[2] = {nullptr, nullptr};
  size_t stage_cap[2] = {0, 0};
  std::map<std::tuple<int, int, int>, std::pair<std::vector<int32_t>*, int32_t*>> offsets;   // (ksize, D, stride)
  // statistics of the last call
  int64_t reads = 0, d2h_bytes = 0, h2d_bytes = 0;
  // profiling of convolution launches
  bool profile = false;
  std::vector<ProfileRec> prof;
  std::vector<cudaEvent_t> event_pool;
  std::vector<cudaEvent_t> stage_marks;        // stage boundaries of the last pair (profiling on)
  std::map<const float*, float*> amax_of;      // activation tensor -> device slot holding max |x| (current network)
  // taps of the last pair (device pointers into the arena, valid until the next call on this context)
  struct Tap {
    const void* p = nullptr;
    int64_t rows = 0;
    int32_t cols = 0, elem = 4;
  } taps[12];
  // what dgr_pair_safeguard needs
  int64_t pair_n0 = 0, pair_n1 = 0;
  double pair_voxel = 0;
  const float* pair_xyz = nullptr;
  const int32_t* pair_idx1 = nullptr;
  const dgr_keyspec_t* pair_spec = nullptr;
  const uint64_t* pair_keys = nullptr;
  const int32_t* pair_vals = nullptr;
  int64_t pair_cap = 0;
};

namespace {

struct Conv {
  const float* w = nullptr;
  float* packed = nullptr;
  const float* scale = nullptr;
  const float* shift = nullptr;
  int cin = 0, cout = 0, ksize = 3, K = 0;
  bool tc = false;
  // 3xFP16 mode of the cta_group::2 kernel (wide layers): fp16 slabs + (1 / weight scale, max |W|)
  bool f16 = false;
  void* packed16 = nullptr;
  float* wscale = nullptr;
};

}  // namespace

struct dgr_net {
  int D = 3, in_ch = 1, out_ch = 32, conv1_ks = 3, normalize = 0;
  int C[5] = {0, 0, 0, 0, 0}, T[5] = {0, 0, 0, 0, 0};
  Conv enc[4], eb1[4], eb2[4], dec[3], db1[3], db2[3];
  const float* conv1_tr_w = nullptr;
  const float* final_w = nullptr;
  const float* final_b = nullptr;
  std::vector<float*> owned;
  int device = 0;
};

namespace {

template <typename T>
int32_t aalloc(dgr_ctx* c, int64_t n, T** out) {
  void* p = nullptr;
  DGR_TRY(c->arena.alloc_raw((size_t)(n > 0 ? n : 1) * sizeof(T), &p));
  *out = (T*)p;
  return DGR_OK;
}

int32_t get_offsets(dgr_ctx* c, int ksize, int D, int stride, const int32_t** out) {
  auto key = std::make_tuple(ksize, D, stride);
  auto it = c->offsets.find(key);
  if (it == c->offsets.end()) {
    int K = 1;
    for (int a = 0; a < D; ++a) K *= ksize;
    auto* host = new std::vector<int32_t>((size_t)K * D);
    for (int kap = 0; kap < K; ++kap) {
      int rem = kap;
      for (int ax = 0; ax < D; ++ax) {      // axis 0 fastest, centred, scaled by the input tensor stride
        (*host)[(size_t)kap * D + ax] = (rem % ksize - ksize / 2) * stride;
        rem /= ksize;
      }
    }
    int32_t* dev = nullptr;
    DGR_CUDA_CHECK(cudaMalloc(&dev, host->size() * sizeof(int32_t)));
    DGR_CUDA_CHECK(cudaMemcpyAsync(dev, host->data(), host->size() * sizeof(int32_t), cudaMemcpyHostToDevice,
                                   c->stream));
    it = c->offsets.emplace(key, std::make_pair(host, dev)).first;
  }
  *out = it->second.second;
  return DGR_OK;
}

int32_t read_meta(dgr_ctx* c, int n_ints) {
  DGR_CUDA_CHECK(cudaMemcpyAsync(c->meta_host, c->meta_dev, (size_t)n_ints * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                 c->stream));
  DGR_CUDA_CHECK(cudaStreamSynchronize(c->stream));
  c->reads += 1;
  c->d2h_bytes += (int64_t)n_ints * 4;
  return DGR_OK;
}

cudaEvent_t pool_event(dgr_ctx* c) {
  if (!c->event_pool.empty()) {
    cudaEvent_t e = c->event_pool.back();
    c->event_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

const char* const kStageNames[] = {"dgr:upload+voxelise", "dgr:fcgf_coordinate_phase", "dgr:read1+fcgf_pair_lists",
                                   "dgr:fcgf_convolutions", "dgr:feature_knn", "dgr:inlier_coordinate_phase",
                                   "dgr:read2+inlier_pair_lists", "dgr:inlier_convolutions",
                                   "dgr:weights+procrustes+refine(+icp)"};

// stage boundary k of dgr_pair_register (0 = start ... 9 = end): NVTX range per stage, CUDA event when profiling
struct StageRanges {             // closes the open NVTX range on every exit path of dgr_pair_register
  bool open = false;
  ~StageRanges() {
    if (open) nvtxRangePop();
  }
};

void mark_stage(dgr_ctx* c, StageRanges& r, int k) {
  if (r.open) nvtxRangePop();
  r.open = k < 9;
  if (r.open) nvtxRangePushA(kStageNames[k]);
  if (!c->profile) return;
  cudaEvent_t e = pool_event(c);
  cudaEventRecord(e, c->stream);
  c->stage_marks.push_back(e);
}

// ---------------------------------------------------------------------------------------
// plan of one forward pass
// ---------------------------------------------------------------------------------------
struct Level {
  int32_t* coords = nullptr;
  int64_t n_max = 0;
  const int32_t* n_dev = nullptr;
  int n = -1;
  uint64_t* keys = nullptr;
  int32_t* vals = nullptr;
  int64_t cap = 0;
  uint32_t* bloom = nullptr;
  int64_t n_bloom = 0;
};

struct KMap {
  int lin = 0, lout = 0, ksize = 3, K = 27;
  bool dense = false;        // dense neighbour table instead of pair lists (conv1 table kernel)
  bool bits_only = false;    // occupancy masks only: conv1 of a network whose single input channel is all ones
  int64_t W = 0;             // mask words per offset
  const int32_t* offsets = nullptr;
  uint32_t* bits = nullptr;
  int32_t* cnt = nullptr;
  int32_t* kofs = nullptr;
  int32_t* meta = nullptr;
  int P = 0, n_tiles = 0, nonempty = 0;
  int32_t *in_idx = nullptr, *out_idx = nullptr, *tile_k = nullptr, *tile_start = nullptr;
  int32_t* nbr = nullptr;
  int64_t nbr_stride = 0;
};

struct Plan {
  int D = 3, ncols = 4;
  const dgr_keyspec_t* spec = nullptr;
  Level lv[4];
  KMap maps[8];
  int n_maps = 0;
  int map_conv1 = 0, map_same[4] = {0, 0, 0, 0}, map_down[3] = {0, 0, 0};
  int meta_base = kMetaNetBase;
  bool input_ones = false;   // the network input is one channel of ones (FCGF / inlier 'ones'): conv1 needs occupancy only
};

bool conv1_table_kernel(const dgr_net* net) {
  return net->D == 3 && net->conv1_ks > 3 && net->in_ch <= 8 && (net->C[1] == 16 || net->C[1] == 32 || net->C[1] == 64);
}

int meta_ints(const Plan& p) { return p.meta_base + 4 + kMetaPerMap * p.n_maps; }

// Coordinate phase: everything up to (not including) the host read.  lv[0] must hold coords / n_max /
// n_dev (or n); its table is built here when keys == nullptr.
int32_t plan_begin(dgr_ctx* c, const dgr_net* net, Plan& p) {
  void* st = c->stream;
  const int ncols = p.ncols;
  Level& l0 = p.lv[0];
  const int64_t n_max = l0.n_max;
  if (l0.keys == nullptr) {
    l0.cap = next_pow2(2 * (n_max > 512 ? n_max : 512));
    DGR_TRY(aalloc(c, l0.cap, &l0.keys));
    DGR_TRY(aalloc(c, l0.cap, &l0.vals));
    DGR_TRY(dgr_table_build_unique(l0.coords, n_max, l0.n_dev, ncols, p.spec, l0.keys, l0.vals, l0.cap, st));
  }
  // coarse maps at strides 2, 4, 8: all derived from the stride-1 rows (floor(c / s) * s composes, and
  // ranking cells by their first stride-1 row reproduces the cascaded first-occurrence order)
  const int64_t cap = next_pow2(2 * (n_max > 512 ? n_max : 512));
  uint64_t* keys;
  int32_t *vals, *coords, *slot, *scan;
  const int64_t nmx = n_max > 0 ? n_max : 1;
  DGR_TRY(aalloc(c, 3 * cap, &keys));
  DGR_TRY(aalloc(c, 3 * cap, &vals));
  DGR_TRY(aalloc(c, 3 * nmx * ncols, &coords));
  DGR_TRY(aalloc(c, 3 * nmx, &slot));
  DGR_TRY(aalloc(c, 3 * dgr_scan_ws_elems(nmx), &scan));
  const int32_t strides[3] = {2, 4, 8};
  int32_t* n_out_dev = c->meta_dev + p.meta_base + 1;
  DGR_TRY(dgr_coarse_maps(l0.coords, n_max, l0.n_dev, ncols, p.spec, 3, strides, keys, vals, cap, coords, n_out_dev,
                          slot, scan, st));
  for (int l = 1; l < 4; ++l) {
    Level& L = p.lv[l];
    L.coords = coords + (int64_t)(l - 1) * nmx * ncols;
    L.n_max = n_max;
    L.n_dev = n_out_dev + (l - 1);
    L.keys = keys + (int64_t)(l - 1) * cap;
    L.vals = vals + (int64_t)(l - 1) * cap;
    L.cap = cap;
  }
  // miss filters for the kernel maps with many offsets per row (6-D: 729)
  const bool use_bloom = p.D > 3;
  if (use_bloom || net->conv1_ks > 3) {
    const int64_t words = dgr_bloom2_words(n_max);
    for (int l = 0; l < (use_bloom ? 4 : 1); ++l) {       // 3-D: only the stride-1 table is probed with 5^3 / 7^3 offsets
      DGR_TRY(aalloc(c, words, &p.lv[l].bloom));
      p.lv[l].n_bloom = words;
      DGR_TRY(dgr_bloom2_build(p.lv[l].keys, p.lv[l].cap, p.lv[l].bloom, words, st));
    }
  }
  // the kernel maps of the network
  p.n_maps = 0;
  auto add_map = [&](int lin, int lout, int ksize, bool dense) {
    KMap& m = p.maps[p.n_maps];
    m = KMap();
    m.lin = lin; m.lout = lout; m.ksize = ksize; m.dense = dense;
    m.K = 1;
    for (int a = 0; a < p.D; ++a) m.K *= ksize;
    return p.n_maps++;
  };
  for (int l = 0; l < 4; ++l) p.map_same[l] = add_map(l, l, 3, false);
  for (int l = 0; l < 3; ++l) p.map_down[l] = add_map(l, l + 1, 3, false);
  if (net->conv1_ks == 3) {
    p.map_conv1 = p.map_same[0];
  } else {
    const bool bits_only = conv1_table_kernel(net) && p.input_ones && net->in_ch == 1;
    p.map_conv1 = add_map(0, 0, net->conv1_ks, conv1_table_kernel(net) && !bits_only);
    p.maps[p.map_conv1].bits_only = bits_only;
  }
  for (int i = 0; i < p.n_maps; ++i) {
    KMap& m = p.maps[i];
    const Level& Lin = p.lv[m.lin];
    const Level& Lout = p.lv[m.lout];
    DGR_TRY(get_offsets(c, m.ksize, p.D, 1 << m.lin, &m.offsets));
    m.meta = c->meta_dev + p.meta_base + 4 + kMetaPerMap * i;
    if (m.dense) {
      m.nbr_stride = nmx;
      DGR_TRY(aalloc(c, (int64_t)m.K * nmx, &m.nbr));
      const bool bloom = Lin.bloom != nullptr && m.K > 27;
      DGR_CUDA_CHECK(cudaMemsetAsync(m.meta, 0, kMetaPerMap * sizeof(int32_t), (cudaStream_t)st));
      DGR_TRY(dgr_kmap_dense(Lout.coords, Lout.n_max, Lout.n_dev, ncols, p.spec, Lin.keys, Lin.vals, Lin.cap,
                             bloom ? Lin.bloom : nullptr, bloom ? Lin.n_bloom : 0, m.offsets, m.K, m.nbr, m.nbr_stride,
                             m.meta, st));          // meta[0] = pairs P (for the roofline bookkeeping)
      continue;
    }
    m.W = dgr_kmap_mask_words(nmx);
    DGR_TRY(aalloc(c, (int64_t)m.K * m.W, &m.bits));
    DGR_TRY(aalloc(c, dgr_kmap_cnt_elems(m.K, nmx), &m.cnt));
    DGR_TRY(aalloc(c, m.K + 2, &m.kofs));
    // same-stride maps probe half the offsets and mirror the rest; down maps enumerate from the input rows
    const bool down = m.lout == m.lin + 1 && m.ksize == 3;
    const int mode = m.lout == m.lin ? DGR_KMAP_SAME : (down ? DGR_KMAP_DOWN : DGR_KMAP_GENERAL);
    const bool bloom = Lin.bloom != nullptr && m.K > 27 && !down;
    DGR_TRY(dgr_kmap_probe_mode(mode, Lout.coords, Lout.n_max, Lout.n_dev, ncols, p.spec, Lin.keys, Lin.vals, Lin.cap,
                                bloom ? Lin.bloom : nullptr, bloom ? Lin.n_bloom : 0, m.offsets, m.K,
                                down ? Lin.coords : nullptr, down ? Lin.n_max : 0, down ? Lin.n_dev : nullptr,
                                down ? 1 << m.lin : 0, down ? Lout.keys : nullptr, down ? Lout.vals : nullptr,
                                down ? Lout.cap : 0, m.bits, m.cnt, m.kofs, m.meta, st));
  }
  return DGR_OK;
}

// After read_meta(): host-side sizes, then pair lists and work lists.
int32_t plan_finish(dgr_ctx* c, Plan& p) {
  void* st = c->stream;
  const int32_t* mh = c->meta_host + p.meta_base;
  for (int l = 1; l < 4; ++l) p.lv[l].n = mh[l];
  for (int i = 0; i < p.n_maps; ++i) {
    KMap& m = p.maps[i];
    const int32_t* mm = mh + 4 + kMetaPerMap * i;
    if (m.dense || m.bits_only) {
      m.P = mm[0];
      m.nonempty = m.dense ? m.K : mm[3];
      continue;
    }
    m.P = mm[0]; m.n_tiles = mm[1]; m.nonempty = mm[3];
    if (mm[4] != 0) {
      dgr_set_error("coordinate extent does not fit a 63-bit packed key");
      return DGR_ERR_ARG;
    }
    const Level& Lin = p.lv[m.lin];
    const Level& Lout = p.lv[m.lout];
    DGR_TRY(aalloc(c, m.P, &m.in_idx));
    DGR_TRY(aalloc(c, m.P, &m.out_idx));
    DGR_TRY(aalloc(c, m.n_tiles, &m.tile_k));
    DGR_TRY(aalloc(c, m.n_tiles, &m.tile_start));
    if (m.P > 0) {
      DGR_TRY(dgr_kmap_fill(m.bits, m.cnt, m.K, Lout.n_max > 0 ? Lout.n_max : 1, Lout.coords, p.ncols, p.spec, Lin.keys,
                            Lin.vals, Lin.cap, m.offsets, m.in_idx, m.out_idx, st));
      DGR_TRY(dgr_kernel_map_tiles(m.kofs, m.K, kTileRows, m.n_tiles, 0, m.tile_k, m.tile_start, st));
    }
  }
  return DGR_OK;
}

// ---------------------------------------------------------------------------------------
// convolution phase (launch-only)
// ---------------------------------------------------------------------------------------
struct LayerExec {
  const Conv* conv;
  const KMap* map;
  bool transposed;
  int n_in, n_out;
  bool table;     // conv1: output-stationary fp32 table kernel (few input channels)
  bool bits;      // conv1 on an all-ones input from the occupancy masks
};

bool tc_f16_enabled() {
  static const bool v = [] {
    const char* e = getenv("DGR_TC_F16");
    return e ? atoi(e) != 0 : true;
  }();
  return v;
}
int tc_f16_min_cout() {
  static const int v = [] {
    const char* e = getenv("DGR_TC_F16_MIN_COUT");
    return e ? atoi(e) : 128;
  }();
  return v;
}

int32_t run_conv(dgr_ctx* c, const LayerExec& L, const float* feat, float* out) {
  void* st = c->stream;
  const Conv& cv = *L.conv;
  const KMap& m = *L.map;
  ProfileRec rec;
  rec.kind = -1;
  const bool prof = c->profile;
  if (prof) {
    rec.e0 = pool_event(c);
    rec.e1 = pool_event(c);
    rec.flops = 2.0 * m.P * cv.cin * cv.cout;
    // SURVEY 8(d): gather read + scatter write + (in, out) index pair + weights of the non-empty offsets
    rec.bytes = (double)m.P * (cv.cin + cv.cout) * 4.0 + 8.0 * m.P + (double)m.nonempty * cv.cin * cv.cout * 4.0;
    cudaEventRecord(rec.e0, c->stream);
  }
  if (L.bits) {
    DGR_TRY(dgr_spconv_ones_bits_fwd(cv.w, cv.cout, m.bits, m.W, m.K, L.n_out, cv.scale, cv.shift, out, st));
    rec.kind = 2;
  } else if (L.table) {
    DGR_TRY(dgr_spconv_table_fwd_strided(feat, cv.cin, cv.w, cv.cout, m.nbr, m.K, L.n_out, m.nbr_stride, cv.scale,
                                         cv.shift, out, st));
    rec.kind = 2;
  } else {
    const int32_t* in_idx = L.transposed ? m.out_idx : m.in_idx;
    const int32_t* out_idx = L.transposed ? m.in_idx : m.out_idx;
    if (m.P > 0) {
      if (cv.f16) {
        // |input| maximum -> the power-of-two activation scale of this launch (read on the device)
        float* amax;
        auto known = c->amax_of.find(feat);
        if (known != c->amax_of.end()) {
          amax = known->second;            // reduced by the elementwise pass that produced `feat`
        } else {
          DGR_TRY(aalloc(c, 1, &amax));
          DGR_TRY(dgr_absmax_f32(feat, (int64_t)L.n_in * cv.cin, amax, st));
          if (prof) cudaEventRecord(rec.e0, c->stream);      // the timed launch is the convolution itself
        }
        DGR_TRY(dgr_spconv_tc_f16_fwd(feat, cv.cin, cv.packed16, cv.cout, in_idx, out_idx, m.kofs, m.tile_k,
                                      m.tile_start, m.n_tiles, kTileRows, amax, cv.wscale, out, st));
        rec.kind = 0;
      } else if (cv.tc) {
        DGR_TRY(dgr_spconv_tc_fwd(feat, cv.cin, cv.packed, cv.cout, in_idx, out_idx, m.kofs, m.tile_k, m.tile_start,
                                  m.n_tiles, kTileRows, 3, out, st));
        rec.kind = 0;
      } else {
        DGR_TRY(dgr_spconv_fwd(feat, cv.cin, cv.w, cv.cout, in_idx, out_idx, m.kofs, m.tile_k, m.tile_start, m.n_tiles,
                               kTileRows, 0, out, st));
        rec.kind = 1;
      }
    }
  }
  if (prof) {
    cudaEventRecord(rec.e1, c->stream);
    c->prof.push_back(rec);
  }
  return DGR_OK;
}

// ResUNet2.forward of the reference (model/resunet.py:598-649) with fused epilogues: eval-BatchNorm folded to
// scale/shift applied together with the residual add and ReLU in one pass after each scatter-add convolution;
// ME.cat fused into the consuming 1x1 convolution; ReLU + bias + L2-normalise fused into the 1x1 epilogues.
// The ReLUs after each block are idempotent (the block already ends in ReLU) and are dropped.
int32_t run_network(dgr_ctx* c, const dgr_net* net, Plan& p, const float* feats_in, float* out) {
  void* st = c->stream;
  std::vector<LayerExec> layers;
  const int n[4] = {p.lv[0].n, p.lv[1].n, p.lv[2].n, p.lv[3].n};
  for (int s = 0; s < 4; ++s) {
    const KMap* m = s == 0 ? &p.maps[p.map_conv1] : &p.maps[p.map_down[s - 1]];
    layers.push_back({&net->enc[s], m, false, s == 0 ? n[0] : n[s - 1], n[s], s == 0 && m->dense, s == 0 && m->bits_only});
    layers.push_back({&net->eb1[s], &p.maps[p.map_same[s]], false, n[s], n[s], false, false});
    layers.push_back({&net->eb2[s], &p.maps[p.map_same[s]], false, n[s], n[s], false, false});
  }
  for (int d = 0; d < 3; ++d) {
    const int lo = 2 - d;       // output level index
    layers.push_back({&net->dec[d], &p.maps[p.map_down[lo]], true, n[lo + 1], n[lo], false, false});
    layers.push_back({&net->db1[d], &p.maps[p.map_same[lo]], false, n[lo], n[lo], false, false});
    layers.push_back({&net->db2[d], &p.maps[p.map_same[lo]], false, n[lo], n[lo], false, false});
  }
  // one slab for every convolution output, zero-filled once (the scatter-add kernels accumulate)
  // (the conv1 table / bits kernels write every row themselves: their outputs live outside the zeroed slab)
  int64_t total = 0, total_direct = 0;
  for (auto& L : layers) (L.table || L.bits ? total_direct : total) += (int64_t)L.n_out * L.conv->cout;
  float *slab, *slab_direct;
  DGR_TRY(aalloc(c, total, &slab));
  DGR_TRY(aalloc(c, total_direct, &slab_direct));
  if (total > 0) DGR_CUDA_CHECK(cudaMemsetAsync(slab, 0, (size_t)total * sizeof(float), c->stream));
  int64_t ofs = 0, ofs_direct = 0;
  auto take = [&](const LayerExec& L) {
    const bool direct = L.table || L.bits;
    float* b = direct ? slab_direct + ofs_direct : slab + ofs;
    (direct ? ofs_direct : ofs) += (int64_t)L.n_out * L.conv->cout;
    return b;
  };
  // max |activation| of every elementwise-pass output, reduced in that pass: the 3xFP16 layers read their
  // input's slot instead of sweeping the tensor again
  float* amax_slots;
  DGR_TRY(aalloc(c, (int64_t)layers.size() + 1, &amax_slots));
  DGR_CUDA_CHECK(cudaMemsetAsync(amax_slots, 0, (layers.size() + 1) * sizeof(float), c->stream));
  int n_slots = 0;
  c->amax_of.clear();
  auto conv_bn = [&](const LayerExec& L, const float* feat, const float* residual, int relu, bool want_amax,
                     float** res) -> int32_t {
    float* o = take(L);
    DGR_TRY(run_conv(c, L, feat, o));
    if (!L.table && !L.bits) {
      float* slot = (want_amax && L.conv->cout % 4 == 0) ? amax_slots + n_slots++ : nullptr;
      DGR_TRY(dgr_affine_act_amax(o, L.n_out, L.conv->cout, L.conv->scale, L.conv->shift, residual, relu, o, slot, st));
      if (slot != nullptr) c->amax_of[o] = slot;
    }
    *res = o;
    return DGR_OK;
  };
  const float* feat = feats_in;
  const float* skips[4] = {nullptr, nullptr, nullptr, nullptr};
  size_t li = 0;
  for (int stage = 0; stage < 7; ++stage) {
    float *a, *h, *b;
    // an output's maximum is reduced in its elementwise pass only when a 3xFP16 layer consumes it
    const bool next_f16 = stage < 6 && stage != 4 && stage != 5 && li + 3 < layers.size() && layers[li + 3].conv->f16;
    DGR_TRY(conv_bn(layers[li], feat, nullptr, 0, layers[li + 1].conv->f16, &a));
    DGR_TRY(conv_bn(layers[li + 1], a, nullptr, 1, layers[li + 2].conv->f16, &h));
    DGR_TRY(conv_bn(layers[li + 2], h, a, 1, next_f16, &b));
    const int n_rows = layers[li + 2].n_out, ch = layers[li + 2].conv->cout;
    li += 3;
    feat = b;
    if (stage < 4) {
      skips[stage] = b;
    } else if (stage < 6) {
      // decoder levels 4 and 3 feed a 3^D transposed convolution: materialise ME.cat(decoder, skip)
      const int sk = 2 - (stage - 4);
      const int csk = net->C[sk + 1];
      float* cat;
      DGR_TRY(aalloc(c, (int64_t)n_rows * (ch + csk), &cat));
      DGR_TRY(dgr_cat2(b, ch, skips[sk], csk, n_rows, cat, st));
      feat = cat;
    }
  }
  // conv1_tr reads (decoder, skip) directly; final adds the bias and (FCGF) L2-normalises
  float* h;
  DGR_TRY(aalloc(c, (int64_t)n[0] * net->T[1], &h));
  DGR_TRY(dgr_linear_fwd(feat, net->T[2], skips[0], net->C[1], n[0], net->conv1_tr_w, net->T[1], nullptr, 1, 0, h, st));
  DGR_TRY(dgr_linear_fwd(h, net->T[1], nullptr, 0, n[0], net->final_w, net->out_ch, net->final_b, 0, net->normalize, out,
                         st));
  return DGR_OK;
}

int32_t ones_features(dgr_ctx* c, int64_t n, float** out) {
  DGR_TRY(aalloc(c, n, out));
  if (n > 0) fill_f32_kernel<<<dgr_blocks(n, 256), 256, 0, c->stream>>>(*out, n, 1.0f);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

void set_tap(dgr_ctx* c, int which, const void* p, int64_t rows, int32_t cols, int32_t elem = 4) {
  c->taps[which].p = p;
  c->taps[which].rows = rows;
  c->taps[which].cols = cols;
  c->taps[which].elem = elem;
}

int32_t stage_input(dgr_ctx* c, int slot, const void* host, size_t bytes, void** dev) {
  if (c->stage_cap[slot] < bytes) {
    if (c->stage[slot]) DGR_CUDA_CHECK(cudaFreeHost(c->stage[slot]));
    c->stage[slot] = nullptr;
    size_t cap = bytes + bytes / 4 + 4096;
    DGR_CUDA_CHECK(cudaHostAlloc(&c->stage[slot], cap, cudaHostAllocDefault));
    c->stage_cap[slot] = cap;
  }
  memcpy(c->stage[slot], host, bytes);
  void* d;
  DGR_TRY(c->arena.alloc_raw(bytes, &d));
  DGR_CUDA_CHECK(cudaMemcpyAsync(d, c->stage[slot], bytes, cudaMemcpyHostToDevice, c->stream));
  c->h2d_bytes += (int64_t)bytes;
  *dev = d;
  return DGR_OK;
}

}  // namespace

// =========================================================================================
// C ABI
// =========================================================================================
extern "C" {

int32_t dgr_ctx_create(int32_t device, void* stream, dgr_ctx_t** out) {
  DGR_ARG_CHECK(out != nullptr, "out is null");
  DGR_TRY(dgr_device_check(device));
  DGR_CUDA_CHECK(cudaSetDevice(device));
  dgr_ctx* c = new dgr_ctx();
  c->device = device;
  if (stream != nullptr) {
    c->stream = (cudaStream_t)stream;
  } else {
    DGR_CUDA_CHECK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  DGR_CUDA_CHECK(cudaMalloc(&c->meta_dev, kMetaInts * sizeof(int32_t)));
  DGR_CUDA_CHECK(cudaMemset(c->meta_dev, 0, kMetaInts * sizeof(int32_t)));
  DGR_CUDA_CHECK(cudaHostAlloc(&c->meta_host, kMetaInts * sizeof(int32_t), cudaHostAllocDefault));
  DGR_CUDA_CHECK(cudaMalloc(&c->res_dev, 64 * sizeof(double)));
  DGR_CUDA_CHECK(cudaMemset(c->res_dev, 0, 64 * sizeof(double)));
  DGR_CUDA_CHECK(cudaHostAlloc(&c->res_host, 64 * sizeof(double), cudaHostAllocDefault));
  *out = c;
  return DGR_OK;
}

int32_t dgr_ctx_destroy(dgr_ctx_t* c) {
  if (c == nullptr) return DGR_OK;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  c->arena.release();
  for (auto& kv : c->offsets) {
    cudaFree(kv.second.second);
    delete kv.second.first;
  }
  for (auto& r : c->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
  for (auto e : c->event_pool) cudaEventDestroy(e);
  for (auto e : c->stage_marks) cudaEventDestroy(e);
  cudaFree(c->meta_dev);
  cudaFreeHost(c->meta_host);
  cudaFree(c->res_dev);
  cudaFreeHost(c->res_host);
  for (int s = 0; s < 2; ++s)
    if (c->stage[s]) cudaFreeHost(c->stage[s]);
  if (c->own_stream) cudaStreamDestroy(c->stream);
  delete c;
  return DGR_OK;
}

void* dgr_ctx_stream(dgr_ctx_t* c) { return c != nullptr ? (void*)c->stream : nullptr; }

/* stats[0..6) = host reads, device-to-host bytes, host-to-device bytes of the last pair / forward call,
 * arena high-water mark [bytes], cudaMalloc calls of the arena so far, arena chunks. */
int32_t dgr_ctx_stats(dgr_ctx_t* c, int64_t* stats) {
  DGR_ARG_CHECK(c != nullptr && stats != nullptr, "null argument");
  stats[0] = c->reads; stats[1] = c->d2h_bytes; stats[2] = c->h2d_bytes;
  stats[3] = (int64_t)c->arena.high; stats[4] = c->arena.n_malloc; stats[5] = (int64_t)c->arena.chunks.size();
  return DGR_OK;
}

int32_t dgr_ctx_profile(dgr_ctx_t* c, int32_t enable) {
  DGR_ARG_CHECK(c != nullptr, "null context");
  for (auto& r : c->prof) { c->event_pool.push_back(r.e0); c->event_pool.push_back(r.e1); }
  c->prof.clear();
  c->profile = enable != 0;
  return DGR_OK;
}

/* Synchronises the context's stream and returns the convolution launches recorded since
 * dgr_ctx_profile(1): rows of (milliseconds, algorithmic flops, gather-scatter-model bytes, kind). */
int64_t dgr_ctx_profile_read(dgr_ctx_t* c, double* rows, int64_t max_rows) {
  if (c == nullptr) return 0;
  cudaStreamSynchronize(c->stream);
  int64_t n = 0;
  for (auto& r : c->prof) {
    if (n >= max_rows) break;
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    rows[4 * n + 0] = ms; rows[4 * n + 1] = r.flops; rows[4 * n + 2] = r.bytes; rows[4 * n + 3] = r.kind;
    ++n;
  }
  return n;
}

/* Stage times [ms] of the last dgr_pair_register with profiling on, in order: upload + voxelisation, FCGF
 * coordinate phase, host read 1 + FCGF pair lists, FCGF convolutions, feature kNN, 6-D coordinate phase, host
 * read 2 + 6-D pair lists, inlier convolutions, weights + Procrustes + refinement (+ ICP).  Returns the count. */
int32_t dgr_ctx_stage_times(dgr_ctx_t* c, double* ms, int32_t max_stages) {
  if (c == nullptr || ms == nullptr) return 0;
  cudaStreamSynchronize(c->stream);
  int n = 0;
  for (size_t i = 1; i < c->stage_marks.size() && n < max_stages; ++i, ++n) {
    float t = 0.f;
    cudaEventElapsedTime(&t, c->stage_marks[i - 1], c->stage_marks[i]);
    ms[n] = t;
  }
  return n;
}

/* ---- network ------------------------------------------------------------------------ */
/* params: 66 device pointers in execution order -
 *   for l = 1..4: conv{l}.kernel, norm{l} scale, shift, block{l}.conv1.kernel, norm1 scale, shift,
 *                 block{l}.conv2.kernel, norm2 scale, shift                                   (36)
 *   for l = 4,3,2: conv{l}_tr.kernel, norm{l}_tr scale, shift, block{l}_tr.conv1.kernel, ... (27)
 *   conv1_tr.kernel, final.kernel, final.bias                                                  (3)
 * kernels in ME layout [K, cin, cout]; scale / shift = eval BatchNorm folded. */
int32_t dgr_net_create(int32_t device, int32_t D, int32_t in_ch, int32_t out_ch, int32_t conv1_ks, int32_t normalize,
                       const int32_t* channels, const int32_t* tr_channels, const float* const* params,
                       int32_t n_params, void* stream, dgr_net_t** out) {
  DGR_ARG_CHECK(out != nullptr && params != nullptr && channels != nullptr && tr_channels != nullptr, "null argument");
  DGR_ARG_CHECK(n_params == 66, "a ResUNet2-family network has 66 parameter tensors (see dgr_b200.h)");
  DGR_ARG_CHECK(D == 3 || D == 6, "D must be 3 or 6");
  DGR_ARG_CHECK(conv1_ks == 3 || conv1_ks == 5 || conv1_ks == 7, "conv1 kernel size must be 3, 5 or 7");
  DGR_CUDA_CHECK(cudaSetDevice(device));
  dgr_net* net = new dgr_net();
  net->device = device;
  net->D = D; net->in_ch = in_ch; net->out_ch = out_ch; net->conv1_ks = conv1_ks; net->normalize = normalize;
  for (int i = 0; i < 5; ++i) { net->C[i] = channels[i]; net->T[i] = tr_channels[i]; }
  const int* C = net->C;
  const int* T = net->T;
  int k3 = 1, k1 = 1;
  for (int a = 0; a < D; ++a) { k3 *= 3; k1 *= conv1_ks; }
  int pi = 0;
  auto set_conv = [&](Conv& cv, int cin, int cout, int ksize, int K) -> int32_t {
    cv.w = params[pi++]; cv.scale = params[pi++]; cv.shift = params[pi++];
    cv.cin = cin; cv.cout = cout; cv.ksize = ksize; cv.K = K;
    cv.tc = dgr_spconv_tc_supported(cin, cout) != 0;
    cv.f16 = cv.tc && tc_f16_enabled() && cout >= tc_f16_min_cout() &&
             dgr_spconv_tc_f16_supported(cin, cout) != 0;
    if (cv.f16) {
      DGR_CUDA_CHECK(cudaMalloc(&cv.packed16, (size_t)4 * K * cin * cout));
      net->owned.push_back((float*)cv.packed16);
      DGR_CUDA_CHECK(cudaMalloc(&cv.wscale, 2 * sizeof(float)));
      net->owned.push_back(cv.wscale);
      DGR_TRY(dgr_pack_weight_f16(cv.w, K, cin, cout, cv.packed16, cv.wscale, stream));
    } else if (cv.tc) {
      DGR_CUDA_CHECK(cudaMalloc(&cv.packed, (size_t)2 * K * cin * cout * sizeof(float)));
      net->owned.push_back(cv.packed);
      DGR_TRY(dgr_pack_weight_tf32(cv.w, K, cin, cout, cv.packed, stream));
    }
    return DGR_OK;
  };
  const int enc_in[4] = {in_ch, C[1], C[2], C[3]};
  int32_t rc = DGR_OK;
  for (int s = 0; s < 4 && rc == DGR_OK; ++s) {
    rc = set_conv(net->enc[s], enc_in[s], C[s + 1], s == 0 ? conv1_ks : 3, s == 0 ? k1 : k3);
    if (rc == DGR_OK) rc = set_conv(net->eb1[s], C[s + 1], C[s + 1], 3, k3);
    if (rc == DGR_OK) rc = set_conv(net->eb2[s], C[s + 1], C[s + 1], 3, k3);
  }
  const int dec_in[3] = {C[4], C[3] + T[4], C[2] + T[3]};
  const int dec_out[3] = {T[4], T[3], T[2]};
  for (int d = 0; d < 3 && rc == DGR_OK; ++d) {
    rc = set_conv(net->dec[d], dec_in[d], dec_out[d], 3, k3);
    if (rc == DGR_OK) rc = set_conv(net->db1[d], dec_out[d], dec_out[d], 3, k3);
    if (rc == DGR_OK) rc = set_conv(net->db2[d], dec_out[d], dec_out[d], 3, k3);
  }
  if (rc != DGR_OK) {
    for (auto p : net->owned) cudaFree(p);
    delete net;
    return rc;
  }
  net->conv1_tr_w = params[pi++];
  net->final_w = params[pi++];
  net->final_b = params[pi++];
  DGR_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  *out = net;
  return DGR_OK;
}

int32_t dgr_net_destroy(dgr_net_t* net) {
  if (net == nullptr) return DGR_OK;
  cudaSetDevice(net->device);
  for (auto p : net->owned) cudaFree(p);
  delete net;
  return DGR_OK;
}

/* Forward pass of one sparse tensor: coords [n, D+1] int32 (distinct rows, column 0 = batch), feats [n, in_ch]
 * (NULL = ones), out [n, out_ch]; device pointers, work on the context's stream; returns after the launches are
 * enqueued (one host read inside).  The arena is reset at entry: results of earlier calls on this context
 * must have been consumed. */
int32_t dgr_net_forward(dgr_ctx_t* c, dgr_net_t* net, const int32_t* coords, int64_t n, const float* feats, float* out) {
  DGR_ARG_CHECK(c != nullptr && net != nullptr && coords != nullptr && out != nullptr, "null argument");
  DGR_ARG_CHECK(n >= 1 && n < (1ll << 30), "row count out of range");
  DGR_CUDA_CHECK(cudaSetDevice(c->device));
  DGR_CUDA_CHECK(cudaStreamSynchronize(c->stream));
  DGR_TRY(c->arena.reset());
  c->reads = c->d2h_bytes = c->h2d_bytes = 0;
  void* st = c->stream;
  Plan p;
  p.D = net->D;
  p.ncols = net->D + 1;
  int32_t* minmax;
  dgr_keyspec_t* spec;
  DGR_TRY(aalloc(c, 2 * DGR_MAX_COLS, &minmax));
  DGR_TRY(aalloc(c, 1, &spec));
  DGR_TRY(dgr_coords_minmax(coords, n, p.ncols, minmax, st));
  DGR_TRY(dgr_keyspec_build(minmax, p.ncols, kKeyMargin, spec, st));
  p.spec = spec;
  p.lv[0].coords = const_cast<int32_t*>(coords);
  p.lv[0].n_max = n;
  p.lv[0].n = (int)n;
  p.input_ones = feats == nullptr;
  DGR_TRY(plan_begin(c, net, p));
  DGR_TRY(read_meta(c, meta_ints(p)));
  DGR_TRY(plan_finish(c, p));
  const float* f = feats;
  if (f == nullptr) {
    DGR_ARG_CHECK(net->in_ch == 1, "feats may be NULL (= ones) only for one input channel");
    float* ones;
    DGR_TRY(ones_features(c, n, &ones));
    f = ones;
  }
  return run_network(c, net, p, f, out);
}

/* ---- scan pair ---------------------------------------------------------------------- */
/* result (host double[64]):
 *   [0..16)  R (9, row-major), t (3), refinement iterations, final loss, break count, active correspondences
 *   [16]     weight sum (the gate of core/deep_global_registration.py:276-281 is the caller's decision)
 *   [17..37) ICP: 4x4 pose, fitness, inlier RMSE, iterations, correspondences (zeros when use_icp == 0)
 *   [40..44) N0, N1 (voxels per cloud), host reads, device-to-host bytes                              */
int32_t dgr_pair_register(dgr_ctx_t* c, dgr_net_t* fcgf, dgr_net_t* inlier, const void* xyz0, int64_t n_raw0,
                          int32_t is_f64_0, const void* xyz1, int64_t n_raw1, int32_t is_f64_1, int32_t on_host,
                          double voxel, float clip, int32_t use_icp, double* result) {
  DGR_ARG_CHECK(c != nullptr && fcgf != nullptr && inlier != nullptr && result != nullptr, "null argument");
  DGR_ARG_CHECK(n_raw0 >= 1 && n_raw1 >= 1 && n_raw0 + n_raw1 < (1ll << 30), "point counts out of range");
  DGR_ARG_CHECK(fcgf->D == 3 && fcgf->in_ch == 1, "FCGF network: D = 3, one input channel");
  DGR_ARG_CHECK(inlier->D == 6 && inlier->in_ch == 1 && inlier->out_ch == 1,
                "inlier network: D = 6, feature type 'ones' (other feature types run stage by stage)");
  DGR_ARG_CHECK(voxel > 0, "voxel size must be positive");
  DGR_CUDA_CHECK(cudaSetDevice(c->device));
  DGR_CUDA_CHECK(cudaStreamSynchronize(c->stream));
  DGR_TRY(c->arena.reset());
  c->reads = c->d2h_bytes = c->h2d_bytes = 0;
  for (auto& t : c->taps) t = dgr_ctx::Tap{};       // the arena is reused: a refused pair leaves no stale taps
  c->pair_xyz = nullptr;
  void* st = c->stream;
  const int64_t n_raw = n_raw0 + n_raw1;
  for (auto e : c->stage_marks) c->event_pool.push_back(e);
  c->stage_marks.clear();
  StageRanges ranges;
  mark_stage(c, ranges, 0);                                // 0: start

  // ---- stage 0: upload + voxelise both scans into ONE batched coordinate set (batch 0 / 1) -------------
  const void *d0 = xyz0, *d1 = xyz1;
  if (on_host) {
    void *a, *b;
    DGR_TRY(stage_input(c, 0, xyz0, (size_t)n_raw0 * 3 * (is_f64_0 ? 8 : 4), &a));
    DGR_TRY(stage_input(c, 1, xyz1, (size_t)n_raw1 * 3 * (is_f64_1 ? 8 : 4), &b));
    d0 = a;
    d1 = b;
  }
  int32_t *raw, *minmax, *mm_scratch, *sel, *inverse, *n_unique, *slot_ws, *scan_ws, *coords;
  dgr_keyspec_t* spec;
  float* xyz;
  DGR_TRY(aalloc(c, n_raw * 4, &raw));
  DGR_TRY(aalloc(c, 8, &minmax));
  DGR_TRY(aalloc(c, 8, &mm_scratch));
  DGR_TRY(aalloc(c, 1, &spec));
  DGR_TRY(dgr_quantize_points(d0, is_f64_0, n_raw0, voxel, 0, raw, mm_scratch, st));
  DGR_TRY(dgr_quantize_points(d1, is_f64_1, n_raw1, voxel, 1, raw + 4 * n_raw0, mm_scratch, st));
  DGR_TRY(dgr_coords_minmax(raw, n_raw, 4, minmax, st));
  DGR_TRY(dgr_keyspec_build(minmax, 4, kKeyMargin, spec, st));
  const int64_t cap = next_pow2(2 * (n_raw > 512 ? n_raw : 512));
  uint64_t* keys;
  int32_t* vals;
  DGR_TRY(aalloc(c, cap, &keys));
  DGR_TRY(aalloc(c, cap, &vals));
  DGR_TRY(aalloc(c, n_raw, &sel));
  DGR_TRY(aalloc(c, n_raw, &inverse));
  DGR_TRY(aalloc(c, 2, &n_unique));
  DGR_TRY(aalloc(c, n_raw, &slot_ws));
  DGR_TRY(aalloc(c, dgr_scan_ws_elems(n_raw), &scan_ws));
  DGR_TRY(dgr_hash_clear(keys, vals, cap, st));
  DGR_TRY(dgr_unique_first(raw, n_raw, 4, spec, keys, vals, cap, sel, inverse, n_unique, slot_ws, scan_ws, st));
  DGR_TRY(aalloc(c, n_raw * 4, &coords));
  DGR_TRY(aalloc(c, n_raw * 3, &xyz));
  DGR_TRY(dgr_compact_voxel_pair(raw, sel, n_unique, n_raw0, n_raw1, d0, is_f64_0, d1, is_f64_1, voxel, coords, xyz,
                                 c->meta_dev, st));

  mark_stage(c, ranges, 1);                                        // 1: upload + voxelisation enqueued
  // ---- stage 1: FCGF features of both clouds in one forward pass ------------------------------------------
  Plan pf;
  pf.D = 3;
  pf.ncols = 4;
  pf.spec = spec;
  pf.lv[0].coords = coords;
  pf.lv[0].n_max = n_raw;
  pf.lv[0].n_dev = c->meta_dev;       // N = meta[0]
  pf.lv[0].keys = keys;
  pf.lv[0].vals = vals;
  pf.lv[0].cap = cap;
  pf.input_ones = true;
  DGR_TRY(plan_begin(c, fcgf, pf));
  mark_stage(c, ranges, 2);                                        // 2: FCGF coordinate phase
  DGR_TRY(read_meta(c, meta_ints(pf)));                 // host read 1
  const int N = c->meta_host[0], N0 = c->meta_host[1], N1 = c->meta_host[2];
  if (c->meta_host[3] != 0) {
    dgr_set_error("coordinates are not finite, or their extent does not fit a 63-bit packed key");
    return DGR_ERR_ARG;
  }
  if (N0 < 1 || N1 < 1) {
    dgr_set_error("empty cloud after voxelisation");
    return DGR_ERR_ARG;
  }
  pf.lv[0].n = N;
  DGR_TRY(plan_finish(c, pf));
  mark_stage(c, ranges, 3);                                        // 3: FCGF pair lists + work lists
  float *ones, *F;
  DGR_TRY(ones_features(c, N, &ones));
  const int Cf = fcgf->out_ch;
  DGR_TRY(aalloc(c, (int64_t)N * Cf, &F));
  DGR_TRY(run_network(c, fcgf, pf, ones, F));
  mark_stage(c, ranges, 4);                                        // 4: FCGF convolution phase

  // ---- stage 2: feature nearest neighbour (core/knn.py:23-74) --------------------------------------------
  int32_t* idx1;
  uint64_t* packed_ws;
  DGR_TRY(aalloc(c, N0, &idx1));
  DGR_TRY(aalloc(c, N0, &packed_ws));
  if (dgr_knn_tc_supported(Cf)) {
    float* fws;
    DGR_TRY(aalloc(c, dgr_knn_tc_ws_elems(N0, N1, Cf), &fws));
    DGR_TRY(dgr_knn_top1_tc(F, N0, F + (int64_t)N0 * Cf, N1, Cf, packed_ws, fws, idx1, nullptr, st));
  } else {
    DGR_TRY(dgr_knn_top1(F, N0, F + (int64_t)N0 * Cf, N1, Cf, packed_ws, idx1, nullptr, st));
  }

  mark_stage(c, ranges, 5);                                        // 5: feature kNN
  // ---- stage 3/4: 6-D coordinates and the inlier network ---------------------------------------------------
  int32_t *coords6, *minmax6;
  dgr_keyspec_t* spec6;
  DGR_TRY(aalloc(c, (int64_t)N0 * 7, &coords6));
  DGR_TRY(aalloc(c, 2 * DGR_MAX_COLS, &minmax6));
  DGR_TRY(aalloc(c, 1, &spec6));
  DGR_TRY(dgr_inlier_coords(coords, coords + 4 * (int64_t)N0, idx1, N0, coords6, st));
  DGR_TRY(dgr_coords_minmax(coords6, N0, 7, minmax6, st));
  DGR_TRY(dgr_keyspec_build(minmax6, 7, kKeyMargin, spec6, st));
  Plan pi;
  pi.D = 6;
  pi.ncols = 7;
  pi.spec = spec6;
  pi.lv[0].coords = coords6;
  pi.lv[0].n_max = N0;
  pi.lv[0].n = N0;
  pi.input_ones = true;
  DGR_TRY(plan_begin(c, inlier, pi));
  mark_stage(c, ranges, 6);                                        // 6: 6-D coordinate phase
  DGR_TRY(read_meta(c, meta_ints(pi)));                 // host read 2
  DGR_TRY(plan_finish(c, pi));
  mark_stage(c, ranges, 7);                                        // 7: 6-D pair lists + work lists
  float *ones6, *logit, *w;
  DGR_TRY(ones_features(c, N0, &ones6));
  DGR_TRY(aalloc(c, N0, &logit));
  DGR_TRY(aalloc(c, N0, &w));
  DGR_TRY(run_network(c, inlier, pi, ones6, logit));
  mark_stage(c, ranges, 8);                                        // 8: inlier convolution phase

  // ---- stage 5: weights, gate sum, weighted Procrustes + SE(3) refinement, ICP ---------------------------
  double *wsum, *icp_res = nullptr;
  float *pack_ws, *se3;
  int32_t* cnt_ws;
  DGR_TRY(aalloc(c, 1, &wsum));
  DGR_TRY(aalloc(c, 7 * (int64_t)N0, &pack_ws));
  DGR_TRY(aalloc(c, 4, &cnt_ws));
  DGR_TRY(aalloc(c, 16, &se3));
  DGR_TRY(dgr_sigmoid_clip_sum(logit, N0, clip, w, wsum, st));
  const float* xyz1p = xyz + 3 * (int64_t)N0;
  DGR_TRY(dgr_se3_register(xyz, xyz1p, idx1, w, N0, (float)(2 * voxel), 1000, 20, 1e-4f, 0.1f, 0.999f, pack_ws,
                           cnt_ws, se3, st));
  if (use_icp) {
    double *T12, *icp_ws;
    int64_t icp_words = 0;
    DGR_TRY(dgr_icp_ws_elems(N0, &icp_words));
    DGR_TRY(aalloc(c, 12, &T12));
    DGR_TRY(aalloc(c, icp_words, &icp_ws));
    DGR_TRY(aalloc(c, 20, &icp_res));
    pose_to_T12_kernel<<<1, 32, 0, c->stream>>>(se3, T12);
    dgr_note_launches(1);
    // nearest target point through the pair's voxel hash: rows of cloud 1 are rows N0.. of `xyz` (batch 1)
    DGR_TRY(dgr_icp(xyz, N0, xyz, nullptr, spec, keys, vals, cap, 1, voxel, 2 * voxel, T12, 30, 1e-6, 1e-6, icp_ws,
                    icp_res, st));
  }
  mark_stage(c, ranges, 9);                                        // 9: weights + Procrustes + refinement (+ ICP)
  pack_result_kernel<<<1, 64, 0, c->stream>>>(se3, wsum, icp_res, c->res_dev);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  DGR_CUDA_CHECK(cudaMemcpyAsync(c->res_host, c->res_dev, 40 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  DGR_CUDA_CHECK(cudaStreamSynchronize(c->stream));       // host read 3
  c->reads += 1;
  c->d2h_bytes += 40 * 8;
  memcpy(result, c->res_host, 40 * sizeof(double));
  result[40] = N0; result[41] = N1; result[42] = (double)c->reads; result[43] = (double)c->d2h_bytes;
  for (int k = 44; k < 64; ++k) result[k] = 0.0;

  set_tap(c, 0, coords, N, 4);
  set_tap(c, 1, xyz, N, 3);
  set_tap(c, 2, F, N, Cf);
  set_tap(c, 3, idx1, N0, 1);
  set_tap(c, 4, coords6, N0, 7);
  set_tap(c, 5, logit, N0, 1);
  set_tap(c, 6, w, N0, 1);
  set_tap(c, 7, sel, N, 1);
  c->pair_n0 = N0; c->pair_n1 = N1; c->pair_voxel = voxel;
  c->pair_xyz = xyz; c->pair_idx1 = idx1; c->pair_spec = spec; c->pair_keys = keys; c->pair_vals = vals;
  c->pair_cap = cap;
  return DGR_OK;
}

/* Safeguard branch (core/deep_global_registration.py:302-315) on the pair the context last registered:
 * RANSAC over its correspondences, then (use_icp) the same ICP from the RANSAC pose.
 * result (host double[40]): RANSAC 20 doubles (pose, fitness, inlier RMSE, hypothesis, inliers), ICP 20. */
int32_t dgr_pair_safeguard(dgr_ctx_t* c, double max_dist, int64_t num_hyp, uint64_t seed, int32_t use_icp,
                           double* result) {
  DGR_ARG_CHECK(c != nullptr && result != nullptr, "null argument");
  DGR_ARG_CHECK(c->pair_xyz != nullptr, "no registered pair on this context");
  DGR_CUDA_CHECK(cudaSetDevice(c->device));
  void* st = c->stream;
  const int64_t N0 = c->pair_n0;
  int64_t words = 0;
  DGR_TRY(dgr_ransac_ws_elems(N0, num_hyp, &words));
  uint64_t* ws;
  double *res, *icp_res = nullptr;
  DGR_TRY(aalloc(c, words, &ws));
  DGR_TRY(aalloc(c, 40, &res));
  DGR_CUDA_CHECK(cudaMemsetAsync(res, 0, 40 * sizeof(double), c->stream));
  DGR_TRY(dgr_ransac_correspondence(c->pair_xyz, c->pair_xyz + 3 * N0, nullptr, c->pair_idx1, N0, max_dist, num_hyp,
                                    seed, ws, res, st));
  if (use_icp) {
    double* icp_ws;
    int64_t icp_words = 0;
    DGR_TRY(dgr_icp_ws_elems(N0, &icp_words));
    DGR_TRY(aalloc(c, icp_words, &icp_ws));
    icp_res = res + 20;
    DGR_TRY(dgr_icp(c->pair_xyz, N0, c->pair_xyz, nullptr, c->pair_spec, c->pair_keys, c->pair_vals, c->pair_cap, 1,
                    c->pair_voxel, 2 * c->pair_voxel, res, 30, 1e-6, 1e-6, icp_ws, icp_res, st));
  }
  DGR_CUDA_CHECK(cudaMemcpyAsync(c->res_host, res, 40 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  DGR_CUDA_CHECK(cudaStreamSynchronize(c->stream));
  c->reads += 1;
  c->d2h_bytes += 40 * 8;
  memcpy(result, c->res_host, 40 * sizeof(double));
  return DGR_OK;
}

/* Intermediate tensors of the last dgr_pair_register on this context: which = 0 coords [N, 4] int32 (both
 * clouds, batch 0 / 1), 1 xyz [N, 3] float32, 2 FCGF features [N, C], 3 correspondences idx1 [N0] int32,
 * 4 6-D coordinates [N0, 7] int32, 5 inlier logits [N0], 6 weights [N0], 7 kept raw-point indices sel [N]
 * int32 (rows of cloud 1 offset by n_raw0).  dst == NULL: only the shape is returned; otherwise the tensor is
 * copied to the DEVICE buffer dst (synchronous). */
int32_t dgr_pair_tap(dgr_ctx_t* c, int32_t which, int64_t* rows, int32_t* cols, void* dst) {
  DGR_ARG_CHECK(c != nullptr && which >= 0 && which < 8, "bad tap");
  const auto& t = c->taps[which];
  DGR_ARG_CHECK(t.p != nullptr, "no registered pair on this context");
  if (rows) *rows = t.rows;
  if (cols) *cols = t.cols;
  if (dst != nullptr) {
    DGR_CUDA_CHECK(cudaMemcpyAsync(dst, t.p, (size_t)t.rows * t.cols * t.elem, cudaMemcpyDeviceToDevice, c->stream));
    DGR_CUDA_CHECK(cudaStreamSynchronize(c->stream));
  }
  return DGR_OK;
}

}  // extern "C"
