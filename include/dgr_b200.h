/*
 * dgr_b200.h - C ABI of libdgr_b200.so: the H100-native (sm_90a) replacement for the
 * native layer underneath Deep Global Registration's pairwise-registration hot path.
 *
 * The reference (chrischoy/DeepGlobalRegistration) has no native code of its own; the
 * native layer on this path is the pybind11 module of MinkowskiEngine 0.5.4
 * (requirements.txt:24) plus a handful of ATen / LAPACK kernels reached through torch.
 * Every entry point below names the reference call site it serves.
 *
 * Conventions
 *   - plain C, no torch types: raw device pointers + extents; the caller owns every
 *     buffer (inputs, outputs, workspaces); the library never allocates, frees or
 *     retains memory beyond one call (exception: the round-2 executor contexts at the end of this
 *     header own a device arena);
 *   - every function enqueues its work on `stream` (a cudaStream_t passed as void*)
 *     and returns without synchronising, unless stated otherwise;
 *   - return value 0 = OK, negative = error; dgr_last_error() returns a thread-local
 *     message for the last failing call;
 *   - all row indices are int32; feature matrices are row-major float32 [rows, channels];
 *     coordinate matrices are row-major int32 [rows, ncols] with column 0 = batch index
 *     (ME.utils.batched_coordinates layout, core/deep_global_registration.py:158);
 *   - there is no CPU fallback: on a machine without an sm_90 device every compute
 *     entry point fails with DGR_ERR_DEVICE.
 */
#ifndef DGR_B200_H_
#define DGR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGR_OK 0
#define DGR_ERR_CUDA (-1)
#define DGR_ERR_ARG (-2)
#define DGR_ERR_DEVICE (-3)

#define DGR_MAX_COLS 8      /* batch + up to 7 spatial columns (DGR uses 4 and 7) */

/* Packing rule of one coordinate row into a 64-bit hash key:
 *   key = sum_i (uint64)(c[i] - lo[i]) << shift[i]
 * Lives in DEVICE memory (written by dgr_keyspec_build, read by every kernel that hashes
 * coordinates) so that building it costs no host round trip.  `overflow` != 0 means the
 * coordinate extent does not fit 63 bits and every later result is invalid; the host
 * checks it at its next natural synchronisation point and raises. */
typedef struct dgr_keyspec {
  int32_t ncols;
  int32_t overflow;
  int32_t lo[DGR_MAX_COLS];
  int32_t shift[DGR_MAX_COLS];
  int32_t bits[DGR_MAX_COLS];
} dgr_keyspec_t;

/* ---- library ------------------------------------------------------------------------ */
int32_t dgr_version(void);
const char* dgr_last_error(void);
/* Number of CUDA kernels this library has launched in this process (all threads). */
int64_t dgr_launch_count(void);
/* 0 if device `device` is sm_90 (H100); DGR_ERR_DEVICE otherwise.  Host-only query. */
int32_t dgr_device_check(int32_t device);

/* ---- voxelisation: ME.utils.sparse_quantize + re-floor of preprocess()
 *      (core/deep_global_registration.py:152-158) ------------------------------------- */
/* coords[r] = (batch, floor(xyz[r] / voxel)) with the division in the input dtype
 * (is_f64 ? double : float), plus per-column min/max into minmax[2*4] (device int32:
 * mins then maxes; initialised by the call). */
int32_t dgr_quantize_points(const void* xyz, int32_t is_f64, int64_t n, double voxel, int32_t batch,
                            int32_t* coords, int32_t* minmax, void* stream);
/* Per-column min/max of an existing coordinate matrix into minmax[2*ncols]. */
int32_t dgr_coords_minmax(const int32_t* coords, int64_t n, int32_t ncols, int32_t* minmax,
                          void* stream);
/* Key spec from min/max with `margin` spare cells on both sides of every spatial axis
 * (kernel offsets and coarser strides stay inside the packed range). */
int32_t dgr_keyspec_build(const int32_t* minmax, int32_t ncols, int32_t margin, dgr_keyspec_t* spec,
                          void* stream);

/* ---- coordinate hash: ME CoordinateMap insert / find (ME.SparseTensor(...),
 *      core/deep_global_registration.py:167,214) ------------------------------------- */
/* keys[cap] (uint64) / vals[cap] (int32) open-addressing table, cap a power of two. */
int32_t dgr_hash_clear(uint64_t* keys, int32_t* vals, int64_t cap, void* stream);
/* Deduplicate rows keeping the FIRST occurrence (smallest row index) of every distinct
 * coordinate, deterministically:
 *   sel[0..m)      ascending first-occurrence rows,
 *   inverse[n]     row -> index into sel of its representative,
 *   n_unique[2]    (m, spec->overflow) device int32 - one host read for both,
 * and leaves the table mapping key -> index into sel.  slot_ws[n], rank_ws[n] and
 * scan_ws[dgr_scan_ws_elems(n)] are int32 workspaces. */
int32_t dgr_unique_first(const int32_t* coords, int64_t n, int32_t ncols, const dgr_keyspec_t* spec,
                         uint64_t* keys, int32_t* vals, int64_t cap, int32_t* sel, int32_t* inverse,
                         int32_t* n_unique, int32_t* slot_ws, int32_t* rank_ws, int32_t* scan_ws,
                         void* stream);
int64_t dgr_scan_ws_elems(int64_t n);
/* rows[i] -> vals of matching key, or -1. */
int32_t dgr_hash_find(const int32_t* coords, int64_t n, int32_t ncols, const dgr_keyspec_t* spec,
                      const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t* rows_out,
                      void* stream);
/* out[i, :] = src[idx[i], :] for int32 row matrices. */
int32_t dgr_gather_rows_i32(const int32_t* src, const int32_t* idx, int64_t n, int32_t ncols,
                            int32_t* out, void* stream);

/* ---- sparse convolution forward: ME.MinkowskiConvolution / ConvolutionTranspose
 *      (model/residual_block.py:38-44,72-80; graph model/resunet.py:598-649) ---------- */
/* out[out_idx[p], :] += in[in_idx[p], :] @ W[kappa(p)]   for all pairs p.
 * `out` must hold the initial value (zeros, or a bias/residual to accumulate onto).
 * W is [K, cin, cout] row-major fp32 (ME's `kernel` parameter layout).  A transposed
 * convolution passes the down-convolution's lists with in_idx/out_idx exchanged.
 * relu_in != 0 applies max(x, 0) to gathered input rows (fuses a preceding MEF.relu). */
int32_t dgr_spconv_fwd(const float* in_feat, int32_t cin, const float* weight, int32_t cout,
                       const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs,
                       const int32_t* tile_k, const int32_t* tile_start, int32_t n_tiles,
                       int32_t tile_rows, int32_t relu_in, float* out, void* stream);
/* Tensor-core (wgmma, TF32 operands, fp32 register accumulator) variant of dgr_spconv_fwd for
 * cin % 32 == 0 and cout in {16, 32, ..., 256} (dgr_spconv_tc_supported returns 1).
 * weight_t is the layer's weight in the packed layout of dgr_pack_weight_tf32
 * ([K][cin/32][2][cout][32]: per offset and 32-channel chunk the TF32 hi tile and the lo
 * residual tile in shared-memory image order; the host caches it per layer; 2 * K * cin * cout
 * floats).  passes = 3 evaluates every
 * product as hi*hi + lo*hi + hi*lo on TF32 splits (fp32-accurate); passes = 1 is plain
 * TF32 (~1e-3 relative), offered as an opt-in fast mode.  One CTA per 128-pair tile; the weight
 * slab of each 32-channel chunk arrives by one bulk copy. */
int32_t dgr_spconv_tc_supported(int32_t cin, int32_t cout);
int32_t dgr_pack_weight_tf32(const float* w, int32_t K, int32_t cin, int32_t cout, float* packed, void* stream);
int32_t dgr_spconv_tc_fwd(const float* in_feat, int32_t cin, const float* weight_t, int32_t cout,
                          const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs,
                          const int32_t* tile_k, const int32_t* tile_start, int32_t n_tiles,
                          int32_t tile_rows, int32_t passes, float* out, void* stream);
/* kernel_size == 1 convolution (conv1_tr / final, model/resunet.py:578-596):
 *   out = act((concat(a, b) @ W[ca+cb, cout]) + bias), b may be NULL (cb = 0): fuses ME.cat.
 * relu != 0 applies ReLU; normalize != 0 divides every row by (||row||_2 + 1e-8)
 * (model/resunet.py:643-647) and requires cout <= 64. */
int32_t dgr_linear_fwd(const float* a, int32_t ca, const float* b, int32_t cb, int64_t n,
                       const float* weight, int32_t cout, const float* bias, int32_t relu,
                       int32_t normalize, float* out, void* stream);

/* ---- elementwise layers ------------------------------------------------------------ */
/* out = act(x * scale[c] + shift[c] + residual): eval-mode ME.MinkowskiBatchNorm
 * (model/common.py:13) folded to scale/shift, the residual add and MEF.relu of
 * BasicBlockBase.forward (model/residual_block.py:118-134).  scale/shift/residual may be
 * NULL; out may alias x. */
int32_t dgr_affine_act(const float* x, int64_t n, int32_t c, const float* scale, const float* shift,
                       const float* residual, int32_t relu, float* out, void* stream);
/* ME.cat(a, b): out[:, :ca] = a, out[:, ca:] = b (model/resunet.py:624,631,638). */
int32_t dgr_cat2(const float* a, int32_t ca, const float* b, int32_t cb, int64_t n, float* out,
                 void* stream);
/* F / (||F||_2 + 1e-8) row-wise (model/resunet.py:643-647). */
int32_t dgr_l2_normalize(const float* x, int64_t n, int32_t c, float* out, void* stream);

/* ---- feature nearest neighbour: find_knn_gpu(knn=1) (core/knn.py:23-74) with pdist
 *      'L2' (core/metrics.py:62-65) ---------------------------------------------------- */
/* idx[i] = argmin_j sqrt(sum_c (F0[i,c]-F1[j,c])^2 + 1e-7), lowest j on ties.
 * packed_ws[n0] is a uint64 workspace; dist (optional) receives the minimum. */
int32_t dgr_knn_top1(const float* f0, int64_t n0, const float* f1, int64_t n1, int32_t c,
                     uint64_t* packed_ws, int32_t* idx, float* dist, void* stream);

/* Tensor-core variant for c in {32, 64} (dgr_knn_tc_supported): two wgmma (TF32) sweeps
 * find, per row, the candidate columns whose approximate distance is within a proven error
 * bound of the row minimum; only those are evaluated with the exact fp32 arithmetic above.
 * Results are bit-identical to dgr_knn_top1.  ws: dgr_knn_tc_ws_elems(n0, n1, c) floats, 16-byte aligned. */
int32_t dgr_knn_tc_supported(int32_t c);
int64_t dgr_knn_tc_ws_elems(int64_t n0, int64_t n1, int32_t c);
int32_t dgr_knn_top1_tc(const float* f0, int64_t n0, const float* f1, int64_t n1, int32_t c,
                        uint64_t* packed_ws, float* ws, int32_t* idx, float* dist, void* stream);

/* ---- correspondences -> 6-D coordinates, weights (core/deep_global_registration.py:261-272) */
/* out[i] = (coords0[i, 0..3], coords1[idx1[i], 1..3]) int32 [n0, 7]. */
int32_t dgr_inlier_coords(const int32_t* coords0, const int32_t* coords1, const int32_t* idx1,
                          int64_t n0, int32_t* out, void* stream);
/* w = sigmoid(logit); w[w < clip] = 0 (if clip > 0); *wsum (device double) = sum w. */
int32_t dgr_sigmoid_clip_sum(const float* logit, int64_t n, float clip, float* w, double* wsum,
                             void* stream);

/* ---- weighted Procrustes + SE(3) refinement (core/registration.py:91-113,135-194,
 *      core/loss.py:42-61) -------------------------------------------------------------- */
/* Correspondence i pairs x[i] with y[idx1[i]] (idx1 may be NULL: y[i]).
 * result (device float[16]): R row-major [0..9), t [9..12), iterations, final loss,
 * break_count, n_active (correspondences with non-zero weight).
 * max_iter == 0 returns the closed-form weighted Procrustes solution only.
 * pack_ws: float workspace of 7 * n elements; cnt_ws: int32[4]. */
int32_t dgr_se3_register(const float* x, const float* y, const int32_t* idx1, const float* w,
                         int64_t n, float quantization_size, int32_t max_iter,
                         int32_t max_break_count, float break_threshold_ratio, float lr, float gamma,
                         float* pack_ws, int32_t* cnt_ws, float* result, void* stream);

/* ---- Normal estimation and ICP: open3d 0.10 EstimateNormals(KDTreeSearchParamHybrid(radius, max_nn)) and
 *      registration_icp with default criteria, point-to-point (the ICP fine-tune, SURVEY 8f rank 1,
 *      core/deep_global_registration.py:317-322) or TransformationEstimationPointToPlane (the ICP (Point-to-plane)
 *      row of the reference's results; util/pointcloud.py:60, scripts/test_3dmatch.py:72-73) ---------------------- */
/* Normals of the cloud xyz[n] through its OWN voxel hash (keys / vals / spec of a dgr_unique_first table at `cell`,
 * at most one point per cell, rows = rows of xyz, `batch` = its batch column; radius / cell <= 4).  Neighbours of
 * point i: the rows j with |p_j - p_i|^2 < radius^2 (strict; i itself included), the max_nn (1..64) smallest by
 * (d^2, row) when more qualify.  Normal: eigenvector of the smallest eigenvalue of E[e e^T] - mu mu^T over the
 * offsets e = p_j - p_i (fp64 cumulants, one-sided Jacobi); (0, 0, 1) for fewer than 3 neighbours or a zero
 * covariance.  Sign: largest-magnitude component positive; with prev (optional float [n, 3]) then flipped where it
 * has a negative dot product with prev[i].  normals: float [n, 3]; counts: int32 [n] = rows within the radius
 * (before the max_nn truncation).  No atomics, the same bits on every run. */
int32_t dgr_estimate_normals(const float* xyz, int64_t n, const dgr_keyspec_t* spec, const uint64_t* keys,
                             const int32_t* vals, int64_t cap, int32_t batch, double cell, double radius,
                             int32_t max_nn, const float* prev, float* normals, int32_t* counts, void* stream);
/* ICP of src onto tgt.  Correspondences: the nearest target point strictly within max_dist of each transformed
 * source point s, through the TARGET cloud's voxel hash (keys / vals / spec of the table dgr_unique_first built at
 * `voxel`; table rows = rows of tgt; `batch` = the batch index those coordinates carry; max_dist / voxel <= 4).
 * Update, in fp64:
 *   tgt_normals == NULL: point-to-point, the Kabsch rotation of the correspondences' centred cross-covariance;
 *   tgt_normals (float [n_tgt, 3]): point-to-plane, r = (s - q).n, J = [s x n, n], J^T J x = -J^T r by Cholesky (a
 *     non-positive pivot gives the identity update), T <- [Rz(x2) Ry(x1) Rx(x0) | x3..5] T.
 * Stop when fitness and the Euclidean inlier RMSE both change by less than the tolerances, or after max_iter
 * updates.  The sums are per-block partials reduced in block order: the same bits on every run.  No host round trip.
 * T_init: device double[12] row-major [R | t]; ws: dgr_icp_ws_elems(n_src) doubles; result: device double[20] =
 * 4x4 pose, fitness, inlier rmse, iterations, correspondences. */
int32_t dgr_icp_ws_elems(int64_t n_src, int64_t* n_elems);
int32_t dgr_icp(const float* src, int64_t n_src, const float* tgt, const float* tgt_normals, const dgr_keyspec_t* spec,
                const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t batch, double voxel, double max_dist,
                const double* T_init, int32_t max_iter, double rel_fitness, double rel_rmse, double* ws,
                double* result, void* stream);

/* ---- Safeguard RANSAC (SURVEY 8f rank 2): open3d registration_ransac_based_on_correspondence as
 *      called at core/deep_global_registration.py:50-64 (from :302-315) ---------------------- */
/* Correspondence i pairs x[idx0[i]] with y[idx1[i]] (a null index array means i itself).
 * num_hyp hypotheses of 4 correspondences each (Umeyama without scaling, fp64), every one scored
 * on ALL correspondences: more inliers (|R p + t - q| < max_dist) wins, then the lower inlier
 * RMSE, then the lower hypothesis number; no early exit (the reference's criteria put 80000 in
 * the confidence slot, which open3d clamps to 1).  Sampling is a counter hash of (seed,
 * hypothesis, slot), so a call is reproducible.
 * ws: dgr_ransac_ws_elems() 8-byte words; result: device double[20] = 4x4 pose (identity when no
 * hypothesis has an inlier), fitness, inlier RMSE (both re-evaluated in fp64), winning hypothesis
 * (-1 if none), its inlier count. */
int32_t dgr_ransac_ws_elems(int64_t n_corr, int64_t num_hyp, int64_t* n_elems);
int32_t dgr_ransac_correspondence(const float* x, const float* y, const int32_t* idx0, const int32_t* idx1,
                                  int64_t n_corr, double max_dist, int64_t num_hyp, uint64_t seed,
                                  uint64_t* ws, double* result, void* stream);

/* ---- Feature-matching RANSAC: open3d 0.10 registration_ransac_based_on_feature_matching as called at
 *      core/deep_global_registration.py:29-47 (the FCGF + RANSAC baseline) ------------------------ */
/* nn[i] = row of the target feature nearest to source feature i (dgr_knn_top1 / dgr_knn_top1_tc).
 * Hypotheses h = 0 .. max_iteration-1 each draw 4 SOURCE points (the counter hash of
 * dgr_ransac_correspondence) paired with their nn; edge_ratio > 0 enables the edge-length checker
 * (every sampled edge |S_a - S_b| >= r |T_a - T_b| and vice versa), then the fp64 Umeyama fit
 * without scaling, then check_dist > 0 the distance checker (every sampled residual <= check_dist).
 * The first max_validation hypotheses that pass are scored on ALL source points: a point matches its
 * nearest target point strictly within max_dist of R s + t, searched through the TARGET's voxel hash
 * (keys / vals / spec of a dgr_unique_first table at `cell`, at most one point per cell, rows = rows of
 * tgt, `batch` = its batch column; max_dist / cell <= 4).  Best = more matches, then a smaller sum of
 * squared distances, then the lower hypothesis.  All fp64, reproducible bit for bit; no host read.
 * ws: dgr_ransac_fm_ws_elems() 8-byte words; result: device double[24] = 4x4 pose (identity when no
 * hypothesis matched a point), fitness, inlier RMSE, winning hypothesis (-1 if none), matched source
 * points, validated hypotheses scored, hypotheses drawn until the max_validation-th validation
 * (max_iteration if it is never reached), 2 zeros. */
int32_t dgr_ransac_fm_ws_elems(int64_t n_src, int64_t max_iteration, int64_t max_validation, int64_t* n_elems);
int32_t dgr_ransac_feature_matching(const float* src, int64_t n_src, const float* tgt, const int32_t* nn,
                                    const dgr_keyspec_t* spec, const uint64_t* keys, const int32_t* vals, int64_t cap,
                                    int32_t batch, double cell, double max_dist, double edge_ratio, double check_dist,
                                    int64_t max_iteration, int64_t max_validation, uint64_t seed, uint64_t* ws,
                                    double* result, void* stream);

/* ---- Fast Global Registration over feature matches: open3d registration_fast_based_on_feature_matching
 *      with FastGlobalRegistrationOption (the FGR row of the reference's results) ---------------------- */
/* nn_st[i] = row of the target feature nearest to source feature i, nn_ts[j] = row of the source feature nearest
 * to target feature j (dgr_knn_top1 / dgr_knn_top1_tc).  Both clouds are centred on their fp64 means and divided by
 * s = the largest centred norm (use_absolute_scale: not divided, mu starts at s instead of 1).  Mutual pairs
 * (nn_ts[nn_st[i]] == i) are listed in the order of the larger cloud's rows (the source's on a tie).  tuple_test:
 * trials k = 0 .. 100 n_mut - 1 draw 3 list positions with the counter hash (draws 3k .. 3k + 2 of `seed`) and
 * pass when every edge has l_s tuple_scale < l_t < l_s / tuple_scale; the first maximum_tuple_count that pass
 * give 3 correspondences each, in order (no trial when n_mut < 3); without tuple_test the correspondences are the
 * mutual list.  With >= 10 correspondences, iteration_number Gauss-Newton steps on the Geman-McClure objective
 * sum (mu / (r^2 + mu))^2-weighted |p - T q|^2 move the target onto the source (mu divided by division_factor
 * when decrease_mu, itr % 4 == 0 and mu > maximum_correspondence_distance; a non-positive Cholesky pivot makes
 * that step the identity).  All fp64, no host read, the same bits on every run.
 * ws: dgr_fgr_ws_elems() 8-byte words.  corres_out (optional): int32 (source, target) pairs, room for
 * tuple_test ? 3 min(maximum_tuple_count, 100 min(n_src, n_tgt)) : min(n_src, n_tgt) of them; the first
 * result[17] are written.  result: device double[24] = 4x4 pose mapping the source into the target, n_mut,
 * correspondences used, trials drawn until the maximum_tuple_count-th acceptance (100 n_mut if it is never
 * reached, 0 without trials), final mu, 1 if the optimiser ran, 1 if the clouds were swapped for the matching
 * order (n_tgt > n_src), 2 zeros. */
int32_t dgr_fgr_ws_elems(int64_t n_src, int64_t n_tgt, int64_t maximum_tuple_count, int32_t tuple_test,
                         int64_t* n_elems);
int32_t dgr_fgr_feature_matching(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt,
                                 const int32_t* nn_st, const int32_t* nn_ts, double division_factor,
                                 int32_t use_absolute_scale, int32_t decrease_mu,
                                 double maximum_correspondence_distance, int32_t iteration_number,
                                 double tuple_scale, int64_t maximum_tuple_count, int32_t tuple_test, uint64_t seed,
                                 uint64_t* ws, int32_t* corres_out, double* result, void* stream);

/* ---- Go-ICP (Yang, Li, Campbell & Jia, TPAMI 2016): globally optimal trimmed ICP by branch and bound (the Go-ICP
 *      row of the reference's results; oracle/goicp.py is the specification) ------------------------------ */
/* Normalisation and distance transform.  Both clouds are centred on their fp64 means and divided by s = the larger
 * largest centred norm (dgr_fgr_feature_matching's statistics): stat = double[8] (source mean, largest norm, target
 * mean, largest norm), tgt_norm = float [n_tgt, 3] normalised target.  dt = int32 [G][G][G] (x fastest) over
 * [-e, e]^3, cell size h = 2e/G: the exact squared Euclidean distance in cell units from each cell to the nearest
 * cell a target point falls in (cell floor((q + e) / h) clamped to the grid); separable exact passes along x, y, z
 * (Felzenszwalb-Huttenlocher in integers), no atomics.  n_src in [1, 1024], G in [16, 512], e > 0. */
int32_t dgr_goicp_dt_build(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, int32_t dt_size,
                           double dt_expand, double* stat, float* tgt_norm, int32_t* dt, void* stream);
/* Globally optimal registration of src onto tgt (normalised as above) for the trimmed objective
 * E(R, t) = sum of the K = max(1, floor(n_src (1 - trim_fraction))) smallest squared distance-transform lookups of
 * R x_i + t (fp32 lookups, fp64 pairwise-tree sums): best-first branch and bound over angle-axis rotation cubes of the
 * cube (rot_min, rot_width) in rounds of the cubes_per_round smallest (LB, key) pool cubes, each child bounded by two
 * nested searches over translation cubes of (trans_min, trans_width); trimmed point-to-point ICP (dgr_knn_top1's fp32
 * correspondences, Kabsch) from the identity and from every child that beats the incumbent.  Stops when the pool is
 * empty or E* - LB_min < eps = mse_thresh K (converged), after max_rounds rounds, or when a round's children would
 * overflow max_rotation_cubes (>= 8 cubes_per_round).  One pinned host read per round; the same bits on every run.
 * ws: dgr_goicp_ws_elems() 8-byte words.  result: device double[32] = 4x4 pose mapping src into tgt, E*, LB_min
 * (normalised units), eps, K, converged, rounds, rotation children searched, translation cubes evaluated, ICP runs,
 * inner searches whose pool overflowed, the pool's high-water mark, s, host reads, 3 zeros.  Arguments out of range
 * are rejected before any device work. */
int32_t dgr_goicp_ws_elems(int64_t n_src, int64_t n_tgt, int32_t dt_size, int64_t max_rotation_cubes,
                           int32_t cubes_per_round, int64_t* n_elems);
int32_t dgr_goicp(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, double mse_thresh,
                  double trim_fraction, int32_t dt_size, double dt_expand, const double* rot_min, double rot_width,
                  const double* trans_min, double trans_width, int32_t cubes_per_round, int32_t max_rounds,
                  int64_t max_rotation_cubes, uint64_t* ws, double* result, void* stream);

/* ---- Super4PCS (Mellado, Aiger & Mitra, SGP 2014): 4-point congruent sets scored by their largest common pointset
 *      (the Super4PCS row of the reference's results; oracle/super4pcs.py is the specification) ------------ */
/* src (n_src in [4, 1024] rows, sampled by the caller) and the whole tgt are normalised as dgr_goicp's are and the
 * target's distance transform is built (dt_size, dt_expand as there).  Q = rows floor(k n_tgt / n_sample_tgt) of the
 * normalised target (n_sample_tgt in [4, 4096], at most n_tgt).  Bases run in rounds of bases_per_round, all rounds
 * enqueued up front: base b draws 32 triplets from the counter-hash stream of seed, completes the largest into a
 * coplanar base within D = overlap 2 max|p| and delta / s of its plane; pairs of Q congruent to its two segments
 * (at most max_pairs each) are joined on their invariant points through a hash of delta-cells, with the angle
 * filter angle_tol (radians; 0: 2 delta / min(d1, d2)); at most max_candidates congruent sets are fitted by Kabsch,
 * prefiltered on 64 source rows, and the verify_per_base best are scored on all of src (the LCP: points within
 * delta of the target through the distance transform).  Stops after max_bases bases or at the end of the first
 * round whose best LCP is >= terminate_fraction n_src.  delta in the input units.  No host read; the same bits on
 * every run.  ws: dgr_super4pcs_ws_elems() 8-byte words.  base_log (optional, int32 [max_bases][16]): per base its
 * 4 source rows, valid, |S1|, |S2|, candidates kept, candidates dropped, candidates verified, best LCP and its
 * candidate, 4 zeros (-1 rows / best when invalid or not run).  result: device double[32] = 4x4 pose mapping src
 * into tgt, LCP fraction, LCP count, bases tried, valid bases, candidates, pairs dropped, candidates dropped, the
 * winning base and candidate (-1: none), rounds, s, host reads (0), 4 zeros.  Arguments out of range are rejected
 * before any device work. */
int32_t dgr_super4pcs_ws_elems(int64_t n_src, int64_t n_tgt, int64_t n_sample_tgt, int32_t dt_size,
                               int32_t bases_per_round, int64_t max_pairs, int64_t max_candidates,
                               int32_t verify_per_base, int64_t* n_elems);
int32_t dgr_super4pcs(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, int64_t n_sample_tgt,
                      double overlap, double delta, double angle_tol, int32_t dt_size, double dt_expand,
                      int32_t max_bases, int32_t bases_per_round, int64_t max_pairs, int64_t max_candidates,
                      int32_t verify_per_base, double terminate_fraction, uint64_t seed, uint64_t* ws,
                      int32_t* base_log, double* result, void* stream);

/* ---- PointNetLK (Aoki, Goforth, Srivatsan & Lucey, CVPR 2019): a PointNet feature under an inverse-compositional
 *      Lucas-Kanade loop (the PointNetLK row of the reference's results; oracle/pointnetlk.py is the specification) */
/* The network phi: five 1x1 layers 3 -> 64 -> 64 -> 64 -> 128 -> 1024, each conv + eval-mode BatchNorm (eps 1e-5)
 * + ReLU, then the max over points of each of the 1024 channels (every feature >= +0).  params: device double
 * [DGR_POINTNET_PARAMS], per layer W [cout][cin], conv bias, BN weight, BN bias, running mean, running var.
 * dgr_pointnet_pack folds each BN into its layer in fp64, rounds to fp32 once and lays layers 2-5 out as TF32 hi / lo
 * tiles in shared-memory image order: packed = DGR_POINTNET_PACKED_BYTES device bytes (16-byte aligned), once per
 * checkpoint. */
#define DGR_POINTNET_PARAMS 154368
#define DGR_POINTNET_PACKED_BYTES 1185792
int32_t dgr_pointnet_pack(const double* params, void* packed, void* stream);
/* features (float [n_poses][1024]) = phi(R_b (p - c) + t_b) for poses (device double [n_poses][12], row-major
 * [R | t]) about the centre c (device double[3]; NULL: the origin).  Each input point is computed in fp64 from the
 * fp32 point, c and the pose, d = p - c, ((R0 d0 + R1 d1) + R2 d2) + t without contraction, and rounded to fp32 once; the layers run as 3xTF32 tensor-core products (fp32-accurate).  The max is
 * exact, so every run gives the same bits.  A NaN input point makes every feature of its pose NaN (the ReLUs and the
 * max keep NaN).  n in [1, 2^31 - 128], n_poses in [1, 65535]. */
int32_t dgr_pointnet_forward(const float* points, int64_t n, const double* centre, const double* poses, int32_t n_poses,
                             const void* packed, float* features, void* stream);
/* PointNetLK of src onto tgt (template T = tgt, source S = src).  Both clouds are centred on their fp64 means
 * (dgr_fgr_feature_matching's statistics).  J[:, i] = (phi(T) - phi(exp(-delta e_i) T)) / delta (one 7-pose forward),
 * H = J^T J; a non-positive pivot of H's Cholesky factorisation ends the call with status 1 and g = I.  Then for
 * k < max_iter: r = phi(g S) - phi(T), dx = -H^-1 J^T r; stop when |dx| < xtol (iterations = k + 1), otherwise
 * g <- exp(dx) g, with exp the SE(3) exponential of the twist (rotation first).  The pose is
 * translate(mean_T) g translate(-mean_S).  J, H, the solve, exp and the pose are fp64, reduced in a fixed order; no
 * host read, the same bits on every run.  ws: dgr_pointnetlk_ws_elems() 8-byte words.  jac_out (optional): double
 * [1024][6].  log (optional, double [max_iter][16]): per iteration run, g before the step (12), |dx|, |r|, 2 zeros
 * (rows of iterations not run are left as they were).  result: device double[32] = 4x4 pose mapping src into tgt,
 * iterations, last |dx|, last |r|, status (0 ok, 1 singular H), n_src, n_tgt, host reads (0), 9 zeros.  delta > 0,
 * max_iter in [1, 1000], xtol >= 0; arguments out of range are rejected before any device work. */
int32_t dgr_pointnetlk_ws_elems(int64_t n_src, int64_t n_tgt, int32_t max_iter, int64_t* n_elems);
int32_t dgr_pointnetlk(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt, const void* packed,
                       double delta, int32_t max_iter, double xtol, uint64_t* ws, double* jac_out, double* log,
                       double* result, void* stream);

/* ======================================================================================
 * Round 2: coordinate planning with device-side counts, and the native executor.
 * ====================================================================================== */

/* Output-stationary variant of dgr_spconv_fwd for few input channels (conv1: cin <= 8): reads the dense
 * neighbour table (rows nbr_stride apart), no atomics, optional fused per-channel affine (eval BatchNorm):
 *   out[j, :] = (sum_kappa in[nbr[kappa * nbr_stride + j], :] @ W[kappa]) * scale + shift. */
int32_t dgr_spconv_table_fwd_strided(const float* in_feat, int32_t cin, const float* weight, int32_t cout,
                                     const int32_t* nbr, int32_t K, int64_t n_out, int64_t nbr_stride,
                                     const float* scale, const float* shift, float* out, void* stream);

/* ---- training (SURVEY 8f rank 3): backward of the sparse convolution
 *      (core/trainer.py:204-264 -> loss.backward() through MinkowskiConvolution) -------------- */
/* dw[K, cin, cout] (overwritten) = weight gradient: dw[kappa] = sum over pairs p of bucket kappa of
 * in_feat[in_idx[p], :]^T (x) grad_out[out_idx[p], :]; deterministic (in-order sums per block).
 * The input gradient is dgr_spconv_fwd(grad_out, W^T) with in_idx / out_idx exchanged. */
int32_t dgr_spconv_wgrad(const float* in_feat, int32_t cin, const float* grad_out, int32_t cout,
                         const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs, int32_t K, float* dw,
                         void* stream);

/* ---- 3xFP16 mode of the tensor-core convolution ----------------------------------------------
 * fp16 has TF32's 11 significant bits at half the bytes and twice the tensor rate; operands are scaled by
 * powers of two (exact) so that the tensor's absolute maximum lands in [2^14, 2^15), then split hi / lo as
 * in the 3xTF32 path: same 2^-21 relative accuracy, 1.5 TF32-MMA equivalents per product instead of 3. */
/* dgr_affine_act that also reduces max |out| into amax[0] (device float, zeroed by the CALLER): the activation
 * scale of the 3xFP16 convolution consuming `out`, computed in the pass that produces it. */
int32_t dgr_affine_act_amax(const float* x, int64_t n, int32_t c, const float* scale, const float* shift,
                            const float* residual, int32_t relu, float* out, float* amax, void* stream);
/* amax[0] (device float, zeroed by the call) = max |x[i]|. */
int32_t dgr_absmax_f32(const float* x, int64_t n, float* amax, void* stream);
int32_t dgr_spconv_tc_f16_supported(int32_t cin, int32_t cout);     /* cin % 64 == 0, cout % 32 == 0, <= 256 */
/* packed: 4 * K * cin * cout bytes ([K][cin/64][hi|lo][cout][64 halves], shared-memory image order);
 * scale_ws: device float[2] = (1 / weight scale, max |W|). */
int32_t dgr_pack_weight_f16(const float* w, int32_t K, int32_t cin, int32_t cout, void* packed, float* scale_ws,
                            void* stream);
/* Same contract as dgr_spconv_tc_fwd (plain or paired tile list).  amax_in: device float >= max |in_feat|
 * (dgr_absmax_f32); w_scale: scale_ws of dgr_pack_weight_f16. */
int32_t dgr_spconv_tc_f16_fwd(const float* in_feat, int32_t cin, const void* weight_h, int32_t cout,
                              const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs,
                              const int32_t* tile_k, const int32_t* tile_start, int32_t n_tiles, int32_t tile_rows,
                              const float* amax_in, const float* w_scale, float* out, void* stream);

/* conv1 of the FCGF network on its actual input - one channel, all ones (core/deep_global_registration.py:96,159)
 * - from the kernel map's occupancy masks (bits[K][mask_words] of dgr_kmap_probe) instead of a dense 343 x N
 * neighbour table: out[j, :] = (sum over kappa with bit (kappa, j) set of weight[kappa, 0, :]) * scale + shift. */
int32_t dgr_spconv_ones_bits_fwd(const float* weight, int32_t cout, const uint32_t* bits, int64_t mask_words, int32_t K,
                                 int64_t n_out, const float* scale, const float* shift, float* out, void* stream);

/* ---- coordinate planning without host round trips (csrc/coordplan.cu) --------------------
 * Convention: `n_max` is a host-side upper bound of a row count (sizes buffers and grids), `n_dev` a
 * device int32* holding the actual count (NULL = n_max).  Replaces the MinkowskiEngine coordinate
 * manager behind ME.SparseTensor / MinkowskiConvolution (core/deep_global_registration.py:167,214,
 * model/residual_block.py:31-80). */
/* After dgr_unique_first over the concatenated raw voxel coordinates [n_raw0 + n_raw1, 4] of a scan pair:
 * coords[i] = raw[sel[i]], xyz[i] = float(point sel[i]) for i < n_unique[0]; counts[4] = (N, N0, N1,
 * key-overflow flag) with N0 = kept points of cloud 0 (sel ascending: cloud 0 rows first). */
int32_t dgr_compact_voxel_pair(const int32_t* raw_coords, const int32_t* sel, const int32_t* n_unique,
                               int64_t n_raw0, int64_t n_raw1, const void* xyz0, int32_t is_f64_0, const void* xyz1,
                               int32_t is_f64_1, int32_t* coords, float* xyz, int32_t* counts, void* stream);
/* Table key -> row index of rows known to be distinct (clears the table first). */
int32_t dgr_table_build_unique(const int32_t* coords, int64_t n_max, const int32_t* n_dev, int32_t ncols,
                               const dgr_keyspec_t* spec, uint64_t* keys, int32_t* vals, int64_t cap, void* stream);
/* Coarse maps of `n_levels` (<= 4) tensor strides in one call, all derived from the same fine rows:
 * level l: coords_out[l][n_max][ncols] (first n_out[l] rows valid, ordered by first occurrence among the
 * fine rows), table keys[l][cap] / vals[l][cap] (key -> coarse row), n_out[l] device counts.
 * slot_ws: n_levels * n_max ints; scan_ws: n_levels * dgr_coarse_scan_elems(n_max) ints. */
int64_t dgr_coarse_scan_elems(int64_t n_max);
int32_t dgr_coarse_maps(const int32_t* fine, int64_t n_max, const int32_t* n_dev, int32_t ncols,
                        const dgr_keyspec_t* spec, int32_t n_levels, const int32_t* strides, uint64_t* keys,
                        int32_t* vals, int64_t cap, int32_t* coords_out, int32_t* n_out, int32_t* slot_ws,
                        int32_t* scan_ws, void* stream);
/* Blocked Bloom filter of a table (both bits of a key in one 32-bit word); n_words a power of two.  Kernel maps
 * with many offsets per row (K > 27: 6-D maps, 5^3 / 7^3 kernels) miss on most probes and use one.
 * dgr_bloom2_words(n_max): the filter size for a table of n_max keys (about 10 bits per key, 1024..16384 words). */
int32_t dgr_bloom2_build(const uint64_t* keys, int64_t cap, uint32_t* words, int64_t n_words, void* stream);
int64_t dgr_bloom2_words(int64_t n_max);
/* Kernel map of KernelGenerator(kernel_size, HYPER_CUBE) (model/residual_block.py:31-44,56-80): the pairs
 * (i, j) with C_in[i] == C_out[j] + offsets[kappa], sorted by (kappa, j).  offsets is a DEVICE int32
 * [K, ncols-1] matrix (already scaled by the input tensor stride), kappa enumerates axis 0 fastest.
 * Phase 1: bits[K][W] (W = dgr_kmap_mask_words(n_out_max)) holds one bit per (offset, output row),
 * block_cnt (dgr_kmap_cnt_elems ints) the exclusive-scanned per-(offset, 256-word block) pair counts,
 * kofs[K + 2] the bucket offsets + key-overflow flag, meta[5] = (pairs P, 128-row tiles, tiles with an even
 * count per offset, non-empty offsets, key overflow).  bloom_words (optional, <= 32768 words) is copied to
 * shared memory and answers most misses there.  No host synchronisation. */
int64_t dgr_kmap_mask_words(int64_t n_out_max);
int64_t dgr_kmap_cnt_elems(int32_t K, int64_t n_out_max);
int32_t dgr_kmap_probe(const int32_t* out_coords, int64_t n_out_max, const int32_t* n_out_dev, int32_t ncols,
                       const dgr_keyspec_t* spec, const uint64_t* in_keys, const int32_t* in_vals, int64_t in_cap,
                       const uint32_t* bloom_words, int64_t n_bloom_words, const int32_t* offsets, int32_t K,
                       uint32_t* bits, int32_t* block_cnt, int32_t* kofs, int32_t* meta, void* stream);
/* Kernel map, phase 2 (after the caller has read P from meta): in_idx[P], out_idx[P] sorted by (kappa, j),
 * the same lists as the oracle's buckets (oracle/sparse_ops.py). */
int32_t dgr_kmap_fill(const uint32_t* bits, const int32_t* block_cnt, int32_t K, int64_t n_out_max,
                      const int32_t* out_coords, int32_t ncols, const dgr_keyspec_t* spec, const uint64_t* in_keys,
                      const int32_t* in_vals, int64_t in_cap, const int32_t* offsets, int32_t* in_idx,
                      int32_t* out_idx, void* stream);
/* Work list of the gather-GEMM-scatter kernel: tile t covers pairs
 * [tile_start[t], min(tile_start[t] + tile_rows, kofs[tile_k[t] + 1])) of bucket tile_k[t].
 * n_tiles = sum_k ceil(count_k / tile_rows) (meta[1] of dgr_kmap_probe).  pair != 0 rounds every offset's tile
 * count up to even (meta[2]; the extra tile is empty); the convolutions skip empty tiles, so either list serves
 * them. */
int32_t dgr_kernel_map_tiles(const int32_t* kofs, int32_t K, int32_t tile_rows, int32_t n_tiles, int32_t pair,
                             int32_t* tile_k, int32_t* tile_start, void* stream);
/* Dense neighbour table nbr[kappa * nbr_stride + j] (-1 = no neighbour) with a device-side row count;
 * bloom_words optional as in dgr_kmap_probe; hit_count (optional device int32, zeroed by the call) receives
 * the number of pairs P. */
int32_t dgr_kmap_dense(const int32_t* out_coords, int64_t n_out_max, const int32_t* n_out_dev, int32_t ncols,
                       const dgr_keyspec_t* spec, const uint64_t* in_keys, const int32_t* in_vals, int64_t in_cap,
                       const uint32_t* bloom_words, int64_t n_bloom_words, const int32_t* offsets, int32_t K,
                       int32_t* nbr, int64_t nbr_stride, int32_t* hit_count, void* stream);

/* ---- native executor (csrc/exec.cu) ------------------------------------------------------
 * A context owns a stream (or uses the one given), a grow-only device arena and pinned staging; calls
 * on one context are serialised by the caller, different contexts may be driven from different host
 * threads (two pairs in flight per GPU).  Unlike the operator-level entry points above, these allocate
 * device memory internally (the arena) and synchronise the context's stream where stated. */
typedef struct dgr_ctx dgr_ctx_t;
typedef struct dgr_net dgr_net_t;
int32_t dgr_ctx_create(int32_t device, void* stream /* NULL: own non-blocking stream */, dgr_ctx_t** out);
int32_t dgr_ctx_destroy(dgr_ctx_t* ctx);
void* dgr_ctx_stream(dgr_ctx_t* ctx);
/* stats[6]: host reads, device-to-host bytes, host-to-device bytes of the last call; arena high-water mark
 * [bytes], cudaMalloc calls of the arena so far, arena chunks. */
int32_t dgr_ctx_stats(dgr_ctx_t* ctx, int64_t* stats);
/* Per-launch CUDA-event timing of the convolution launches (bench.py's live roofline):
 * dgr_ctx_profile(ctx, 1) starts recording, dgr_ctx_profile_read synchronises and returns rows of
 * (milliseconds, algorithmic flops, gather-scatter-model bytes, kind: 0 tensor-core / 1 fp32 / 2 table). */
int32_t dgr_ctx_profile(dgr_ctx_t* ctx, int32_t enable);
int64_t dgr_ctx_profile_read(dgr_ctx_t* ctx, double* rows, int64_t max_rows);
/* Stage times [ms] of the last dgr_pair_register with profiling on (CUDA events on the context's stream):
 * upload + voxelisation, FCGF coordinate phase, host read 1 + FCGF pair lists, FCGF convolutions, feature kNN,
 * 6-D coordinate phase, host read 2 + 6-D pair lists, inlier convolutions, weights + Procrustes + refinement
 * (+ ICP).  Returns the number of stages written. */
int32_t dgr_ctx_stage_times(dgr_ctx_t* ctx, double* ms, int32_t max_stages);

/* A ResUNet2-family network (model/resunet.py:419-665) from 66 DEVICE parameter pointers in execution order:
 *   for l = 1..4:   conv{l}.kernel, norm{l} scale, shift, block{l}.conv1.kernel, block{l}.norm1 scale, shift,
 *                   block{l}.conv2.kernel, block{l}.norm2 scale, shift
 *   for l = 4,3,2:  conv{l}_tr.kernel, norm{l}_tr scale, shift, block{l}_tr.conv1.kernel, ... (same 9)
 *   conv1_tr.kernel, final.kernel, final.bias
 * kernels in ME layout [K, cin, cout]; scale / shift = eval-mode BatchNorm folded (model/common.py:13).
 * channels / tr_channels: CHANNELS / TR_CHANNELS of the model class (5 ints each, index 0 unused).  The
 * parameters must outlive the network; the TF32 weight slabs are packed here, once. */
int32_t dgr_net_create(int32_t device, int32_t D, int32_t in_ch, int32_t out_ch, int32_t conv1_ks, int32_t normalize,
                       const int32_t* channels, const int32_t* tr_channels, const float* const* params,
                       int32_t n_params, void* stream, dgr_net_t** out);
int32_t dgr_net_destroy(dgr_net_t* net);
/* Forward pass (model/resunet.py:598-649) of one sparse tensor: coords [n, D+1] int32 (distinct rows),
 * feats [n, in_ch] (NULL = ones), out [n, out_ch]; device pointers.  Resets the context's arena, ONE host
 * read inside, returns with the convolution phase enqueued on the context's stream. */
int32_t dgr_net_forward(dgr_ctx_t* ctx, dgr_net_t* net, const int32_t* coords, int64_t n, const float* feats,
                        float* out);

/* DeepGlobalRegistration.register() (core/deep_global_registration.py:238-324) for inlier_feature_type 'ones':
 * xyz0 / xyz1 = raw points [n, 3] (float64 or float32; host pointers when on_host, else device pointers).
 * Three host reads.  result (host double[64]):
 *   [0..16)  R (9, row-major), t (3), refinement iterations, final loss, break count, active correspondences
 *   [16]     weight sum (the gate of :276-281 and the safeguard call are the caller's: dgr_pair_safeguard)
 *   [17..37) ICP (use_icp): 4x4 pose, fitness, inlier RMSE, iterations, correspondences
 *   [40..44) N0, N1 (voxels per cloud), host reads, device-to-host bytes */
int32_t dgr_pair_register(dgr_ctx_t* ctx, dgr_net_t* fcgf, dgr_net_t* inlier, const void* xyz0, int64_t n_raw0,
                          int32_t is_f64_0, const void* xyz1, int64_t n_raw1, int32_t is_f64_1, int32_t on_host,
                          double voxel, float clip, int32_t use_icp, double* result);
/* Safeguard branch (:302-315) on the pair this context registered last: RANSAC over its correspondences, then
 * (use_icp) ICP from that pose.  result (host double[40]): RANSAC 20 doubles, ICP 20 doubles. */
int32_t dgr_pair_safeguard(dgr_ctx_t* ctx, double max_dist, int64_t num_hyp, uint64_t seed, int32_t use_icp,
                           double* result);
/* Intermediate tensors of the last pair: which = 0 coords [N, 4] i32, 1 xyz [N, 3] f32, 2 FCGF features
 * [N, C] f32, 3 idx1 [N0] i32, 4 6-D coords [N0, 7] i32, 5 logits [N0] f32, 6 weights [N0] f32, 7 sel [N] i32.
 * dst NULL: shape only; else a synchronous copy into the DEVICE buffer dst. */
int32_t dgr_pair_tap(dgr_ctx_t* ctx, int32_t which, int64_t* rows, int32_t* cols, void* dst);

#ifdef __cplusplus
}
#endif
#endif /* DGR_B200_H_ */
