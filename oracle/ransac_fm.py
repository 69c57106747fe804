"""ORACLE (test infrastructure only) - the FCGF + RANSAC baseline of the reference:
``o3d.registration.registration_ransac_based_on_feature_matching(pcd0, pcd1, source_feat, target_feat,
distance_threshold, TransformationEstimationPointToPoint(False), 4,
[CorrespondenceCheckerBasedOnDistance(distance_threshold)], RANSACConvergenceCriteria(num_iterations, 1000))``
(core/deep_global_registration.py:29-47; open3d 0.10 API, where the criteria are (max_iteration,
max_validation)).

PARITY UNPINNED: open3d is not installed in the build container and not vendored, so this restates
open3d 0.10's loop, and the boundary conventions below are pinned here rather than measured against it:

1. nn[i] = the target feature nearest to source feature i (L2, lowest row on ties).  open3d searches a
   float64 KD-tree; the library computes nn in fp32 (dgr_knn_top1), so near-ties may pick differently.
2. Hypotheses h = 0 .. max_iteration-1 in order.  Each draws 4 SOURCE rows with the counter hash of
   oracle/ransac.py (sample_indices) and pairs them with nn.  Checkers: edge length (every one of the 6
   edges: |S_a - S_b| >= r |T_a - T_b| and |T_a - T_b| >= r |S_a - S_b|) before the fit, Umeyama without
   scaling, then distance (every sampled residual <= c).  A hypothesis passing all is VALIDATED and
   scored on all source points: a point matches its nearest target point strictly within d of R s + t;
   fitness = matched / n_s, inlier_rmse = sqrt(sum d^2 / matched).  A hypothesis is kept when its
   fitness is higher, or equal with a strictly lower RMSE (the earliest keeps a tie).  The loop stops
   after max_validation validated hypotheses.
3. Nothing better than the initial result (fitness 0) -> identity, hypothesis -1.

open3d draws from per-thread mt19937s seeded by std::random_device and validates in parallel, so its
draws are not reproducible; what is exact here is the search given the draws.  All float64."""
import numpy as np
from scipy.spatial import cKDTree

from .ransac import kabsch_batch, sample_indices


def feature_nn(feat_src, feat_tgt, chunk=2048):
  """Row of the nearest target feature of every source feature (L2, lowest row on ties), float64."""
  fs, ft = np.asarray(feat_src, np.float64), np.asarray(feat_tgt, np.float64)
  out = np.empty(len(fs), np.int64)
  for lo in range(0, len(fs), chunk):
    d2 = ((fs[lo:lo + chunk, None, :] - ft[None]) ** 2).sum(-1)
    out[lo:lo + chunk] = d2.argmin(1)
  return out


def edge_check(P, Q, ratio):
  """[B] CorrespondenceCheckerBasedOnEdgeLength over samples P, Q [B, 4, 3]."""
  ok = np.ones(len(P), bool)
  for a in range(1, 4):
    for b in range(a):
      ds = np.sqrt(((P[:, a] - P[:, b]) ** 2).sum(-1))
      dt = np.sqrt(((Q[:, a] - Q[:, b]) ** 2).sum(-1))
      ok &= ~((ds < ratio * dt) | (dt < ratio * ds))
  return ok


def score(R, t, src, tree, tgt, max_dist):
  """(matched, sum d^2) of pose (R, t): nearest target point strictly within max_dist of every R s + t."""
  X = src @ R.T + t
  _, j = tree.query(X, k=1, distance_upper_bound=max_dist * 1.000001)
  hit = j < len(tgt)
  d2 = ((X[hit] - tgt[j[hit]]) ** 2).sum(-1)
  keep = d2 < max_dist * max_dist
  return int(keep.sum()), float(d2[keep].sum())


def ransac_feature_matching(src, tgt, nn, max_dist, max_iteration, max_validation, edge_ratio=0.0, check_dist=0.0,
                            seed=0, chunk=1024):
  """src [n_s, 3], tgt [n_t, 3], nn [n_s] (feature_nn) -> (T 4x4 float64, info).  edge_ratio 0 / check_dist
  <= 0 switch the checkers off."""
  S = np.asarray(src, np.float64)
  Tg = np.asarray(tgt, np.float64)
  nn = np.asarray(nn, np.int64)
  n = len(S)
  tree = cKDTree(Tg)
  best = (0, 0.0, -1, np.eye(3), np.zeros(3))      # matched, sum d^2, hypothesis, R, t
  validated, drawn = 0, max_iteration
  for lo in range(0, max_iteration, chunk):
    hyp = np.arange(lo, min(lo + chunk, max_iteration))
    s = sample_indices(seed, hyp, n)
    P, Q = S[s], Tg[nn[s]]
    ok = edge_check(P, Q, edge_ratio) if edge_ratio > 0 else np.ones(len(hyp), bool)
    R, t = kabsch_batch(P, Q)
    if check_dist > 0:
      res = np.sqrt(((np.einsum('bij,bmj->bmi', R, P) + t[:, None] - Q) ** 2).sum(-1))
      ok &= (res <= check_dist).all(1)
    for b in np.flatnonzero(ok):
      cnt, err = score(R[b], t[b], S, tree, Tg, max_dist)
      # IsBetterRANSACThan: higher fitness, or the same with a lower RMSE (strict: the earliest keeps a tie)
      if cnt > 0 and (cnt > best[0] or (cnt == best[0] and err < best[1])):
        best = (cnt, err, int(hyp[b]), R[b], t[b])
      validated += 1
      if validated == max_validation:
        drawn = int(hyp[b]) + 1
        break
    if validated == max_validation:
      break
  T = np.eye(4)
  T[:3, :3], T[:3, 3] = best[3], best[4]
  info = dict(fitness=best[0] / n if n else 0.0, inlier_rmse=float(np.sqrt(best[1] / best[0])) if best[0] else 0.0,
              hypothesis=best[2], matched=best[0], validated=validated, drawn=drawn)
  return T, info
