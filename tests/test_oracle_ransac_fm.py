"""The feature-matching RANSAC oracle (oracle/ransac_fm.py: open3d 0.10's
registration_ransac_based_on_feature_matching, core/deep_global_registration.py:29-47) and the open3d
stand-in's argument handling for it, on the CPU."""
import numpy as np
import pytest

from deepglobalregistration_b200 import o3d_registration as reg
from deepglobalregistration_b200 import shims
from deepglobalregistration_b200 import synthetic as syn
from oracle import ransac_fm as orf


def test_feature_nn_identifies_the_built_matches():
  P, Q, fs, ft, T, perm, ident = syn.feature_matching_pair(0, n=800, match_frac=0.4)
  nn = orf.feature_nn(fs, ft)
  assert np.array_equal(nn == perm, ident)
  # lowest row on ties
  assert np.array_equal(orf.feature_nn(np.zeros((2, 3)), np.zeros((4, 3))), [0, 0])


@pytest.mark.parametrize('seed,frac', [(1, 0.3), (2, 0.5)])
def test_recovers_the_ground_truth(seed, frac):
  P, Q, fs, ft, T_gt, perm, ident = syn.feature_matching_pair(seed, n=1500, match_frac=frac)
  nn = orf.feature_nn(fs, ft)
  T, info = orf.ransac_feature_matching(P, Q, nn, 0.03, 4000, 1000, check_dist=0.03, seed=seed)
  te, re = syn.rte_rre(T, T_gt)
  assert te < 0.01 and re < 0.01, (te, re, info)
  assert info['fitness'] > 0.95 and info['matched'] == round(info['fitness'] * len(P))
  assert 0 <= info['hypothesis'] < info['drawn'] and 0 < info['inlier_rmse'] < 0.03
  # the winner is the fit of its own four draws
  s = orf.sample_indices(seed, [info['hypothesis']], len(P))
  R, t = orf.kabsch_batch(P[s].astype(np.float64), Q[nn[s]].astype(np.float64))
  np.testing.assert_allclose(T[:3, :3], R[0], atol=1e-12)
  np.testing.assert_allclose(T[:3, 3], t[0], atol=1e-12)


def test_stops_after_exactly_max_validation():
  P, Q, fs, ft, _, _, _ = syn.feature_matching_pair(3, n=600, match_frac=0.5)
  nn = orf.feature_nn(fs, ft)
  # no checker: every hypothesis validates, so V validations take V draws
  _, info = orf.ransac_feature_matching(P, Q, nn, 0.03, 500, 7)
  assert info['validated'] == 7 and info['drawn'] == 7
  # with the distance checker only some validate; the V-th validation is hypothesis drawn - 1
  _, info = orf.ransac_feature_matching(P, Q, nn, 0.03, 20000, 5, check_dist=0.03)
  assert info['validated'] == 5 and 5 < info['drawn'] <= 20000
  _, short = orf.ransac_feature_matching(P, Q, nn, 0.03, info['drawn'] - 1, 5, check_dist=0.03)
  assert short['validated'] == 4 and short['drawn'] == info['drawn'] - 1
  _, exact = orf.ransac_feature_matching(P, Q, nn, 0.03, info['drawn'], 5, check_dist=0.03)
  assert exact['validated'] == 5 and exact['hypothesis'] == info['hypothesis']
  # V never reached: every hypothesis was drawn
  _, big = orf.ransac_feature_matching(P, Q, nn, 0.03, 300, 10 ** 6, check_dist=0.03)
  assert big['drawn'] == 300 and big['validated'] < 300


def test_edge_checker_rejects_an_inconsistent_sample():
  S = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]]], np.float64)
  R = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], np.float64)
  T = S @ R.T + 0.5
  assert orf.edge_check(S, T, 0.9).all()
  bad = T.copy()
  bad[0, 3] = [0.5, 0.5, 3.0]                      # one edge of the target three times too long
  assert not orf.edge_check(S, bad, 0.9).any()
  assert orf.edge_check(S, bad, 0.0).all()         # ratio 0 accepts anything
  # inside the loop: nothing validates when every sampled target is off, so the identity comes back
  P, Q, fs, ft, _, _, _ = syn.feature_matching_pair(4, n=300)
  rng = np.random.default_rng(0)
  Qs = rng.uniform(-50, 50, size=Q.shape)
  Tid, info = orf.ransac_feature_matching(P, Qs, orf.feature_nn(fs, ft), 0.03, 200, 10, edge_ratio=0.99)
  assert info['validated'] == 0 and info['hypothesis'] == -1 and np.array_equal(Tid, np.eye(4))


def test_stand_in_feature_and_criteria():
  f = reg.Feature()
  f.resize(32, 100)
  assert f.data.shape == (32, 100) and f.data.dtype == np.float64 and f.dimension() == 32 and f.num() == 100
  feats = np.random.default_rng(0).normal(size=(50, 8)).astype(np.float32)
  f.data = feats.astype('d').transpose()          # what the reference does (:33-34)
  assert f.dimension() == 8 and f.num() == 50
  c = reg.RANSACConvergenceCriteria(80000, 1000)    # the reference's call (:44)
  assert (c.max_iteration, c.confidence, c.max_validation) == (80000, 1.0, 1000)
  c = reg.RANSACConvergenceCriteria(4000000, 80000)
  assert (c.max_iteration, c.confidence, c.max_validation) == (4000000, 1.0, 80000)
  for args, want in (((), 1000), ((100, 0.999), 1000), ((100, 1.0), 1000), ((100, 0), 1000), ((100, 5), 5),
                     ((100, np.int64(7)), 7), ((100, True), 1000)):
    assert reg.RANSACConvergenceCriteria(*args).max_validation == want, args
  assert reg.CorrespondenceCheckerBasedOnEdgeLength().similarity_threshold == 0.9
  o3d = shims._open3d_stub()
  assert o3d.registration is o3d.pipelines.registration
  assert o3d.registration.Feature is reg.Feature
  assert o3d.registration.registration_ransac_based_on_feature_matching is reg.registration_ransac_based_on_feature_matching


def test_stand_in_rejects_what_is_not_built():
  """All raised before a device is needed."""
  f = reg.Feature()
  f.resize(4, 10)
  pts = np.zeros((10, 3))
  est = reg.TransformationEstimationPointToPoint(False)
  dist = [reg.CorrespondenceCheckerBasedOnDistance(0.1)]
  crit = reg.RANSACConvergenceCriteria(100, 10)
  call = reg.registration_ransac_based_on_feature_matching
  with pytest.raises(NotImplementedError, match='mutual_filter'):
    call(pts, pts, f, f, True, 0.1, est, 4, dist, crit)            # >= 0.12: a bool in the 5th slot
  with pytest.raises(NotImplementedError, match='mutual_filter'):
    call(pts, pts, f, f, mutual_filter=False, max_correspondence_distance=0.1, estimation_method=est, ransac_n=4,
         checkers=dist, criteria=crit)
  with pytest.raises(NotImplementedError, match='ransac_n'):
    call(pts, pts, f, f, 0.1, est, 3, dist, crit)

  class CorrespondenceCheckerBasedOnNormal:
    normal_angle_threshold = 0.5
  with pytest.raises(NotImplementedError, match='CorrespondenceCheckerBasedOnNormal'):
    call(pts, pts, f, f, 0.1, est, 4, dist + [CorrespondenceCheckerBasedOnNormal()], crit)
  assert reg._feature_checkers([reg.CorrespondenceCheckerBasedOnEdgeLength(0.9), dist[0],
                                reg.CorrespondenceCheckerBasedOnDistance(0.05)]) == (0.9, 0.05)
  assert reg._feature_checkers(None) == (0.0, 0.0)
