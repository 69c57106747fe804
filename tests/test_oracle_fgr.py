"""The Fast Global Registration oracle (oracle/fgr.py: open3d's registration_fast_based_on_feature_matching) and the
open3d stand-in's argument handling for it, on the CPU."""
import numpy as np
import pytest

from deepglobalregistration_b200 import o3d_registration as reg
from deepglobalregistration_b200 import shims
from deepglobalregistration_b200 import synthetic as syn
from oracle import fgr as ofg
from oracle import ransac_fm as orf


def rigid_copy(seed, n=400, dim=16):
  """Target = an exact rigid motion of the source, rows shuffled; every source feature equals its partner's."""
  g = np.random.default_rng(seed)
  P = g.uniform(-1.5, 1.5, size=(n, 3))
  T = syn.random_se3(g, 40.0, 0.5)
  perm = g.permutation(n)
  Q = np.empty_like(P)
  Q[perm] = syn.apply_se3(T, P)
  ft = g.normal(size=(n, dim))
  return P, Q, ft[perm], ft, T, perm


def gnc_mu(mu0=1.0, iterations=64, factor=1.4, limit=0.025):
  mu = mu0
  for itr in range(iterations):
    if itr % 4 == 0 and mu > limit:
      mu /= factor
  return mu


def test_known_answer_rigid_copy():
  P, Q, fs, ft, T_gt, perm = rigid_copy(0)
  T, info = ofg.fgr_feature_matching(P, Q, fs, ft)
  assert info['n_mut'] == len(P) and info['ran'] and not info['swapped']
  assert np.array_equal(info['mutual'], np.stack([np.arange(len(P)), perm], 1))
  assert info['n_corr'] == 3000 and np.array_equal(info['corres'][:, 1], perm[info['corres'][:, 0]])
  np.testing.assert_allclose(T, T_gt, atol=1e-10)
  assert info['mu'] == gnc_mu()


def test_relative_scale_keeps_rotation_and_scales_translation():
  P, Q, fs, ft, _, _ = rigid_copy(1)
  T1, i1 = ofg.fgr_feature_matching(P, Q, fs, ft)
  c = 3.7
  Tc, ic = ofg.fgr_feature_matching(c * P, c * Q, fs, ft)
  assert np.array_equal(i1['corres'], ic['corres'])
  np.testing.assert_allclose(Tc[:3, :3], T1[:3, :3], atol=1e-12)
  np.testing.assert_allclose(Tc[:3, 3], c * T1[:3, 3], atol=1e-11)


def test_mutual_set_does_not_depend_on_direction():
  P, Q, fs, ft, _, _, _ = syn.feature_matching_pair(2, n=900, match_frac=0.4)
  keep = np.random.default_rng(0).random(len(Q)) < 0.8            # the target is the smaller cloud
  Q, ft = Q[keep], ft[keep]
  nn_st, nn_ts = orf.feature_nn(fs, ft), orf.feature_nn(ft, fs)
  a, sw_a = ofg.mutual_pairs(nn_st, nn_ts)
  b, sw_b = ofg.mutual_pairs(nn_ts, nn_st)
  assert not sw_a and sw_b and len(a) > 100
  assert np.array_equal(a, b[:, ::-1])                          # the same pairs, listed by the larger cloud's rows
  assert np.all(np.diff(a[:, 0]) > 0)


def test_tuple_test_rejects_repeated_draws_and_stops_at_the_count():
  P, Q, fs, ft, _, _ = rigid_copy(3, n=50)
  Sn, Tn = ofg.normalise(P, Q)[:2]
  pairs, _ = ofg.mutual_pairs(orf.feature_nn(fs, ft), orf.feature_nn(ft, fs))
  k = np.arange(100 * len(pairs))
  pos = ofg.tuple_positions(7, k, len(pairs))
  distinct = (pos[:, 0] != pos[:, 1]) & (pos[:, 1] != pos[:, 2]) & (pos[:, 0] != pos[:, 2])
  assert 0 < (~distinct).sum() < len(k)
  # an exact rigid copy passes every edge test, so exactly the trials with three distinct draws are accepted
  acc, drawn = ofg.tuple_test(Sn, Tn, pairs, 0.95, 10 ** 9, 7, chunk=1000)
  assert np.array_equal(acc, k[distinct]) and drawn == len(k)
  acc, drawn = ofg.tuple_test(Sn, Tn, pairs, 0.95, 25, 7, chunk=7)
  assert np.array_equal(acc, k[distinct][:25]) and drawn == k[distinct][24] + 1
  T, info = ofg.fgr(P, Q, orf.feature_nn(fs, ft), orf.feature_nn(ft, fs), seed=7, maximum_tuple_count=25)
  assert info['n_corr'] == 75 and info['drawn'] == drawn
  # a 3-slot trial is draws 3k .. 3k + 2 of the stream RANSAC reads 4 at a time
  flat = orf.sample_indices(7, np.arange(30), len(pairs)).reshape(-1)
  assert np.array_equal(ofg.tuple_positions(7, np.arange(40), len(pairs)).reshape(-1), flat[:120])


def pinned_translation(P, Q):
  T = np.eye(4)
  T[:3, 3] = np.asarray(Q, np.float64).mean(0) - np.asarray(P, np.float64).mean(0)
  return T


def test_fewer_than_3_mutual_pairs_and_fewer_than_10_correspondences():
  P, Q, fs, ft, _, _ = rigid_copy(4, n=5)
  # 2 mutual pairs: no trial, no correspondence, the optimiser returns the identity
  nn_st, nn_ts = np.array([0, 1, 0, 0, 0]), np.array([0, 1, 3, 3, 3])
  T, info = ofg.fgr(P, Q, nn_st, nn_ts)
  assert (info['n_mut'], info['n_corr'], info['drawn'], info['ran']) == (2, 0, 0, False)
  assert np.array_equal(T, pinned_translation(P, Q)) and info['mu'] == 1.0
  # 5 mutual pairs without the tuple test, 9 correspondences from 3 tuples: both below 10
  nn = orf.feature_nn(fs, ft)
  T, info = ofg.fgr(P, Q, nn, orf.feature_nn(ft, fs), tuple_test=False)
  assert (info['n_mut'], info['n_corr'], info['ran']) == (5, 5, False)
  assert np.array_equal(T, pinned_translation(P, Q))
  T, info = ofg.fgr(P, Q, nn, orf.feature_nn(ft, fs), maximum_tuple_count=3)
  assert info['n_corr'] == 9 and not info['ran'] and np.array_equal(T, pinned_translation(P, Q))


def test_options():
  P, Q, fs, ft, T_gt, perm = rigid_copy(5, n=300)
  nn_st, nn_ts = orf.feature_nn(fs, ft), orf.feature_nn(ft, fs)
  T, info = ofg.fgr(P, Q, nn_st, nn_ts, tuple_test=False)
  assert np.array_equal(info['corres'], info['mutual']) and info['drawn'] == 0 and info['n_corr'] == 300
  np.testing.assert_allclose(T, T_gt, atol=1e-10)
  T, info = ofg.fgr(P, Q, nn_st, nn_ts, decrease_mu=False)
  assert info['mu'] == 1.0
  np.testing.assert_allclose(T, T_gt, atol=1e-10)
  T, info = ofg.fgr(P, Q, nn_st, nn_ts, use_absolute_scale=True)
  s = max(np.linalg.norm(P - P.mean(0), axis=1).max(), np.linalg.norm(Q - Q.mean(0), axis=1).max())
  assert info['scale'] == 1.0 and info['mu0'] == pytest.approx(s, rel=1e-15)
  assert info['mu'] == gnc_mu(info['mu0'])
  np.testing.assert_allclose(T, T_gt, atol=1e-10)
  # a larger target swaps the matching order but not the pose
  T, info = ofg.fgr(P[40:], Q, nn_st[40:], orf.feature_nn(ft, fs[40:]))
  assert info['swapped'] and np.all(np.diff(info['mutual'][:, 1]) > 0)
  np.testing.assert_allclose(T, T_gt, atol=1e-10)
  with pytest.raises(TypeError):
    ofg.fgr(P, Q, nn_st, nn_ts, tuple_count=5)


def test_stand_in_option_and_names():
  o = reg.FastGlobalRegistrationOption()
  assert (o.division_factor, o.use_absolute_scale, o.decrease_mu, o.maximum_correspondence_distance,
          o.iteration_number, o.tuple_scale, o.maximum_tuple_count, o.tuple_test, o.seed) == \
      (1.4, False, True, 0.025, 64, 0.95, 1000, True, 0)
  assert reg.FastGlobalRegistrationOption(maximum_correspondence_distance=0.05).maximum_correspondence_distance == 0.05
  o3d = shims._open3d_stub()
  for mod in (o3d.pipelines.registration, o3d.registration):
    assert mod.FastGlobalRegistrationOption is reg.FastGlobalRegistrationOption
    assert mod.registration_fast_based_on_feature_matching is reg.registration_fast_based_on_feature_matching


def test_stand_in_rejects_bad_arguments_without_a_device():
  f4, f5 = reg.Feature(), reg.Feature()
  f4.resize(4, 10)
  f5.resize(5, 10)
  pts = np.zeros((10, 3))
  call = reg.registration_fast_based_on_feature_matching
  with pytest.raises(ValueError, match='dimensions'):
    call(pts, pts, f4, f5, reg.FastGlobalRegistrationOption())
  with pytest.raises(ValueError, match='one feature per point'):
    call(pts[:9], pts, f4, f4, reg.FastGlobalRegistrationOption())
  for kw in (dict(tuple_scale=0.0), dict(tuple_scale=1.5), dict(division_factor=1.0), dict(iteration_number=-1),
             dict(maximum_tuple_count=0), dict(maximum_correspondence_distance=0.0)):
    with pytest.raises(ValueError):
      call(pts, pts, f4, f4, reg.FastGlobalRegistrationOption(**kw))
  with pytest.raises(TypeError):
    call(pts, pts, f4, f4, reg.FastGlobalRegistrationOption(), max_correspondence_distance=0.1)
  with pytest.raises(TypeError):
    reg.FastGlobalRegistrationOption(tuple_count=5)
  # empty clouds need no device either: the identity, like open3d's initial result
  e = reg.Feature()
  e.resize(4, 0)
  r = call(np.zeros((0, 3)), pts, e, f4)
  assert np.array_equal(r.transformation, np.eye(4)) and r.fitness == 0 and len(r.correspondence_set) == 0
