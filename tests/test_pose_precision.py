"""oracle/pose64.py on the CPU: its references recover known poses, its floor is the Kabsch rotation's real
sensitivity, the numpy restatement of csrc/kabsch.cuh meets the criterion on every constructed spectrum that
tests/test_gpu_pose_fp64.py gives the kernel, and the criterion rejects S rounded to bfloat16 or a Jacobi stopped after
one sweep by at least 10x."""
import numpy as np
import pytest
import torch

from oracle import pose64 as P
from oracle import registration as oreg

SPECTRA = {
    'generic': dict(sig=[1.0, 0.6, 0.3]),
    's3=1e-3': dict(sig=[1.0, 0.5, 1e-3]),
    's3=2^-24': dict(sig=[1.0, 0.5, 2.0 ** -24]),
    's3=1e-9': dict(sig=[1.0, 0.5, 1e-9]),
    'rank2': dict(sig=[1.0, 0.5, 0.0]),
    's1=s2': dict(sig=[1.0, 1.0, 0.3]),
    's2=s3': dict(sig=[1.0, 0.4, 0.4]),
    'all-equal': dict(sig=[1.0, 1.0, 1.0]),
    'rank1': dict(sig=[1.0, 0.0, 0.0]),
    'reflect-s3-small': dict(sig=[1.0, 0.5, 1e-3], det_u=-1.0),
    'reflect-s3=s2': dict(sig=[1.0, 0.5, 0.5], det_u=-1.0),
    'scale-1e-4': dict(sig=[1.0, 0.6, 0.3], scale=1e-4),
    'scale-1e4': dict(sig=[1.0, 0.6, 0.3], scale=1e4),
    'far-1e4': dict(sig=[1.0, 0.6, 0.3], offset=1e4),
}
NON_UNIQUE = {'rank1', 'reflect-s3=s2'}


def spectrum_case(name, seed=0, n=512):
  return P.prescribed(np.random.default_rng([seed, sorted(SPECTRA).index(name)]), n=n, **SPECTRA[name])


def test_references_recover_a_known_pose():
  g = np.random.default_rng(1)
  R_gt = P.random_orthogonal(g)
  t_gt = np.array([0.3, -1.2, 2.0])
  X = g.normal(size=(300, 3)).astype(np.float32)
  Y = (X.astype(np.float64) @ R_gt.T + t_gt).astype(np.float32)
  w = g.uniform(0.1, 1.0, 300).astype(np.float32)
  ref = P.procrustes64(X, Y, w)
  assert np.abs(ref['R'] - R_gt).max() < 1e-6 and np.abs(ref['t'] - t_gt).max() < 1e-5
  pp = P.kabsch_pairs64(X, Y)
  assert np.abs(pp['R'] - R_gt).max() < 1e-6 and np.abs(pp['t'] - t_gt).max() < 1e-5
  assert np.abs(P.kabsch_rotation(pp['S']) - pp['R']).max() < 1e-12
  # the refinement's first loss is evaluated at the Procrustes pose: an exact fit up to the float32 rows
  assert 0 <= P.refine64(X, Y, w, 0.1, 1)[2] < 1e-9
  # the 6x6 step: a known small motion of points on three planes is recovered to first order
  Q = g.normal(size=(200, 3))
  N = np.zeros_like(Q)
  N[np.arange(200), np.arange(200) % 3] = 1.0
  x_gt = np.array([1e-4, -2e-4, 3e-4, 1e-3, -2e-3, 5e-4])
  Pm = (P.zyx_update_left(-x_gt, np.eye(4))[:3, :3] @ Q.T).T - x_gt[3:]    # approximately the inverse motion
  A, gv = P.plane_system(Pm, Q, N)
  x, cond = P.gn_step64(A, gv)
  assert np.abs(x - x_gt).max() < 1e-5 and 1 <= cond < 1e3
  # an exact plane: J^T J is singular
  N1 = np.tile([0.0, 0.0, 1.0], (200, 1))
  assert P.gn_step64(*P.plane_system(Pm, Q, N1))[0] is None


@pytest.mark.parametrize('sig,s', [([1.0, 0.6, 0.3], 1.0), ([1.0, 0.5, 1e-3], 1.0), ([1.0, 0.5, 0.3], -1.0),
                                   ([1.0, 1e-2, 1e-2], 1.0)])
def test_floor_matches_finite_difference_sensitivity(sig, s):
  """The worst rotation change per unit |dS|_2 over the six pair directions U (e_i e_j^T -+ e_j e_i^T) V^T matches
  |S|_2 / min(s~i + s~j) to within a factor 2 (the antisymmetric direction turns R by 2 |dS| / (s~i + s~j) about the
  pair's axis, which moves entries of R by between 1x and 2x that angle)."""
  g = np.random.default_rng(7)
  U, V = P.random_orthogonal(g, s), P.random_orthogonal(g)
  S = U @ np.diag(sig) @ V.T
  R0 = P.kabsch64(S)[0]
  h = 1e-9
  worst = 0.0
  for i in range(3):
    for j in range(i + 1, 3):
      for sgn in (1.0, -1.0):
        E = np.zeros((3, 3))
        E[i, j], E[j, i] = h, sgn * h
        worst = max(worst, np.abs(P.kabsch64(S + U @ E @ V.T)[0] - R0).max() / h)
  predicted = P.sensitivity_floor(S) / P.U32 / sig[0]
  assert 0.5 <= worst / predicted <= 2.0, (worst, predicted)


@pytest.mark.parametrize('name', sorted(SPECTRA))
def test_restated_kabsch_meets_the_criterion(name):
  """A different fp32 summation order (rows permuted) through the numpy kabsch.cuh stands in for the kernel."""
  X, Y, w = spectrum_case(name)
  ref = P.procrustes64(X, Y, w)
  R32, t32 = P.oracle32(X, Y, w)
  perm = np.random.default_rng(3).permutation(len(X))
  R, t = P.restated(X[perm], Y[perm], w[perm])
  c = P.check(R, t, R32, t32, ref)
  assert c['unique'] == (name not in NON_UNIQUE), (name, ref['floor'])
  assert c['ok'], (name, c)


def test_zero_covariance_gives_the_identity():
  """X at the origin: S = 0 exactly, and kabsch.cuh returns the identity as LAPACK's SVD does for the oracle."""
  g = np.random.default_rng(2)
  X = np.zeros((50, 3), np.float32)
  Y = g.normal(size=(50, 3)).astype(np.float32)
  w = np.ones(50, np.float32)
  R, t = P.restated(X, Y, w)
  R32, _ = P.oracle32(X, Y, w)
  assert np.array_equal(R, np.eye(3)) and np.array_equal(R32, np.eye(3))


@pytest.mark.parametrize('name', ['generic', 's3=1e-3', 'reflect-s3-small', 'scale-1e4', 'far-1e4'])
def test_negative_controls_miss_the_criterion(name):
  """S rounded to bfloat16, and the Jacobi stopped after one sweep, exceed the bound by >= 10x: the criterion can
  fail."""
  X, Y, w = spectrum_case(name)
  ref = P.procrustes64(X, Y, w)
  R32, t32 = P.oracle32(X, Y, w)
  for kw in (dict(round_S=P.bf16_round), dict(max_sweeps=1)):
    c = P.check(*P.restated(X, Y, w, **kw), R32, t32, ref)
    assert c['e'] >= 10 * c['bound'], (name, kw, c)


@pytest.mark.parametrize('name', sorted(P.PLANE_CASES))
def test_plane_step_criterion(name):
  """The kernel's 6x6 step restated (fp64 row-by-row sums, cholesky6_step) meets the step criterion at every
  cond(J^T J); the same step with J^T J summed in fp32, and the step fp32 end to end, miss it by >= 10x.  The
  systems are badly scaled rather than near-singular: their scaled condition stays below 100."""
  Ps, Q, N = P.plane_case(name)
  c = P.plane_check(P.plane_restated(Ps, Q, N), Ps, Q, N)
  assert c['ok'] and c['scaled_cond'] < 100, c
  for T in (P.plane_restated(Ps, Q, N, np.float32), P.plane_fp32(Ps, Q, N)):
    assert P.plane_check(T, Ps, Q, N)['e'] >= 10 * c['bound']


def test_refine64_is_the_reference_loop_in_fp64():
  """refine64 and oracle.se3_refine (fp32, break rule off) take the same k Adam steps: they agree to fp32 round-off,
  and the loss both report is the one at step k - 1."""
  g = np.random.default_rng(4)
  X = g.normal(size=(400, 3)).astype(np.float32)
  R_gt = P.random_orthogonal(g)
  Y = (X @ R_gt.T + [0.1, 0.2, -0.3] + g.normal(scale=0.05, size=X.shape)).astype(np.float32)
  w = g.uniform(0.1, 1.0, 400).astype(np.float32)
  w[7] = -0.5
  for k in (1, 10):
    R, t, loss = P.refine64(X, Y, w, 0.1, k)
    Ro, to, io = oreg.se3_refine(X, Y, w, 0.1, max_iter=k, break_threshold_ratio=0.0)
    assert io['iterations'] == k - 1 and io['break_count'] == 0
    assert np.abs(Ro.double().numpy() - R).max() < 1e-5 and np.abs(to.double().numpy().reshape(3) - t).max() < 1e-5
    assert abs(io['loss'] - loss) <= 1e-5 * abs(loss)
  # the loss is normalised by sum w, not sum |w|
  R0, t0 = torch.from_numpy(P.procrustes64(X, Y, w)['R']), torch.from_numpy(P.procrustes64(X, Y, w)['t'])
  Xd, Yd, wd = (torch.from_numpy(a.astype(np.float64)) for a in (X, Y, w))
  s = (((Xd @ R0.T + t0 - Yd) / 0.1) ** 2).sum(1)
  rho = torch.where(s < 1, 0.5 * s, 0.5 * (torch.sqrt(s + P.F32_EPS) - 0.5))
  assert abs(float((rho * wd).sum() / wd.sum()) - P.refine64(X, Y, w, 0.1, 1)[2]) < 1e-12
