"""ORACLE (test infrastructure only) - Fast Global Registration over feature matches, open3d's
``registration_fast_based_on_feature_matching(source, target, source_feature, target_feature,
FastGlobalRegistrationOption(...))``: the ``FGR`` row of the reference's published comparison.

PARITY UNPINNED: open3d is not installed in the build container and not vendored, so this restates the algorithm
of Zhou, Park & Koltun, "Fast Global Registration" (ECCV 2016) with open3d's documented options (division_factor
1.4, use_absolute_scale False, decrease_mu True, maximum_correspondence_distance 0.025, iteration_number 64,
tuple_scale 0.95, maximum_tuple_count 1000, tuple_test True; ``seed`` is this library's addition).  The boundary
conventions below are pinned here rather than measured against open3d:

1. Normalise: each cloud is centred on its own float64 mean; s = the largest centred norm over both clouds (1 if
   that is 0).  Unless use_absolute_scale, both clouds are divided by s and mu starts at 1; with it the clouds keep
   their scale and mu starts at s.  This follows the original FGR code; whether open3d starts mu the same way
   could not be checked.
2. Mutual matching: nn_st[i] = target feature nearest to source feature i, nn_ts[j] = source feature nearest to
   target feature j (L2, lowest row on ties; the library computes both in fp32, so near-ties may differ from
   open3d's float64 KD-tree).  (i, j) is kept when j = nn_st[i] and nn_ts[j] = i.  The kept pairs are listed in
   the row order of the cloud with more points (open3d swaps that cloud to the front; on a tie the source stays
   first).
3. Tuple test (tuple_test on): trials k = 0 .. 100 n_mut - 1 in order; trial k takes the list positions of draws
   3k, 3k + 1, 3k + 2 of the counter hash of oracle/ransac.py (the stream whose draws 4h .. 4h + 3 are RANSAC
   hypothesis h, so ``sample_indices`` serves both) with n = n_mut.  It is accepted when each edge (0, 1), (1, 2),
   (2, 0) has l_s * tuple_scale < l_t < l_s / tuple_scale, in float64 on the normalised points (a repeated draw
   gives two zero lengths and is rejected).  The first maximum_tuple_count accepted trials, in trial order, give
   their 3 pairs each, in draw order: those are the correspondences.  n_mut < 3: no trial.  With tuple_test off
   the correspondences are the mutual list.
4. Graduated non-convexity: fewer than 10 correspondences -> the optimiser returns the identity.  Otherwise
   iteration_number Gauss-Newton steps on sum rho(|p - T q|) (p source, q target: the TARGET moves onto the
   source) with Geman-McClure weights (mu / (r^2 + mu))^2.  Before the weights of step itr, when decrease_mu and
   itr % 4 == 0 and mu > maximum_correspondence_distance, mu is divided by division_factor (mu itself is compared,
   not mu^2, as in FGR).  The 6x6 normal equations are solved by Cholesky in float64; a non-positive pivot makes
   that step the identity.  The step (alpha, beta, gamma, t) is applied as [Rz(gamma) Ry(beta) Rx(alpha) | t],
   composed on the left.
5. Result: target -> source in the input frame is [R | -R m_t + scale t + m_s] (scale = s, or 1 with
   use_absolute_scale); the pose returned is its inverse, mapping source into target.  With fewer than 10
   correspondences that is the translation m_t - m_s.

The sums of the GPU kernel run in a different order than numpy's, so its pose agrees to round-off, not bit for
bit; the mutual list and the tuple correspondences agree exactly unless an edge ratio lies within round-off of
tuple_scale."""
import numpy as np

from .ransac import sample_indices
from .ransac_fm import feature_nn

OPTION_DEFAULTS = dict(division_factor=1.4, use_absolute_scale=False, decrease_mu=True,
                       maximum_correspondence_distance=0.025, iteration_number=64, tuple_scale=0.95,
                       maximum_tuple_count=1000, tuple_test=True)


def _norm(d):
  """Row norms of [m, 3] as sqrt((x x + y y) + z z) (the GPU evaluates the same expression)."""
  return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def normalise(src, tgt, use_absolute_scale=False):
  """-> (normalised source, normalised target, m_s, m_t, scale, mu0)."""
  S, T = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
  ms, mt = S.mean(0), T.mean(0)
  Sc, Tc = S - ms, T - mt
  s = max(_norm(Sc).max(), _norm(Tc).max())
  s = s if s > 0 else 1.0
  scale = 1.0 if use_absolute_scale else s
  return Sc / scale, Tc / scale, ms, mt, scale, (s if use_absolute_scale else 1.0)


def mutual_pairs(nn_st, nn_ts):
  """-> ([n_mut, 2] (source, target) rows in the larger cloud's row order, swapped = target larger)."""
  nn_st, nn_ts = np.asarray(nn_st, np.int64), np.asarray(nn_ts, np.int64)
  swapped = len(nn_ts) > len(nn_st)
  if swapped:
    j = np.arange(len(nn_ts))
    keep = nn_st[nn_ts] == j
    return np.stack([nn_ts[keep], j[keep]], 1), swapped
  i = np.arange(len(nn_st))
  keep = nn_ts[nn_st] == i
  return np.stack([i[keep], nn_st[keep]], 1), swapped


def tuple_positions(seed, trials, n):
  """[len(trials), 3] list positions of tuple trials: draws 3k .. 3k + 2 of the counter-hash stream."""
  d = 3 * np.asarray(trials, np.int64)[:, None] + np.arange(3)
  pos = sample_indices(seed, (d // 4).reshape(-1), n)
  return pos[np.arange(pos.shape[0]), (d % 4).reshape(-1)].reshape(-1, 3)


def tuple_test(Sn, Tn, pairs, tuple_scale, maximum_tuple_count, seed, chunk=1 << 16):
  """-> (accepted trial numbers, trials drawn until the maximum_tuple_count-th acceptance (100 n_mut if it is
  never reached, 0 without trials))."""
  n_mut = len(pairs)
  if n_mut < 3:
    return np.zeros(0, np.int64), 0
  n_trials = 100 * n_mut
  accepted = []
  for lo in range(0, n_trials, chunk):
    k = np.arange(lo, min(lo + chunk, n_trials))
    pos = tuple_positions(seed, k, n_mut)
    ps, pt = Sn[pairs[pos, 0]], Tn[pairs[pos, 1]]            # [m, 3, 3]
    ok = np.ones(len(k), bool)
    for a, b in ((0, 1), (1, 2), (2, 0)):
      ls, lt = _norm(ps[:, a] - ps[:, b]), _norm(pt[:, a] - pt[:, b])
      ok &= (ls * tuple_scale < lt) & (lt < ls / tuple_scale)
    accepted.extend(k[ok][:maximum_tuple_count - len(accepted)].tolist())
    if len(accepted) == maximum_tuple_count:
      return np.array(accepted, np.int64), accepted[-1] + 1
  return np.array(accepted, np.int64), n_trials


def cholesky_step(A, g):
  """x = -(A^-1 g) by Cholesky, or None on a non-positive pivot."""
  L = np.zeros((6, 6))
  for j in range(6):
    d = A[j, j] - L[j, :j] @ L[j, :j]
    if not d > 0:
      return None
    L[j, j] = np.sqrt(d)
    for i in range(j + 1, 6):
      L[i, j] = (A[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
  y = np.zeros(6)
  for i in range(6):
    y[i] = (-g[i] - L[i, :i] @ y[:i]) / L[i, i]
  x = np.zeros(6)
  for i in range(5, -1, -1):
    x[i] = (y[i] - L[i + 1:, i] @ x[i + 1:]) / L[i, i]
  return x


def step_pose(x):
  """[Rz(gamma) Ry(beta) Rx(alpha) | t] of a step x = (alpha, beta, gamma, t)."""
  ca, sa, cb, sb, cc, sc = np.cos(x[0]), np.sin(x[0]), np.cos(x[1]), np.sin(x[1]), np.cos(x[2]), np.sin(x[2])
  Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1.0]])
  Ry = np.array([[cb, 0, sb], [0, 1.0, 0], [-sb, 0, cb]])
  Rx = np.array([[1.0, 0, 0], [0, ca, -sa], [0, sa, ca]])
  D = np.eye(4)
  D[:3, :3], D[:3, 3] = Rz @ Ry @ Rx, x[3:]
  return D


def optimise(P, Q, mu0, division_factor, decrease_mu, maximum_correspondence_distance, iteration_number):
  """Graduated non-convexity on correspondences P[k] (source) <- Q[k] (target), normalised.
  -> (4x4 target -> source, final mu, ran)."""
  T, mu = np.eye(4), mu0
  if len(P) < 10:
    return T, mu, False
  for itr in range(iteration_number):
    if decrease_mu and itr % 4 == 0 and mu > maximum_correspondence_distance:
      mu /= division_factor
    q = Q @ T[:3, :3].T + T[:3, 3]
    r = P - q
    w = (mu / ((r * r).sum(1) + mu)) ** 2
    z, one = np.zeros(len(q)), np.ones(len(q))
    J = np.stack([np.stack([z, -q[:, 2], q[:, 1], -one, z, z], 1),            # d r_x
                  np.stack([q[:, 2], z, -q[:, 0], z, -one, z], 1),            # d r_y
                  np.stack([-q[:, 1], q[:, 0], z, z, z, -one], 1)], 1)        # d r_z   -> [m, 3, 6]
    A = np.einsum('m,mka,mkb->ab', w, J, J)
    g = np.einsum('m,mka,mk->a', w, J, r)
    x = cholesky_step(A, g)
    T = (step_pose(x) if x is not None else np.eye(4)) @ T
  return T, mu, True


def fgr(src, tgt, nn_st, nn_ts, seed=0, **option):
  """src [n_s, 3], tgt [n_t, 3], nn_st [n_s], nn_ts [n_t] -> (T 4x4 float64 mapping src into tgt, info)."""
  unknown = set(option) - set(OPTION_DEFAULTS)
  if unknown:
    raise TypeError(f'unknown options {sorted(unknown)}')
  o = dict(OPTION_DEFAULTS, **option)
  Sn, Tn, ms, mt, scale, mu0 = normalise(src, tgt, o['use_absolute_scale'])
  pairs, swapped = mutual_pairs(nn_st, nn_ts)
  trials, drawn = np.zeros(0, np.int64), 0
  if o['tuple_test']:
    trials, drawn = tuple_test(Sn, Tn, pairs, o['tuple_scale'], o['maximum_tuple_count'], seed)
    corres = pairs[tuple_positions(seed, trials, len(pairs)).reshape(-1)] if len(trials) else np.zeros((0, 2), np.int64)
  else:
    corres = pairs
  Tts, mu, ran = optimise(Sn[corres[:, 0]], Tn[corres[:, 1]], mu0, o['division_factor'], o['decrease_mu'],
                          o['maximum_correspondence_distance'], o['iteration_number'])
  R = Tts[:3, :3]
  t = -R @ mt + scale * Tts[:3, 3] + ms
  T = np.eye(4)
  T[:3, :3], T[:3, 3] = R.T, -R.T @ t
  info = dict(n_mut=len(pairs), n_corr=len(corres), drawn=drawn, mu=mu, ran=ran, swapped=swapped, mutual=pairs,
              corres=corres, trials=trials, scale=scale, mu0=mu0)
  return T, info


def fgr_feature_matching(src, tgt, feat_src, feat_tgt, seed=0, **option):
  """fgr() with both nearest-feature directions computed here (float64)."""
  return fgr(src, tgt, feature_nn(feat_src, feat_tgt), feature_nn(feat_tgt, feat_src), seed=seed, **option)
