"""``open3d.pipelines.registration`` stand-in backed by libdgr_b200 - the three calls the reference's
``core/deep_global_registration.py`` makes into open3d, with open3d's signatures and result objects:

  registration_icp(source, target, max_correspondence_distance, init, ...)             (:317-322)
      -> dgr_icp (point-to-point): nearest target point through a voxel hash of the target, fp64 Kabsch
         update, open3d's default stopping rule (relative fitness / RMSE 1e-6, 30 iterations);
  registration_ransac_based_on_correspondence(source, target, corres, ...)              (:50-64)
      -> dgr_ransac_correspondence: criteria.max_iteration four-point hypotheses, each scored on all
         correspondences (the reference passes its 80000 into the confidence slot, so open3d >= 0.12 never
         exits early; under 0.10 / 0.11 the same argument bounded the VALIDATED hypotheses instead - this
         stand-in follows the >= 0.12 reading, INTEGRATION.md).
  registration_ransac_based_on_feature_matching(source, target, source_feature, target_feature, ...)  (:29-47)
      -> dgr_knn_top1 + dgr_ransac_feature_matching: open3d 0.10's form (RANSACConvergenceCriteria(max_iteration,
         max_validation)), the edge-length and distance checkers, every validated hypothesis scored on all source
         points through a voxel hash of the target.

It also carries the calls open3d users make beyond DGR's own: point-to-plane ICP (``registration_icp`` with
``TransformationEstimationPointToPlane``, -> dgr_icp) on target normals from
``PointCloud.estimate_normals(KDTreeSearchParamHybrid(radius, max_nn))`` (-> dgr_estimate_normals), and

  registration_colored_icp(source, target, max_distance, init, criteria, lambda_geometric)           (open3d 0.10)
  registration_colored_icp(source, target, max_correspondence_distance, init, estimation_method, criteria) (>= 0.12)
      -> dgr_color_gradient on the target, then dgr_colored_icp: ICP with a geometric and a photometric row per
         correspondence (Park, Zhou & Koltun 2017), the local refinement of open3d's reconstruction system;

  registration_generalized_icp(source, target, max_correspondence_distance, init, estimation_method, criteria)
      -> dgr_generalized_icp on covariances from estimate_covariances (-> dgr_estimate_covariances) or built from
         normals (-> dgr_covariances_from_normals): plane-to-plane ICP (Segal, Haehnel & Thrun 2009);
  L2Loss / L1Loss / HuberLoss / CauchyLoss / GMLoss / TukeyLoss as the kernel of the point-to-plane, colored and
  generalized estimators -> dgr_icp_loss, dgr_colored_icp_loss, dgr_generalized_icp;

  registration_fast_based_on_feature_matching(source, target, source_feature, target_feature, option)
      -> dgr_knn_top1 both ways + dgr_fgr_feature_matching: Fast Global Registration (mutual matches, tuple
         test, graduated non-convexity) with FastGlobalRegistrationOption's fields and defaults;
  compute_fpfh_feature(input, KDTreeSearchParamHybrid(radius, max_nn))
      -> dgr_compute_fpfh: FPFH descriptors of a cloud with normals, the features open3d's global-registration
         recipe feeds to the two searches above;
  get_information_matrix_from_point_clouds(source, target, max_correspondence_distance, transformation)
      -> dgr_information_matrix: the 6x6 information matrix of a registered pair;
  PoseGraph / PoseGraphNode / PoseGraphEdge and global_optimization(pose_graph, method, criteria, option)
      -> dgr_pose_graph_optimize: multiway registration (Levenberg-Marquardt with line processes, pruning,
         compensation to the reference node) with GlobalOptimizationConvergenceCriteria's and
         GlobalOptimizationOption's fields and defaults.

With ``shims.install()`` these are reachable as ``open3d.pipelines.registration`` (and the pre-0.12 alias
``open3d.registration``) whenever the real open3d is absent, so the reference's own class runs on this stack
without a line changed.  There is no CPU path: the functions raise without an sm_90 device.
"""
import math

import numpy as np
import torch

from . import _abi


class TransformationEstimationPointToPoint:
  def __init__(self, with_scaling=False):
    if with_scaling:
      raise NotImplementedError('with_scaling=True is not used by DGR and not built')
    self.with_scaling = False


class RobustKernel:
  """open3d >= 0.12's robust loss: each residual row r of an estimator is weighted by Weight(r) (_abi.LOSS_IDS)."""
  loss = None

  def __init__(self, k=1.0):
    k = float(k)
    if self.loss in ('Huber', 'Cauchy', 'GM', 'Tukey') and not 0.0 < k < math.inf:
      raise ValueError(f'{type(self).__name__}: k must be finite and positive, got {k}')
    self.k = k

  def __repr__(self):
    return f'{type(self).__name__}(k={self.k})'


class L2Loss(RobustKernel):
  """Weight 1: the estimator without a kernel."""
  loss = 'L2'

  def __init__(self):
    super().__init__(1.0)


class L1Loss(RobustKernel):
  """Weight 1 / |r| (0 at r = 0, where open3d's is infinite)."""
  loss = 'L1'

  def __init__(self):
    super().__init__(1.0)


class HuberLoss(RobustKernel):
  """Weight 1 for |r| <= k, else k / |r|."""
  loss = 'Huber'


class CauchyLoss(RobustKernel):
  """Weight 1 / (1 + (r / k)^2)."""
  loss = 'Cauchy'


class GMLoss(RobustKernel):
  """Geman-McClure: weight k / (k + r^2)^2."""
  loss = 'GM'


class TukeyLoss(RobustKernel):
  """Weight (1 - min(1, |r| / k)^2)^2: 0 beyond k."""
  loss = 'Tukey'


def _kernel_check(kernel):
  """None or one of the six losses; any other object raises NotImplementedError."""
  if kernel is not None and not isinstance(kernel, RobustKernel):
    raise NotImplementedError(f'{type(kernel).__name__}: only L2Loss, L1Loss, HuberLoss, CauchyLoss, GMLoss and '
                              'TukeyLoss are built')
  return kernel


def _loss_args(kernel):
  """(loss, loss_k) of the _abi ICP wrappers: (None, 1.0) without a kernel."""
  return (None, 1.0) if kernel is None else (kernel.loss, kernel.k)


class TransformationEstimationPointToPlane:
  def __init__(self, kernel=None):
    self.kernel = _kernel_check(kernel)


class TransformationEstimationForColoredICP:
  """lambda_geometric weighs the geometric rows against the photometric ones; outside [0, 1] it falls back to 0.968,
  as open3d's constructor does."""

  def __init__(self, lambda_geometric=0.968, kernel=None):
    self.kernel = _kernel_check(kernel)
    lam = float(lambda_geometric)
    self.lambda_geometric = lam if 0.0 <= lam <= 1.0 else 0.968


class TransformationEstimationForGeneralizedICP:
  """Generalized ICP (Segal, Haehnel & Thrun 2009): plane-to-plane residuals weighted by both clouds' surface
  covariances.  epsilon: the covariance built from a normal n is R diag(epsilon, 1, 1) R^T (flat along n)."""

  def __init__(self, epsilon=1e-3, kernel=None):
    self.kernel = _kernel_check(kernel)
    epsilon = float(epsilon)
    if not 0.0 < epsilon < math.inf:
      raise ValueError(f'epsilon must be finite and positive, got {epsilon}')
    self.epsilon = epsilon


class KDTreeSearchParamHybrid:
  """Neighbours within `radius`, at most `max_nn` of them: what estimate_normals searches on the GPU."""

  def __init__(self, radius, max_nn):
    self.radius, self.max_nn = float(radius), int(max_nn)


class KDTreeSearchParamKNN:
  """open3d's unbounded k-nearest search: accepted as a name, not built (the voxel-hash search needs a radius)."""

  def __init__(self, knn=30):
    self.knn = int(knn)


class KDTreeSearchParamRadius:
  """open3d's radius search without a neighbour bound: accepted as a name, not built."""

  def __init__(self, radius):
    self.radius = float(radius)


def _hybrid_check(search_param, max_nn=_abi.MAX_NN):
  """A KDTreeSearchParamHybrid with a positive radius and 1 <= max_nn <= the caller's bound (64 for normals, 128 for
  FPFH)."""
  if isinstance(search_param, (KDTreeSearchParamKNN, KDTreeSearchParamRadius)):
    raise NotImplementedError(f'{type(search_param).__name__}: only KDTreeSearchParamHybrid(radius, max_nn) is built '
                              '(a bounded radius the voxel hash can search)')
  if not isinstance(search_param, KDTreeSearchParamHybrid):
    raise TypeError(f'expected KDTreeSearchParamHybrid, got {type(search_param).__name__}')
  if not search_param.radius > 0.0:
    raise ValueError(f'radius must be positive, got {search_param.radius}')
  if not 1 <= search_param.max_nn <= max_nn:
    raise ValueError(f'max_nn must lie in [1, {max_nn}], got {search_param.max_nn}')


def estimate_normals(points, search_param, prev=None):
  """Normals of points [N, 3] (float64 [N, 3], as open3d stores them) from KDTreeSearchParamHybrid neighbours,
  through a voxel hash of the cloud (dgr_estimate_normals); prev [N, 3]: the normals to orient against."""
  _hybrid_check(search_param)
  pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
  if prev is not None and np.asarray(prev).shape != pts.shape:
    raise ValueError('previous normals must hold one row per point')
  if len(pts) == 0:
    return np.zeros((0, 3))
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  p64 = torch.from_numpy(np.ascontiguousarray(pts)).to(dev)
  cell, spec, table, p32 = _target_hash(p64, search_param.radius, rows=True)
  prev_d = None if prev is None else torch.from_numpy(np.ascontiguousarray(prev, dtype=np.float32)).to(dev)
  nrm = _abi.estimate_normals(p32, (spec, table), cell, search_param.radius, search_param.max_nn, prev=prev_d)
  return nrm.cpu().numpy().astype(np.float64)


def estimate_covariances(points, search_param):
  """Per-point covariances of points [N, 3] (open3d's EstimatePerPointCovariances) from KDTreeSearchParamHybrid
  neighbours, through a voxel hash of the cloud (dgr_estimate_covariances).  -> float64 [N, 3, 3]."""
  _hybrid_check(search_param)
  pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
  if len(pts) == 0:
    return np.zeros((0, 3, 3))
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  p64 = torch.from_numpy(np.ascontiguousarray(pts)).to(dev)
  cell, spec, table, p32 = _target_hash(p64, search_param.radius, rows=True)
  cov = _abi.estimate_covariances(p32, (spec, table), cell, search_param.radius, search_param.max_nn)
  return _cov33(cov.cpu().numpy())


def _cov33(c6):
  """[N, 6] (xx, xy, xz, yy, yz, zz) -> [N, 3, 3]."""
  return np.ascontiguousarray(np.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], axis=1))


class ICPConvergenceCriteria:
  def __init__(self, relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=30):
    self.relative_fitness, self.relative_rmse, self.max_iteration = relative_fitness, relative_rmse, max_iteration


class RANSACConvergenceCriteria:
  def __init__(self, max_iteration=100000, confidence=0.999):
    self.max_iteration = int(max_iteration)
    self.confidence = min(float(confidence), 1.0)       # open3d clamps; DGR passes 80000 here
    # open3d 0.10 / 0.11 read the second argument as max_validation (what the feature-matching RANSAC uses;
    # DGR passes 1000 there at core/deep_global_registration.py:44); 1000 was that version's default
    is_count = isinstance(confidence, (int, np.integer)) and not isinstance(confidence, bool) and confidence >= 1
    self.max_validation = int(confidence) if is_count else 1000


class CorrespondenceCheckerBasedOnDistance:
  def __init__(self, distance_threshold):
    self.distance_threshold = distance_threshold


class CorrespondenceCheckerBasedOnEdgeLength:
  def __init__(self, similarity_threshold=0.9):
    self.similarity_threshold = similarity_threshold


class Feature:
  """Per-point feature vectors, stored as open3d does: data [dimension, num] float64."""

  def __init__(self):
    self.data = np.zeros((0, 0), dtype=np.float64)

  def resize(self, dim, n):
    self.data = np.zeros((int(dim), int(n)), dtype=np.float64)

  def dimension(self):
    return int(np.asarray(self.data).shape[0])

  def num(self):
    return int(np.asarray(self.data).shape[1])


class RegistrationResult:
  def __init__(self, transformation, fitness=0.0, inlier_rmse=0.0, n_corr=0):
    self.transformation = np.asarray(transformation, dtype=np.float64).reshape(4, 4).copy()
    self.fitness, self.inlier_rmse = float(fitness), float(inlier_rmse)
    self.correspondence_set = np.zeros((int(n_corr), 2), dtype=np.int32)   # count only; pairs stay on the device

  def __repr__(self):
    return (f'RegistrationResult with fitness={self.fitness:e}, inlier_rmse={self.inlier_rmse:e}, and '
            f'correspondence_set size of {len(self.correspondence_set)}')


def _points(pcd, device):
  pts = np.asarray(getattr(pcd, 'points', pcd), dtype=np.float64).reshape(-1, 3)
  return torch.from_numpy(np.ascontiguousarray(pts)).to(device)


def _target_hash(tgt64, max_dist, max_reach=4, what='max_correspondence_distance', rows=False):
  """Voxel hash of the target with at most one point per cell (what the ICP, normal and FPFH kernels search): cell =
  max_dist / 2 as in DGR (voxelised clouds, radius 2 voxels); a cloud with several points per cell gets finer
  cells up to the kernel's reach (4 for ICP and normals, 6 for FPFH, whose 5-voxel radius needs cell = max_dist / 5).
  A cell whose quotient max_dist / cell rounds above the reach is widened by one ulp.  -> (cell, spec, table), and with
  rows=True also the target as the float32 rows a search of this table must read (_abi.float32_in_cells of the
  table's cells)."""
  for div in range(2, max_reach + 1):
    cell = max_dist / div
    if math.ceil(max_dist / cell) > max_reach:
      cell = float(np.nextafter(cell, np.inf))
    raw, spec, table, _, _, n = _abi.voxelise(tgt64, cell)
    if n == tgt64.shape[0]:                 # every row kept: raw row i is target row i
      return (cell, spec, table, _abi.float32_in_cells(tgt64, raw[:, 1:], cell)) if rows else (cell, spec, table)
  raise NotImplementedError(f'target has several points within {what} / {max_reach} of each other: '
                            'voxel-downsample it first (DGR always passes voxelised clouds)')


def compute_fpfh_feature(input, search_param):
  """open3d's ``registration.compute_fpfh_feature(pcd, KDTreeSearchParamHybrid(radius, max_nn))``: FPFH features of a
  cloud with normals, through a voxel hash of the cloud (dgr_compute_fpfh; max_nn <= 128, the point itself
  included).  -> Feature with data float64 [33, N]."""
  _hybrid_check(search_param, _abi.FPFH_MAX_NN)
  pts = np.asarray(getattr(input, 'points', input), dtype=np.float64).reshape(-1, 3)
  nrm = getattr(input, 'normals', None)
  if nrm is None:
    raise RuntimeError('compute_fpfh_feature needs normals: call '
                       'pcd.estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) first')
  nrm = np.asarray(nrm, dtype=np.float32).reshape(-1, 3)
  if len(nrm) != len(pts):
    raise RuntimeError('normals must hold one row per point')
  feature = Feature()
  feature.resize(_abi.FPFH_DIM, len(pts))
  if len(pts) == 0:
    return feature
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  p64 = torch.from_numpy(np.ascontiguousarray(pts)).to(dev)
  cell, spec, table, p32 = _target_hash(p64, search_param.radius, max_reach=6, what='the radius', rows=True)
  f = _abi.compute_fpfh(p32, torch.from_numpy(np.ascontiguousarray(nrm)).to(dev), (spec, table),
                        cell, search_param.radius, search_param.max_nn)
  feature.data = f.cpu().numpy().astype(np.float64).T.copy()
  return feature


def registration_icp(source, target, max_correspondence_distance, init=None, estimation_method=None, criteria=None):
  """Point-to-point (the default, what DGR calls), point-to-plane or generalized ICP; point-to-plane needs target
  normals (``target.estimate_normals(KDTreeSearchParamHybrid(radius, max_nn))``), generalized ICP covariances on both
  clouds (``estimate_covariances``; unlike open3d, which returns ``init`` unchanged, it raises without them)."""
  if isinstance(estimation_method, TransformationEstimationForGeneralizedICP):
    for pcd, which in ((source, 'source'), (target, 'target')):
      if getattr(pcd, 'covariances', None) is None:
        raise RuntimeError(f'registration_icp with TransformationEstimationForGeneralizedICP needs covariances on the '
                           f'{which} cloud: call estimate_covariances(KDTreeSearchParamHybrid(radius, max_nn)) first, '
                           'or use registration_generalized_icp')
    return registration_generalized_icp(source, target, max_correspondence_distance, init, estimation_method,
                                        criteria)
  plane = isinstance(estimation_method, TransformationEstimationPointToPlane)
  if not (plane or estimation_method is None or isinstance(estimation_method, TransformationEstimationPointToPoint)):
    raise NotImplementedError('only point-to-point, point-to-plane and generalized ICP are built')
  tgt_normals = getattr(target, 'normals', None) if plane else None
  if plane and tgt_normals is None:
    raise RuntimeError('TransformationEstimationPointToPlane needs target normals: call '
                       'target.estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) first')
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  criteria = criteria or ICPConvergenceCriteria()
  src64, tgt64 = _points(source, dev), _points(target, dev)
  T0 = np.eye(4) if init is None else np.asarray(init, dtype=np.float64).reshape(4, 4)
  if len(src64) == 0 or len(tgt64) == 0:
    return RegistrationResult(T0)
  cell, spec, table, tgt = _target_hash(tgt64, float(max_correspondence_distance), rows=True)
  src = src64.float().contiguous()
  T12 = torch.from_numpy(np.ascontiguousarray(T0[:3])).to(dev)
  args = (float(max_correspondence_distance), T12, int(criteria.max_iteration), float(criteria.relative_fitness),
          float(criteria.relative_rmse))
  if plane:
    nrm = np.asarray(tgt_normals, dtype=np.float32).reshape(-1, 3)
    if len(nrm) != len(tgt):
      raise RuntimeError('target normals must hold one row per target point')
    loss, loss_k = _loss_args(estimation_method.kernel)
    res = _abi.icp_point_to_plane(src, tgt, torch.from_numpy(np.ascontiguousarray(nrm)).to(dev), (spec, table), cell,
                                  *args, loss=loss, loss_k=loss_k)
  else:
    res = _abi.icp_point_to_point(src, tgt, (spec, table), cell, *args)
  r = res.cpu().numpy()
  return RegistrationResult(r[:16], r[16], r[17], r[19])


_COLORED_ICP_FORMS = (('max_distance', 'init', 'criteria', 'lambda_geometric'),                   # open3d 0.10
                      ('max_correspondence_distance', 'init', 'estimation_method', 'criteria'))  # >= 0.12


def _colored_icp_arguments(args, kwargs):
  """(max_distance, init, criteria, lambda_geometric) of either argument form; the fifth argument (or a keyword only
  one form has) tells them apart."""
  new = ((len(args) >= 3 and isinstance(args[2], TransformationEstimationForColoredICP)) or
         'estimation_method' in kwargs or 'max_correspondence_distance' in kwargs)
  names = _COLORED_ICP_FORMS[new]
  if len(args) > len(names):
    raise TypeError(f'registration_colored_icp takes at most {len(names) + 2} positional arguments')
  bound = dict(zip(names, args))
  for k, v in kwargs.items():
    if k not in names or k in bound:
      raise TypeError(f'registration_colored_icp got an unexpected or repeated argument {k!r}')
    bound[k] = v
  if names[0] not in bound:
    raise TypeError(f'registration_colored_icp needs {names[0]}')
  if new:
    est = bound.get('estimation_method') or TransformationEstimationForColoredICP()
    if not isinstance(est, TransformationEstimationForColoredICP):
      raise NotImplementedError('registration_colored_icp takes TransformationEstimationForColoredICP')
    lam = est.lambda_geometric
  else:
    lam = TransformationEstimationForColoredICP(bound.get('lambda_geometric', 0.968)).lambda_geometric
  return float(bound[names[0]]), bound.get('init'), bound.get('criteria'), lam


def _colors(pcd, which):
  c = getattr(pcd, 'colors', None)
  n = len(np.asarray(getattr(pcd, 'points', pcd)).reshape(-1, 3))
  if c is None or len(np.asarray(c).reshape(-1, 3)) != n or n == 0:
    raise RuntimeError(f'colored ICP needs colours on the {which} cloud (PointCloud.colors, one row per point)')
  return np.asarray(c, dtype=np.float64).reshape(-1, 3)


def intensity(colors):
  """open3d's colored-ICP intensity (r + g + b) / 3 of colours [n, 3] in [0, 1], as the float32 the kernels read."""
  c = np.asarray(colors, dtype=np.float64).reshape(-1, 3)
  return ((c[:, 0] + c[:, 1] + c[:, 2]) / 3.0).astype(np.float32)


def registration_colored_icp(source, target, *args, **kwargs):
  """open3d's colored ICP (Park, Zhou & Koltun, ICCV 2017) in either argument form: 0.10's (source, target,
  max_distance, init, criteria, lambda_geometric) or >= 0.12's (source, target, max_correspondence_distance, init,
  estimation_method, criteria).  The target needs normals and both clouds colours.  As open3d does, the target's
  colour gradients come from its normals and colours at KDTreeSearchParamHybrid(2 max_distance, 30)
  (dgr_color_gradient); the ICP (dgr_colored_icp) searches a voxel hash of the target whose cell serves both radii."""
  max_distance, init, criteria, lam = _colored_icp_arguments(args, kwargs)
  est = kwargs.get('estimation_method', args[2] if len(args) >= 3 else None)
  kernel = est.kernel if isinstance(est, TransformationEstimationForColoredICP) else None     # the >= 0.12 form
  if not max_distance > 0.0:
    raise ValueError(f'max_distance must be positive, got {max_distance}')
  tgt_normals = getattr(target, 'normals', None)
  if tgt_normals is None:
    raise RuntimeError('colored ICP needs target normals: call '
                       'target.estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) first')
  c_src, c_tgt = _colors(source, 'source'), _colors(target, 'target')
  nrm = np.asarray(tgt_normals, dtype=np.float32).reshape(-1, 3)
  if len(nrm) != len(c_tgt):
    raise RuntimeError('target normals must hold one row per target point')
  criteria = criteria or ICPConvergenceCriteria()
  T0 = np.eye(4) if init is None else np.asarray(init, dtype=np.float64).reshape(4, 4)
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  src64, tgt64 = _points(source, dev), _points(target, dev)
  cell, spec, table, tgt = _target_hash(tgt64, 2.0 * max_distance, what='2 max_distance', rows=True)
  src = src64.float().contiguous()
  nrm_d = torch.from_numpy(np.ascontiguousarray(nrm)).to(dev)
  i_src = torch.from_numpy(intensity(c_src)).to(dev)
  i_tgt = torch.from_numpy(intensity(c_tgt)).to(dev)
  grad = _abi.color_gradient(tgt, nrm_d, i_tgt, (spec, table), cell, 2.0 * max_distance, 30)
  T12 = torch.from_numpy(np.ascontiguousarray(T0[:3])).to(dev)
  loss, loss_k = _loss_args(kernel)
  r = _abi.icp_colored(src, i_src, tgt, nrm_d, i_tgt, grad, (spec, table), cell, max_distance, lam, T12,
                       int(criteria.max_iteration), float(criteria.relative_fitness),
                       float(criteria.relative_rmse), loss=loss, loss_k=loss_k).cpu().numpy()
  return RegistrationResult(r[:16], r[16], r[17], r[19])


def _gicp_covariances(pcd, which, epsilon, dev):
  """The cloud's covariances as the device float64 [N, 6] dgr_generalized_icp reads: its own if it has them, else
  built from its normals with epsilon (dgr_covariances_from_normals); open3d's precedence."""
  n = len(np.asarray(getattr(pcd, 'points', pcd)).reshape(-1, 3))
  cov = getattr(pcd, 'covariances', None)
  if cov is not None:
    cov = np.asarray(cov, dtype=np.float64).reshape(-1, 3, 3)
    if len(cov) != n:
      raise RuntimeError(f'{which} covariances must hold one [3, 3] matrix per point')
    c6 = np.stack([cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]], axis=1)
    return torch.from_numpy(np.ascontiguousarray(c6)).to(dev)
  nrm = getattr(pcd, 'normals', None)
  if nrm is None:
    raise RuntimeError(f'generalized ICP needs covariances or normals on the {which} cloud: call '
                       'estimate_covariances(KDTreeSearchParamHybrid(radius, max_nn)) or '
                       'estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) first')
  nrm = np.asarray(nrm, dtype=np.float32).reshape(-1, 3)
  if len(nrm) != n:
    raise RuntimeError(f'{which} normals must hold one row per point')
  return _abi.covariances_from_normals(torch.from_numpy(np.ascontiguousarray(nrm)).to(dev), epsilon)


def registration_generalized_icp(source, target, max_correspondence_distance, init=None, estimation_method=None,
                                 criteria=None):
  """open3d's generalized ICP (Segal, Haehnel & Thrun 2009; plane-to-plane).  Each cloud uses its own covariances
  if it has them, else covariances built from its normals with estimation_method.epsilon; a cloud with neither is an
  error (open3d would estimate normals with KDTreeSearchParamKNN, which is not built).  dgr_generalized_icp searches
  a voxel hash of the target as registration_icp does."""
  est = TransformationEstimationForGeneralizedICP() if estimation_method is None else estimation_method
  if not isinstance(est, TransformationEstimationForGeneralizedICP):
    raise NotImplementedError('registration_generalized_icp takes TransformationEstimationForGeneralizedICP')
  d = float(max_correspondence_distance)
  if not d > 0.0:
    raise ValueError(f'max_correspondence_distance must be positive, got {max_correspondence_distance}')
  for pcd, which in ((source, 'source'), (target, 'target')):
    if getattr(pcd, 'covariances', None) is None and getattr(pcd, 'normals', None) is None:
      raise RuntimeError(f'generalized ICP needs covariances or normals on the {which} cloud: call '
                         'estimate_covariances(KDTreeSearchParamHybrid(radius, max_nn)) or '
                         'estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) first')
  criteria = criteria or ICPConvergenceCriteria()
  T0 = np.eye(4) if init is None else np.asarray(init, dtype=np.float64).reshape(4, 4)
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  src64, tgt64 = _points(source, dev), _points(target, dev)
  if len(src64) == 0 or len(tgt64) == 0:
    return RegistrationResult(T0)
  c_src = _gicp_covariances(source, 'source', est.epsilon, dev)
  c_tgt = _gicp_covariances(target, 'target', est.epsilon, dev)
  cell, spec, table, tgt = _target_hash(tgt64, d, rows=True)
  T12 = torch.from_numpy(np.ascontiguousarray(T0[:3])).to(dev)
  loss, loss_k = _loss_args(est.kernel)
  r = _abi.icp_generalized(src64.float().contiguous(), c_src, tgt, c_tgt, (spec, table), cell, d, T12,
                           int(criteria.max_iteration), float(criteria.relative_fitness),
                           float(criteria.relative_rmse), loss=loss, loss_k=loss_k).cpu().numpy()
  return RegistrationResult(r[:16], r[16], r[17], r[19])


def registration_ransac_based_on_correspondence(source, target, corres, max_correspondence_distance,
                                                estimation_method=None, ransac_n=3, checkers=None, criteria=None,
                                                seed=0):
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  if int(ransac_n) != 4:
    raise NotImplementedError('ransac_n = 4 (what DGR passes) is the built sample size')
  criteria = criteria or RANSACConvergenceCriteria()
  corres = np.asarray(corres).reshape(-1, 2)
  src, tgt = _points(source, dev).float().contiguous(), _points(target, dev).float().contiguous()
  if len(corres) < 4:
    return RegistrationResult(np.eye(4))
  idx0 = torch.from_numpy(np.ascontiguousarray(corres[:, 0], dtype=np.int32)).to(dev)
  idx1 = torch.from_numpy(np.ascontiguousarray(corres[:, 1], dtype=np.int32)).to(dev)
  r = _abi.ransac_correspondence(src, tgt, idx0, idx1, float(max_correspondence_distance),
                                 num_hyp=criteria.max_iteration, seed=seed).cpu().numpy()
  return RegistrationResult(r[:16], r[16], r[17], r[19])


def _feature_checkers(checkers):
  """(edge_ratio, check_dist) of the checker list (0 = that checker is off); several of one kind combine to the
  strictest."""
  edge, dist = 0.0, 0.0
  for c in checkers or ():
    if isinstance(c, CorrespondenceCheckerBasedOnEdgeLength):
      edge = max(edge, float(c.similarity_threshold))
    elif isinstance(c, CorrespondenceCheckerBasedOnDistance):
      d = float(c.distance_threshold)
      dist = d if dist == 0.0 else min(dist, d)
    else:
      raise NotImplementedError(f'{type(c).__name__}: only the edge-length and distance checkers are built')
  return edge, dist


def registration_ransac_based_on_feature_matching(source, target, source_feature, target_feature,
                                                  max_correspondence_distance, estimation_method=None, ransac_n=3,
                                                  checkers=None, criteria=None, seed=0, **kwargs):
  """open3d 0.10's argument order (the reference's :29-47).  Every source point's nearest target feature
  (dgr_knn_top1, fp32) proposes its match; dgr_ransac_feature_matching draws criteria.max_iteration
  hypotheses of 4 source points, and the first criteria.max_validation that pass the checkers are scored on
  every source point."""
  if 'mutual_filter' in kwargs or isinstance(max_correspondence_distance, (bool, np.bool_)):
    raise NotImplementedError('the open3d >= 0.12 form (mutual_filter) is not built; DGR calls the 0.10 form')
  if kwargs:
    raise TypeError(f'unexpected arguments {sorted(kwargs)}')
  if int(ransac_n) != 4:
    raise NotImplementedError('ransac_n = 4 (what DGR passes) is the built sample size')
  if not (estimation_method is None or isinstance(estimation_method, TransformationEstimationPointToPoint)):
    raise NotImplementedError('only point-to-point estimation is built (what DGR calls)')
  edge_ratio, check_dist = _feature_checkers(checkers)
  criteria = criteria or RANSACConvergenceCriteria()
  fs = np.asarray(source_feature.data, dtype=np.float32).T
  ft = np.asarray(target_feature.data, dtype=np.float32).T
  if fs.shape[1] != ft.shape[1]:
    raise ValueError(f'feature dimensions differ: {fs.shape[1]} vs {ft.shape[1]}')
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  src64, tgt64 = _points(source, dev), _points(target, dev)
  if len(fs) != len(src64) or len(ft) != len(tgt64):
    raise ValueError('one feature per point is required')
  if len(src64) == 0 or len(tgt64) == 0:
    return RegistrationResult(np.eye(4))
  d = float(max_correspondence_distance)
  cell, spec, table, tgt = _target_hash(tgt64, d, rows=True)
  nn = _abi.knn_top1(torch.from_numpy(np.ascontiguousarray(fs)).to(dev), torch.from_numpy(np.ascontiguousarray(ft)).to(dev))
  r = _abi.ransac_feature_matching(src64.float().contiguous(), tgt, nn, spec, table, cell, d,
                                   edge_ratio, check_dist, criteria.max_iteration, criteria.max_validation,
                                   seed=seed).cpu().numpy()
  return RegistrationResult(r[:16], r[16], r[17], r[19])


class FastGlobalRegistrationOption:
  """open3d's option object for Fast Global Registration, with its field names and defaults.  ``seed`` (not an
  open3d field in every release) makes the tuple test's draws reproducible."""

  def __init__(self, division_factor=1.4, use_absolute_scale=False, decrease_mu=True,
               maximum_correspondence_distance=0.025, iteration_number=64, tuple_scale=0.95,
               maximum_tuple_count=1000, tuple_test=True, seed=0):
    self.division_factor = float(division_factor)
    self.use_absolute_scale = bool(use_absolute_scale)
    self.decrease_mu = bool(decrease_mu)
    self.maximum_correspondence_distance = float(maximum_correspondence_distance)
    self.iteration_number = int(iteration_number)
    self.tuple_scale = float(tuple_scale)
    self.maximum_tuple_count = int(maximum_tuple_count)
    self.tuple_test = bool(tuple_test)
    self.seed = int(seed)

  def __repr__(self):
    return ('FastGlobalRegistrationOption(' + ', '.join(f'{k}={v}' for k, v in vars(self).items()) + ')')


def _fgr_option_check(o):
  if not o.division_factor > 1.0:
    raise ValueError(f'division_factor must be > 1, got {o.division_factor}')
  if not o.maximum_correspondence_distance > 0.0:
    raise ValueError(f'maximum_correspondence_distance must be positive, got {o.maximum_correspondence_distance}')
  if o.iteration_number < 0:
    raise ValueError(f'iteration_number must be >= 0, got {o.iteration_number}')
  if not 0.0 < o.tuple_scale <= 1.0:
    raise ValueError(f'tuple_scale must lie in (0, 1], got {o.tuple_scale}')
  if o.maximum_tuple_count < 1:
    raise ValueError(f'maximum_tuple_count must be >= 1, got {o.maximum_tuple_count}')


def registration_fast_based_on_feature_matching(source, target, source_feature, target_feature,
                                                option=None):
  """Fast Global Registration (Zhou, Park & Koltun 2016) on feature matches.  Both nearest-feature directions
  come from dgr_knn_top1 (fp32); dgr_fgr_feature_matching keeps the mutual matches, runs the tuple test and the
  graduated non-convexity optimiser.  Like open3d's, the result carries the transformation only (fitness 0, no
  correspondence set)."""
  option = FastGlobalRegistrationOption() if option is None else option
  _fgr_option_check(option)
  fs = np.asarray(source_feature.data, dtype=np.float32).T
  ft = np.asarray(target_feature.data, dtype=np.float32).T
  if fs.shape[1] != ft.shape[1]:
    raise ValueError(f'feature dimensions differ: {fs.shape[1]} vs {ft.shape[1]}')
  n_s = len(np.asarray(getattr(source, 'points', source)).reshape(-1, 3))
  n_t = len(np.asarray(getattr(target, 'points', target)).reshape(-1, 3))
  if len(fs) != n_s or len(ft) != n_t:
    raise ValueError('one feature per point is required')
  if n_s == 0 or n_t == 0:
    return RegistrationResult(np.eye(4))
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  src, tgt = _points(source, dev).float().contiguous(), _points(target, dev).float().contiguous()
  fs_d = torch.from_numpy(np.ascontiguousarray(fs)).to(dev)
  ft_d = torch.from_numpy(np.ascontiguousarray(ft)).to(dev)
  r = _abi.fgr_feature_matching(src, tgt, _abi.knn_top1(fs_d, ft_d), _abi.knn_top1(ft_d, fs_d),
                                option.division_factor, option.use_absolute_scale, option.decrease_mu,
                                option.maximum_correspondence_distance, option.iteration_number, option.tuple_scale,
                                option.maximum_tuple_count, option.tuple_test, seed=option.seed).cpu().numpy()
  return RegistrationResult(r[:16])


def get_information_matrix_from_point_clouds(source, target, max_correspondence_distance, transformation):
  """open3d's ``get_information_matrix_from_point_clouds``: sum of G^T G over the nearest target point of every
  transformed source point strictly within the radius (dgr_information_matrix, through a voxel hash of the target as
  registration_icp searches it).  -> float64 [6, 6]; entry [5, 5] is the correspondence count."""
  d = float(max_correspondence_distance)
  if not d > 0.0:
    raise ValueError(f'max_correspondence_distance must be positive, got {max_correspondence_distance}')
  T = np.asarray(transformation, dtype=np.float64).reshape(4, 4)
  if not np.isfinite(T).all():
    raise ValueError('transformation must be finite')
  n_s = len(np.asarray(getattr(source, 'points', source)).reshape(-1, 3))
  n_t = len(np.asarray(getattr(target, 'points', target)).reshape(-1, 3))
  if n_s == 0 or n_t == 0:
    return np.zeros((6, 6))
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  src64, tgt64 = _points(source, dev), _points(target, dev)
  cell, spec, table, tgt = _target_hash(tgt64, d, rows=True)
  out = _abi.information_matrix(src64.float().contiguous(), tgt, (spec, table), cell, d, T)
  return out.cpu().numpy()[:36].reshape(6, 6).copy()


class PoseGraphNode:
  def __init__(self, pose=None):
    self.pose = np.eye(4) if pose is None else np.asarray(pose, dtype=np.float64).reshape(4, 4).copy()

  def __repr__(self):
    return 'PoseGraphNode, access pose to get its current pose.'


class PoseGraphEdge:
  def __init__(self, source_node_id=-1, target_node_id=-1, transformation=None, information=None, uncertain=False,
               confidence=1.0):
    self.source_node_id, self.target_node_id = int(source_node_id), int(target_node_id)
    self.transformation = np.eye(4) if transformation is None else \
        np.asarray(transformation, dtype=np.float64).reshape(4, 4).copy()
    self.information = np.eye(6) if information is None else \
        np.asarray(information, dtype=np.float64).reshape(6, 6).copy()
    self.uncertain = bool(uncertain)
    self.confidence = float(confidence)

  def __repr__(self):
    return (f'PoseGraphEdge from nodes {self.source_node_id} to {self.target_node_id}, access transformation to get '
            'relative transformation')


class PoseGraph:
  def __init__(self):
    self.nodes = []
    self.edges = []

  def __repr__(self):
    return f'PoseGraph with {len(self.nodes)} nodes and {len(self.edges)} edges.'


class GlobalOptimizationLevenbergMarquardt:
  pass


class GlobalOptimizationGaussNewton:
  """Accepted as a name; global_optimization raises NotImplementedError when it is passed."""


class GlobalOptimizationConvergenceCriteria:
  def __init__(self, max_iteration=100, min_relative_increment=1e-6, min_relative_residual_increment=1e-6,
               min_right_term=1e-6, min_residual=1e-6, max_iteration_lm=20, upper_scale_factor=2. / 3.,
               lower_scale_factor=1. / 3.):
    self.max_iteration = int(max_iteration)
    self.min_relative_increment = float(min_relative_increment)
    self.min_relative_residual_increment = float(min_relative_residual_increment)
    self.min_right_term = float(min_right_term)
    self.min_residual = float(min_residual)
    self.max_iteration_lm = int(max_iteration_lm)
    self.upper_scale_factor = float(upper_scale_factor)
    self.lower_scale_factor = float(lower_scale_factor)


class GlobalOptimizationOption:
  def __init__(self, max_correspondence_distance=0.075, edge_prune_threshold=0.25, preference_loop_closure=1.0,
               reference_node=-1):
    self.max_correspondence_distance = float(max_correspondence_distance)
    self.edge_prune_threshold = float(edge_prune_threshold)
    self.preference_loop_closure = float(preference_loop_closure)
    self.reference_node = int(reference_node)


def _pose_graph_arrays(pose_graph, option):
  """Host arrays of a PoseGraph, every argument checked as the library checks it."""
  n, m = len(pose_graph.nodes), len(pose_graph.edges)
  if n == 0:
    raise ValueError('the pose graph has no node')
  if n > _abi.POSE_GRAPH_MAX_NODES:
    raise ValueError(f'{n} nodes: at most {_abi.POSE_GRAPH_MAX_NODES} are supported (a dense solver)')
  if m > _abi.POSE_GRAPH_MAX_EDGES:
    raise ValueError(f'{m} edges: at most {_abi.POSE_GRAPH_MAX_EDGES} are supported')
  if not option.max_correspondence_distance > 0.0:
    raise ValueError(f'max_correspondence_distance must be positive, got {option.max_correspondence_distance}')
  if not -1 <= option.reference_node < n:
    raise ValueError(f'reference_node must lie in [-1, {n}), got {option.reference_node}')
  poses = np.stack([np.asarray(v.pose, dtype=np.float64).reshape(4, 4) for v in pose_graph.nodes])
  ends = np.array([[e.source_node_id, e.target_node_id] for e in pose_graph.edges], dtype=np.int64).reshape(m, 2)
  if m and (ends.min() < 0 or ends.max() >= n):
    raise ValueError('an edge names a node that is not in the graph')
  if m and (ends[:, 0] == ends[:, 1]).any():
    raise ValueError('an edge joins a node to itself')
  T = np.stack([np.asarray(e.transformation, dtype=np.float64).reshape(4, 4) for e in pose_graph.edges]) if m else \
      np.zeros((0, 4, 4))
  info = np.stack([np.asarray(e.information, dtype=np.float64).reshape(6, 6) for e in pose_graph.edges]) if m else \
      np.zeros((0, 6, 6))
  unc = np.array([bool(e.uncertain) for e in pose_graph.edges], dtype=bool)
  conf = np.array([float(e.confidence) for e in pose_graph.edges], dtype=np.float64)
  for name, a in (('node poses', poses), ('edge transformations', T), ('information matrices', info),
                  ('confidences', conf)):
    if not np.isfinite(a).all():
      raise ValueError(f'{name} must be finite')
  return poses, ends.astype(np.int32), T, info, unc, conf


def global_optimization(pose_graph, method=None, criteria=None, option=None):
  """open3d's ``global_optimization``: Levenberg-Marquardt on the pose graph with line processes on the uncertain
  edges, the uncertain edges whose line process ends below option.edge_prune_threshold removed, a second run on the
  rest, then every pose moved so the reference node keeps its pose (dgr_pose_graph_optimize, one launch).  In place:
  node poses updated, uncertain edges' confidence set to their final line process, pruned edges removed.  Returns
  the library's statistics (open3d returns None)."""
  if isinstance(method, GlobalOptimizationGaussNewton):
    raise NotImplementedError('GlobalOptimizationGaussNewton is not built; use GlobalOptimizationLevenbergMarquardt')
  if not (method is None or isinstance(method, GlobalOptimizationLevenbergMarquardt)):
    raise TypeError(f'expected a global optimisation method, got {type(method).__name__}')
  criteria = GlobalOptimizationConvergenceCriteria() if criteria is None else criteria
  option = GlobalOptimizationOption() if option is None else option
  poses, ends, T, info, unc, conf = _pose_graph_arrays(pose_graph, option)
  out, kept, lp, stats = _abi.pose_graph_optimize(
      poses, ends, T, info, unc, conf, option.max_correspondence_distance, option.edge_prune_threshold,
      option.preference_loop_closure, option.reference_node, criteria.max_iteration, criteria.min_relative_increment,
      criteria.min_relative_residual_increment, criteria.min_right_term, criteria.min_residual,
      criteria.max_iteration_lm, criteria.upper_scale_factor, criteria.lower_scale_factor)
  for node, P in zip(pose_graph.nodes, out):
    node.pose = P.copy()
  for edge, l in zip(pose_graph.edges, lp):
    if edge.uncertain:
      edge.confidence = float(l)
  pose_graph.edges = [e for e, k in zip(pose_graph.edges, kept) if k]
  return stats
