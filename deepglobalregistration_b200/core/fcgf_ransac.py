"""``FCGFRansac``: the classical FCGF + RANSAC registration DGR is measured against (the ``RANSAC`` row of the
reference's results; the ``'ransac'`` method of scripts/test_kitti.py's FCGFWrapper), on the same features,
GPU and evaluation protocol as ``DeepGlobalRegistration``.

    dgr = DeepGlobalRegistration(config)
    T = FCGFRansac(dgr).register(xyz0, xyz1)

Voxelise both clouds -> FCGF features of both in one pass -> nearest target feature of every source point
(dgr_knn_top1) -> feature-matching RANSAC (dgr_ransac_feature_matching; what
core/deep_global_registration.py:29-47 asks of open3d 0.10) -> optionally point-to-point ICP, as the
stagewise path does.  The wrapped object's preprocessing, FCGF network, voxel size and ``use_icp`` are
used as they are: no second checkpoint is loaded.

``FCGFBaseline`` is that skeleton with the search step left to the subclass (core/fcgf_fgr.py uses it too) and
the descriptor in one overridable step, ``_features`` (core/fpfh_baseline.py swaps FCGF for FPFH there).
"""
import numpy as np
import torch

from .. import _abi
from ..util.timer import Timer


class FCGFBaseline:
  """Voxelise -> ``_features`` (FCGF on both clouds in one pass) -> ``_search`` (device result whose first 12 entries are the
  [R | t] rows of the pose) -> optional ICP from that pose -> one readback."""
  branch = None      # last_branch after a call
  label = None       # name in the timing log line

  def __init__(self, dgr):
    self.dgr = dgr
    self.reg_timer = Timer()
    self.last_branch = None
    self.last_info = {}

  @property
  def voxel_size(self):
    return self.dgr.voxel_size

  @property
  def use_icp(self):
    return self.dgr.use_icp

  def _features(self, p0, p1, c0, c1):
    """-> per-point features (f0, f1) of the voxelised clouds p0 / p1 (coords c0 / c1 from preprocess): FCGF of both
    in one pass."""
    return self.dgr.fcgf_feature_extraction_pair(c0, c1)

  def _search(self, p0, p1, f0, f1, manager1):
    """-> device double result of the global search; manager1: cloud 1's coordinate manager (voxel hash)."""
    raise NotImplementedError

  def _info(self, res):
    """last_info entries of the search's host result."""
    raise NotImplementedError

  def register(self, xyz0, xyz1):
    """-> 4x4 float64 ndarray mapping cloud 0 into cloud 1's frame."""
    d = self.dgr
    self.reg_timer.tic()
    _abi.refresh_stream()
    vs = self.voxel_size
    with torch.no_grad():
      p0, c0, _ = d.preprocess(xyz0, 0, _batch=0)
      p1, c1, _ = d.preprocess(xyz1, 1, _batch=1)
      f0, f1 = self._features(p0, p1, c0, c1)
      m = c1._dgr_manager
      res = self._search(p0, p1, f0.contiguous(), f1.contiguous(), m)
      parts = [res]
      if self.use_icp:
        parts.append(_abi.icp_point_to_point(p0, p1, m, vs, 2 * vs, res[:12].contiguous(), batch=1))
      host = torch.cat(parts).cpu().numpy()
    n_res = res.numel()
    T = host[:16].reshape(4, 4).copy()
    self.last_branch = self.branch
    self.last_info = dict(n0=len(p0), n1=len(p1), **self._info(host[:n_res]))
    if self.use_icp:
      icp = host[n_res:n_res + 20]
      T = icp[:16].reshape(4, 4).copy()
      self.last_info.update(icp_fitness=float(icp[16]), icp_inlier_rmse=float(icp[17]), icp_iterations=int(icp[18]))
    d._log(f'=> {self.label} takes {self.reg_timer.toc():.2} s')
    return np.asarray(T, dtype=np.float64)


class FCGFRansac(FCGFBaseline):
  branch = 'ransac'
  label = 'FCGF + RANSAC'

  def __init__(self, dgr):
    super().__init__(dgr)
    # what the reference's function receives from its safeguard call (:306-313, :43-44):
    # RANSACConvergenceCriteria(num_iterations = 80000, 1000) and only the distance checker
    self.max_iteration = 80000
    self.max_validation = 1000
    self.edge_ratio = 0.0         # CorrespondenceCheckerBasedOnEdgeLength threshold; 0 = not used
    self.seed = 0                 # open3d draws from std::random_device; here a call is reproducible

  def _search(self, p0, p1, f0, f1, manager1):
    vs = self.voxel_size
    nn = _abi.knn_top1(f0, f1)
    return _abi.ransac_feature_matching(p0, p1, nn, manager1.spec, manager1._maps[1].table, vs, 2 * vs,
                                        self.edge_ratio, 2 * vs, self.max_iteration, self.max_validation,
                                        seed=self.seed, batch=1)

  def _info(self, res):
    return dict(ransac_fitness=float(res[16]), ransac_inlier_rmse=float(res[17]), ransac_hypothesis=int(res[18]),
                ransac_inliers=int(res[19]), ransac_validated=int(res[20]), ransac_drawn=int(res[21]))
