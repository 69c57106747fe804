"""``ICPBaseline``: ICP from a fixed initial pose (identity by default), the ``ICP (Point-to-point)`` and
``ICP (Point-to-plane)`` rows of the reference's results and generalized ICP, on the same voxelisation, GPU and
evaluation protocol as ``DeepGlobalRegistration``.

    dgr = DeepGlobalRegistration(config)
    T = ICPBaseline(dgr, method='point_to_plane').register(xyz0, xyz1)

Voxelise both clouds (the wrapped object's ``preprocess`` and ``voxel_size``; no FCGF) -> point_to_plane: target
normals from neighbours within 2 voxels, at most 30 (dgr_estimate_normals, util/pointcloud.py:60's setting), through
cloud 1's voxel table -> ICP from ``init`` through the same table (dgr_icp, with or without the normals)
-> one readback.  generalized: both clouds' normals at the same setting, each through its own table, covariances
R diag(1e-3, 1, 1) R^T from them (dgr_covariances_from_normals) -> dgr_generalized_icp.
"""
import numpy as np
import torch

from .. import _abi
from ..util.timer import Timer

METHODS = {'point_to_point': 'icp', 'point_to_plane': 'icp_plane', 'generalized': 'icp_generalized'}


class ICPBaseline:
  normal_radius_voxels = 2.0
  normal_max_nn = 30
  gicp_epsilon = 1e-3

  def __init__(self, dgr, method='point_to_plane', max_correspondence_distance=None, max_iteration=30, init=None):
    if method not in METHODS:
      raise ValueError(f'method must be one of {sorted(METHODS)}, got {method!r}')
    self.dgr = dgr
    self.method = method
    self.max_correspondence_distance = max_correspondence_distance
    self.max_iteration = int(max_iteration)
    self.init = np.eye(4) if init is None else np.asarray(init, dtype=np.float64).reshape(4, 4)
    self._check()
    self.reg_timer = Timer()
    self.last_branch = None
    self.last_info = {}

  @property
  def voxel_size(self):
    return self.dgr.voxel_size

  def _distance(self):
    d = self.max_correspondence_distance
    return 2.0 * self.voxel_size if d is None else float(d)

  def _check(self):
    d, vs = self._distance(), self.voxel_size
    if not 0.0 < d <= 4.0 * vs:
      raise ValueError(f'max_correspondence_distance must lie in (0, 4 voxels = {4 * vs}], got {d} (the voxel-hash '
                       'search reaches 4 cells)')
    if self.max_iteration < 0:
      raise ValueError(f'max_iteration must be >= 0, got {self.max_iteration}')

  def register(self, xyz0, xyz1):
    """-> 4x4 float64 ndarray mapping cloud 0 into cloud 1's frame."""
    self._check()
    d = self.dgr
    self.reg_timer.tic()
    _abi.refresh_stream()
    vs, dist = self.voxel_size, self._distance()
    with torch.no_grad():
      p0, c0, _ = d.preprocess(xyz0, 0, _batch=0)
      p1, c1, _ = d.preprocess(xyz1, 1, _batch=1)
      m = c1._dgr_manager
      T0 = torch.from_numpy(np.ascontiguousarray(self.init[:3])).to(p0.device)
      radius = self.normal_radius_voxels * vs
      if self.method == 'generalized':
        n0 = _abi.estimate_normals(p0, c0._dgr_manager, vs, radius, self.normal_max_nn, batch=0)
        n1 = _abi.estimate_normals(p1, m, vs, radius, self.normal_max_nn, batch=1)
        res = _abi.icp_generalized(p0, _abi.covariances_from_normals(n0, self.gicp_epsilon), p1,
                                   _abi.covariances_from_normals(n1, self.gicp_epsilon), m, vs, dist, T0,
                                   self.max_iteration, batch=1)
      elif self.method == 'point_to_plane':
        normals = _abi.estimate_normals(p1, m, vs, radius, self.normal_max_nn, batch=1)
        res = _abi.icp_point_to_plane(p0, p1, normals, m, vs, dist, T0, self.max_iteration, batch=1)
      else:
        res = _abi.icp_point_to_point(p0, p1, m, vs, dist, T0, self.max_iteration, batch=1)
      host = res.cpu().numpy()
    self.last_branch = METHODS[self.method]
    self.last_info = dict(n0=len(p0), n1=len(p1), icp_fitness=float(host[16]), icp_inlier_rmse=float(host[17]),
                          icp_iterations=int(host[18]), icp_correspondences=int(host[19]))
    d._log(f'=> ICP ({self.method}) takes {self.reg_timer.toc():.2} s')
    return host[:16].reshape(4, 4).copy()
