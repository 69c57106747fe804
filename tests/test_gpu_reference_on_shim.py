"""Boundary b2 (SURVEY 8b): the open3d stand-in's registration pipeline (o3d_registration.py: registration_icp /
registration_ransac_based_on_correspondence behind `open3d.pipelines.registration`) called the way
core/deep_global_registration.py:50-64,317-322 and util/pointcloud.py:15-23 of the reference call open3d, against
the library entry points and the oracle."""
import sys
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
EXTENT = (1.8, 1.5, 1.25)


@pytest.fixture(scope='module')
def setup():
  from deepglobalregistration_b200 import _abi, shims
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  _abi.require_device('cuda')
  state = syn.make_checkpoint(0)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False))
  saved = sys.modules.pop('open3d', None)
  o3d = shims._open3d_stub()
  if saved is not None:
    sys.modules['open3d'] = saved
  return d, state, o3d, _abi


def _pcd(o3d, xyz_t):
  """util/pointcloud.py:15-23 make_open3d_point_cloud"""
  pcd = o3d.geometry.PointCloud()
  pcd.points = o3d.utility.Vector3dVector(xyz_t.cpu().detach().numpy())
  return pcd


def test_standin_icp_equals_library_and_oracle(setup):
  from oracle import icp as oicp
  d, state, o3d, abi = setup
  xyz0, xyz1, T_gt = syn.room_pair(4, n_raw=20000, extent=EXTENT)
  with torch.no_grad():
    p0, c0, _ = d.preprocess(xyz0, 0, _batch=0)
    p1, c1, _ = d.preprocess(xyz1, 1, _batch=0)
  T0 = T_gt.copy()
  T0[:3, 3] += 0.02                                        # a perturbed start, as after the refinement
  # the reference's call (core/deep_global_registration.py:317-322)
  res = o3d.pipelines.registration.registration_icp(source=_pcd(o3d, p0), target=_pcd(o3d, p1),
                                                    max_correspondence_distance=d.voxel_size * 2, init=T0)
  lib = abi.icp_point_to_point(p0, p1, c1._dgr_manager, d.voxel_size, 2 * d.voxel_size, T0, batch=0).cpu().numpy()
  assert np.allclose(res.transformation, lib[:16].reshape(4, 4), atol=1e-9)
  assert abs(res.fitness - lib[16]) < 1e-12 and abs(res.inlier_rmse - lib[17]) < 1e-12
  T_o, info = oicp.icp_point_to_point(p0.cpu().numpy(), p1.cpu().numpy(), 2 * d.voxel_size, T0)
  te, re = syn.rte_rre(res.transformation, T_o)
  assert te <= 1e-5 and re <= 1e-5, (te, re)
  assert abs(res.fitness - info['fitness']) <= 1e-9 and len(res.correspondence_set) == info['n_corr']
  # a target that is NOT voxelised (several raw points within a quarter of the search radius): refused loudly
  dense = torch.from_numpy(xyz1[:30000]).float().cuda()
  with pytest.raises(NotImplementedError):
    o3d.pipelines.registration.registration_icp(_pcd(o3d, p0), _pcd(o3d, dense), 0.04, T0)


def test_standin_ransac_equals_library(setup):
  d, state, o3d, abi = setup
  P, Q, idx0, idx1, T_gt, inl = syn.correspondence_set(3, n=3000)
  corres = o3d.utility.Vector2iVector(np.stack((idx0, idx1), axis=1))       # :52-53
  res = o3d.pipelines.registration.registration_ransac_based_on_correspondence(
      source=_pcd(o3d, torch.from_numpy(P)), target=_pcd(o3d, torch.from_numpy(Q)), corres=corres,
      max_correspondence_distance=0.1,
      estimation_method=o3d.pipelines.registration.TransformationEstimationPointToPoint(False), ransac_n=4,
      criteria=o3d.pipelines.registration.RANSACConvergenceCriteria(50000, 80000))
  lib = abi.ransac_correspondence(torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda(),
                                  torch.from_numpy(idx0.astype(np.int32)).cuda(),
                                  torch.from_numpy(idx1.astype(np.int32)).cuda(), 0.1, num_hyp=50000, seed=0).cpu().numpy()
  assert np.allclose(res.transformation, lib[:16].reshape(4, 4), atol=1e-12)
  te, re = syn.rte_rre(res.transformation, T_gt)
  assert te <= 0.02 and re <= 0.02 and res.fitness > 0.25
