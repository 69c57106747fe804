"""``FPFHRansac`` / ``FPFHFastGlobal``: FPFH + RANSAC and FPFH + FGR, the classical global registrations that need no
trained network, on the same voxelisation, GPU and evaluation protocol as ``DeepGlobalRegistration``.

    dgr = DeepGlobalRegistration(config)
    T = FPFHRansac(dgr).register(xyz0, xyz1)

open3d's global-registration recipe with DGR's own voxelisation: voxelise both clouds (the wrapped object's
``preprocess`` and ``voxel_size``) -> normals of each cloud from neighbours within 2 voxels, at most 30
(dgr_estimate_normals) -> FPFH from neighbours within 5 voxels, at most 100 (dgr_compute_fpfh, rows padded to 64
columns for the tensor-core kNN), each cloud through its own voxel table -> the search of ``FCGFRansac`` /
``FCGFFastGlobal`` with its settings -> optionally point-to-point ICP.  Only the descriptor differs from the FCGF
rows.
"""
from .. import _abi
from .fcgf_fgr import FCGFFastGlobal
from .fcgf_ransac import FCGFRansac


class _FPFHFeatures:
  normal_radius_voxels = 2.0
  normal_max_nn = 30
  feature_radius_voxels = 5.0
  feature_max_nn = 100
  feature_ld = 64          # 33 FPFH columns + zeros: the channel count dgr_knn_top1_tc takes

  def _features(self, p0, p1, c0, c1):
    vs = self.voxel_size
    out = []
    for batch, (p, c) in enumerate(((p0, c0), (p1, c1))):
      m = c._dgr_manager
      normals = _abi.estimate_normals(p, m, vs, self.normal_radius_voxels * vs, self.normal_max_nn, batch=batch)
      out.append(_abi.compute_fpfh(p, normals, m, vs, self.feature_radius_voxels * vs, self.feature_max_nn,
                                   batch=batch, ld=self.feature_ld))
    return out


class FPFHRansac(_FPFHFeatures, FCGFRansac):
  label = 'FPFH + RANSAC'


class FPFHFastGlobal(_FPFHFeatures, FCGFFastGlobal):
  label = 'FPFH + FGR'
