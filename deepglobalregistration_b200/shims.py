"""Register the drop-in modules the reference imports by name.

    from deepglobalregistration_b200 import shims; shims.install()
    import MinkowskiEngine as ME          # -> deepglobalregistration_b200.me
    from easydict import EasyDict         # -> attribute dict (checkpoint configs unpickle)

    import open3d as o3d                  # -> only if the real one is missing: the few names
                                          #    demo.py needs (io.read_point_cloud, geometry.PointCloud,
                                          #    utility.Vector3dVector, visualization.draw_geometries)

After install() the reference's own ``model/resunet.py`` / ``model/residual_block.py`` /
``model/common.py`` import and run unchanged on top of libdgr_b200 (the plugin
boundary of SURVEY.md §8b).
"""
import sys
import types

from .synthetic import AttrDict


def install(force=False):
  from . import me
  if force or 'MinkowskiEngine' not in sys.modules:
    sys.modules['MinkowskiEngine'] = me
    sys.modules['MinkowskiEngine.MinkowskiFunctional'] = me.MinkowskiFunctional
    sys.modules['MinkowskiEngine.utils'] = me.utils
  if force or 'easydict' not in sys.modules:
    try:
      import easydict  # noqa: F401
    except ImportError:
      mod = types.ModuleType('easydict')
      mod.EasyDict = AttrDict
      sys.modules['easydict'] = mod
  if force or 'open3d' not in sys.modules:
    try:
      import open3d  # noqa: F401
    except ImportError:
      sys.modules['open3d'] = _open3d_stub()
  return me


def _open3d_stub():
  """The part of open3d the reference touches on the registration path: demo.py:10-48 (I/O, PointCloud, a no-op
  viewer, backed by io.py) and core/deep_global_registration.py:29-64,317-322 + util/pointcloud.py:15-23
  (pipelines.registration.registration_icp / registration_ransac_based_on_correspondence /
  registration_ransac_based_on_feature_matching, Feature, utility vectors; plus
  registration_fast_based_on_feature_matching / FastGlobalRegistrationOption / compute_fpfh_feature for FGR and
  FPFH users, the pose graph and global_optimization for multiway registration, and
  TransformationEstimationPointToPlane with geometry.KDTreeSearchParamHybrid for point-to-plane ICP users, and
  registration_colored_icp / TransformationEstimationForColoredICP for colored-ICP refinement,
  registration_generalized_icp / TransformationEstimationForGeneralizedICP / estimate_covariances and the six robust
  losses) backed
  by libdgr_b200 (o3d_registration.py), and what util/integration.py fuses RGB-D frames with
  (pipelines.integration.ScalableTSDFVolume, camera.PinholeCameraIntrinsic, geometry.Image / RGBDImage /
  TriangleMesh, io.read_image / write_triangle_mesh; o3d_integration.py) and poses raw frames with
  (pipelines.odometry.compute_rgbd_odometry; o3d_odometry.py) - so the reference's OWN
  DeepGlobalRegistration class, demo.py and util/integration.py run on this stack unmodified.  This package's
  DeepGlobalRegistration does not go through here: it calls the library."""
  import numpy as np

  from . import io as dio
  o3d = types.ModuleType('open3d')
  o3d.__dgr_stub__ = True
  o3d.io = types.ModuleType('open3d.io')
  o3d.io.read_point_cloud = dio.read_point_cloud
  o3d.io.write_point_cloud = lambda path, pcd, **kw: (dio.write_ply(path, pcd.points, dtype='double'), True)[1]
  o3d.geometry = types.ModuleType('open3d.geometry')
  o3d.geometry.PointCloud = dio.PointCloud
  o3d.utility = types.ModuleType('open3d.utility')
  o3d.utility.Vector3dVector = lambda a: np.asarray(a, dtype=np.float64).reshape(-1, 3)
  o3d.utility.Vector2iVector = lambda a: np.asarray(a, dtype=np.int32).reshape(-1, 2)
  from . import o3d_registration as reg
  o3d.pipelines = types.ModuleType('open3d.pipelines')
  o3d.pipelines.registration = types.ModuleType('open3d.pipelines.registration')
  for name in ('KDTreeSearchParamHybrid', 'KDTreeSearchParamKNN', 'KDTreeSearchParamRadius'):
    setattr(o3d.geometry, name, getattr(reg, name))
    setattr(o3d, name, getattr(reg, name))               # the pre-0.10 top-level path (util/pointcloud.py:60)
  for name in ('TransformationEstimationPointToPoint', 'TransformationEstimationPointToPlane', 'ICPConvergenceCriteria',
               'RANSACConvergenceCriteria',
               'CorrespondenceCheckerBasedOnDistance', 'CorrespondenceCheckerBasedOnEdgeLength', 'Feature',
               'RegistrationResult', 'registration_icp', 'registration_ransac_based_on_correspondence',
               'registration_ransac_based_on_feature_matching', 'FastGlobalRegistrationOption',
               'registration_fast_based_on_feature_matching', 'compute_fpfh_feature',
               'get_information_matrix_from_point_clouds', 'PoseGraph', 'PoseGraphNode', 'PoseGraphEdge',
               'GlobalOptimizationLevenbergMarquardt', 'GlobalOptimizationGaussNewton',
               'GlobalOptimizationConvergenceCriteria', 'GlobalOptimizationOption', 'global_optimization',
               'TransformationEstimationForColoredICP', 'registration_colored_icp',
               'TransformationEstimationForGeneralizedICP', 'registration_generalized_icp', 'estimate_covariances',
               'RobustKernel', 'L2Loss', 'L1Loss', 'HuberLoss', 'CauchyLoss', 'GMLoss', 'TukeyLoss'):
    setattr(o3d.pipelines.registration, name, getattr(reg, name))
  o3d.registration = o3d.pipelines.registration          # the pre-0.12 module path
  sys.modules['open3d.pipelines'] = o3d.pipelines
  sys.modules['open3d.pipelines.registration'] = o3d.pipelines.registration
  sys.modules['open3d.registration'] = o3d.pipelines.registration
  # RGB-D fusion (util/integration.py): pipelines.integration (integration before 0.12), camera, images, meshes
  from . import o3d_integration as integ
  o3d.pipelines.integration = types.ModuleType('open3d.pipelines.integration')
  for name in ('ScalableTSDFVolume', 'TSDFVolumeColorType'):
    setattr(o3d.pipelines.integration, name, getattr(integ, name))
  o3d.integration = o3d.pipelines.integration
  sys.modules['open3d.pipelines.integration'] = o3d.pipelines.integration
  sys.modules['open3d.integration'] = o3d.pipelines.integration
  # RGB-D odometry (make_fragments): pipelines.odometry (odometry before 0.12)
  from . import o3d_odometry as odo
  o3d.pipelines.odometry = types.ModuleType('open3d.pipelines.odometry')
  for name in ('OdometryOption', 'RGBDOdometryJacobianFromHybridTerm', 'RGBDOdometryJacobianFromColorTerm',
               'compute_rgbd_odometry'):
    setattr(o3d.pipelines.odometry, name, getattr(odo, name))
  o3d.odometry = o3d.pipelines.odometry
  sys.modules['open3d.pipelines.odometry'] = o3d.pipelines.odometry
  sys.modules['open3d.odometry'] = o3d.pipelines.odometry
  o3d.camera = types.ModuleType('open3d.camera')
  o3d.camera.PinholeCameraIntrinsic = integ.PinholeCameraIntrinsic
  sys.modules['open3d.camera'] = o3d.camera
  o3d.geometry.Image = dio.Image
  o3d.geometry.RGBDImage = integ.RGBDImage
  o3d.geometry.TriangleMesh = dio.TriangleMesh
  o3d.io.read_image = dio.read_image
  o3d.io.write_triangle_mesh = dio.write_triangle_mesh
  o3d.utility.VerbosityLevel = types.SimpleNamespace(Error=0, Warning=1, Info=2, Debug=3)
  o3d.utility.set_verbosity_level = lambda level: None
  o3d.visualization = types.ModuleType('open3d.visualization')

  def draw_geometries(geometries, *args, **kwargs):
    print('[open3d stub] draw_geometries: ' + ', '.join(repr(g) for g in geometries) + ' (no display)')
  o3d.visualization.draw_geometries = draw_geometries
  for sub in ('io', 'geometry', 'utility', 'visualization'):
    sys.modules['open3d.' + sub] = getattr(o3d, sub)
  return o3d
