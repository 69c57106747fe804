"""``FCGFFastGlobal``: FCGF + Fast Global Registration (the ``FGR`` row of the reference's results) on the same
checkpoint, GPU and evaluation protocol as ``DeepGlobalRegistration``.

    dgr = DeepGlobalRegistration(config)
    method = FCGFFastGlobal(dgr)
    method.option.tuple_scale = 0.9          # open3d's FastGlobalRegistrationOption fields
    T = method.register(xyz0, xyz1)

Voxelise both clouds -> FCGF features of both in one pass -> nearest feature in both directions (dgr_knn_top1) ->
FGR (dgr_fgr_feature_matching: mutual matches, tuple test, graduated non-convexity) -> optionally point-to-point
ICP (the wrapped object's ``use_icp``) -> one readback.  FGR runs on the checkpoint's FCGF features, as the
RANSAC baseline does.
"""
from .. import _abi
from ..o3d_registration import FastGlobalRegistrationOption, _fgr_option_check
from .fcgf_ransac import FCGFBaseline


class FCGFFastGlobal(FCGFBaseline):
  branch = 'fgr'
  label = 'FCGF + FGR'

  def __init__(self, dgr):
    super().__init__(dgr)
    self.option = FastGlobalRegistrationOption()

  def _search(self, p0, p1, f0, f1, manager1):
    o = self.option
    _fgr_option_check(o)
    return _abi.fgr_feature_matching(p0, p1, _abi.knn_top1(f0, f1), _abi.knn_top1(f1, f0), o.division_factor,
                                     o.use_absolute_scale, o.decrease_mu, o.maximum_correspondence_distance,
                                     o.iteration_number, o.tuple_scale, o.maximum_tuple_count, o.tuple_test,
                                     seed=o.seed)

  def _info(self, res):
    return dict(fgr_mutual=int(res[16]), fgr_correspondences=int(res[17]), fgr_trials=int(res[18]),
                fgr_mu=float(res[19]), fgr_ran=bool(res[20]), fgr_swapped=bool(res[21]))
