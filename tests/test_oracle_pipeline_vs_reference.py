"""oracle/pipeline.py::register against the reference's OWN DeepGlobalRegistration.register():
core/deep_global_registration.py, core/knn.py, core/registration.py, model/*.py, util/*.py of the reference
run unmodified end to end on the CPU, with
* MinkowskiEngine  -> oracle/me_cpu.py (sparse operators of oracle/sparse_ops.py),
* open3d           -> the I/O stand-in of shims.py + registration_icp backed by oracle/icp.py,
recorded in tests/golden/reference_cpu.npz by tests/golden/make_golden_reference_cpu.py.
The sparse operators and ICP are therefore the oracle's on both sides; what this pins is everything
else the oracle restates by hand: the order of the stages, dtypes, voxelisation and re-flooring, the
6-D coordinate assembly, feature types, the sigmoid / clip / weight-sum gate and its thresholds, the
arguments handed to GlobalRegistration and to ICP."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import pipeline as op


@pytest.fixture(scope='module')
def ref():
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_cpu.npz'))


@pytest.mark.parametrize('feature_type,dtype', [('ones', np.float64), ('coords', np.float32)])
def test_reference_register_equals_oracle_pipeline(ref, feature_type, dtype):
  state = syn.make_checkpoint(1, inlier_feature_type=feature_type)
  xyz0, xyz1, _ = syn.room_pair(7, n_raw=5000, extent=(1.2, 1.0, 0.8))
  xyz0, xyz1 = xyz0.astype(dtype), xyz1.astype(dtype)
  g = lambda k: ref[f'pipe_{feature_type}_{k}']
  # the reference's register() ran with its default (use_icp = True); the pose it handed to open3d's ICP is tap A
  T_o, taps = op.register(state, xyz0, xyz1, clip_weight_thresh=0.05, use_icp=True)
  assert taps['branch'] == 'procrustes'
  assert f"=> Weighted sum {taps['wsum']:.2f} >=" in str(g('gate'))          # same gate value, same branch
  assert float(g('icp_max_dist')) == 2 * state['config']['voxel_size'] and int(g('icp_n_source')) == len(taps['coords0']) \
      and int(g('icp_n_target')) == len(taps['coords1'])
  te, re = syn.rte_rre(g('icp_init'), taps['T_refined'])                 # tap A: before ICP
  assert te <= 1e-3 and re <= 1e-3, (te, re, taps['refine'])
  te, re = syn.rte_rre(g('T'), T_o)                                      # tap B: the literal return value
  assert te <= 1e-3 and re <= 1e-3, (te, re, taps['icp'])
  # stage taps through the reference's own methods: preprocess(xyz0), fcgf_feature_extraction of its result
  p0, c0, F0 = g('p0'), g('c0'), g('F0')
  assert np.array_equal(c0, taps['coords0']) and np.array_equal(p0, taps['xyz0'])
  assert p0.dtype == np.float32 and c0.dtype == np.int32 and F0.shape == (len(c0), 32)
  assert float(np.abs(F0 - np.asarray(taps['feat0'])).max()) <= 1e-6


def test_public_surface_matches_the_reference_class(ref):
  """Same public methods with the same parameter names (and defaults where the reference has them) on
  deepglobalregistration_b200's DeepGlobalRegistration - the drop-in boundary of SURVEY.md 8(b)."""
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration as Ours
  ref_methods = json.loads(str(ref['surface']))
  assert set(ref_methods) == {'__init__', 'preprocess', 'fcgf_feature_extraction', 'fcgf_feature_matching',
                              'inlier_feature_generation', 'inlier_prediction', 'safeguard_registration', 'register'}
  for name, want in ref_methods.items():
    ours = getattr(Ours, name, None)
    assert ours is not None, f'missing method {name}'
    got = inspect.signature(ours).parameters
    public = [p for p in got if not p.startswith('_')]          # ours may add private keyword-only helpers
    assert public == [p for p, _ in want], (name, public, want)
    for p, default in want:
      if default is not None and name != '__init__':
        assert repr(got[p].default) == default, (name, p)
  assert str(inspect.signature(Ours.__init__).parameters['device'].default) == 'cuda'
