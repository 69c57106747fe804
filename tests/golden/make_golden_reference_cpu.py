"""Generate tests/golden/reference_cpu.npz by running the UNMODIFIED reference (chrischoy/DeepGlobalRegistration,
checked out at REF) on the CPU over oracle/me_cpu.py (MinkowskiEngine) and the open3d stand-in of shims.py with
ICP backed by oracle/icp.py - the setups of tests/test_oracle_graph_vs_reference.py and
tests/test_oracle_pipeline_vs_reference.py, which compare the oracle against what is stored here:

  graph_<i>                      ResUNetBN2C forward of the reference's model/*.py, case i of the graph test
  pipe_<tag>_T                   register() return value (use_icp = True)
  pipe_<tag>_icp_init, _icp_max_dist, _icp_n_source, _icp_n_target   what register() handed to open3d's ICP
  pipe_<tag>_gate                the weight-sum line register() printed
  pipe_<tag>_p0, _c0, _F0        preprocess(xyz0) and fcgf_feature_extraction of its result
  surface                        JSON: public methods of DeepGlobalRegistration -> [(parameter, default repr)]

    python tests/golden/make_golden_reference_cpu.py /path/to/DeepGlobalRegistration
"""
import contextlib
import inspect
import io
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from deepglobalregistration_b200 import shims  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402
from oracle import icp as oicp  # noqa: E402
from oracle import me_cpu  # noqa: E402

GRAPH_CASES = [(3, 1, 32, 7, True, 600, 7), (3, 1, 32, 5, True, 500, 9), (6, 1, 1, 3, False, 300, 2),
               (6, 6, 1, 3, False, 250, 2)]
PIPE_CASES = [('ones', np.float64), ('coords', np.float32)]


def graph_cloud(seed, n, D, extent):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-extent, extent, size=(n, D)), axis=0)
  return np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)


def graph_inputs(D, cin, cout, k1, n, extent):
  """State dict, coordinates and features of one graph case (shared with the test)."""
  sd = syn.resunet_state_dict(D + k1, cin, cout, k1, D)
  g = torch.Generator().manual_seed(1)
  for k in sd:                                  # non-trivial BN statistics so a misplaced norm shows
    if k.endswith('running_mean'):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
    if k.endswith('bn.bias'):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
  coords = graph_cloud(D, n, D, extent)
  feats = torch.ones(len(coords), cin) if cin == 1 else torch.randn(len(coords), cin, generator=g)
  return sd, coords, feats


def pipe_inputs(feature_type, dtype):
  state = syn.make_checkpoint(1, inlier_feature_type=feature_type)
  xyz0, xyz1, _ = syn.room_pair(7, n_raw=5000, extent=(1.2, 1.0, 0.8))
  return state, xyz0.astype(dtype), xyz1.astype(dtype)


def main(ref):
  out = {}
  restore_me = me_cpu.install()
  sys.path.insert(0, ref)
  try:
    from model import load_model
    for i, (D, cin, cout, k1, normalize, n, extent) in enumerate(GRAPH_CASES):
      sd, coords, feats = graph_inputs(D, cin, cout, k1, n, extent)
      net = load_model('ResUNetBN2C')(cin, cout, bn_momentum=0.05, conv1_kernel_size=k1, normalize_feature=normalize, D=D)
      net.load_state_dict(sd, strict=True)
      net.eval()
      import MinkowskiEngine as ME
      with torch.no_grad():
        out[f'graph_{i}'] = net(ME.SparseTensor(feats, coordinates=coords)).F.numpy()

    o3d = shims._open3d_stub()
    o3d.pipelines = types.ModuleType('open3d.pipelines')
    o3d.pipelines.registration = types.ModuleType('open3d.pipelines.registration')
    icp_calls = []

    def registration_icp(source, target, max_correspondence_distance, init=np.eye(4), *a, **k):
      icp_calls.append(dict(init=np.array(init), max_dist=max_correspondence_distance, n_source=len(source.points),
                            n_target=len(target.points)))
      T, info = oicp.icp_point_to_point(np.asarray(source.points), np.asarray(target.points),
                                        max_correspondence_distance, init)
      return types.SimpleNamespace(transformation=T, fitness=info['fitness'], inlier_rmse=info['inlier_rmse'])
    o3d.pipelines.registration.registration_icp = registration_icp
    sys.modules['open3d'] = o3d
    preloaded = {}
    real_load = torch.load
    torch.load = lambda f, *a, **k: preloaded[str(f)] if str(f) in preloaded else real_load(f, *a, **k)
    from core.deep_global_registration import DeepGlobalRegistration
    ckpt = os.path.join(tempfile.mkdtemp(), 'ckpt.pth')     # register() asserts the path exists
    open(ckpt, 'wb').close()
    for feature_type, dtype in PIPE_CASES:
      tag = feature_type
      state, xyz0, xyz1 = pipe_inputs(feature_type, dtype)
      preloaded[ckpt] = state
      dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=ckpt, clip_weight_thresh=0.05),
                                   device=torch.device('cpu'))
      icp_calls.clear()
      buf = io.StringIO()
      with contextlib.redirect_stdout(buf):
        T = dgr.register(xyz0, xyz1)
      call, = icp_calls
      out[f'pipe_{tag}_T'] = np.asarray(T, np.float64)
      out[f'pipe_{tag}_icp_init'] = call['init']
      out[f'pipe_{tag}_icp_max_dist'] = np.float64(call['max_dist'])
      out[f'pipe_{tag}_icp_n_source'] = np.int64(call['n_source'])
      out[f'pipe_{tag}_icp_n_target'] = np.int64(call['n_target'])
      out[f'pipe_{tag}_gate'] = np.array([ln for ln in buf.getvalue().splitlines() if 'Weighted sum' in ln][0])
      p0, c0, f0 = dgr.preprocess(xyz0)
      with torch.no_grad():
        F0 = dgr.fcgf_feature_extraction(f0, c0)
      out[f'pipe_{tag}_p0'], out[f'pipe_{tag}_c0'], out[f'pipe_{tag}_F0'] = p0.numpy(), c0.numpy(), F0.numpy()
    surface = {n: [(p, repr(q.default) if q.default is not inspect.Parameter.empty else None)
                   for p, q in inspect.signature(f).parameters.items()]
               for n, f in inspect.getmembers(DeepGlobalRegistration, inspect.isfunction)
               if not n.startswith('_') or n == '__init__'}
    out['surface'] = np.array(json.dumps(surface, sort_keys=True))
  finally:
    sys.path.remove(ref)
    restore_me()
  np.savez_compressed(os.path.join(HERE, 'reference_cpu.npz'), **out)


if __name__ == '__main__':
  main(sys.argv[1])
