"""``PointNetLKBaseline``: PointNetLK (Aoki, Goforth, Srivatsan & Lucey, CVPR 2019), the ``PointNetLK`` row of the
reference's results, on the same voxelisation, GPU and evaluation protocol as ``DeepGlobalRegistration``.

    dgr = DeepGlobalRegistration(config)
    T = PointNetLKBaseline(dgr, 'pointnetlk.pth').register(xyz0, xyz1)

Voxelise both clouds (the wrapped object's ``preprocess``; no FCGF), keep every voxel -> dgr_pointnetlk (a 7-pose
forward for the Jacobian at the target, then the Lucas-Kanade loop on the source) -> one readback.  The weights are
packed once, at construction.  ``delta`` 1e-2, ``xtol`` 1e-7 and ``max_iter`` 10 are the defaults of the authors'
released code as remembered (whether its iteration cap is 10 or 20 cannot be checked offline).
"""
import numpy as np
import torch

from .. import _abi
from ..util.timer import Timer

WIDTHS = ((3, 64), (64, 64), (64, 64), (64, 128), (128, 1024))
# (conv, BatchNorm) module names of the published ``PointNet_features`` (h1 = Sequential(Conv1d, BN, ReLU, Conv1d, BN,
# ReLU), h2 the same with three layers)
MODULES = (('h1.0', 'h1.1'), ('h1.3', 'h1.4'), ('h2.0', 'h2.1'), ('h2.3', 'h2.4'), ('h2.6', 'h2.7'))
PREFIXES = ('module.', 'ptnet.')
IGNORED = ('dt',)                  # PointLK's learnable twist step: the call takes delta as an argument


def expected_keys():
  """{key: shape} of a PointNet_features state dict (``*.num_batches_tracked`` is accepted and ignored)."""
  keys = {}
  for (conv, bn), (cin, cout) in zip(MODULES, WIDTHS):
    keys[conv + '.weight'] = (cout, cin, 1)
    keys[conv + '.bias'] = (cout,)
    for k in ('weight', 'bias', 'running_mean', 'running_var'):
      keys[f'{bn}.{k}'] = (cout,)
  return keys


def load_pointnet_weights(weights):
  """Parameters of a PointNetLK feature network, fp64 in ``dgr_pointnet_pack``'s order (per layer W [cout][cin],
  conv bias, BN weight, BN bias, running mean, running var).

  ``weights``: a path (``torch.load``) or a state dict in the published ``PointNet_features`` layout, optionally under
  ``ptnet.`` and / or ``module.`` prefixes (a whole PointLK state dict also carries ``dt``, ignored).  Expected keys
  (Conv1d(cin, cout, 1) then BatchNorm1d(cout), ReLU between them in the Sequential):

      h1.0.weight [64, 3, 1]     h1.0.bias [64]      h1.1.{weight, bias, running_mean, running_var} [64]
      h1.3.weight [64, 64, 1]    h1.3.bias [64]      h1.4.{...} [64]
      h2.0.weight [64, 64, 1]    h2.0.bias [64]      h2.1.{...} [64]
      h2.3.weight [128, 64, 1]   h2.3.bias [128]     h2.4.{...} [128]
      h2.6.weight [1024, 128, 1] h2.6.bias [1024]    h2.7.{...} [1024]

  These names are the published code's as remembered; they cannot be checked offline.  Raises ValueError naming
  every missing, unexpected or mis-shaped key: the architecture is fixed."""
  sd = torch.load(weights, map_location='cpu', weights_only=False) if not isinstance(weights, dict) else weights
  if 'state_dict' in sd and isinstance(sd['state_dict'], dict):
    sd = sd['state_dict']
  clean = {}
  for k, v in sd.items():
    name = k
    changed = True
    while changed:
      changed = False
      for p in PREFIXES:
        if name.startswith(p):
          name, changed = name[len(p):], True
    clean[name] = v
  want = expected_keys()
  missing = sorted(k for k in want if k not in clean)
  unexpected = sorted(k for k in clean if k not in want and k not in IGNORED and not k.endswith('.num_batches_tracked'))
  shaped = sorted(f'{k} {tuple(clean[k].shape)} (expected {want[k]})' for k in want
                  if k in clean and tuple(clean[k].shape) != want[k])
  if missing or unexpected or shaped:
    raise ValueError(f'not a PointNetLK feature network: missing {missing}, unexpected {unexpected}, '
                     f'mis-shaped {shaped}')
  parts = []
  for (conv, bn), (cin, cout) in zip(MODULES, WIDTHS):
    parts.append(torch.as_tensor(clean[conv + '.weight'], dtype=torch.float64).reshape(-1))
    parts.append(torch.as_tensor(clean[conv + '.bias'], dtype=torch.float64))
    for k in ('weight', 'bias', 'running_mean', 'running_var'):
      parts.append(torch.as_tensor(clean[f'{bn}.{k}'], dtype=torch.float64))
  return torch.cat(parts).numpy()


class PointNetLKBaseline:
  def __init__(self, dgr, weights, delta=1e-2, max_iter=10, xtol=1e-7):
    self.dgr = dgr
    self.delta, self.max_iter, self.xtol = float(delta), int(max_iter), float(xtol)
    params = torch.as_tensor(load_pointnet_weights(weights), device=dgr.device)
    self.packed = _abi.pointnet_pack(params)
    self.reg_timer = Timer()
    self.last_branch = None
    self.last_info = {}

  def register(self, xyz0, xyz1):
    """-> 4x4 float64 ndarray mapping cloud 0 into cloud 1's frame."""
    d = self.dgr
    self.reg_timer.tic()
    _abi.refresh_stream()
    with torch.no_grad():
      p0, _, _ = d.preprocess(xyz0, 0, _batch=0)
      p1, _, _ = d.preprocess(xyz1, 1, _batch=1)
      src = p0.to(torch.float32).contiguous()
      tgt = p1.to(torch.float32).contiguous()
      res = _abi.pointnetlk(src, tgt, self.packed, delta=self.delta, max_iter=self.max_iter, xtol=self.xtol)
      host = res.cpu().numpy()
    self.last_branch = 'pointnetlk'
    self.last_info = dict(delta=self.delta, max_iter=self.max_iter, xtol=self.xtol,
                          **{k: float(v) for k, v in zip(_abi.POINTNETLK_RESULT, host[16:23])})
    d._log(f'=> PointNetLK takes {self.reg_timer.toc():.2} s')
    return host[:16].reshape(4, 4).copy()
