"""``GoICPBaseline``: Go-ICP (Yang, Li, Campbell & Jia, TPAMI 2016), the ``Go-ICP`` row of the reference's results, on
the same voxelisation, GPU and evaluation protocol as ``DeepGlobalRegistration``.

    dgr = DeepGlobalRegistration(config)
    T = GoICPBaseline(dgr).register(xyz0, xyz1)

Voxelise both clouds (the wrapped object's ``preprocess``; no FCGF) -> source rows floor(k n0 / n_data) for
k < n_data (all of them when there are fewer) -> dgr_goicp against the whole target (its distance transform,
branch and bound over rotation and translation cubes, trimmed ICP for incumbents) -> one readback.  The search runs
in the normalised frame (both clouds centred, divided by the larger largest centred norm), so the default
translation cube [-1, 1]^3 covers every offset of the two centres.
"""
import math

import numpy as np
import torch

from .. import _abi
from ..util.timer import Timer


class GoICPBaseline:
  def __init__(self, dgr, mse_thresh=1e-3, trim_fraction=0.0, n_data=1000, dt_size=300, dt_expand=2.0,
               rot_min=(-math.pi,) * 3, rot_width=2 * math.pi, trans_min=(-1.0,) * 3, trans_width=2.0,
               cubes_per_round=64, max_rounds=100000, max_rotation_cubes=1 << 20):
    self.dgr = dgr
    self.mse_thresh, self.trim_fraction = float(mse_thresh), float(trim_fraction)
    self.n_data = int(n_data)
    if not 1 <= self.n_data <= 1024:
      raise ValueError(f'n_data must lie in [1, 1024], got {n_data}')
    self.search = dict(mse_thresh=self.mse_thresh, trim_fraction=self.trim_fraction, dt_size=dt_size,
                       dt_expand=dt_expand, rot_min=rot_min, rot_width=rot_width, trans_min=trans_min,
                       trans_width=trans_width, cubes_per_round=cubes_per_round, max_rounds=max_rounds,
                       max_rotation_cubes=max_rotation_cubes)
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
      n0 = len(p0)
      if n0 > self.n_data:
        rows = torch.arange(self.n_data, device=p0.device, dtype=torch.int64) * n0 // self.n_data
        p0 = p0[rows]
      src = p0.to(torch.float32).contiguous()
      res = _abi.goicp(src, p1.to(torch.float32).contiguous(), **self.search)
      host = res.cpu().numpy()
    self.last_branch = 'goicp'
    self.last_info = dict(n0=n0, n_data=len(src), n1=len(p1),
                          **{k: float(v) for k, v in zip(_abi.GOICP_RESULT, host[16:29])})
    d._log(f'=> Go-ICP takes {self.reg_timer.toc():.2} s')
    return host[:16].reshape(4, 4).copy()
