"""``Super4PCSBaseline``: Super4PCS (Mellado, Aiger & Mitra, SGP 2014), the ``Super4PCS`` row of the reference's
results, on the same voxelisation, GPU and evaluation protocol as ``DeepGlobalRegistration``.

    dgr = DeepGlobalRegistration(config)
    T = Super4PCSBaseline(dgr).register(xyz0, xyz1)

Voxelise both clouds (the wrapped object's ``preprocess``; no FCGF) -> source rows floor(k n0 / sample_size) for
k < sample_size (all of them when there are fewer) -> dgr_super4pcs against the whole target (its distance
transform, bases in rounds, congruent sets, LCP verification) -> one readback.  The congruence and LCP tolerance
``delta`` defaults to 2 voxels, the correspondence radius of the other baselines.  The reference's settings for its
Super4PCS row (overlap, delta, sample size, time budget) are not published; the defaults here are this project's.
"""
import numpy as np
import torch

from .. import _abi
from ..util.timer import Timer


class Super4PCSBaseline:
  def __init__(self, dgr, overlap=0.5, delta=None, sample_size=512, n_sample_tgt=None, angle_tol=0.0, dt_size=300,
               dt_expand=2.0, max_bases=256, bases_per_round=64, max_pairs=262144, max_candidates=65536,
               verify_per_base=64, terminate_fraction=0.9, seed=0):
    self.dgr = dgr
    self.delta = None if delta is None else float(delta)
    self.sample_size = int(sample_size)
    if not 4 <= self.sample_size <= 1024:
      raise ValueError(f'sample_size must lie in [4, 1024], got {sample_size}')
    self.n_sample_tgt = min(4096, 2 * self.sample_size) if n_sample_tgt is None else int(n_sample_tgt)
    self.search = dict(overlap=overlap, angle_tol=angle_tol, dt_size=dt_size, dt_expand=dt_expand,
                       max_bases=max_bases, bases_per_round=bases_per_round, max_pairs=max_pairs,
                       max_candidates=max_candidates, verify_per_base=verify_per_base,
                       terminate_fraction=terminate_fraction, seed=seed)
    self.reg_timer = Timer()
    self.last_branch = None
    self.last_info = {}

  def register(self, xyz0, xyz1):
    """-> 4x4 float64 ndarray mapping cloud 0 into cloud 1's frame."""
    d = self.dgr
    self.reg_timer.tic()
    _abi.refresh_stream()
    delta = 2.0 * d.voxel_size if self.delta is None else self.delta
    with torch.no_grad():
      p0, _, _ = d.preprocess(xyz0, 0, _batch=0)
      p1, _, _ = d.preprocess(xyz1, 1, _batch=1)
      n0 = len(p0)
      if n0 > self.sample_size:
        rows = torch.arange(self.sample_size, device=p0.device, dtype=torch.int64) * n0 // self.sample_size
        p0 = p0[rows]
      src = p0.to(torch.float32).contiguous()
      tgt = p1.to(torch.float32).contiguous()
      res = _abi.super4pcs(src, tgt, n_sample_tgt=min(self.n_sample_tgt, len(tgt)), delta=delta, **self.search)
      host = res.cpu().numpy()
    self.last_branch = 'super4pcs'
    self.last_info = dict(n0=n0, n_sample=len(src), n1=len(p1), n_sample_tgt=min(self.n_sample_tgt, len(tgt)),
                          delta=delta, **{k: float(v) for k, v in zip(_abi.SUPER4PCS_RESULT, host[16:28])})
    d._log(f'=> Super4PCS takes {self.reg_timer.toc():.2} s')
    return host[:16].reshape(4, 4).copy()
