"""``MultiwayRegistration``: a sequence of fragments into one consistent trajectory, with any pairwise method of this
package (DGR or a baseline) behind the pose-graph pipeline of Choi, Zhou & Koltun (*Robust reconstruction of indoor
scenes*, CVPR 2015) as open3d's reconstruction system runs it.

    method = DeepGlobalRegistration(config)          # or FPFHFastGlobal(dgr), FCGFRansac(dgr), ...
    poses, report = MultiwayRegistration(method).register_sequence(clouds)

Steps, each a method of its own:
  1. ``pairwise``: every pair i < j through ``sharding.register_pairs`` (so under torchrun too); register(i, j) maps
     fragment i into fragment j, which is edge (s = i, t = j, X).
  2. ``edges``: the information matrix of every pair on the voxelised fragments (dgr_information_matrix, radius
     ``info_radius_voxels`` voxels; each fragment's voxel hash built once).  Odometry edges (j = i + 1) are kept as
     certain; a loop closure is kept as uncertain when Lambda[5, 5] / min(n_i, n_j) >= ``overlap_thresh``.
  3. ``refine`` (only with ``refine='colored_icp'``): open3d's refine_registration / multiscale_icp on every kept
     edge (s, t): colored ICP of fragment s onto fragment t from the edge's pose at scales v, v / 2, v / 4 with 50, 30
     and 14 iterations (max_distance sigma, normals and colour gradients at radius 2 sigma with max_nn 30, hash cell
     sigma).  Each fragment is voxelised and its normals, intensities and gradients computed once per scale, shared by
     every edge.  The refined pose replaces the edge's and its information matrix is recomputed as in ``edges``; the
     edge selection is not redone.  DEPARTURE: a voxel keeps the colour of its first point (this package's
     voxelisation), where open3d's voxel_down_sample averages.
  4. ``optimise``: from the odometry chain P_0 = I, P_{i+1} = P_i X_{i,i+1}^-1, open3d's global_optimization
     (dgr_pose_graph_optimize) with reference node 0 and max_correspondence_distance = the information radius.
The information matrices, the refinement and the optimisation run on rank 0 after the gather: a scene fits one GPU.
Refinement needs coloured fragments: io.PointCloud objects with colours, or files that io.read_point_cloud reads with
colours (PLY red / green / blue).
"""
import time

import numpy as np
import torch

from .. import _abi
from .. import sharding


def odometry_chain(n, edges):
  """P_0 = I, P_{i+1} = P_i X_{i,i+1}^-1 from the odometry edges."""
  X = {(e['s'], e['t']): e['T'] for e in edges}
  P = [np.eye(4)]
  for i in range(n - 1):
    P.append(P[-1] @ np.linalg.inv(X[(i, i + 1)]))
  return np.stack(P)


def select_edges(edges, n_points, overlap_thresh):
  """Marks every edge dict: odometry edges certain and kept, loop closures kept (uncertain) when their overlap
  Lambda[5, 5] / min(n_s, n_t) reaches overlap_thresh.  Returns the kept edges in input order."""
  kept = []
  for e in edges:
    e['odometry'] = e['t'] == e['s'] + 1
    e['overlap'] = float(e['info'][5, 5]) / max(min(n_points[e['s']], n_points[e['t']]), 1)
    e['uncertain'] = not e['odometry']
    e['kept'] = e['odometry'] or e['overlap'] >= overlap_thresh
    if e['kept']:
      kept.append(e)
  return kept


REFINE_SCALES = (1.0, 0.5, 0.25)        # open3d's multiscale_icp: voxel, voxel / 2, voxel / 4
REFINE_ITERATIONS = (50, 30, 14)
REFINE_LAMBDA = 0.968                   # TransformationEstimationForColoredICP's default


def coloured_fragments(clouds):
  """(points float64 [n, 3], colours float64 [n, 3]) of every fragment: a path is read with io.read_point_cloud, an
  object needs ``points`` and ``colors``.  Raises ValueError, before any device work, for a fragment without colours."""
  from .. import io as dio
  out = []
  for k, c in enumerate(clouds):
    if isinstance(c, (str, bytes)) or hasattr(c, '__fspath__'):
      c = dio.read_point_cloud(str(c) if not isinstance(c, bytes) else c.decode())
    pts = np.asarray(getattr(c, 'points', c), dtype=np.float64).reshape(-1, 3)
    col = getattr(c, 'colors', None)
    if col is None or np.asarray(col).reshape(-1, 3).shape != pts.shape or len(pts) == 0:
      raise ValueError(f'fragment {k} has no colours: colored ICP refinement needs one colour per point')
    out.append((pts, np.asarray(col, dtype=np.float64).reshape(-1, 3)))
  return out


def absolute_trajectory_error(poses, gt):
  """RMS translation error after expressing both trajectories relative to node 0."""
  A = np.linalg.inv(poses[0]) @ poses
  G = np.linalg.inv(gt[0]) @ gt
  return float(np.sqrt(np.mean(np.sum((A[:, :3, 3] - G[:, :3, 3]) ** 2, axis=1))))


class MultiwayRegistration:

  def __init__(self, method, voxel_size=None, overlap_thresh=0.3, info_radius_voxels=2, refine=None):
    if refine not in (None, 'colored_icp'):
      raise ValueError(f"refine must be None or 'colored_icp', got {refine!r}")
    self.method = method
    self.refine = refine
    self.voxel_size = float(voxel_size if voxel_size is not None else method.voxel_size)
    self.overlap_thresh = float(overlap_thresh)
    self.info_radius_voxels = float(info_radius_voxels)
    if not self.voxel_size > 0.0:
      raise ValueError(f'voxel_size must be positive, got {self.voxel_size}')
    if not 0 < self.info_radius_voxels <= 4:
      raise ValueError(f'info_radius_voxels must lie in (0, 4], got {info_radius_voxels}')

  @property
  def info_radius(self):
    return self.info_radius_voxels * self.voxel_size

  @staticmethod
  def pair_list(n):
    return [(i, j) for i in range(n) for j in range(i + 1, n)]

  def pairwise(self, clouds, device=None):
    """-> (pairs [(i, j)], X [M, 4, 4] mapping i into j), identical on every rank."""
    pairs = self.pair_list(len(clouds))
    rows = sharding.register_pairs(self.method, [(clouds[i], clouds[j]) for i, j in pairs], device=device)
    return pairs, rows.numpy()[:, :16].reshape(-1, 4, 4).astype(np.float64)

  def _voxelised(self, cloud, dev):
    if isinstance(cloud, (str, bytes)) or hasattr(cloud, '__fspath__'):
      cloud = sharding._cloud(cloud)
    x64 = torch.from_numpy(np.ascontiguousarray(np.asarray(cloud, dtype=np.float64).reshape(-1, 3))).to(dev)
    raw, spec, table, sel, _, n = _abi.voxelise(x64, self.voxel_size)
    sel = sel.long()
    return _abi.float32_in_cells(x64[sel], raw[sel, 1:], self.voxel_size), (spec, table), n

  def edges(self, clouds, pairs, X, device='cuda'):
    """The information matrix of every pair (i, j) under X[k], on the voxelised fragments.
    -> (edge dicts (s, t, T, info), voxels per fragment)."""
    dev = _abi.require_device(device)
    _abi.refresh_stream()
    vox = [self._voxelised(c, dev) for c in clouds]
    out = []
    for (i, j), T in zip(pairs, X):
      src, (tgt, hash_t, _) = vox[i][0], vox[j]
      lam = _abi.information_matrix(src, tgt, hash_t, self.voxel_size, self.info_radius, T)
      out.append(dict(s=i, t=j, T=np.asarray(T, np.float64).reshape(4, 4), info_dev=lam))
    for e in out:                                       # one host read per edge, after every launch is queued
      e['info'] = e.pop('info_dev').cpu().numpy()[:36].reshape(6, 6).copy()
    return out, [v[2] for v in vox]

  def _colored_scale(self, pts, colors, sigma, dev):
    """One fragment at scale sigma: voxelised (first point per voxel), its hash at cell sigma, normals, intensities
    and colour gradients at radius 2 sigma, max_nn 30."""
    from ..o3d_registration import intensity
    x64 = torch.from_numpy(np.ascontiguousarray(pts)).to(dev)
    raw, spec, table, sel, _, _ = _abi.voxelise(x64, sigma)
    x = _abi.float32_in_cells(x64[sel.long()], raw[sel.long(), 1:], sigma)
    inten = torch.from_numpy(intensity(colors)).to(dev)[sel.long()].contiguous()
    nrm = _abi.estimate_normals(x, (spec, table), sigma, 2 * sigma, 30)
    grad = _abi.color_gradient(x, nrm, inten, (spec, table), sigma, 2 * sigma, 30)
    return x, inten, nrm, grad, (spec, table)

  def refine_edges(self, coloured, edges, device='cuda'):
    """Multi-scale colored ICP of every edge from its pose (open3d's multiscale_icp).  Each scale's launches are
    chained on the device (one scale's result seeds the next), with one host read per edge at the end.
    -> [(refined 4x4, fitness, inlier RMSE)] in edge order."""
    dev = _abi.require_device(device)
    _abi.refresh_stream()
    used = sorted({e[k] for e in edges for k in ('s', 't')})
    T = [torch.from_numpy(np.ascontiguousarray(np.asarray(e['T'], np.float64).reshape(4, 4)[:3])).to(dev)
         for e in edges]
    res = [None] * len(edges)
    for scale, iters in zip(REFINE_SCALES, REFINE_ITERATIONS):
      sigma = self.voxel_size * scale
      frag = {k: self._colored_scale(*coloured[k], sigma, dev) for k in used}
      for m, e in enumerate(edges):
        src, i_src = frag[e['s']][:2]
        tgt, i_tgt, nrm, grad, hashed = frag[e['t']]
        res[m] = _abi.icp_colored(src, i_src, tgt, nrm, i_tgt, grad, hashed, sigma, sigma, REFINE_LAMBDA, T[m],
                                  max_iter=iters)
        T[m] = res[m][:12]
    out = []
    for r in res:
      r = r.cpu().numpy()
      out.append((r[:16].reshape(4, 4).copy(), float(r[16]), float(r[17])))
    return out

  def optimise(self, n, edges, reference_node=0):
    """open3d's global_optimization over the kept edges from the odometry chain.
    -> (poses [n, 4, 4], kept-after-pruning [len(edges)] bool, line process [len(edges)], stats)."""
    P0 = odometry_chain(n, edges)
    if not edges:
      return P0, np.zeros(0, bool), np.zeros(0), {}
    return _abi.pose_graph_optimize(
        P0, [(e['s'], e['t']) for e in edges], np.stack([e['T'] for e in edges]),
        np.stack([e['info'] for e in edges]), [e['uncertain'] for e in edges], [1.0] * len(edges),
        max_correspondence_distance=self.info_radius, reference_node=reference_node)

  def register_sequence(self, clouds, device=None):
    """-> (poses [N, 4, 4] mapping each fragment into fragment 0's frame, report); on ranks other than 0 of a
    process group the poses are None (the pairwise results are gathered, the graph is solved on rank 0)."""
    n = len(clouds)
    if n < 2:
      raise ValueError('multiway registration needs at least two fragments')
    coloured = None
    if self.refine is not None:
      coloured = coloured_fragments(clouds)
      clouds = [c[0] for c in coloured]
    t0 = time.perf_counter()
    pairs, X = self.pairwise(clouds, device=device)
    t1 = time.perf_counter()
    report = dict(n_fragments=n, pairs=len(pairs), pairwise_poses=X, seconds=dict(pairwise=t1 - t0))
    rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
    if rank != 0:
      return None, report
    edges, n_points = self.edges(clouds, pairs, X, device=device if device is not None else 'cuda')
    kept = select_edges(edges, n_points, self.overlap_thresh)
    t2 = time.perf_counter()
    if coloured is not None and kept:
      dev = device if device is not None else 'cuda'
      refined = self.refine_edges(coloured, kept, device=dev)
      infos, _ = self.edges(clouds, [(e['s'], e['t']) for e in kept], [r[0] for r in refined], device=dev)
      for e, (T, fit, rmse), f in zip(kept, refined, infos):
        e['T_pairwise'], e['T'], e['info'] = e['T'], T, f['info']
        e['refine_fitness'], e['refine_rmse'] = fit, rmse
      report['seconds']['refine'] = time.perf_counter() - t2
      t2 = time.perf_counter()
    poses, alive, lp, stats = self.optimise(n, kept)
    t3 = time.perf_counter()
    for e in edges:
      e['pruned'], e['line_process'] = False, None
    for e, a, l in zip(kept, alive, lp):
      e['pruned'], e['line_process'] = not bool(a), float(l)
    report.update(
        n_points=n_points, edges=edges, optimiser=stats,
        odometry=sum(e['odometry'] for e in edges), loop_candidates=sum(not e['odometry'] for e in edges),
        kept=len(kept), pruned=sum(e['pruned'] for e in edges))
    report['seconds'].update(information=t2 - t1 - report['seconds'].get('refine', 0.0), optimise=t3 - t2,
                             total=t3 - t0)
    return poses, report
