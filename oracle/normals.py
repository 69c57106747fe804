"""ORACLE (test infrastructure only) - normal estimation as the reference calls it:
``pcd.estimate_normals(o3d.geometry.KDTreeSearchParamHybrid(radius=2 * voxel, max_nn=30))`` (util/pointcloud.py:60;
radius 0.1 at scripts/test_3dmatch.py:72-73), i.e. open3d 0.10's EstimateNormals with a hybrid search.

PARITY UNPINNED: open3d is not installable offline, so this restates its published algorithm in float64 and pins
every boundary convention the GPU kernel (csrc/icp.cu, dgr_estimate_normals) follows:

* strict radius: neighbours of point i are the rows j with |p_j - p_i|^2 < radius^2 (nanoflann's radius search),
  i itself included; d^2 = (ex ex + ey ey) + ez ez of the offset e = p_j - p_i, evaluated in that order;
* tie order: when more than max_nn rows qualify, the max_nn smallest by (d^2, row index) are kept;
* covariance: the cumulant form open3d uses, E[e e^T] - mu mu^T, here over the offsets from p_i (the covariance does
  not depend on the origin; offsets keep the fp64 cancellation small);
* the normal is the eigenvector of the smallest eigenvalue; fewer than 3 neighbours, or a covariance that is
  exactly zero, give (0, 0, 1);
* sign, NOT open3d's (its eigen solver's sign is arbitrary): the largest-magnitude component is made positive (the
  first one on a tie);
* orientation against previous normals (open3d's rule when the cloud already has normals): a normal whose dot
  product with the previous one is negative is flipped.
"""
import numpy as np
from scipy.spatial import cKDTree


def neighbours(xyz, radius, max_nn):
  """-> (list of neighbour row arrays, ordered by (d^2, row) and truncated to max_nn; counts within the radius)."""
  xyz = np.asarray(xyz, np.float64)
  tree = cKDTree(xyz)
  r2 = float(radius) * float(radius)
  out, counts = [], np.zeros(len(xyz), np.int64)
  for i, cand in enumerate(tree.query_ball_point(xyz, r=float(radius) * (1 + 1e-9))):
    cand = np.asarray(cand, np.int64)
    e = xyz[cand] - xyz[i]
    d2 = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
    keep = d2 < r2
    cand, d2 = cand[keep], d2[keep]
    counts[i] = len(cand)
    order = np.lexsort((cand, d2))[:max_nn]
    out.append(cand[order])
  return out, counts


def estimate_normals(xyz, radius, max_nn, prev=None):
  """-> (normals float64 [n, 3], counts within the radius int [n], eigenvalues ascending float64 [n, 3]; zeros where
  the normal is the (0, 0, 1) default)."""
  xyz = np.asarray(xyz, np.float64)
  nbrs, counts = neighbours(xyz, radius, max_nn)
  normals = np.zeros((len(xyz), 3))
  eig = np.zeros((len(xyz), 3))
  for i, nb in enumerate(nbrs):
    n = np.array([0.0, 0.0, 1.0])
    if len(nb) >= 3:
      e = xyz[nb] - xyz[i]
      mu = e.sum(0) / len(nb)
      C = (e.T @ e) / len(nb) - np.outer(mu, mu)
      if np.any(C != 0.0):
        w, V = np.linalg.eigh(C)
        eig[i] = w
        n = V[:, 0].copy()
        big = int(np.argmax(np.abs(n)))
        if n[big] < 0:
          n = -n
    if prev is not None and float(n @ np.asarray(prev[i], np.float64)) < 0.0:
      n = -n
    normals[i] = n
  return normals, counts, eig
