"""Pair sharding across the GPUs of one box (SURVEY.md §8e).

Scan pairs are independent (the reference's evaluation loops are per pair,
scripts/test_3dmatch.py:99-127, scripts/test_kitti.py:67-84), so the path shards with no
data-path collective: every rank holds a replica of both checkpoints and registers pairs
rank, rank + W, ...; the only exchange is one all-gather of the per-pair results
([4x4 pose, weight sum, iterations, branch, milliseconds] = 20 float64: the pose keeps the
precision register() returns) at the end - NCCL over
NVLink on GPUs, gloo in the CPU tests."""
import time

import numpy as np
import torch
import torch.distributed as dist

RESULT_WIDTH = 20
BRANCH_CODE = {'procrustes': 0.0, 'safeguard': 1.0, 'ransac': 2.0, 'fgr': 3.0, 'icp': 4.0, 'icp_plane': 5.0,
               'goicp': 6.0, 'super4pcs': 7.0, 'pointnetlk': 8.0, 'icp_generalized': 9.0, None: -1.0}


def shard_indices(n_pairs, rank, world):
  """Round-robin ownership: pair i belongs to rank i % world."""
  return list(range(rank, n_pairs, world))


def pack_result(T, wsum=0.0, iterations=0, branch=None, ms=0.0):
  row = np.zeros(RESULT_WIDTH, np.float64)
  row[:16] = np.asarray(T, np.float64).reshape(16)
  row[16:] = (wsum, iterations, BRANCH_CODE.get(branch, -1.0), ms)
  return row


def gather_results(local_rows, n_pairs, device=None):
  """All-gather the per-rank result rows and return them in pair order [n_pairs, 20].
  Works without an initialised process group (world size 1)."""
  world = dist.get_world_size() if dist.is_initialized() else 1
  rank = dist.get_rank() if dist.is_initialized() else 0
  per_rank = (n_pairs + world - 1) // world
  buf = torch.zeros(per_rank, RESULT_WIDTH, dtype=torch.float64)
  mine = shard_indices(n_pairs, rank, world)
  if len(mine):
    buf[:len(mine)] = torch.from_numpy(np.stack(local_rows).astype(np.float64))
  if device is not None:
    buf = buf.to(device)
  if world > 1:
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf)
  else:
    parts = [buf]
  out = torch.zeros(n_pairs, RESULT_WIDTH, dtype=torch.float64)
  for r, part in enumerate(parts):
    idx = shard_indices(n_pairs, r, world)
    out[idx] = part[:len(idx)].cpu()
  return out


def _cloud(item):
  """A pair member is an array / tensor / point-cloud object, or the path of a file to read when
  its turn comes (so a rank only ever loads its own share)."""
  if isinstance(item, (str, bytes)) or hasattr(item, '__fspath__'):
    from . import io as dio
    return dio.read_points(str(item) if not isinstance(item, bytes) else item.decode())
  return item


def register_pairs(dgr, pairs, device=None, inflight=4):
  """Register this rank's share of `pairs` ([(xyz0, xyz1), ...]; members may be file paths) with
  `dgr` and gather all results.  Returns [len(pairs), 20] float64, identical on every rank.  With a
  DeepGlobalRegistration that has register_batch, `inflight` pairs are kept in flight on the GPU (one host
  thread, stream and arena each); file members are read by the worker that registers them, so a rank only
  ever loads its own share.  The milliseconds column is the time between consecutive completions on this
  rank (its inverse is the rank's throughput), file reads included."""
  world = dist.get_world_size() if dist.is_initialized() else 1
  rank = dist.get_rank() if dist.is_initialized() else 0
  mine = shard_indices(len(pairs), rank, world)
  rows = []
  if hasattr(dgr, 'register_batch'):
    t0 = time.perf_counter()
    out = dgr.register_batch([(lambda i=i: (_cloud(pairs[i][0]), _cloud(pairs[i][1]))) for i in mine],
                             inflight=inflight)
    done = sorted(info.get('t_done', t0) for _, _, info in out)
    gaps = dict(zip(done, np.diff([t0] + done))) if done else {}
    for T, branch, info in out:
      rows.append(pack_result(T, info.get('wsum', 0.0), info.get('iterations', 0), branch,
                              1e3 * gaps.get(info.get('t_done'), 0.0)))
  else:
    for i in mine:
      xyz0, xyz1 = _cloud(pairs[i][0]), _cloud(pairs[i][1])
      t = time.perf_counter()
      T = dgr.register(xyz0, xyz1)
      info = getattr(dgr, 'last_info', {})
      rows.append(pack_result(T, info.get('wsum', 0.0), info.get('iterations', 0),
                              getattr(dgr, 'last_branch', None), 1e3 * (time.perf_counter() - t)))
  return gather_results(rows, len(pairs), device)
