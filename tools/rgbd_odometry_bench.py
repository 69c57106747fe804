"""Time RGB-D odometry (csrc/odometry.cu) on 640x480 ray-cast pairs, consecutive and 5 frames apart: CUDA-event
medians of one compute_rgbd_odometry call and of each level's step (project, accumulate, update), a bytes model per
step from the measured correspondence counts, one call of the fp64 oracle, and one 50-frame fragment through
``integration --poses odometry`` split into pairs, pose graph and integration.  Prints one JSON line; numbers belong
with the card's name and power limit, read in the same run.

    python tools/rgbd_odometry_bench.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import integration  # noqa: E402
from deepglobalregistration_b200 import o3d_integration as integ  # noqa: E402
from deepglobalregistration_b200 import o3d_odometry as odo  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402
from oracle import rgbd_odometry as ro  # noqa: E402


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return out or torch.cuda.get_device_name(0)


def events(fn, reps):
  ts = []
  for _ in range(reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
  return float(np.median(ts))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  args = ap.parse_args()
  dev = _abi.require_device('cuda')
  cols, deps, poses, intr = syn.rgbd_sequence(3, 50, turn=0.1, radius=0.05)   # 0.72 degrees, 6 mm per frame
  cam = integ.PinholeCameraIntrinsic(640, 480, *intr)
  opt = odo.OdometryOption()
  its = opt.iteration_number_per_pyramid_level
  L = len(its)
  out = {'card': card(), 'size': [640, 480], 'iterations': its}
  for name, (s, t) in (('consecutive', (10, 11)), ('five_apart', (10, 15))):
    src = integ.RGBDImage.create_from_color_and_depth(cols[s], deps[s], depth_trunc=4.0)
    tgt = integ.RGBDImage.create_from_color_and_depth(cols[t], deps[t], depth_trunc=4.0)
    a = odo.odometry_arguments(src, tgt, cam, np.eye(4), None, opt)
    _abi.refresh_stream()
    imgs = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in a[0]]
    res = torch.empty(_abi.ODOMETRY_RESULT, dtype=torch.float64, device=dev)
    call = lambda lv=its: _abi.rgbd_odometry(*imgs, a[1], a[2], 'hybrid', lv, result=res)   # noqa: E731
    call()
    torch.cuda.synchronize()
    t_call = events(call, args.reps)
    r = res.cpu().numpy()
    counts = r[55:55 + int(r[17])]
    # per level: a call with one more step at that level minus the call without it (the steps of a level are equal
    # launches on equal-size images)
    per_level = {}
    for li in range(L):
      more = list(its)
      more[li] += 1
      t_more = events(lambda m=tuple(more): call(m), args.reps)
      per_level[f'level{L - 1 - li}'] = round(t_more - t_call, 4)
    # bytes per step at level 0: source depth read (4 B / px), z-buffer atomics and reads (8 B / match, twice),
    # 8 B / px z-buffer read and reset, per match 6 floats of target images and 2 of source, partials
    n0 = 640 * 480
    m = float(counts[-1]) if len(counts) else 0.0
    bytes0 = 4 * n0 + 8 * n0 + 2 * 8 * m + 8 * 4 * m + 2368 * 32 * 8
    t0 = time.perf_counter()
    Is, Ds, It, Dt = a[0]
    ro.compute_rgbd_odometry(Is, Ds, It, Dt, tuple(a[1]), hybrid=True, iterations=its)
    t_oracle = time.perf_counter() - t0
    out[name] = {'call_ms': round(t_call, 3), 'step_ms': per_level, 'success': bool(r[16]),
                 'counts_first_last': [int(counts[0]), int(counts[-1])] if len(counts) else [],
                 'level0_step_bytes_model': int(bytes0),
                 'level0_step_GBps_model': round(bytes0 / (per_level['level0'] * 1e-3) / 1e9, 1)
                 if per_level['level0'] > 0 else None,
                 'oracle_s': round(t_oracle, 2)}
  # one 50-frame fragment: pairs + pose graph, then integration
  with tempfile.TemporaryDirectory() as tmp:
    seq = syn.write_rgbd_sequence(tmp, 'room', cols, deps, poses, intr)
    frames = integration.sequence_frames(seq, need_poses=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    P, st = integration.odometry_poses(seq, frames, cam, 0, 50)
    t1 = time.perf_counter()
    integration.integrate_fragment(seq, frames, cam, 0, 50, poses=P)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    gt = np.linalg.inv(poses[0]) @ poses
    from deepglobalregistration_b200.core.multiway import absolute_trajectory_error
    out['fragment'] = {'frames': 50, 'pairs_and_pose_graph_s': round(t1 - t0, 3), 'integration_s': round(t2 - t1, 3),
                       'ate_m': round(absolute_trajectory_error(P, gt), 5), **st}
  print(json.dumps(out))


if __name__ == '__main__':
  main()
