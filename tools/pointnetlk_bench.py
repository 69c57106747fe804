"""Time PointNetLK on the bench's full-size pair syn.room_pair(0) (voxel 0.05 m, about 51k / 40k voxels) with a seeded
random network: CUDA-event times of one forward, the 7-pose Jacobian forward, one LK iteration and the whole call
(10 iterations, xtol 0 so none stops early), the achieved rate of the forwards from their shapes, and the card's name
and power limit read in the same run.  One JSON line.

The forward's useful work is 2 n (3*64 + 64*64 + 64*64 + 64*128 + 128*1024) FLOP per pose.  It runs as 3xTF32: three
TF32 tensor-core products per useful product on layers 2-5, so the tensor pipe executes about 3x those FLOP.  The
data-sheet rate it is compared with is the H100 SXM's dense TF32 rate, 495 TFLOP/s, for a card allowed 700 W.

    python tools/pointnetlk_bench.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402

TF32_DENSE_TFLOPS = 495.0
MACS_PER_POINT = 3 * 64 + 64 * 64 + 64 * 64 + 64 * 128 + 128 * 1024
TC_MACS_PER_POINT = MACS_PER_POINT - 3 * 64


def card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  return out or torch.cuda.get_device_name()


def timed(fn, reps):
  fn()
  torch.cuda.synchronize()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  ev[0].record()
  for _ in range(reps):
    fn()
  ev[1].record()
  torch.cuda.synchronize()
  return ev[0].elapsed_time(ev[1]) / reps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  args = ap.parse_args()
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.pointnetlk import PointNetLKBaseline
  from oracle.pointnetlk import jacobian_poses
  dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=0.05),
                                                     clip_weight_thresh=0.05, verbose=False))
  b = PointNetLKBaseline(dgr, syn.pointnetlk_state_dict(0))
  xyz0, xyz1, _ = syn.room_pair(0)
  name = card()
  with torch.no_grad():
    p0, _, _ = dgr.preprocess(xyz0, 0, _batch=0)
    p1, _, _ = dgr.preprocess(xyz1, 1, _batch=1)
  src, tgt = p0.float().contiguous(), p1.float().contiguous()
  eye = torch.eye(4, dtype=torch.float64, device=src.device)[None]
  jp = torch.as_tensor(np.stack(jacobian_poses(1e-2)), device=src.device)
  fwd_ms = timed(lambda: _abi.pointnet_forward(src, eye, b.packed), args.reps)
  jac_ms = timed(lambda: _abi.pointnet_forward(tgt, jp, b.packed), args.reps)
  call_ms = timed(lambda: _abi.pointnetlk(src, tgt, b.packed, max_iter=10, xtol=0.0), args.reps)
  one_ms = timed(lambda: _abi.pointnetlk(src, tgt, b.packed, max_iter=1, xtol=0.0), args.reps)
  iter_ms = (call_ms - one_ms) / 9

  def rate(n, poses, ms):
    useful = 2.0 * n * poses * MACS_PER_POINT / (ms * 1e-3) / 1e12
    tc = 3 * 2.0 * n * poses * TC_MACS_PER_POINT / (ms * 1e-3) / 1e12
    return dict(useful_tflops=round(useful, 1), tc_tf32_tflops=round(tc, 1),
                tc_share_of_datasheet=round(tc / TF32_DENSE_TFLOPS, 3))

  print(json.dumps(dict(card=name, n_src=len(src), n_tgt=len(tgt), forward_ms=round(fwd_ms, 4),
                        forward=rate(len(src), 1, fwd_ms), jacobian_7pose_ms=round(jac_ms, 4),
                        jacobian=rate(len(tgt), 7, jac_ms), lk_iteration_ms=round(iter_ms, 4),
                        call_10_iterations_ms=round(call_ms, 3), call_1_iteration_ms=round(one_ms, 3),
                        tf32_datasheet_tflops=TF32_DENSE_TFLOPS)), flush=True)


if __name__ == '__main__':
  main()
