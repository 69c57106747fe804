"""Time RGB-D fusion on the GPU: a synthetic 640 x 480, 50-frame sequence (syn.rgbd_sequence) integrated at
voxel_length 0.008 m / sdf_trunc 0.04 m with RGB8 colour, then extracted.  Reports, with the card's name and power
limit read in the same run:
  * integrate ms per frame (ScalableTSDFVolume.integrate: upload, touch pass, its host read, integration; CUDA events,
    median and p90 over the 50 frames after a warm-up sequence);
  * the integration kernel alone on the last frame's touched units (CUDA events over repeated launches);
  * touched units per frame and total units; extract ms (count, host read, write), vertices, triangles;
  * a bytes model: touched units x 4096 x 20 B read and again written per frame, plus the depth and colour images;
    extraction reads every unit and its +1 halo (tsdf and weight), then tsdf and colour again, and writes the mesh;
  * achieved GB/s against the H100's 3.35 TB/s;
  * the CPU oracle's time on two frames, for context only.
One JSON line.

    python tools/tsdf_bench.py [--frames 50] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import o3d_integration as integ  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402
from oracle import tsdf as ot  # noqa: E402

HBM_BPS = 3.35e12


def card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  return out or f'{torch.cuda.get_device_name()}, power limit unknown'


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--frames', type=int, default=50)
  ap.add_argument('--reps', type=int, default=20)
  args = ap.parse_args()
  W, H, VL, TR = 640, 480, 0.008, 0.04
  t0 = time.time()
  c, d, P, K = syn.rgbd_sequence(0, args.frames, W, H)
  t_gen = time.time() - t0
  intr = integ.PinholeCameraIntrinsic(W, H, *K)
  rgbd = [integ.RGBDImage.create_from_color_and_depth(integ.Image(c[k]), integ.Image(d[k]), depth_trunc=4.5,
                                                      convert_rgb_to_intensity=False) for k in range(len(P))]
  ext = [np.linalg.inv(p) for p in P]

  def run(vol, times=None, touched=None):
    for k in range(len(P)):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      vol.integrate(rgbd[k], intr, ext[k])
      e1.record()
      if times is not None:
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        touched.append(vol.n_touched)

  run(integ.ScalableTSDFVolume(VL, TR, integ.TSDFVolumeColorType.RGB8))     # warm-up
  torch.cuda.synchronize()
  vol = integ.ScalableTSDFVolume(VL, TR, integ.TSDFVolumeColorType.RGB8)
  times, touched = [], []
  run(vol, times, touched)

  # the integration kernel alone, on the last frame's touched units (the slabs change; the work does not)
  dev = vol.device
  depth = torch.from_numpy(np.asarray(rgbd[-1].depth)).to(dev)
  color = torch.from_numpy(np.asarray(rgbd[-1].color)).to(dev)
  kargs = (depth, color, intr._params(), ext[-1], VL, TR, vol._unit_keys, vol._touched, vol.n_touched, vol._tsdf,
           vol._weight, vol._rgb)
  _abi.tsdf_integrate(*kargs)
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(args.reps):
    _abi.tsdf_integrate(*kargs)
  e1.record()
  torch.cuda.synchronize()
  k_ms = e0.elapsed_time(e1) / args.reps

  vol.extract_triangle_mesh_tensors()                  # warm-up
  torch.cuda.synchronize()
  ex = []
  for _ in range(5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    v, cc, t = vol.extract_triangle_mesh_tensors()
    e1.record()
    torch.cuda.synchronize()
    ex.append(e0.elapsed_time(e1))
  x_ms = float(np.median(ex))

  img_bytes = W * H * (4 + 3)
  per_frame = [n * 4096 * 20 * 2 + img_bytes for n in touched]
  n_units, nv, nt = vol.n_units, v.shape[0], t.shape[0]
  ext_bytes = n_units * 17 ** 3 * 8 + n_units * 4096 * 16 + nv * 48 + nt * 12
  med, p90 = float(np.median(times)), float(np.percentile(times, 90))
  kbytes = vol.n_touched * 4096 * 20 * 2 + img_bytes

  t0 = time.time()
  ov = ot.Volume(VL, TR, color=True)
  for k in range(2):
    ov.integrate(np.asarray(rgbd[k].depth), (W, H) + tuple(K), ext[k], np.asarray(rgbd[k].color))
  oracle_s = (time.time() - t0) / 2

  res = {
      'card': card(), 'frames': len(P), 'width': W, 'height': H, 'voxel_length': VL, 'sdf_trunc': TR,
      'integrate_ms_median': round(med, 4), 'integrate_ms_p90': round(p90, 4),
      'touched_units_median': int(np.median(touched)), 'touched_units_max': int(max(touched)), 'total_units': n_units,
      'frame_bytes_median': int(np.median(per_frame)),
      'integrate_GBps_median_frame': round(float(np.median(per_frame)) / (med * 1e-3) / 1e9, 1),
      'kernel_ms_last_frame': round(k_ms, 4), 'kernel_units_last_frame': vol.n_touched,
      'kernel_GBps': round(kbytes / (k_ms * 1e-3) / 1e9, 1),
      'kernel_share_of_hbm': round(kbytes / (k_ms * 1e-3) / HBM_BPS, 3),
      'extract_ms': round(x_ms, 3), 'vertices': int(nv), 'triangles': int(nt), 'extract_bytes': int(ext_bytes),
      'extract_GBps': round(ext_bytes / (x_ms * 1e-3) / 1e9, 1),
      'oracle_cpu_s_per_frame': round(oracle_s, 2), 'sequence_gen_s': round(t_gen, 1),
  }
  print(json.dumps(res))


if __name__ == '__main__':
  main()
