"""Fuse 3DMatch raw RGB-D sequences into fragment meshes on the GPU: the layout and defaults of the reference's
util/integration.py, on o3d_integration.ScalableTSDFVolume.

    python -m deepglobalregistration_b200.integration /data/3dmatch-raw/7-scenes-redkitchen out/

For every ``seq-*`` directory of DATASET (frames ``*.color.png`` / ``*.depth.png`` / ``*.pose.txt``, intrinsics in
``intrinsics.txt`` beside them or ``camera-intrinsics.txt`` one level up), every run of ``--frames_per_fragment``
frames is integrated (voxel 0.008 m, sdf_trunc 0.04 m, depth truncated at 4.5 m, RGB8 colour) and its mesh written to
``OUTPUT/<scene>/<seq>/fragment-<k>.ply``.  An existing ``OUTPUT/<scene>`` is an error unless ``--overwrite`` is
given.  One JSON summary line goes to stdout."""
import argparse
import json
import os
import sys
import time

import numpy as np

from . import io as dio
from . import o3d_integration as integ


def read_intrinsics(path):
  K = np.loadtxt(path)
  return K[0, 0], K[1, 1], K[0, 2], K[1, 2]


def sequence_frames(seq_path):
  files = os.listdir(seq_path)
  color = sorted(f for f in files if f.endswith('.color.png'))
  depth = sorted(f for f in files if f.endswith('.depth.png'))
  pose = sorted(f for f in files if f.endswith('.pose.txt'))
  if not color or not (len(color) == len(depth) == len(pose)):
    raise ValueError(f'{seq_path}: expected matching .color.png / .depth.png / .pose.txt frames, found '
                     f'{len(color)} / {len(depth)} / {len(pose)}')
  return color, depth, pose


def sequence_intrinsic(seq_path, width, height):
  own = os.path.join(seq_path, 'intrinsics.txt')
  fx, fy, cx, cy = read_intrinsics(own if os.path.exists(own) else os.path.join(seq_path, '..',
                                                                                 'camera-intrinsics.txt'))
  return integ.PinholeCameraIntrinsic(int(width), int(height), fx, fy, cx, cy)


def integrate_fragment(seq_path, frames, intrinsic, start, end, voxel_length=0.008, sdf_trunc=0.04, max_depth=4.5):
  """Mesh of frames [start, end) of a sequence (util/integration.py:44-71)."""
  color, depth, pose = frames
  volume = integ.ScalableTSDFVolume(voxel_length=voxel_length, sdf_trunc=sdf_trunc,
                                    color_type=integ.TSDFVolumeColorType.RGB8)
  for i in range(start, end):
    rgbd = integ.RGBDImage.create_from_color_and_depth(
        dio.read_image(os.path.join(seq_path, color[i])), dio.read_image(os.path.join(seq_path, depth[i])),
        depth_trunc=max_depth, convert_rgb_to_intensity=False)
    volume.integrate(rgbd, intrinsic, np.linalg.inv(np.loadtxt(os.path.join(seq_path, pose[i]))))
  return volume.extract_triangle_mesh(), volume.n_units


def main(argv=None):
  ap = argparse.ArgumentParser(description='RGB-D integration of a 3DMatch raw scene into fragment meshes (GPU)')
  ap.add_argument('dataset', help='scene directory holding seq-* sub-directories')
  ap.add_argument('output', help='output root; fragments go to OUTPUT/<scene>/<seq>/fragment-<k>.ply')
  ap.add_argument('--frames_per_fragment', type=int, default=50)
  ap.add_argument('--voxel_length', type=float, default=0.008)
  ap.add_argument('--sdf_trunc', type=float, default=0.04)
  ap.add_argument('--max_depth', type=float, default=4.5)
  ap.add_argument('--overwrite', action='store_true', help='write into an existing OUTPUT/<scene>')
  args = ap.parse_args(argv)
  if args.frames_per_fragment < 1:
    ap.error('--frames_per_fragment must be >= 1')
  scene = os.path.basename(os.path.normpath(args.dataset))
  out_scene = os.path.join(args.output, scene)
  if os.path.exists(out_scene) and not args.overwrite:
    print(f'error: {out_scene} exists; pass --overwrite to write into it', file=sys.stderr)
    return 2
  seqs = sorted(s for s in os.listdir(args.dataset) if s.startswith('seq')
                and os.path.isdir(os.path.join(args.dataset, s)))
  if not seqs:
    print(f'error: no seq-* directory under {args.dataset}', file=sys.stderr)
    return 2
  t0 = time.time()
  written, n_frames, n_vertices, n_triangles = [], 0, 0, 0
  for seq in seqs:
    seq_path = os.path.join(args.dataset, seq)
    frames = sequence_frames(seq_path)
    width, height = dio.read_image(os.path.join(seq_path, frames[0][0])).get_max_bound()
    intrinsic = sequence_intrinsic(seq_path, width, height)
    out_seq = os.path.join(out_scene, seq)
    os.makedirs(out_seq, exist_ok=True)
    n = len(frames[0])
    for k in range((n + args.frames_per_fragment - 1) // args.frames_per_fragment):
      start, end = k * args.frames_per_fragment, min((k + 1) * args.frames_per_fragment, n)
      mesh, _ = integrate_fragment(seq_path, frames, intrinsic, start, end, args.voxel_length, args.sdf_trunc,
                                   args.max_depth)
      path = os.path.join(out_seq, f'fragment-{k}.ply')
      dio.write_triangle_mesh(path, mesh)
      written.append(path)
      n_frames += end - start
      n_vertices += len(mesh.vertices)
      n_triangles += len(mesh.triangles)
  print(json.dumps({'scene': scene, 'sequences': len(seqs), 'frames': n_frames, 'fragments': len(written),
                    'vertices': n_vertices, 'triangles': n_triangles, 'seconds': round(time.time() - t0, 3),
                    'output': out_scene}))
  return 0


if __name__ == '__main__':
  sys.exit(main())
