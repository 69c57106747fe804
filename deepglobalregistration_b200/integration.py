"""Fuse 3DMatch raw RGB-D sequences into fragment meshes on the GPU: the layout and defaults of the reference's
util/integration.py, on o3d_integration.ScalableTSDFVolume.

    python -m deepglobalregistration_b200.integration /data/3dmatch-raw/7-scenes-redkitchen out/

For every ``seq-*`` directory of DATASET (frames ``*.color.png`` / ``*.depth.png`` / ``*.pose.txt``, intrinsics in
``intrinsics.txt`` beside them or ``camera-intrinsics.txt`` one level up), every run of ``--frames_per_fragment``
frames is integrated (voxel 0.008 m, sdf_trunc 0.04 m, depth truncated at 4.5 m, RGB8 colour) and its mesh written to
``OUTPUT/<scene>/<seq>/fragment-<k>.ply``.  An existing ``OUTPUT/<scene>`` is an error unless ``--overwrite`` is
given.  One JSON summary line goes to stdout.

With ``--poses odometry`` the ``.pose.txt`` files are optional: each fragment's frames are posed as open3d's
reconstruction system (make_fragments) poses them - RGB-D odometry between consecutive frames (certain edges, chained
into the node poses) and between keyframes every ``--keyframe_every`` frames (uncertain loop closures, kept when the
odometry succeeds), then the pose graph's global optimisation - and the fragment's trajectory is written beside its
mesh as ``fragment-<k>.log``.  The mesh is then in the frame of the fragment's first camera.  open3d starts a loop
closure from OpenCV's 5-point ORB pose (and skips it without OpenCV); here it starts from the odometry chain's relative
pose.

With ``--poses model`` (a project extension) each frame is instead tracked against the model fused so far, as
KinectFusion and open3d's dense SLAM do: the fragment's volume is ray-cast at the previous pose and the frame is
registered to that rendering by RGB-D odometry, then fused (track_model).  There is no pose graph, so
``--frames_per_fragment`` is not capped; the mesh and ``fragment-<k>.log`` come from the tracker's own volume, and
the summary reports ``tracked_frames`` and ``tracking_failures``."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

from . import _abi
from . import io as dio
from . import o3d_integration as integ
from . import o3d_odometry as odo
from . import o3d_registration as reg
from .core.multiway import absolute_trajectory_error

# open3d's reconstruction-system defaults for make_fragments (config: max_depth 3.0, max_depth_diff 0.07,
# preference_loop_closure_odometry 0.1; the odometry's min_depth 0.3)
ODOMETRY_OPTION = dict(min_depth=0.3, max_depth=3.0, max_depth_diff=0.07)


def read_intrinsics(path):
  K = np.loadtxt(path)
  return K[0, 0], K[1, 1], K[0, 2], K[1, 2]


def sequence_frames(seq_path, need_poses=True):
  """-> (colour, depth, pose) file lists; without need_poses the pose list is None unless every frame has one."""
  files = os.listdir(seq_path)
  color = sorted(f for f in files if f.endswith('.color.png'))
  depth = sorted(f for f in files if f.endswith('.depth.png'))
  pose = sorted(f for f in files if f.endswith('.pose.txt'))
  if not need_poses:
    if not color or len(color) != len(depth):
      raise ValueError(f'{seq_path}: expected matching .color.png / .depth.png frames, found {len(color)} / '
                       f'{len(depth)}')
    return color, depth, pose if len(pose) == len(color) else None
  if not color or not (len(color) == len(depth) == len(pose)):
    raise ValueError(f'{seq_path}: expected matching .color.png / .depth.png / .pose.txt frames, found '
                     f'{len(color)} / {len(depth)} / {len(pose)}')
  return color, depth, pose


def sequence_intrinsic(seq_path, width, height):
  own = os.path.join(seq_path, 'intrinsics.txt')
  fx, fy, cx, cy = read_intrinsics(own if os.path.exists(own) else os.path.join(seq_path, '..',
                                                                                 'camera-intrinsics.txt'))
  return integ.PinholeCameraIntrinsic(int(width), int(height), fx, fy, cx, cy)


def odometry_poses(seq_path, frames, intrinsic, start, end, keyframe_every=5):
  """Node poses (frame k -> the fragment's first camera) of frames [start, end), as open3d's make_fragments builds
  and optimises the fragment's pose graph.  All pairs of one stage are enqueued and read back once: the consecutive
  pairs, then the keyframe pairs (whose initial poses come from the chain).  -> (poses [n, 4, 4], stats dict)."""
  color, depth = frames[0], frames[1]
  option = odo.OdometryOption(**ODOMETRY_OPTION)
  rgbd = [integ.RGBDImage.create_from_color_and_depth(
      dio.read_image(os.path.join(seq_path, color[i])), dio.read_image(os.path.join(seq_path, depth[i])),
      depth_trunc=option.max_depth, convert_rgb_to_intensity=True) for i in range(start, end)]
  n = end - start
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()

  def run(pairs, inits):
    if not pairs:
      return []
    out = torch.empty(len(pairs), _abi.ODOMETRY_RESULT, dtype=torch.float64, device=dev)
    for k, ((s, t), init) in enumerate(zip(pairs, inits)):
      args = odo.odometry_arguments(rgbd[s], rgbd[t], intrinsic, init, None, option)
      odo.enqueue_rgbd_odometry(*args, dev, result=out[k])
    return [odo.unpack_result(r) for r in out.cpu().numpy()]

  chain = [(s, s + 1) for s in range(n - 1)]
  graph = reg.PoseGraph()
  trans_odometry = np.eye(4)
  graph.nodes.append(reg.PoseGraphNode(trans_odometry))
  for (s, t), (_, trans, info) in zip(chain, run(chain, [np.eye(4)] * len(chain))):
    trans_odometry = trans @ trans_odometry
    graph.nodes.append(reg.PoseGraphNode(np.linalg.inv(trans_odometry)))
    graph.edges.append(reg.PoseGraphEdge(s, t, trans, info, uncertain=False))
  loops = [(s, t) for s in range(n) for t in range(s + 2, n)
           if (start + s) % keyframe_every == 0 and (start + t) % keyframe_every == 0]
  inits = [np.linalg.inv(graph.nodes[t].pose) @ graph.nodes[s].pose for s, t in loops]
  n_loops = 0
  for (s, t), (ok, trans, info) in zip(loops, run(loops, inits)):
    if ok:
      graph.edges.append(reg.PoseGraphEdge(s, t, trans, info, uncertain=True))
      n_loops += 1
  if graph.edges:
    reg.global_optimization(graph, reg.GlobalOptimizationLevenbergMarquardt(),
                            reg.GlobalOptimizationConvergenceCriteria(),
                            reg.GlobalOptimizationOption(max_correspondence_distance=option.max_depth_diff,
                                                         edge_prune_threshold=0.25, preference_loop_closure=0.1,
                                                         reference_node=0))
  kept = sum(1 for e in graph.edges if e.uncertain)
  return np.stack([v.pose for v in graph.nodes]), dict(odometry_pairs=len(chain) + len(loops),
                                                        loop_closures=n_loops, loop_closures_kept=kept)


def track_model(images, intrinsic, voxel_length=0.008, sdf_trunc=0.04, max_depth=4.5):
  """Frame-to-model tracking, as open3d's dense SLAM (t.pipelines.slam.Model) tracks: frame 0 is fused at the
  identity; every later frame k is registered by RGB-D odometry (hybrid Jacobian, ODOMETRY_OPTION, from the identity)
  against the model ray-cast at P_{k-1} with weight_threshold min(k, 3) over [min_depth, max_depth] of the option,
  posed P_k = P_{k-1} T and fused at P_k.  A failed odometry keeps P_k = P_{k-1} and the frame is not fused.
  images: (colour [H, W, 3] uint8, depth [H, W] uint16 mm) per frame.  One result read per tracked frame, besides the
  integration's own.  -> (poses [n, 4, 4] (frame k -> the first camera), the RGB8 volume, stats dict)."""
  option = odo.OdometryOption(**ODOMETRY_OPTION)
  volume = integ.ScalableTSDFVolume(voxel_length=voxel_length, sdf_trunc=sdf_trunc,
                                    color_type=integ.TSDFVolumeColorType.RGB8)
  dev = volume.device
  intr = intrinsic._params()
  its = option.iteration_number_per_pyramid_level
  poses, failures = [], 0
  for k, (color, depth) in enumerate(images):
    fuse = integ.RGBDImage.create_from_color_and_depth(color, depth, depth_trunc=max_depth,
                                                       convert_rgb_to_intensity=False)
    if k == 0:
      poses.append(np.eye(4))
      volume.integrate(fuse, intrinsic, np.eye(4))
      continue
    src = integ.RGBDImage.create_from_color_and_depth(color, depth, depth_trunc=option.max_depth,
                                                      convert_rgb_to_intensity=True)
    Is, Ds = (torch.from_numpy(np.ascontiguousarray(np.asarray(a))).to(dev) for a in (src.color, src.depth))
    P = poses[-1]
    model = volume.raycast_tensors(intrinsic, np.linalg.inv(P), option.min_depth, option.max_depth,
                                   float(min(k, 3)), outputs=('depth', 'intensity'))
    r = _abi.rgbd_odometry(Is, Ds, model['intensity'], model['depth'], intr, np.eye(4), 'hybrid', its,
                           option.max_depth_diff, option.min_depth, option.max_depth)
    ok, T, _ = odo.unpack_result(r.cpu().numpy())
    if not ok:
      failures += 1
      poses.append(P)
      continue
    poses.append(P @ T)
    volume.integrate(fuse, intrinsic, np.linalg.inv(poses[-1]))
  n = len(poses)
  return np.stack(poses), volume, dict(tracked_frames=max(n - 1, 0) - failures, tracking_failures=failures)


def model_poses(seq_path, frames, intrinsic, start, end, voxel_length=0.008, sdf_trunc=0.04, max_depth=4.5):
  """track_model over frames [start, end) of a sequence: -> (poses [n, 4, 4], volume, stats)."""
  color, depth = frames[0], frames[1]
  images = ((dio.read_image(os.path.join(seq_path, color[i])), dio.read_image(os.path.join(seq_path, depth[i])))
            for i in range(start, end))
  return track_model(images, intrinsic, voxel_length, sdf_trunc, max_depth)


def integrate_fragment(seq_path, frames, intrinsic, start, end, voxel_length=0.008, sdf_trunc=0.04, max_depth=4.5,
                       poses=None):
  """Mesh of frames [start, end) of a sequence (util/integration.py:44-71); poses: camera-to-world poses of the
  frames (default: their .pose.txt files)."""
  color, depth, pose = frames
  volume = integ.ScalableTSDFVolume(voxel_length=voxel_length, sdf_trunc=sdf_trunc,
                                    color_type=integ.TSDFVolumeColorType.RGB8)
  for i in range(start, end):
    rgbd = integ.RGBDImage.create_from_color_and_depth(
        dio.read_image(os.path.join(seq_path, color[i])), dio.read_image(os.path.join(seq_path, depth[i])),
        depth_trunc=max_depth, convert_rgb_to_intensity=False)
    P = np.loadtxt(os.path.join(seq_path, pose[i])) if poses is None else poses[i - start]
    volume.integrate(rgbd, intrinsic, np.linalg.inv(P))
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
  ap.add_argument('--poses', choices=('file', 'odometry', 'model'), default='file',
                  help='frame poses: the .pose.txt files, RGB-D odometry and a pose graph per fragment, or each frame '
                       'tracked against the fragment\'s fused model')
  ap.add_argument('--keyframe_every', type=int, default=5, help='--poses odometry: loop closures between keyframes')
  args = ap.parse_args(argv)
  if args.frames_per_fragment < 1:
    ap.error('--frames_per_fragment must be >= 1')
  if args.poses == 'odometry' and args.frames_per_fragment > _abi.POSE_GRAPH_MAX_NODES:
    ap.error(f'--poses odometry: --frames_per_fragment must be <= {_abi.POSE_GRAPH_MAX_NODES} (pose-graph nodes)')
  if args.keyframe_every < 1:
    ap.error('--keyframe_every must be >= 1')
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
  odo_stats = dict(odometry_pairs=0, loop_closures_kept=0, tracked_frames=0, tracking_failures=0, ate=[])
  for seq in seqs:
    seq_path = os.path.join(args.dataset, seq)
    frames = sequence_frames(seq_path, need_poses=args.poses == 'file')
    width, height = dio.read_image(os.path.join(seq_path, frames[0][0])).get_max_bound()
    intrinsic = sequence_intrinsic(seq_path, width, height)
    out_seq = os.path.join(out_scene, seq)
    os.makedirs(out_seq, exist_ok=True)
    n = len(frames[0])
    for k in range((n + args.frames_per_fragment - 1) // args.frames_per_fragment):
      start, end = k * args.frames_per_fragment, min((k + 1) * args.frames_per_fragment, n)
      poses, volume = None, None
      if args.poses == 'odometry':
        poses, st = odometry_poses(seq_path, frames, intrinsic, start, end, args.keyframe_every)
        odo_stats['odometry_pairs'] += st['odometry_pairs']
        odo_stats['loop_closures_kept'] += st['loop_closures_kept']
      elif args.poses == 'model':                       # the tracker's own volume gives the mesh
        poses, volume, st = model_poses(seq_path, frames, intrinsic, start, end, args.voxel_length, args.sdf_trunc,
                                        args.max_depth)
        odo_stats['tracked_frames'] += st['tracked_frames']
        odo_stats['tracking_failures'] += st['tracking_failures']
      if poses is not None:
        dio.write_trajectory(os.path.join(out_seq, f'fragment-{k}.log'),
                            [((i, i, len(poses)), P) for i, P in enumerate(poses)])
        if frames[2] is not None:                       # ATE against the first frame's frame of the files
          gt = np.stack([np.loadtxt(os.path.join(seq_path, frames[2][i])) for i in range(start, end)])
          gt = np.linalg.inv(gt[0]) @ gt
          odo_stats['ate'].append(float(absolute_trajectory_error(poses, gt)))
      if volume is not None:
        mesh = volume.extract_triangle_mesh()
      else:
        mesh, _ = integrate_fragment(seq_path, frames, intrinsic, start, end, args.voxel_length, args.sdf_trunc,
                                     args.max_depth, poses)
      path = os.path.join(out_seq, f'fragment-{k}.ply')
      dio.write_triangle_mesh(path, mesh)
      written.append(path)
      n_frames += end - start
      n_vertices += len(mesh.vertices)
      n_triangles += len(mesh.triangles)
  summary = {'scene': scene, 'sequences': len(seqs), 'frames': n_frames, 'fragments': len(written),
             'vertices': n_vertices, 'triangles': n_triangles, 'seconds': round(time.time() - t0, 3),
             'output': out_scene}
  if args.poses == 'odometry':
    summary.update(odometry_pairs=odo_stats['odometry_pairs'], loop_closures_kept=odo_stats['loop_closures_kept'])
  elif args.poses == 'model':
    summary.update(tracked_frames=odo_stats['tracked_frames'], tracking_failures=odo_stats['tracking_failures'])
  if odo_stats['ate']:
    summary['fragment_ate'] = odo_stats['ate']
  print(json.dumps(summary))
  return 0


if __name__ == '__main__':
  sys.exit(main())
