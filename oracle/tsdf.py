"""ORACLE (test infrastructure only) - RGB-D fusion as open3d's legacy ``ScalableTSDFVolume`` runs it: ``integrate``
and ``extract_triangle_mesh`` (``integration`` in open3d 0.10, ``pipelines.integration`` from 0.12 on), restated in
numpy.  This module is the arithmetic contract of csrc/tsdf.cu: the kernels must meet it bit for bit, so it fixes the
order of every floating-point operation.  "fp64" below means numpy float64 element-wise ops, "fp32" numpy float32
scalar/array ops; numpy rounds every op to nearest and never contracts a multiply-add.

PARITY UNPINNED: open3d is not installed here and not vendored, so every reading below is a restatement from memory of
open3d's published ScalableTSDFVolume.cpp / UniformTSDFVolume.cpp / MarchingCubesConst.h, recorded as an assumption.

Assumptions (readings of open3d):
  * Images.  RGBDImage.create_from_color_and_depth(color, depth, depth_scale=1000, depth_trunc=3.0,
    convert_rgb_to_intensity=True): float depth = float32(raw) / float32(depth_scale), 0 where >= depth_trunc.  An RGB8
    volume accepts 3-channel uint8 colour only and a depth image of the intrinsic's size; anything else is a ValueError.
  * Multiplier of pixel (u = column, v = row): sqrt(1 + ((u - cx) / fx)^2 + ((v - cy) / fy)^2), fp64, rounded once to
    fp32 (here: a = (u - cx) / fx, b = (v - cy) / fy, sqrt((1 + a a) + b b)).
  * Touched units.  L = voxel_length * volume_unit_resolution.  The depth image is sampled every depth_sampling_stride
    rows and columns in row-major order, keeping d > 0; each sample is back-projected in fp64 (x = ((j - cx) d) / fx,
    y = ((i - cy) d) / fy, z = d), moved to the world by camera_pose = inv(extrinsic) (np.linalg.inv, once, on the
    host; row r: ((P[r,0] x + P[r,1] y) + P[r,2] z) + P[r,3]) and touches every unit from floor((p - sdf_trunc) / L)
    to floor((p + sdf_trunc) / L) per axis, x outermost, then y, then z.  The touched list is the first occurrence of
    each unit in that order; a unit never seen before gets the next slot number in the same order.
  * Voxel update, for every voxel (x, y, z) of every touched unit (linear index (x R + y) R + z), centre
    unit L + (i + 0.5) voxel_length per axis in fp64:
      1. camera point c = extrinsic . centre, row r: ((E[r,0] X + E[r,1] Y) + E[r,2] Z) + E[r,3];
      2. skip if c_z <= 0;
      3. u_f = ((c_x fx) / c_z + cx) + 0.5, v_f the same with fy, cy;
      4. skip unless 0.0001 <= u_f < W - 0.0001 and 0.0001 <= v_f < H - 0.0001;
      5. u = int(u_f), v = int(v_f), d = depth[v, u]; skip if d <= 0;
      6. sdf = float32(d - c_z) * mult[v, u] in fp32;
      7. if sdf > -float32(sdf_trunc), in fp32: tsdf_new = min(1, sdf * float32(1 / sdf_trunc)),
         tsdf <- (tsdf w + tsdf_new) / (w + 1), each colour channel c <- (c w + rgb) / (w + 1) with rgb in 0..255,
         w <- w + 1.
  * Mesh.  Voxel g (global lattice index) lies at (g + 0.5) voxel_length.  A cube is voxel g and its 7 neighbours at
    +1, corners 0..7 = (000, 100, 110, 010, 001, 101, 111, 011); it is skipped when a corner has weight 0 (a corner in a
    missing unit has weight 0) or its index (bit i set when f_i < 0) is 0 or 255.  A vertex sits on each sign-changing
    edge of a kept cube, keyed by (lower endpoint g, axis), at g + |f0| voxel_length / (|f0| + |f1|) along the axis
    (fp64: ((|f0| vl) / (|f0| + |f1|)) added to the endpoint's coordinate), with colour
    ((|f1| c0 + |f0| c1) / (|f0| + |f1|)) / 255 (fp64).  Triangles come from the Lorensen / Bourke tables below
    (TRI_TABLE; EDGE_TABLE bit e set when edge e's ends differ in sign), each emitted with open3d's winding
    (e[i], e[i+2], e[i+1]).

Departures:
  * open3d transforms voxels in fp32 with incremental z steps; here every voxel is projected directly in fp64.  The
    two differ only for voxels whose projection lands within fp32 rounding of a pixel edge.
  * open3d emits vertices and triangles in hash-map order, which is not fixed.  Here both come in a canonical order:
    vertices by (unit slot, voxel linear index, axis), triangles by (unit slot, voxel, table order).
  * Gray32 colour, extract_point_cloud and extract_voxel_point_cloud are not restated.
"""
import numpy as np

RES = 16
SENTINEL_RANGE = (-(1 << 20), (1 << 20) - 2)     # unit coordinates the library's 21-bit keys can hold

# corner offsets (x, y, z) of corners 0..7, the two corners of edges 0..11
CORNERS = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]])
EDGE_CORNERS = np.array([[0, 1], [1, 2], [2, 3], [3, 0], [4, 5], [5, 6], [6, 7], [7, 4], [0, 4], [1, 5], [2, 6],
                         [3, 7]])
# owner of edge e: its lower endpoint (offset from the cube's voxel) and its axis
EDGE_OWNER = np.minimum(CORNERS[EDGE_CORNERS[:, 0]], CORNERS[EDGE_CORNERS[:, 1]])
EDGE_AXIS = np.argmax(np.abs(CORNERS[EDGE_CORNERS[:, 0]] - CORNERS[EDGE_CORNERS[:, 1]]), axis=1)
EDGE_TABLE = np.array([sum(1 << e for e in range(12)
                           if ((i >> EDGE_CORNERS[e, 0]) ^ (i >> EDGE_CORNERS[e, 1])) & 1) for i in range(256)],
                      dtype=np.int32)

_TRI = [
    [], [0, 8, 3], [0, 1, 9], [1, 8, 3, 9, 8, 1], [1, 2, 10], [0, 8, 3, 1, 2, 10], [9, 2, 10, 0, 2, 9],
    [2, 8, 3, 2, 10, 8, 10, 9, 8], [3, 11, 2], [0, 11, 2, 8, 11, 0], [1, 9, 0, 2, 3, 11],
    [1, 11, 2, 1, 9, 11, 9, 8, 11], [3, 10, 1, 11, 10, 3], [0, 10, 1, 0, 8, 10, 8, 11, 10],
    [3, 9, 0, 3, 11, 9, 11, 10, 9], [9, 8, 10, 10, 8, 11], [4, 7, 8], [4, 3, 0, 7, 3, 4], [0, 1, 9, 8, 4, 7],
    [4, 1, 9, 4, 7, 1, 7, 3, 1], [1, 2, 10, 8, 4, 7], [3, 4, 7, 3, 0, 4, 1, 2, 10], [9, 2, 10, 9, 0, 2, 8, 4, 7],
    [2, 10, 9, 2, 9, 7, 2, 7, 3, 7, 9, 4], [8, 4, 7, 3, 11, 2], [11, 4, 7, 11, 2, 4, 2, 0, 4],
    [9, 0, 1, 8, 4, 7, 2, 3, 11], [4, 7, 11, 9, 4, 11, 9, 11, 2, 9, 2, 1], [3, 10, 1, 3, 11, 10, 7, 8, 4],
    [1, 11, 10, 1, 4, 11, 1, 0, 4, 7, 11, 4], [4, 7, 8, 9, 0, 11, 9, 11, 10, 11, 0, 3],
    [4, 7, 11, 4, 11, 9, 9, 11, 10], [9, 5, 4], [9, 5, 4, 0, 8, 3], [0, 5, 4, 1, 5, 0], [8, 5, 4, 8, 3, 5, 3, 1, 5],
    [1, 2, 10, 9, 5, 4], [3, 0, 8, 1, 2, 10, 4, 9, 5], [5, 2, 10, 5, 4, 2, 4, 0, 2],
    [2, 10, 5, 3, 2, 5, 3, 5, 4, 3, 4, 8], [9, 5, 4, 2, 3, 11], [0, 11, 2, 0, 8, 11, 4, 9, 5],
    [0, 5, 4, 0, 1, 5, 2, 3, 11], [2, 1, 5, 2, 5, 8, 2, 8, 11, 4, 8, 5], [10, 3, 11, 10, 1, 3, 9, 5, 4],
    [4, 9, 5, 0, 8, 1, 8, 10, 1, 8, 11, 10], [5, 4, 0, 5, 0, 11, 5, 11, 10, 11, 0, 3],
    [5, 4, 8, 5, 8, 10, 10, 8, 11], [9, 7, 8, 5, 7, 9], [9, 3, 0, 9, 5, 3, 5, 7, 3], [0, 7, 8, 0, 1, 7, 1, 5, 7],
    [1, 5, 3, 3, 5, 7], [9, 7, 8, 9, 5, 7, 10, 1, 2], [10, 1, 2, 9, 5, 0, 5, 3, 0, 5, 7, 3],
    [8, 0, 2, 8, 2, 5, 8, 5, 7, 10, 5, 2], [2, 10, 5, 2, 5, 3, 3, 5, 7], [7, 9, 5, 7, 8, 9, 3, 11, 2],
    [9, 5, 7, 9, 7, 2, 9, 2, 0, 2, 7, 11], [2, 3, 11, 0, 1, 8, 1, 7, 8, 1, 5, 7], [11, 2, 1, 11, 1, 7, 7, 1, 5],
    [9, 5, 8, 8, 5, 7, 10, 1, 3, 10, 3, 11], [5, 7, 0, 5, 0, 9, 7, 11, 0, 1, 0, 10, 11, 10, 0],
    [11, 10, 0, 11, 0, 3, 10, 5, 0, 8, 0, 7, 5, 7, 0], [11, 10, 5, 7, 11, 5], [10, 6, 5], [0, 8, 3, 5, 10, 6],
    [9, 0, 1, 5, 10, 6], [1, 8, 3, 1, 9, 8, 5, 10, 6], [1, 6, 5, 2, 6, 1], [1, 6, 5, 1, 2, 6, 3, 0, 8],
    [9, 6, 5, 9, 0, 6, 0, 2, 6], [5, 9, 8, 5, 8, 2, 5, 2, 6, 3, 2, 8], [2, 3, 11, 10, 6, 5],
    [11, 0, 8, 11, 2, 0, 10, 6, 5], [0, 1, 9, 2, 3, 11, 5, 10, 6], [5, 10, 6, 1, 9, 2, 9, 11, 2, 9, 8, 11],
    [6, 3, 11, 6, 5, 3, 5, 1, 3], [0, 8, 11, 0, 11, 5, 0, 5, 1, 5, 11, 6], [3, 11, 6, 0, 3, 6, 0, 6, 5, 0, 5, 9],
    [6, 5, 9, 6, 9, 11, 11, 9, 8], [5, 10, 6, 4, 7, 8], [4, 3, 0, 4, 7, 3, 6, 5, 10], [1, 9, 0, 5, 10, 6, 8, 4, 7],
    [10, 6, 5, 1, 9, 7, 1, 7, 3, 7, 9, 4], [6, 1, 2, 6, 5, 1, 4, 7, 8], [1, 2, 5, 5, 2, 6, 3, 0, 4, 3, 4, 7],
    [8, 4, 7, 9, 0, 5, 0, 6, 5, 0, 2, 6], [7, 3, 9, 7, 9, 4, 3, 2, 9, 5, 9, 6, 2, 6, 9],
    [3, 11, 2, 7, 8, 4, 10, 6, 5], [5, 10, 6, 4, 7, 2, 4, 2, 0, 2, 7, 11], [0, 1, 9, 4, 7, 8, 2, 3, 11, 5, 10, 6],
    [9, 2, 1, 9, 11, 2, 9, 4, 11, 7, 11, 4, 5, 10, 6], [8, 4, 7, 3, 11, 5, 3, 5, 1, 5, 11, 6],
    [5, 1, 11, 5, 11, 6, 1, 0, 11, 7, 11, 4, 0, 4, 11], [0, 5, 9, 0, 6, 5, 0, 3, 6, 11, 6, 3, 8, 4, 7],
    [6, 5, 9, 6, 9, 11, 4, 7, 9, 7, 11, 9], [10, 4, 9, 6, 4, 10], [4, 10, 6, 4, 9, 10, 0, 8, 3],
    [10, 0, 1, 10, 6, 0, 6, 4, 0], [8, 3, 1, 8, 1, 6, 8, 6, 4, 6, 1, 10], [1, 4, 9, 1, 2, 4, 2, 6, 4],
    [3, 0, 8, 1, 2, 9, 2, 4, 9, 2, 6, 4], [0, 2, 4, 4, 2, 6], [8, 3, 2, 8, 2, 4, 4, 2, 6],
    [10, 4, 9, 10, 6, 4, 11, 2, 3], [0, 8, 2, 2, 8, 11, 4, 9, 10, 4, 10, 6], [3, 11, 2, 0, 1, 6, 0, 6, 4, 6, 1, 10],
    [6, 4, 1, 6, 1, 10, 4, 8, 1, 2, 1, 11, 8, 11, 1], [9, 6, 4, 9, 3, 6, 9, 1, 3, 11, 6, 3],
    [8, 11, 1, 8, 1, 0, 11, 6, 1, 9, 1, 4, 6, 4, 1], [3, 11, 6, 3, 6, 0, 0, 6, 4], [6, 4, 8, 11, 6, 8],
    [7, 10, 6, 7, 8, 10, 8, 9, 10], [0, 7, 3, 0, 10, 7, 0, 9, 10, 6, 7, 10], [10, 6, 7, 1, 10, 7, 1, 7, 8, 1, 8, 0],
    [10, 6, 7, 10, 7, 1, 1, 7, 3], [1, 2, 6, 1, 6, 8, 1, 8, 9, 8, 6, 7],
    [2, 6, 9, 2, 9, 1, 6, 7, 9, 0, 9, 3, 7, 3, 9], [7, 8, 0, 7, 0, 6, 6, 0, 2], [7, 3, 2, 6, 7, 2],
    [2, 3, 11, 10, 6, 8, 10, 8, 9, 8, 6, 7], [2, 0, 7, 2, 7, 11, 0, 9, 7, 6, 7, 10, 9, 10, 7],
    [1, 8, 0, 1, 7, 8, 1, 10, 7, 6, 7, 10, 2, 3, 11], [11, 2, 1, 11, 1, 7, 10, 6, 1, 6, 7, 1],
    [8, 9, 6, 8, 6, 7, 9, 1, 6, 11, 6, 3, 1, 3, 6], [0, 9, 1, 11, 6, 7], [7, 8, 0, 7, 0, 6, 3, 11, 0, 11, 6, 0],
    [7, 11, 6], [7, 6, 11], [3, 0, 8, 11, 7, 6], [0, 1, 9, 11, 7, 6], [8, 1, 9, 8, 3, 1, 11, 7, 6],
    [10, 1, 2, 6, 11, 7], [1, 2, 10, 3, 0, 8, 6, 11, 7], [2, 9, 0, 2, 10, 9, 6, 11, 7],
    [6, 11, 7, 2, 10, 3, 10, 8, 3, 10, 9, 8], [7, 2, 3, 6, 2, 7], [7, 0, 8, 7, 6, 0, 6, 2, 0],
    [2, 7, 6, 2, 3, 7, 0, 1, 9], [1, 6, 2, 1, 8, 6, 1, 9, 8, 8, 7, 6], [10, 7, 6, 10, 1, 7, 1, 3, 7],
    [10, 7, 6, 1, 7, 10, 1, 8, 7, 1, 0, 8], [0, 3, 7, 0, 7, 10, 0, 10, 9, 6, 10, 7], [7, 6, 10, 7, 10, 8, 8, 10, 9],
    [6, 8, 4, 11, 8, 6], [3, 6, 11, 3, 0, 6, 0, 4, 6], [8, 6, 11, 8, 4, 6, 9, 0, 1],
    [9, 4, 6, 9, 6, 3, 9, 3, 1, 11, 3, 6], [6, 8, 4, 6, 11, 8, 2, 10, 1], [1, 2, 10, 3, 0, 11, 0, 6, 11, 0, 4, 6],
    [4, 11, 8, 4, 6, 11, 0, 2, 9, 2, 10, 9], [10, 9, 3, 10, 3, 2, 9, 4, 3, 11, 3, 6, 4, 6, 3],
    [8, 2, 3, 8, 4, 2, 4, 6, 2], [0, 4, 2, 4, 6, 2], [1, 9, 0, 2, 3, 4, 2, 4, 6, 4, 3, 8], [1, 9, 4, 1, 4, 2, 2, 4, 6],
    [8, 1, 3, 8, 6, 1, 8, 4, 6, 6, 10, 1], [10, 1, 0, 10, 0, 6, 6, 0, 4],
    [4, 6, 3, 4, 3, 8, 6, 10, 3, 0, 3, 9, 10, 9, 3], [10, 9, 4, 6, 10, 4], [4, 9, 5, 7, 6, 11],
    [0, 8, 3, 4, 9, 5, 11, 7, 6], [5, 0, 1, 5, 4, 0, 7, 6, 11], [11, 7, 6, 8, 3, 4, 3, 5, 4, 3, 1, 5],
    [9, 5, 4, 10, 1, 2, 7, 6, 11], [6, 11, 7, 1, 2, 10, 0, 8, 3, 4, 9, 5], [7, 6, 11, 5, 4, 10, 4, 2, 10, 4, 0, 2],
    [3, 4, 8, 3, 5, 4, 3, 2, 5, 10, 5, 2, 11, 7, 6], [7, 2, 3, 7, 6, 2, 5, 4, 9],
    [9, 5, 4, 0, 8, 6, 0, 6, 2, 6, 8, 7], [3, 6, 2, 3, 7, 6, 1, 5, 0, 5, 4, 0],
    [6, 2, 8, 6, 8, 7, 2, 1, 8, 4, 8, 5, 1, 5, 8], [9, 5, 4, 10, 1, 6, 1, 7, 6, 1, 3, 7],
    [1, 6, 10, 1, 7, 6, 1, 0, 7, 8, 7, 0, 9, 5, 4], [4, 0, 10, 4, 10, 5, 0, 3, 10, 6, 10, 7, 3, 7, 10],
    [7, 6, 10, 7, 10, 8, 5, 4, 10, 4, 8, 10], [6, 9, 5, 6, 11, 9, 11, 8, 9], [3, 6, 11, 0, 6, 3, 0, 5, 6, 0, 9, 5],
    [0, 11, 8, 0, 5, 11, 0, 1, 5, 5, 6, 11], [6, 11, 3, 6, 3, 5, 5, 3, 1], [1, 2, 10, 9, 5, 11, 9, 11, 8, 11, 5, 6],
    [0, 11, 3, 0, 6, 11, 0, 9, 6, 5, 6, 9, 1, 2, 10], [11, 8, 5, 11, 5, 6, 8, 0, 5, 10, 5, 2, 0, 2, 5],
    [6, 11, 3, 6, 3, 5, 2, 10, 3, 10, 5, 3], [5, 8, 9, 5, 2, 8, 5, 6, 2, 3, 8, 2], [9, 5, 6, 9, 6, 0, 0, 6, 2],
    [1, 5, 8, 1, 8, 0, 5, 6, 8, 3, 8, 2, 6, 2, 8], [1, 5, 6, 2, 1, 6],
    [1, 3, 6, 1, 6, 10, 3, 8, 6, 5, 6, 9, 8, 9, 6], [10, 1, 0, 10, 0, 6, 9, 5, 0, 5, 6, 0], [0, 3, 8, 5, 6, 10],
    [10, 5, 6], [11, 5, 10, 7, 5, 11], [11, 5, 10, 11, 7, 5, 8, 3, 0], [5, 11, 7, 5, 10, 11, 1, 9, 0],
    [10, 7, 5, 10, 11, 7, 9, 8, 1, 8, 3, 1], [11, 1, 2, 11, 7, 1, 7, 5, 1], [0, 8, 3, 1, 2, 7, 1, 7, 5, 7, 2, 11],
    [9, 7, 5, 9, 2, 7, 9, 0, 2, 2, 11, 7], [7, 5, 2, 7, 2, 11, 5, 9, 2, 3, 2, 8, 9, 8, 2],
    [2, 5, 10, 2, 3, 5, 3, 7, 5], [8, 2, 0, 8, 5, 2, 8, 7, 5, 10, 2, 5], [9, 0, 1, 5, 10, 3, 5, 3, 7, 3, 10, 2],
    [9, 8, 2, 9, 2, 1, 8, 7, 2, 10, 2, 5, 7, 5, 2], [1, 3, 5, 3, 7, 5], [0, 8, 7, 0, 7, 1, 1, 7, 5],
    [9, 0, 3, 9, 3, 5, 5, 3, 7], [9, 8, 7, 5, 9, 7], [5, 8, 4, 5, 10, 8, 10, 11, 8],
    [5, 0, 4, 5, 11, 0, 5, 10, 11, 11, 3, 0], [0, 1, 9, 8, 4, 10, 8, 10, 11, 10, 4, 5],
    [10, 11, 4, 10, 4, 5, 11, 3, 4, 9, 4, 1, 3, 1, 4], [2, 5, 1, 2, 8, 5, 2, 11, 8, 4, 5, 8],
    [0, 4, 11, 0, 11, 3, 4, 5, 11, 2, 11, 1, 5, 1, 11], [0, 2, 5, 0, 5, 9, 2, 11, 5, 4, 5, 8, 11, 8, 5],
    [9, 4, 5, 2, 11, 3], [2, 5, 10, 3, 5, 2, 3, 4, 5, 3, 8, 4], [5, 10, 2, 5, 2, 4, 4, 2, 0],
    [3, 10, 2, 3, 5, 10, 3, 8, 5, 4, 5, 8, 0, 1, 9], [5, 10, 2, 5, 2, 4, 1, 9, 2, 9, 4, 2],
    [8, 4, 5, 8, 5, 3, 3, 5, 1], [0, 4, 5, 1, 0, 5], [8, 4, 5, 8, 5, 3, 9, 0, 5, 0, 3, 5], [9, 4, 5],
    [4, 11, 7, 4, 9, 11, 9, 10, 11], [0, 8, 3, 4, 9, 7, 9, 11, 7, 9, 10, 11], [1, 10, 11, 1, 11, 4, 1, 4, 0, 7, 4, 11],
    [3, 1, 4, 3, 4, 8, 1, 10, 4, 7, 4, 11, 10, 11, 4], [4, 11, 7, 9, 11, 4, 9, 2, 11, 9, 1, 2],
    [9, 7, 4, 9, 11, 7, 9, 1, 11, 2, 11, 1, 0, 8, 3], [11, 7, 4, 11, 4, 2, 2, 4, 0],
    [11, 7, 4, 11, 4, 2, 8, 3, 4, 3, 2, 4], [2, 9, 10, 2, 7, 9, 2, 3, 7, 7, 4, 9],
    [9, 10, 7, 9, 7, 4, 10, 2, 7, 8, 7, 0, 2, 0, 7], [3, 7, 10, 3, 10, 2, 7, 4, 10, 1, 10, 0, 4, 0, 10],
    [1, 10, 2, 8, 7, 4], [4, 9, 1, 4, 1, 7, 7, 1, 3], [4, 9, 1, 4, 1, 7, 0, 8, 1, 8, 7, 1], [4, 0, 3, 7, 4, 3],
    [4, 8, 7], [9, 10, 8, 10, 11, 8], [3, 0, 9, 3, 9, 11, 11, 9, 10], [0, 1, 10, 0, 10, 8, 8, 10, 11],
    [3, 1, 10, 11, 3, 10], [1, 2, 11, 1, 11, 9, 9, 11, 8], [3, 0, 9, 3, 9, 11, 1, 2, 9, 2, 11, 9], [0, 2, 11, 8, 0, 11],
    [3, 2, 11], [2, 3, 8, 2, 8, 10, 10, 8, 9], [9, 10, 2, 0, 9, 2], [2, 3, 8, 2, 8, 10, 0, 1, 8, 1, 10, 8],
    [1, 10, 2], [1, 3, 8, 9, 1, 8], [0, 9, 1], [0, 3, 8], [],
]
TRI_TABLE = np.full((256, 16), -1, dtype=np.int32)
for _i, _row in enumerate(_TRI):
  TRI_TABLE[_i, :len(_row)] = _row
TRI_COUNT = (TRI_TABLE >= 0).sum(axis=1) // 3
del _i, _row


def multiplier(width, height, fx, fy, cx, cy):
  """[H, W] fp32 depth-to-camera-distance multiplier (fp64, rounded once)."""
  a = (np.arange(width, dtype=np.float64) - cx) / fx
  b = (np.arange(height, dtype=np.float64) - cy) / fy
  m = np.sqrt((1.0 + a[None, :] * a[None, :]) + b[:, None] * b[:, None])
  return m.astype(np.float32)


def _affine(M, x, y, z):
  return tuple(((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3] for r in range(3))


def touched_units(depth, intrinsic, pose, voxel_length, sdf_trunc, res=RES, stride=4):
  """[n, 3] int64 unit coordinates touched by the depth image, in first-occurrence order."""
  W, H, fx, fy, cx, cy = intrinsic
  L = voxel_length * res
  ii, jj = np.meshgrid(np.arange(0, H, stride), np.arange(0, W, stride), indexing='ij')
  d = depth[ii, jj].astype(np.float64).ravel()
  i, j = ii.ravel().astype(np.float64), jj.ravel().astype(np.float64)
  keep = d > 0
  d, i, j = d[keep], i[keep], j[keep]
  x = ((j - cx) * d) / fx
  y = ((i - cy) * d) / fy
  p = np.stack(_affine(pose, x, y, d), axis=1)
  lo = np.floor((p - sdf_trunc) / L).astype(np.int64)
  hi = np.floor((p + sdf_trunc) / L).astype(np.int64)
  side = int(np.floor(2 * sdf_trunc / L)) + 2
  assert (hi - lo < side).all()
  o = np.stack(np.meshgrid(np.arange(side), np.arange(side), np.arange(side), indexing='ij'), -1).reshape(-1, 3)
  cand = lo[:, None, :] + o[None, :, :]                          # [n, side^3, 3], x outermost
  ok = (cand <= hi[:, None, :]).all(axis=2)
  cand = cand[ok]
  if len(cand) == 0:
    return np.zeros((0, 3), np.int64)
  if cand.min() < SENTINEL_RANGE[0] or cand.max() > SENTINEL_RANGE[1]:
    raise ValueError('unit coordinate outside the 21-bit key range')
  _, first = np.unique(cand, axis=0, return_index=True)
  return cand[np.sort(first)]


class Volume:
  """The state of one ScalableTSDFVolume: unit keys in slot order and the fp32 slabs [n, R^3] (colour [n, 3, R^3])."""

  def __init__(self, voxel_length, sdf_trunc, color=False, res=RES, stride=4):
    if res != RES:
      raise ValueError('volume_unit_resolution must be 16')
    self.voxel_length, self.sdf_trunc, self.color, self.res, self.stride = voxel_length, sdf_trunc, color, res, stride
    self.keys = np.zeros((0, 3), np.int64)
    self.slot = {}
    self.tsdf = np.zeros((0, RES ** 3), np.float32)
    self.weight = np.zeros((0, RES ** 3), np.float32)
    self.rgb = np.zeros((0, 3, RES ** 3), np.float32)
    self.last_touched = np.zeros(0, np.int64)

  def integrate(self, depth, intrinsic, extrinsic, color=None):
    """depth: [H, W] float32 metres (0 = none); intrinsic (W, H, fx, fy, cx, cy); extrinsic 4x4 world-to-camera;
    color: [H, W, 3] uint8 (RGB8 volumes)."""
    W, H, fx, fy, cx, cy = intrinsic
    depth = np.asarray(depth, np.float32)
    if depth.shape != (H, W):
      raise ValueError('depth size differs from the intrinsic')
    if self.color and (color is None or color.dtype != np.uint8 or color.shape != (H, W, 3)):
      raise ValueError('an RGB8 volume needs [H, W, 3] uint8 colour')
    E = np.asarray(extrinsic, np.float64)
    pose = np.linalg.inv(E)
    units = touched_units(depth, intrinsic, pose, self.voxel_length, self.sdf_trunc, self.res, self.stride)
    new = [u for u in map(tuple, units) if u not in self.slot]
    for u in new:
      self.slot[u] = len(self.slot)
    if new:
      k = len(new)
      self.keys = np.concatenate([self.keys, np.array(new, np.int64)])
      self.tsdf = np.concatenate([self.tsdf, np.zeros((k, RES ** 3), np.float32)])
      self.weight = np.concatenate([self.weight, np.zeros((k, RES ** 3), np.float32)])
      self.rgb = np.concatenate([self.rgb, np.zeros((k, 3, RES ** 3), np.float32)])
    slots = np.array([self.slot[u] for u in map(tuple, units)], np.int64)
    self.last_touched = slots
    if len(slots) == 0:
      return
    vl, L = self.voxel_length, self.voxel_length * RES
    loc = np.stack(np.meshgrid(np.arange(RES), np.arange(RES), np.arange(RES), indexing='ij'), -1).reshape(-1, 3)
    cen = self.keys[slots][:, None, :].astype(np.float64) * L + (loc[None].astype(np.float64) + 0.5) * vl
    X, Y, Z = cen[..., 0], cen[..., 1], cen[..., 2]
    cx_, cy_, cz_ = _affine(E, X, Y, Z)
    ok = cz_ > 0
    zs = np.where(ok, cz_, 1.0)
    uf = ((cx_ * fx) / zs + cx) + 0.5
    vf = ((cy_ * fy) / zs + cy) + 0.5
    ok &= (uf >= 0.0001) & (uf < W - 0.0001) & (vf >= 0.0001) & (vf < H - 0.0001)
    u = np.where(ok, uf, 0).astype(np.int64)
    v = np.where(ok, vf, 0).astype(np.int64)
    d = depth[v, u]
    ok &= d > 0
    mult = multiplier(W, H, fx, fy, cx, cy)
    sdf = (d.astype(np.float64) - cz_).astype(np.float32) * mult[v, u]
    trunc32 = np.float32(self.sdf_trunc)
    inv32 = np.float32(1.0 / self.sdf_trunc)
    ok &= sdf > -trunc32
    tsdf_new = np.minimum(np.float32(1), sdf * inv32)
    t0, w0 = self.tsdf[slots], self.weight[slots]
    w1 = w0 + np.float32(1)
    self.tsdf[slots] = np.where(ok, (t0 * w0 + tsdf_new) / w1, t0)
    if self.color:
      for c in range(3):
        c0 = self.rgb[slots, c]
        rgb = color[v, u, c].astype(np.float32)
        self.rgb[slots, c] = np.where(ok, (c0 * w0 + rgb) / w1, c0)
    self.weight[slots] = np.where(ok, w1, w0)

  def extract_triangle_mesh(self):
    """-> (vertices [nv, 3] fp64, colours [nv, 3] fp64 or None, triangles [nt, 3] int32), canonical order."""
    n = len(self.keys)
    if n == 0:
      return np.zeros((0, 3)), (np.zeros((0, 3)) if self.color else None), np.zeros((0, 3), np.int32)
    R = RES
    nb = np.full((n, 2, 2, 2), -1, np.int64)
    for s, k in enumerate(map(tuple, self.keys)):
      for dx in (0, 1):
        for dy in (0, 1):
          for dz in (0, 1):
            nb[s, dx, dy, dz] = self.slot.get((k[0] + dx, k[1] + dy, k[2] + dz), -1)
    # [n, 17, 17, 17] halo of tsdf / weight
    E = R + 1
    ax = np.arange(E)
    bx, lx = ax // R, ax % R
    B = nb[:, bx[:, None, None], bx[None, :, None], bx[None, None, :]]          # [n, E, E, E]
    lin = (lx[:, None, None] * R + lx[None, :, None]) * R + lx[None, None, :]
    Bc = np.maximum(B, 0)
    ft = np.where(B >= 0, self.tsdf[Bc, np.broadcast_to(lin, B.shape)], np.float32(0))
    fw = np.where(B >= 0, self.weight[Bc, np.broadcast_to(lin, B.shape)], np.float32(0))
    idx = np.zeros((n, R, R, R), np.int32)
    kept = np.ones((n, R, R, R), bool)
    for c, (ox, oy, oz) in enumerate(CORNERS):
      f = ft[:, ox:ox + R, oy:oy + R, oz:oz + R]
      w = fw[:, ox:ox + R, oy:oy + R, oz:oz + R]
      kept &= w != 0
      idx |= (f < 0).astype(np.int32) << c
    kept &= (idx != 0) & (idx != 255)
    idx = np.where(kept, idx, 0)
    # vertex keys: (owner unit slot, owner voxel, axis) of every sign-changing edge of a kept cube
    g = (self.keys[:, None, None, None, :] * R
         + np.stack(np.meshgrid(ax[:R], ax[:R], ax[:R], indexing='ij'), -1)[None])          # [n, R, R, R, 3]
    keyset = set()
    s_i, x_i, y_i, z_i = np.nonzero(kept)
    cube_idx = idx[s_i, x_i, y_i, z_i]
    for e in range(12):
      has = (EDGE_TABLE[cube_idx] >> e) & 1 == 1
      o = EDGE_OWNER[e]
      own = g[s_i[has], x_i[has], y_i[has], z_i[has]] + o
      for q in map(tuple, own):
        keyset.add(q + (int(EDGE_AXIS[e]),))
    verts_key = []
    for q in keyset:
      unit = tuple(np.floor_divide(q[:3], R))
      loc = np.mod(q[:3], R)
      verts_key.append((self.slot[unit], (loc[0] * R + loc[1]) * R + loc[2], q[3], q[:3]))
    verts_key.sort()
    vid = {(k[3], k[2]): i for i, k in enumerate(verts_key)}
    nv = len(verts_key)
    V = np.zeros((nv, 3))
    Cc = np.zeros((nv, 3)) if self.color else None
    vl = self.voxel_length
    for i, (s, lv, a, q) in enumerate(verts_key):
      q1 = list(q)
      q1[a] += 1
      s1 = self.slot[tuple(np.floor_divide(q1, R))]
      l1 = np.mod(q1, R)
      lv1 = (l1[0] * R + l1[1]) * R + l1[2]
      f0, f1 = float(self.tsdf[s, lv]), float(self.tsdf[s1, lv1])
      a0, a1 = abs(f0), abs(f1)
      p = [(float(q[k]) + 0.5) * vl for k in range(3)]
      p[a] = p[a] + (a0 * vl) / (a0 + a1)
      V[i] = p
      if self.color:
        for c in range(3):
          c0, c1 = float(self.rgb[s, c, lv]), float(self.rgb[s1, c, lv1])
          Cc[i, c] = ((a1 * c0 + a0 * c1) / (a0 + a1)) / 255.0
    tris = []
    order = np.lexsort((z_i, y_i, x_i, s_i))
    for t in order:
      s, x, y, z, ci = s_i[t], x_i[t], y_i[t], z_i[t], cube_idx[t]
      gg = g[s, x, y, z]
      row = TRI_TABLE[ci]
      for k in range(TRI_COUNT[ci]):
        e = row[3 * k:3 * k + 3]
        ids = [vid[(tuple(int(c) for c in gg + EDGE_OWNER[ee]), int(EDGE_AXIS[ee]))] for ee in e]
        tris.append((ids[0], ids[2], ids[1]))
    T = np.array(tris, np.int32).reshape(-1, 3)
    return V, Cc, T


def depth_from_raw(raw, depth_scale=1000.0, depth_trunc=3.0):
  """open3d's float depth of create_from_color_and_depth: float32(raw) / float32(scale), 0 where >= trunc."""
  d = np.asarray(raw).astype(np.float32) / np.float32(depth_scale)
  d[d >= np.float32(depth_trunc)] = 0
  return d
