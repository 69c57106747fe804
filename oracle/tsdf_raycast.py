"""ORACLE (test infrastructure only) - ray casting a TSDF volume: raycast(vol, ...) renders depth, intensity and
colour from an oracle/tsdf.py Volume.  This module is the arithmetic contract of csrc/tsdf.cu's dgr_tsdf_raycast: the
kernel must meet it bit for bit, so it fixes the order of every floating-point operation ("fp64": numpy float64
element-wise ops, "fp32": numpy float32 ops; numpy rounds every op to nearest and never contracts a multiply-add).

PARITY UNPINNED: open3d is not installed here and not vendored; every reading of open3d below is a restatement from
memory, recorded as an assumption.

Ray casting is a project extension: legacy open3d's ScalableTSDFVolume has none.  Readings of open3d's tensor
VoxelBlockGrid.ray_cast / t.pipelines.slam.Model, recorded as assumptions: the defaults depth_min 0.1, depth_max 3.0, weight_threshold 3.0; a sample counts only where its
weight reaches weight_threshold; a missing block is jumped over; inside the band the ray advances by max(tsdf
sdf_trunc, voxel_length); the surface is the first + to - crossing, its t interpolated linearly; the dense SLAM
model renders frame k with weight_threshold min(k, 3).  The contract, fp64 unless stated:
  * Ray of pixel (u, v): a = (u - cx) / fx, b = (v - cy) / fy; with P = camera_pose = inv(extrinsic) (np.linalg.inv on
    the host), d_r = (P[r,0] a + P[r,1] b) + P[r,2], C_r = P[r,3], s = sqrt((d0 d0 + d1 d1) + d2 d2) (world length of
    one unit of t).  p(t)_r = C_r + t d_r; t is the depth along the optical axis.  Pixel u's centre is u, as in
    integration (pixel u covers projections [u - 0.5, u + 0.5)).
  * Sample at t: voxel g_r = floor(p(t)_r / voxel_length) (centre (g + 0.5) voxel_length), unit U_r = floor(g_r *
    0.0625), local index ((g0 - 16 U0) 16 + (g1 - 16 U1)) 16 + (g2 - 16 U2).  A unit outside SENTINEL_RANGE is
    missing.  Known: the unit exists and float64(weight) >= weight_threshold.
  * March from t = depth_min while t <= depth_max (a NaN t ends the ray):
      - missing unit: t_e = the least (((U_r 16) + (16 if d_r > 0 else 0)) voxel_length - C_r) / d_r over axes with
        d_r != 0; t <- max(t_e, t) + (0.5 voxel_length) / s.  No sample of the jumped segment lies outside that unit
        except in its last half voxel (world length), so the jump can cut the corner of an allocated unit by at most
        half a voxel, never skip more of it;
      - existing unit, unknown voxel: t <- t + voxel_length / s;
      - known voxel f (fp32): if the previous sample was known with f_prev > 0 and f <= 0, the hit is t_h = t_prev +
        (t - t_prev) (f_prev / (f_prev - f)), reported when depth_min <= t_h <= depth_max, and the ray ends; else
        t_prev, f_prev <- t, f and t <- t + max(f sdf_trunc, voxel_length) / s.
    The pair is the last known sample and the current one: an unknown voxel in between keeps it (a voxel at the
    surface can stay unobserved), a missing-unit jump breaks it (open3d's kernel, as read, keeps the previous tsdf
    across a skipped block too; here no surface is interpolated across a unit nobody observed).
  * Termination.  Every step is at least (0.5 voxel_length) / s in t, so a ray takes at most ceil(2 s (depth_max -
    depth_min) / voxel_length) + 1 steps.  s = |R (a, b, 1)| is convex in (a, b), so its largest value over the image,
    s_max, is at one of the four corner pixels (u in {0, W - 1}, v in {0, H - 1}, the same formulas); max_steps =
    ceil(((2 s_max) depth_max) / voxel_length) + 1 (about 900 for VGA at 8 mm and depth_max 3) bounds every ray.
    Arguments whose max_steps exceeds MAX_STEPS (DGR_TSDF_RAYCAST_MAX_STEPS) are refused before anything runs: a tiny
    focal length, a far principal point or a shrinking extrinsic would otherwise make s, and the march, unbounded.
    Within the limit every step is at least depth_max / 65535, far above t's rounding, so t always moves.  A ray also
    stops after max_steps samples; by the bound this never cuts a ray short, it only makes termination structural.
  * Colour (RGB8) at p(t_h): q_r = p_r / voxel_length - 0.5, g0 = floor(q), fr = q - g0; corners c = 0..7 at g0 +
    (c >> 2, (c >> 1) & 1, c & 1) in that order, each present when its unit exists and its weight > 0, weighted
    ((w0 w1) w2) with w_r = fr_r or 1 - fr_r; acc += w rgb, wsum += w in corner order; rgb = float32(acc / wsum) (0
    when wsum is 0).  intensity = ((r 0.299 + g 0.587) + b 0.114) / 255 in fp32 (create_from_color_and_depth's
    formula on the float colour), colour = rgb / 255 in fp32.  Depth float32(t_h).  0 everywhere without a hit.
"""
import numpy as np

from .tsdf import RES, SENTINEL_RANGE

MAX_STEPS = 65536          # DGR_TSDF_RAYCAST_MAX_STEPS


def max_steps(intrinsic, pose, voxel_length, depth_max):
  """The launch's step bound ceil(((2 s_max) depth_max) / voxel_length) + 1; pose = camera_pose (4x4)."""
  W, H, fx, fy, cx, cy = intrinsic
  s_max = 0.0
  for c in range(4):
    a = (float(W - 1 if c & 1 else 0) - cx) / fx
    b = (float(H - 1 if c & 2 else 0) - cy) / fy
    d = [(pose[r, 0] * a + pose[r, 1] * b) + pose[r, 2] for r in range(3)]
    s = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    s_max = s if s > s_max else s_max
  return np.ceil(((2.0 * s_max) * depth_max) / voxel_length) + 1.0


def _ray_units(g, table):
  """g [m, 3] fp64 lattice voxels -> (slot [m] (-1: missing), U [m, 3] fp64, local index [m])."""
  U = np.floor(g * 0.0625)
  ok = ((U >= SENTINEL_RANGE[0]) & (U <= SENTINEL_RANGE[1])).all(axis=1)
  Ui = np.where(ok[:, None], U, 0).astype(np.int64)
  gi = np.where(ok[:, None], g, 0).astype(np.int64)
  lv = ((gi[:, 0] - RES * Ui[:, 0]) * RES + (gi[:, 1] - RES * Ui[:, 1])) * RES + (gi[:, 2] - RES * Ui[:, 2])
  packed, order = table
  slot = np.full(len(g), -1, np.int64)
  if len(packed):
    key = _pack(Ui)
    at = np.minimum(np.searchsorted(packed, key), len(packed) - 1)
    found = ok & (packed[at] == key)
    slot[found] = order[at[found]]
  return slot, U, lv

def raycast(vol, intrinsic, extrinsic, depth_min=0.1, depth_max=3.0, weight_threshold=3.0, trace=None):
  """Render an oracle/tsdf.py Volume `vol` seen by a camera (intrinsic (W, H, fx, fy, cx, cy), extrinsic 4x4 world to camera) -> (depth [H, W] fp32,
  intensity [H, W] fp32, colour [H, W, 3] fp32), the last two None for NoColor.  trace: a dict that receives
  'probes' [H W] (unit lookups per ray, the colour's 8 included) and 'steps' [(ray, t, t_next, kind)] arrays per
  march iteration (kind 0: missing unit, 1: unknown voxel, 2: known voxel)."""
  W, H, fx, fy, cx, cy = intrinsic
  P = np.linalg.inv(np.asarray(extrinsic, np.float64))
  vl, trunc = vol.voxel_length, vol.sdf_trunc
  packed = _pack(vol.keys)
  order = np.argsort(packed, kind='stable')
  table = (packed[order], order)
  vv, uu = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
  a = (uu.ravel() - cx) / fx
  b = (vv.ravel() - cy) / fy
  d = np.stack([(P[r, 0] * a + P[r, 1] * b) + P[r, 2] for r in range(3)], axis=1)
  C = P[:3, 3].copy()
  s = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
  dt_vox, dt_half = vl / s, (0.5 * vl) / s
  n = H * W
  t = np.full(n, float(depth_min))
  tp, t_hit = np.zeros(n), np.zeros(n)
  fp = np.zeros(n, np.float32)
  prev, hit, done = np.zeros(n, bool), np.zeros(n, bool), np.zeros(n, bool)
  probes = np.zeros(n, np.int64)
  steps = []
  cap = max_steps(intrinsic, P, vl, depth_max)
  if not cap <= MAX_STEPS:
    raise ValueError(f'a ray could take {cap} steps, more than {MAX_STEPS}')
  iters = np.zeros(n, np.int64)
  active = np.arange(n)
  with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
    while True:
      active = active[~done[active] & (iters[active] < cap) & (t[active] <= depth_max)]
      if active.size == 0:
        break
      t0 = t[active].copy()
      g = np.floor((C[None, :] + t[active][:, None] * d[active]) / vl)
      slot, U, lv = _ray_units(g, table)
      probes[active] += 1
      iters[active] += 1
      kind = np.full(active.size, 2)
      miss = slot < 0
      m = active[miss]
      if m.size:
        dm = d[m]
        bnd = (U[miss] * 16.0 + np.where(dm > 0.0, 16.0, 0.0)) * vl
        tk = np.where(dm != 0.0, (bnd - C[None, :]) / dm, np.inf)
        te = np.full(m.size, np.inf)
        for r in range(3):
          te = np.where(tk[:, r] < te, tk[:, r], te)
        t[m] = np.where(te > t[m], te, t[m]) + dt_half[m]
        prev[m] = False
        kind[miss] = 0
      e, se, le = active[~miss], slot[~miss], lv[~miss]
      known = vol.weight[se, le].astype(np.float64) >= weight_threshold
      unk = e[~known]
      t[unk] = t[unk] + dt_vox[unk]
      kind[np.flatnonzero(~miss)[~known]] = 1
      k = e[known]
      f = vol.tsdf[se[known], le[known]]
      cross = prev[k] & (fp[k] > 0) & (f <= 0)
      c = k[cross]
      if c.size:
        fpc, fc = fp[c].astype(np.float64), f[cross].astype(np.float64)
        th = tp[c] + (t[c] - tp[c]) * (fpc / (fpc - fc))
        t_hit[c] = th
        hit[c] = (th >= depth_min) & (th <= depth_max)
        done[c] = True
      go, fg = k[~cross], f[~cross]
      prev[go] = True
      fp[go] = fg
      tp[go] = t[go]
      step = fg.astype(np.float64) * trunc
      t[go] = t[go] + np.where(step > vl, step, vl) / s[go]
      if trace is not None:
        moved = ~done[active]
        steps.append((active[moved], t0[moved], t[active[moved]], kind[moved]))
    depth = np.where(hit, t_hit.astype(np.float32), np.float32(0)).reshape(H, W)
    if not vol.color:
      if trace is not None:
        trace.update(probes=probes, steps=steps)
      return depth, None, None
    c32 = np.zeros((n, 3), np.float32)
    h = np.flatnonzero(hit)
    if h.size:
      q = (C[None, :] + t_hit[h][:, None] * d[h]) / vl - 0.5
      g0 = np.floor(q)
      fr = q - g0
      acc, wsum = np.zeros((h.size, 3)), np.zeros(h.size)
      for cc in range(8):
        o = np.array([cc >> 2, (cc >> 1) & 1, cc & 1], np.float64)
        slot, _, lv = _ray_units(g0 + o[None, :], table)
        sl = np.maximum(slot, 0)
        present = (slot >= 0) & (vol.weight[sl, lv] > 0)
        wr = [fr[:, r] if o[r] else 1.0 - fr[:, r] for r in range(3)]
        tw = (wr[0] * wr[1]) * wr[2]
        for r in range(3):
          acc[:, r] = np.where(present, acc[:, r] + tw * vol.rgb[sl, r, lv].astype(np.float64), acc[:, r])
        wsum = np.where(present, wsum + tw, wsum)
      probes[h] += 8
      c32[h] = np.where(wsum[:, None] > 0, (acc / wsum[:, None]).astype(np.float32), np.float32(0))
  intensity = ((c32[:, 0] * np.float32(0.299) + c32[:, 1] * np.float32(0.587)) + c32[:, 2] * np.float32(0.114)) \
      / np.float32(255.0)
  colour = c32 / np.float32(255.0)
  if trace is not None:
    trace.update(probes=probes, steps=steps)
  return depth, intensity.astype(np.float32).reshape(H, W), colour.astype(np.float32).reshape(H, W, 3)


def _pack(U):
  """[m, 3] int unit coordinates in the key range -> int64 keys (3 x 21 bits, as the library packs them)."""
  U = np.asarray(U, np.int64).reshape(-1, 3) + (1 << 20)
  return U[:, 0] | (U[:, 1] << 21) | (U[:, 2] << 42)
