"""oracle/tsdf_raycast.py on the CPU: a fused volume renders the synthetic renderer's depth, every march step
is positive and within the documented bound, and a missing-unit jump leaves its unit only in its last half voxel."""
import numpy as np
import pytest

from deepglobalregistration_b200 import synthetic as syn
from oracle import tsdf as ot
from oracle import tsdf_raycast as orc

VL, TRUNC = 0.02, 0.06


@pytest.fixture(scope='module')
def fused():
  c, d, P, K = syn.rgbd_sequence(3, 8, width=160, height=120, turn=0.05, radius=0.05)
  ov = ot.Volume(VL, TRUNC, color=True)
  for k in range(len(P)):
    ov.integrate(ot.depth_from_raw(d[k], 1000.0, 4.5), (160, 120) + tuple(K), np.linalg.inv(P[k]), c[k])
  return c, d, P, K, ov


def test_depth_matches_the_renderer(fused):
  # 160 x 120, 2 cm voxels, 8 frames fused, weight_threshold 3.  Measured (frames 0, 4, 7): hit share 0.89 / 0.95 /
  # 0.91, median |error| 5.8 / 6.3 / 5.8 mm, 95th percentile 19 / 21 / 20 mm.  The sample is the voxel
  # holding p, not an interpolation, so the crossing is off by up to half a voxel; the share is lowest at the ends
  # of the path, whose view edges fewer than 3 frames saw.
  c, d, P, K, ov = fused
  for k in (0, 4, 7):
    D, I, Col = orc.raycast(ov, (160, 120) + tuple(K), np.linalg.inv(P[k]))
    gt = d[k].astype(np.float32) / np.float32(1000.0)
    both = (D > 0) & (gt > 0)
    err = np.abs(D - gt)[both]
    share = both.sum() / max((gt > 0).sum(), 1)
    print(f'[oracle raycast] frame {k}: hit share {share:.4f}, median {np.median(err) * 1e3:.2f} mm, '
          f'p95 {np.percentile(err, 95) * 1e3:.2f} mm')
    assert share >= 0.85
    assert np.median(err) <= 0.01 and np.percentile(err, 95) <= 0.035
    assert ((I > 0) == (D > 0)).mean() >= 0.99           # a hit has colour (every face colour is non-black)
    assert I.dtype == Col.dtype == D.dtype == np.float32 and 0 <= Col.min() and Col.max() <= 1


def _trace(ov, K, P, **kw):
  tr = {}
  orc.raycast(ov, (160, 120) + tuple(K), np.linalg.inv(P), trace=tr, **kw)
  return tr


@pytest.mark.parametrize('where', ['fused', 'outside'])
def test_steps_positive_and_bounded(fused, where):
  c, d, P, K, ov = fused
  pose = P[2].copy()
  if where == 'outside':                          # 6 m behind the first camera: a long run of missing units first
    pose[:3, 3] -= 6.0 * pose[:3, 2]
  depth_min, depth_max = 0.1, 9.0
  tr = _trace(ov, K, pose, depth_min=depth_min, depth_max=depth_max)
  W, H, fx, fy, cx, cy = (160, 120) + tuple(K)
  vv, uu = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
  a, b = (uu.ravel() - cx) / fx, (vv.ravel() - cy) / fy
  s = np.linalg.norm(np.stack([a, b, np.ones_like(a)], 1) @ pose[:3, :3].T, axis=1)
  n_steps = np.zeros(H * W, np.int64)
  for ray, t0, t1, kind in tr['steps']:
    assert (t1 - t0 > 0).all()
    assert (t1 - t0 >= (0.5 * VL) / s[ray] * (1 - 1e-9)).all()
    n_steps[ray] += 1
  bound = np.ceil(2 * s * (depth_max - depth_min) / VL) + 1
  cap = orc.max_steps((W, H, fx, fy, cx, cy), pose, VL, depth_max)
  print(f'[oracle raycast] {where}: steps per ray mean {n_steps.mean():.1f}, max {n_steps.max()}, '
        f'bound min {bound.min():.0f}, launch cap {cap:.0f}; probes per ray {tr["probes"].mean():.1f}')
  assert (n_steps <= bound).all() and bound.max() <= cap


def test_step_bound():
  # s_max sits at a corner pixel: no pixel's ray is longer per unit of t
  rng = np.random.default_rng(0)
  K = (640, 480, 585.0, 585.0, 320.0, 240.0)
  for _ in range(20):
    pose = np.eye(4)
    pose[:3, :3] = syn.random_se3(rng, max_angle_deg=180.0, max_trans=0.0)[:3, :3] * rng.uniform(0.5, 2.0)
    vv, uu = np.meshgrid(np.arange(480.0), np.arange(640.0), indexing='ij')
    dirs = np.stack([(uu.ravel() - 320.0) / 585.0, (vv.ravel() - 240.0) / 585.0, np.ones(640 * 480)], 1) @ pose[:3, :3].T
    s_all = np.linalg.norm(dirs, axis=1).max()
    assert orc.max_steps(K, pose, 0.008, 3.0) == np.ceil(2 * s_all * 3.0 / 0.008) + 1
  # VGA at 8 mm to depth 3 m: about 900 steps, far below the limit
  assert 900 <= orc.max_steps(K, np.eye(4), 0.008, 3.0) <= 920
  # a tiny focal length, a far principal point or a shrinking extrinsic make s unbounded: refused, not marched
  vol = ot.Volume(VL, TRUNC)
  for k, ext in (((640, 480, 1e-30, 1e-30, 320.0, 240.0), np.eye(4)), ((640, 480, 585.0, 585.0, 1e9, 240.0), np.eye(4)),
                 (K, np.diag([1e-4, 1e-4, 1e-4, 1.0]))):
    with pytest.raises(ValueError):
      orc.raycast(vol, k, ext)


def test_missing_unit_jump_stays_in_its_unit(fused):
  # The jump goes to the unit's exit plus half a voxel: every point of the jumped segment except its last half
  # voxel lies in the missing unit, so an allocated unit is never skipped by more than half a voxel's length.
  c, d, P, K, ov = fused
  pose = P[5].copy()
  pose[:3, 3] -= 6.0 * pose[:3, 2]
  tr = _trace(ov, K, pose, depth_min=0.1, depth_max=9.0)
  W, H, fx, fy, cx, cy = (160, 120) + tuple(K)
  vv, uu = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
  a, b = (uu.ravel() - cx) / fx, (vv.ravel() - cy) / fy
  dirs = np.stack([a, b, np.ones_like(a)], 1) @ pose[:3, :3].T
  s = np.linalg.norm(dirs, axis=1)
  jumps = 0
  for ray, t0, t1, kind in tr['steps']:
    m = kind == 0
    ray, t0, t1 = ray[m], t0[m], t1[m]
    if not len(ray):
      continue
    jumps += len(ray)
    end = t1 - (0.5 * VL) / s[ray]
    unit0 = np.floor(np.floor((pose[:3, 3] + t0[:, None] * dirs[ray]) / VL) / 16)
    for j in range(16):
      tj = t0 + (end - t0) * (j / 16)
      u = np.floor(np.floor((pose[:3, 3] + tj[:, None] * dirs[ray]) / VL) / 16)
      assert (u == unit0).all()
      assert not any(tuple(int(x) for x in q) in ov.slot for q in u[:4096])
  assert jumps > 10_000
