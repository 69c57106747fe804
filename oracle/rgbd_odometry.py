"""ORACLE (test infrastructure only) - RGB-D odometry as open3d's legacy ``compute_rgbd_odometry`` runs it
(``odometry`` in open3d 0.10-0.12, ``pipelines.odometry`` in 0.12-0.17: RGBDOdometry.cpp, RGBDOdometryJacobian.cpp),
restated in numpy.  This module is the arithmetic contract of csrc/odometry.cu: the images (preprocessed, normalised,
pyramid, gradients) and the correspondence sets are met bit for bit, so their order of operations is fixed here.
"fp32" means numpy float32 element-wise ops, "fp64" numpy float64 element-wise ops; numpy rounds every op to nearest
and never contracts a multiply-add.  The Gauss-Newton sums and the information matrix are fp64 in numpy's order; the
device adds the same terms in another fixed order, so poses agree to rounding, not bit for bit.

PARITY UNPINNED: open3d is not installed here and not vendored, so every reading below is a restatement from memory of
open3d's published sources, recorded as an assumption.

Assumptions (readings of open3d):
  * Options.  OdometryOption(iteration_number_per_pyramid_level=[20, 10, 5], max_depth_diff=0.03, min_depth=0.0,
    max_depth=4.0); the list runs from the coarsest level to the finest.  An all-zero odo_init reads as the identity
    (open3d's ``init_odo.isZero()`` test), here for the normalisation too.
  * Initialisation (InitializeRGBDOdometry).  Depth d with d < min_depth, d > max_depth or d <= 0 (compared in fp64)
    becomes NaN.  Gaussian3 runs on both intensities and both depths: a horizontal pass, then a vertical one, each
    out = fp32(((0 + fp32(a k0)) + fp32(b k1)) + fp32(c k2)) with the sum in fp64, k = (0.25, 0.5, 0.25) and the
    border replicated (open3d's FilterHorizontal: float products added to a double, rounded once).  NaN spreads.
  * NormalizeIntensity.  The correspondences at odo_init on the full-resolution filtered depths; with n of them,
    mean = (sum of the filtered intensity at each match, fp64) / n per image, then every pixel v of that image becomes
    fp32(0.5 / mean * v + 0.0) (LinearTransformImage).
  * Pyramid (CreatePyramid(levels, false)).  Level l + 1 is fp32((((p00 + p10) + p01) + p11) / 4) of level l, size
    (W // 2, H // 2); the camera of level l is K / 2^l with K[2, 2] = 1.
  * Gradients (Sobel3Dx / Sobel3Dy on the target's intensity and depth at every level): d/dx is the horizontal pass
    (-1, 0, 1) then the vertical (1, 2, 1); d/dy the horizontal (1, 2, 1) then the vertical (-1, 0, 1), each pass as
    Gaussian3's.  They are scaled by SOBEL_SCALE = 0.125 (fp64) where used; a NaN depth gradient counts as 0.
  * Points (ConvertDepthImageToXYZImage).  Pixel (u, v) with depth d: x = fp32(((u - cx) d) / fx) computed as
    ((u - cx) d) (1 / fx) in fp64, y likewise, z = d; stored as float, as open3d's XYZ image.
  * Correspondences (ComputeCorrespondence).  For a source pixel with depth d: q = R p + t in fp64 (row a:
    ((R[a,0] x + R[a,1] y) + R[a,2] z) + t[a]); u_t = int((fx q_x + cx q_z) / q_z + 0.5), v_t likewise, int()
    truncating; kept if (u_t, v_t) lies in the image, the target depth there d_t is not NaN and |q_z - d_t| <=
    max_depth_diff.
  * Jacobians, at a match (source pixel s, target pixel t, q = T p_s, invz = 1 / q_z):
      c0 = (0.125 dI/dx fx) invz, c1 = (0.125 dI/dy fy) invz, c2 = -(c0 q_x + c1 q_y) invz;
      colour (RGBDOdometryJacobianFromColorTerm, Steinbruecker et al. 2011): r = fp32(I_t[t] - I_s[s]),
        J = [-q_z c1 + q_y c2, q_z c0 - q_x c2, -q_y c0 + q_x c1, c0, c1, c2];
      hybrid (RGBDOdometryJacobianFromHybridTerm, Park, Zhou & Koltun 2017): that row scaled by sqrt(1 - 0.968), and
        a geometric row scaled by sqrt(0.968) with d0, d1, d2 formed as c0, c1, c2 from the depth gradients:
        r = D_t[t] - q_z, J = [(-q_z d1 + q_y d2) - q_y, (q_z d0 - q_x d2) + q_x, -q_y d0 + q_x d1, d0, d1, d2 - 1].
  * Step.  J^T J x = -J^T r over all rows; T <- [Rz(x2) Ry(x1) Rx(x0) | x3..5] T.  Every level runs all its
    iterations (open3d has no convergence test); a failed solve ends the call with (False, I4, I6).
  * Information (CreateInformationMatrix).  The full-resolution correspondences at the final pose; the sum of G^T G
    over each match's TARGET point (x, y, z) (the float XYZ image of the target depth), G = [[0, z, -y, 1, 0, 0],
    [-z, 0, x, 0, 1, 0], [y, -x, 0, 0, 0, 1]] - the form of get_information_matrix_from_point_clouds.

Open point, reading taken.  open3d keys its correspondence map and depth buffer by the SOURCE pixel, which every pass
visits once, so the buffer never compares and several source pixels may claim one target pixel.  The buffer's evident
purpose is occlusion, so it is read here as a TARGET-pixel z-buffer: among the source pixels that land on a target
pixel the one with the smallest fp32(q_z) wins, a tie going to the lowest source pixel index (row-major); the set is
listed in target row-major order.

Departures (deliberate):
  * A transformed depth q_z <= 0 is rejected before the division (open3d divides; its depth test only lets such a
    pixel through when the target depth is below max_depth_diff).  It also keeps every z-buffer key positive.
  * The projection uses the float XYZ point the Jacobian uses; open3d projects d K R K^-1 (u, v, 1) + K t from the
    unrounded depth, which is the same point up to rounding.
  * The 6x6 solve is a Cholesky that fails on a pivot that is not positive (open3d: LDLT), as dgr_icp's.
  * A pair with no correspondence at odo_init fails (open3d divides by zero in NormalizeIntensity).
  * The normalisation sums are added in the device's order (norm_sums below): per target row, lane l of 32 adds
    columns l, l + 32, ... in order, the lanes are combined by an xor butterfly 16, 8, 4, 2, 1, and the rows are added
    in order.
"""
import math

import numpy as np

SOBEL_SCALE = 0.125
LAMBDA_HYBRID_DEPTH = 0.968
GAUSS = (0.25, 0.5, 0.25)
DIFF = (-1.0, 0.0, 1.0)
SMOOTH = (1.0, 2.0, 1.0)


def preprocess_depth(depth, min_depth, max_depth):
  d = np.array(depth, np.float32)
  dd = d.astype(np.float64)
  d[(dd < min_depth) | (dd > max_depth) | (dd <= 0.0)] = np.nan
  return d


def filter_pass(img, kernel, vertical):
  """One FilterHorizontal pass (vertical: along rows), replicated border: fp32 products summed in fp64 from +0."""
  a = np.asarray(img, np.float32)
  ax = 0 if vertical else 1
  n = a.shape[ax]
  acc = np.zeros(a.shape, np.float64)
  for q, k in zip((-1, 0, 1), kernel):
    idx = np.clip(np.arange(n) + q, 0, n - 1)
    src = a[idx, :] if vertical else a[:, idx]
    acc = acc + (src * np.float32(k)).astype(np.float64)
  return acc.astype(np.float32)


def filter2(img, kh, kv):
  return filter_pass(filter_pass(img, kh, False), kv, True)


def gaussian3(img):
  return filter2(img, GAUSS, GAUSS)


def sobel_dx(img):
  return filter2(img, DIFF, SMOOTH)


def sobel_dy(img):
  return filter2(img, SMOOTH, DIFF)


def downsample(img):
  a = np.asarray(img, np.float32)
  H, W = a.shape[0] // 2, a.shape[1] // 2
  p00, p10 = a[0:2 * H:2, 0:2 * W:2], a[0:2 * H:2, 1:2 * W:2]
  p01, p11 = a[1:2 * H:2, 0:2 * W:2], a[1:2 * H:2, 1:2 * W:2]
  return (((p00 + p10) + p01) + p11) / np.float32(4.0)


def level_camera(intr, level):
  """(fx, fy, cx, cy) of pyramid level `level`: K / 2^level."""
  s = 0.5 ** level
  return tuple(float(v) * s for v in intr)


def points(depth, cam):
  """open3d's float XYZ image of a depth image -> fp64 [H*W, 3] (NaN where the depth is)."""
  d = np.asarray(depth, np.float32)
  H, W = d.shape
  fx, fy, cx, cy = cam
  v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
  dd = d.astype(np.float64)
  x = (((u - cx) * dd) * (1.0 / fx)).astype(np.float32).astype(np.float64)
  y = (((v - cy) * dd) * (1.0 / fy)).astype(np.float32).astype(np.float64)
  return np.stack([x.ravel(), y.ravel(), dd.ravel()], 1)


def move(T, p):
  T = np.asarray(T, np.float64)
  return np.stack([((T[a, 0] * p[:, 0] + T[a, 1] * p[:, 1]) + T[a, 2] * p[:, 2]) + T[a, 3] for a in range(3)], 1)


def correspondences(depth_s, depth_t, cam, T, max_depth_diff):
  """-> (src pixel, tgt pixel) int64 arrays in target row-major order: the target-pixel z-buffer reading."""
  ds, dt = np.asarray(depth_s, np.float32), np.asarray(depth_t, np.float32)
  H, W = ds.shape
  fx, fy, cx, cy = cam
  src = np.flatnonzero(~np.isnan(ds.ravel()))
  q = move(T, points(ds, cam)[src])
  ok = q[:, 2] > 0.0
  src, q = src[ok], q[ok]
  with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
    uf = (fx * q[:, 0] + cx * q[:, 2]) / q[:, 2] + 0.5
    vf = (fy * q[:, 1] + cy * q[:, 2]) / q[:, 2] + 0.5
  ok = (uf > -1.0) & (uf < W) & (vf > -1.0) & (vf < H)
  src, q, uf, vf = src[ok], q[ok], uf[ok], vf[ok]
  tgt = np.trunc(vf).astype(np.int64) * W + np.trunc(uf).astype(np.int64)
  d_t = dt.ravel()[tgt].astype(np.float64)
  ok = ~np.isnan(d_t)
  ok[ok] = np.abs(q[ok, 2] - d_t[ok]) <= max_depth_diff
  src, tgt, z = src[ok], tgt[ok], q[ok, 2].astype(np.float32)
  order = np.lexsort((src, z, tgt))                    # by target pixel, then nearest depth, then lowest source
  src, tgt = src[order], tgt[order]
  first = np.ones(len(tgt), bool)
  first[1:] = tgt[1:] != tgt[:-1]
  return src[first], tgt[first]


def norm_sums(values, tgt, W, H):
  """The device's fixed-order sum of values[k] placed at target pixel tgt[k] (norm_rows / scale kernels)."""
  img = np.zeros(H * W, np.float64)
  img[tgt] = values
  cols = -(-W // 32) * 32
  img = np.pad(img.reshape(H, W), ((0, 0), (0, cols - W))).reshape(H, cols // 32, 32)
  acc = np.zeros((H, 32))
  for k in range(cols // 32):
    acc = acc + img[:, k, :]
  lanes = np.arange(32)
  for d in (16, 8, 4, 2, 1):
    acc = acc + acc[:, lanes ^ d]
  total = 0.0
  for y in range(H):
    total += float(acc[y, 0])
  return total


def jacobian_rows(q, dIx, dIy, dDx, dDy, I_t, I_s, D_t, cam, hybrid):
  """Residuals r [n, k] and rows J [n, k, 6] (k = 2 hybrid: photometric, geometric; k = 1 colour) of matches with
  moved source points q [n, 3] and the target's unscaled Sobel gradients, intensities and depth at the matches."""
  fx, fy = cam[0], cam[1]
  invz = 1.0 / q[:, 2]
  c0 = SOBEL_SCALE * np.asarray(dIx, np.float64) * fx * invz
  c1 = SOBEL_SCALE * np.asarray(dIy, np.float64) * fy * invz
  c2 = -(c0 * q[:, 0] + c1 * q[:, 1]) * invz
  photo = (np.asarray(I_t, np.float32) - np.asarray(I_s, np.float32)).astype(np.float64)
  x, y, z = q[:, 0], q[:, 1], q[:, 2]
  Jc = np.stack([-z * c1 + y * c2, z * c0 - x * c2, -y * c0 + x * c1, c0, c1, c2], 1)
  if not hybrid:
    return photo[:, None], Jc[:, None, :]
  si, sd = math.sqrt(1.0 - LAMBDA_HYBRID_DEPTH), math.sqrt(LAMBDA_HYBRID_DEPTH)
  gx = SOBEL_SCALE * np.asarray(dDx, np.float64)
  gy = SOBEL_SCALE * np.asarray(dDy, np.float64)
  gx, gy = np.where(np.isnan(gx), 0.0, gx), np.where(np.isnan(gy), 0.0, gy)
  d0, d1 = gx * fx * invz, gy * fy * invz
  d2 = -(d0 * x + d1 * y) * invz
  Jg = np.stack([(-z * d1 + y * d2) - y, (z * d0 - x * d2) + x, -y * d0 + x * d1, d0, d1, d2 - 1.0], 1)
  r = np.stack([si * photo, sd * (np.asarray(D_t, np.float64) - z)], 1)
  return r, np.stack([si * Jc, sd * Jg], 1)


def cholesky_step(A, b):
  """x = -(A^-1 b) by Cholesky; None on a pivot that is not positive (cholesky6_step's rule)."""
  n = len(b)
  L = np.zeros((n, n))
  for j in range(n):
    d = A[j, j] - L[j, :j] @ L[j, :j]
    if not d > 0.0:
      return None
    L[j, j] = math.sqrt(d)
    for i in range(j + 1, n):
      L[i, j] = (A[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
  y = np.zeros(n)
  for i in range(n):
    y[i] = (-b[i] - L[i, :i] @ y[:i]) / L[i, i]
  x = np.zeros(n)
  for i in range(n - 1, -1, -1):
    x[i] = (y[i] - L[i + 1:, i] @ x[i + 1:]) / L[i, i]
  return x


def zyx(x):
  """open3d's TransformVector6dToMatrix4d: [Rz(x2) Ry(x1) Rx(x0) | x3..5]."""
  ca, sa, cb, sb, cc, sc = (math.cos(x[0]), math.sin(x[0]), math.cos(x[1]), math.sin(x[1]), math.cos(x[2]),
                            math.sin(x[2]))
  Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1.0]])
  Ry = np.array([[cb, 0, sb], [0, 1.0, 0], [-sb, 0, cb]])
  Rx = np.array([[1.0, 0, 0], [0, ca, -sa], [0, sa, ca]])
  T = np.eye(4)
  T[:3, :3] = (Rz @ Ry) @ Rx
  T[:3, 3] = x[3:]
  return T


def information(src, tgt, depth_t, cam):
  q = points(depth_t, cam)[tgt]
  S, Q = q.sum(0), q.T @ q
  Sx = np.array([[0, -S[2], S[1]], [S[2], 0, -S[0]], [-S[1], S[0], 0]])
  G = np.zeros((6, 6))
  G[:3, :3] = np.trace(Q) * np.eye(3) - Q
  G[:3, 3:], G[3:, :3] = Sx, Sx.T
  G[3:, 3:] = len(q) * np.eye(3)
  return G


def prepare(intensity_s, depth_s, intensity_t, depth_t, intr, odo_init, levels, max_depth_diff, min_depth,
            max_depth):
  """The images of InitializeRGBDOdometry and the pyramids -> dict (None for 'levels' when no match at odo_init)."""
  Gs, Gt = gaussian3(intensity_s), gaussian3(intensity_t)
  Ds0 = gaussian3(preprocess_depth(depth_s, min_depth, max_depth))
  Dt0 = gaussian3(preprocess_depth(depth_t, min_depth, max_depth))
  H, W = Ds0.shape
  src, tgt = correspondences(Ds0, Dt0, level_camera(intr, 0), odo_init, max_depth_diff)
  out = dict(Gs=Gs, Gt=Gt, Ds0=Ds0, Dt0=Dt0, norm_src=src, norm_tgt=tgt, levels=None)
  n = len(src)
  if n == 0:
    return out
  ss = norm_sums(Gs.ravel()[src].astype(np.float64), tgt, W, H)
  st = norm_sums(Gt.ravel()[tgt].astype(np.float64), tgt, W, H)
  scale_s, scale_t = 0.5 / (ss / n), 0.5 / (st / n)
  out['scale'] = (scale_s, scale_t)
  Is0 = (scale_s * Gs.astype(np.float64) + 0.0).astype(np.float32)
  It0 = (scale_t * Gt.astype(np.float64) + 0.0).astype(np.float32)
  lv = [dict(Is=Is0, Ds=Ds0, It=It0, Dt=Dt0)]
  for _ in range(1, levels):
    lv.append({k: downsample(v) for k, v in lv[-1].items()})
  for d in lv:
    d.update(dIx=sobel_dx(d['It']), dIy=sobel_dy(d['It']), dDx=sobel_dx(d['Dt']), dDy=sobel_dy(d['Dt']))
  out['levels'] = lv
  return out


def compute_rgbd_odometry(intensity_s, depth_s, intensity_t, depth_t, intr, odo_init=None, hybrid=True,
                          iterations=(20, 10, 5), max_depth_diff=0.03, min_depth=0.0, max_depth=4.0):
  """-> (success, T [4, 4], info [6, 6], trace): trace['counts'] the correspondence count of every step (coarse to
  fine), trace['prep'] the images of prepare().  intr: (fx, fy, cx, cy) of the full-resolution camera."""
  T = np.eye(4) if odo_init is None or not np.any(odo_init) else np.array(odo_init, np.float64).reshape(4, 4)
  L = len(iterations)
  prep = prepare(intensity_s, depth_s, intensity_t, depth_t, intr, T, L, max_depth_diff, min_depth, max_depth)
  trace = dict(counts=[], prep=prep, steps=[])
  fail = (False, np.eye(4), np.eye(6), trace)
  if prep['levels'] is None:
    return fail
  for li, iters in enumerate(iterations):
    level = L - 1 - li
    d = prep['levels'][level]
    cam = level_camera(intr, level)
    for _ in range(iters):
      src, tgt = correspondences(d['Ds'], d['Dt'], cam, T, max_depth_diff)
      trace['counts'].append(len(src))
      q = move(T, points(d['Ds'], cam)[src])
      r, J = jacobian_rows(q, d['dIx'].ravel()[tgt], d['dIy'].ravel()[tgt], d['dDx'].ravel()[tgt],
                           d['dDy'].ravel()[tgt], d['It'].ravel()[tgt], d['Is'].ravel()[src], d['Dt'].ravel()[tgt],
                           cam, hybrid)
      J = J.reshape(-1, 6)
      r = r.reshape(-1)
      x = cholesky_step(J.T @ J, J.T @ r)
      if x is None:
        return fail
      trace['steps'].append(x)
      T = zyx(x) @ T
  src, tgt = correspondences(prep['Ds0'], prep['Dt0'], level_camera(intr, 0), T, max_depth_diff)
  trace['info_src'], trace['info_tgt'] = src, tgt
  return True, T, information(src, tgt, prep['Dt0'], level_camera(intr, 0)), trace
