"""``DeepGlobalRegistration`` with the reference's constructor, attributes and methods
(core/deep_global_registration.py:68-324), every stage on libdgr_b200.

Built path: voxelise -> FCGF features -> feature kNN -> 6-D inlier network -> weights ->
weighted Procrustes + SE(3) refinement -> point-to-point ICP (``use_icp``, default True as
in the reference).  When the weight sum is below the gate (:276-281) the pair goes to the
safeguard branch (:302-315): RANSAC over the correspondences on the GPU
(dgr_ransac_correspondence), followed by the same ICP.
"""
import os

import numpy as np
import torch

import threading
import time

from .. import _abi, native, shims
from ..me.coords import CoordinateManager
from ..model import load_model
from ..util.timer import Timer


class DeepGlobalRegistration:
  def __init__(self, config, device=torch.device('cuda')):
    self.config = config
    self.clip_weight_thresh = self.config.clip_weight_thresh
    self.device = _abi.require_device(device)
    self.safeguard_method = 'correspondence'
    # The reference calls RANSACConvergenceCriteria(4000000, num_iterations) (:62): 4 M hypotheses,
    # and the 80000 it passes lands in open3d's confidence slot (clamped to 1 = no early exit).
    self.safeguard_max_iteration = 4000000
    self.safeguard_seed = 0       # open3d draws from std::random_device; here a call is reproducible
    self.use_icp = True           # as the reference; GPU point-to-point ICP (dgr_icp)
    self.verbose = getattr(config, 'verbose', True)
    self.feat_timer = Timer()
    self.reg_timer = Timer()
    self.last_branch = None
    self.last_info = {}

    weights = config.weights
    if isinstance(weights, dict):
      state = weights               # already-loaded checkpoint (tests / benchmarks)
    else:
      self._log(f"=> loading checkpoint '{weights}'")
      assert os.path.exists(weights)
      shims.install()               # the checkpoint pickles an EasyDict config
      state = torch.load(weights, map_location='cpu', weights_only=False)
    network_config = state['config']
    self.network_config = network_config
    self.config.inlier_feature_type = network_config.inlier_feature_type
    self.voxel_size = network_config.voxel_size
    self._log(f'=> Setting voxel size to {self.voxel_size}')

    # FCGF extractor: current key names first, then the legacy ones of older checkpoints
    # (reference :95-112); one dummy input channel (:96)
    nc = network_config
    legacy = 'feat_model' not in nc
    self.fcgf_model = self._build_network(
        nc['model' if legacy else 'feat_model'], state['state_dict'], in_channels=1,
        out_channels=nc['model_n_out' if legacy else 'feat_model_n_out'],
        conv1_kernel_size=nc['conv1_kernel_size' if legacy else 'feat_conv1_kernel_size'],
        normalize_feature=nc['normalize_feature'], D=3)
    # 6-D inlier network: 6 input channels only for the 'coords' feature type (:119)
    self.inlier_model = self._build_network(
        nc['inlier_model'], state['state_dict_inlier'],
        in_channels=6 if nc.inlier_feature_type == 'coords' else 1, out_channels=1,
        conv1_kernel_size=nc['inlier_conv1_kernel_size'], normalize_feature=False, D=6)
    self._pinned = {}
    # native executor (csrc/exec.cu): one C call per pair; built lazily, rebuilt when the weights change
    self._native_nets = None
    self._native_ctx = []
    self._stage_ctx = None          # the stage methods' own context: they never overwrite a register() call's taps
    self._last_ctx = None
    self._last_sel_value = None
    self._log('=> loading finished')

  @property
  def _last_sel(self):
    """Indices of the raw points kept by the last voxelisation: of the cloud preprocess() saw last, or - after
    a native register() - of both clouds of the pair (cloud 1's offset by the size of cloud 0)."""
    if self._last_ctx is not None:
      return self._last_ctx.tap('sel')
    return self._last_sel_value

  def _build_network(self, name, weights, in_channels, out_channels, conv1_kernel_size, normalize_feature, D):
    cls = load_model(name)
    if cls is None:
      raise KeyError(f'unknown model {name!r}')
    net = cls(in_channels, out_channels, bn_momentum=self.network_config['bn_momentum'],
              conv1_kernel_size=conv1_kernel_size, normalize_feature=normalize_feature, D=D)
    net.load_state_dict(weights)
    return net.to(self.device).eval()

  def _log(self, msg):
    if self.verbose:
      print(msg)

  # ---------------------------------------------------------------------------------------
  def _upload(self, xyz, slot):
    """numpy -> device through a reused pinned staging buffer (async H2D)."""
    xyz = np.ascontiguousarray(xyz)
    if xyz.dtype not in (np.float32, np.float64):
      xyz = xyz.astype(np.float64)
    key = (slot, xyz.dtype)
    buf = self._pinned.get(key)
    if buf is None or buf.shape[0] < xyz.shape[0]:
      buf = torch.empty((max(xyz.shape[0], 1), 3), dtype=torch.from_numpy(xyz[:0]).dtype).pin_memory()
      self._pinned[key] = buf
    view = buf[:xyz.shape[0]]
    view.numpy()[...] = xyz
    return view.to(self.device, non_blocking=True)

  def preprocess(self, pcd, _slot=0, _batch=0):
    """Stage 0: voxelise.  -> (xyz float32 [N,3], coords int32 [N,4], feats [N,1]).
    One GPU pass replaces sparse_quantize + the re-flooring of the reference (:134-161):
    floor(xyz / voxel) in the input dtype, first point per voxel, ascending indices."""
    _abi.refresh_stream()
    if isinstance(pcd, np.ndarray):
      xyz = pcd
    elif isinstance(pcd, torch.Tensor):
      xyz = pcd
    elif hasattr(pcd, 'points'):          # open3d.geometry.PointCloud
      xyz = np.asarray(pcd.points)
    else:
      raise Exception('Unrecognized pcd type')
    if isinstance(xyz, torch.Tensor):
      dxyz = xyz.to(self.device).contiguous()
      if dxyz.dtype not in (torch.float32, torch.float64):
        dxyz = dxyz.double()
    else:
      dxyz = self._upload(xyz, _slot)
    raw_coords, spec, table, sel, _, npts = _abi.voxelise(dxyz, self.voxel_size, batch=_batch)
    coords = _abi.gather_rows_i32(raw_coords, sel, npts)
    # float32 rows the ICP refine and the baselines search this table with: in the cells they are stored under
    xyz_sel = _abi.float32_in_cells(dxyz[sel.long()], coords[:, 1:], self.voxel_size)
    # the dedup table already maps voxel key -> row of `coords`: hand it to SparseTensor
    coords._dgr_manager = CoordinateManager(_parts=(coords, spec, table))
    self._last_sel_value, self._last_ctx = sel, None
    feats = torch.ones(npts, 1, device=self.device)
    return xyz_sel, coords, feats

  def _stage_forward(self, net, coords, feats=None, unique=False):
    """`net` (a native.Net) over coords CUDA int32 [n, D+1] and feats float32 [n, in_channels] (None = ones) on the
    stage context.  The executor assumes distinct rows and cannot detect duplicates, so rows not known to be
    distinct (from preprocess(), which attaches `_dgr_manager`, or `unique`) are checked first."""
    _abi.refresh_stream()
    coords = coords.to(self.device, torch.int32).contiguous()
    if not unique and getattr(coords, '_dgr_manager', None) is None:
      CoordinateManager(coords)         # raises ValueError on duplicate rows
    if feats is not None:
      feats = feats.to(self.device, torch.float32).contiguous()
    if self._stage_ctx is None:
      self._stage_ctx = native.Context(self.device)
    return net.forward(self._stage_ctx, coords, feats)

  def fcgf_feature_extraction(self, feats, coords):
    """Step 1: FCGF feature per voxel."""
    return self._stage_forward(self.native_networks()[0], coords, feats)

  def fcgf_feature_extraction_pair(self, coords0, coords1):
    """Both clouds of a pair in ONE sparse tensor (batch indices 0 / 1): the hash keys carry the
    batch column, so neighbourhoods never cross clouds and the features equal two separate
    forward passes - at half the launches and host synchronisations."""
    n0 = coords0.shape[0]
    F = self._stage_forward(self.native_networks()[0], torch.cat((coords0, coords1), 0), unique=True)
    return F[:n0], F[n0:]

  def fcgf_feature_matching(self, feats0, feats1):
    """Step 2: nearest neighbour of every feats0 row in feats1."""
    idx1 = _abi.knn_top1(feats0.contiguous(), feats1.contiguous())
    corres_idx0 = torch.arange(len(idx1), device=self.device)
    return corres_idx0, idx1.long()

  def inlier_feature_generation(self, xyz0, xyz1, coords0, coords1, fcgf_feats0, fcgf_feats1,
                                corres_idx0, corres_idx1):
    """Step 3: input features of the inlier network."""
    assert len(corres_idx0) == len(corres_idx1)
    feat_type = self.config.inlier_feature_type
    assert feat_type in ['ones', 'feats', 'coords']
    corres_idx0 = corres_idx0.to(self.device)
    corres_idx1 = corres_idx1.to(self.device)
    if feat_type == 'ones':
      feat = torch.ones((len(corres_idx0), 1), device=self.device)
    elif feat_type == 'feats':
      feat = torch.cat((fcgf_feats0[corres_idx0], fcgf_feats1[corres_idx1]), dim=1)
    else:
      feat = torch.cat((torch.cos(xyz0[corres_idx0]), torch.cos(xyz1[corres_idx1])), dim=1)
    return feat

  def inlier_prediction(self, inlier_feats, coords):
    """Step 4: inlier logit per correspondence."""
    return self._stage_forward(self.native_networks()[1], coords, inlier_feats)

  def safeguard_registration(self, pcd0, pcd1, idx0, idx1, feats0, feats1, distance_threshold,
                             num_iterations):
    """Reference :219-236.  pcd0 / pcd1: [N, 3] points (CUDA float32 tensors, or anything
    np.asarray takes); idx0 / idx1: correspondence indices (idx0 None = arange).  As in the
    reference, ``num_iterations`` does not bound the search (it lands in open3d's confidence
    slot, :62); ``self.safeguard_max_iteration`` hypotheses are evaluated.  -> 4x4 float64."""
    if self.safeguard_method == 'fcgf_feature_matching':
      raise NotImplementedError("safeguard_method 'fcgf_feature_matching' (open3d feature-matching RANSAC, "
                                'core/deep_global_registration.py:27-46) is not built; the default '
                                "'correspondence' is")
    if self.safeguard_method != 'correspondence':
      raise ValueError('Undefined')
    res = self._safeguard_launch(pcd0, pcd1, idx0, idx1, distance_threshold)
    self.last_safeguard = res = res.cpu().numpy()
    return res[:16].reshape(4, 4).copy()

  def _safeguard_launch(self, pcd0, pcd1, idx0, idx1, distance_threshold):
    def points(p):
      if not isinstance(p, torch.Tensor):
        p = torch.from_numpy(np.ascontiguousarray(np.asarray(getattr(p, 'points', p)), dtype=np.float32))
      return p.to(self.device, torch.float32).contiguous()

    def index(i):
      return None if i is None else torch.as_tensor(i).to(self.device, torch.int32).contiguous()

    return _abi.ransac_correspondence(points(pcd0), points(pcd1), index(idx0), index(idx1), distance_threshold,
                                      num_hyp=self.safeguard_max_iteration, seed=self.safeguard_seed)

  # ---------------------------------------------------------------------------------------
  # ---------------------------------------------------------------------------------------
  # native path: the whole pair in one C call (three host reads), see csrc/exec.cu
  # ---------------------------------------------------------------------------------------
  def _param_version(self):
    # in-place updates bump _version; .to() / re-assignment changes the storage address the native table points at
    return tuple((p._version, p.data_ptr()) for m in (self.fcgf_model, self.inlier_model)
                 for p in list(m.parameters()) + list(m.buffers()))

  def native_networks(self):
    """(fcgf, inlier) native layer tables, rebuilt when a parameter or BatchNorm statistic changed."""
    ver = self._param_version()
    if self._native_nets is None or self._native_nets[0] != ver:
      if self._native_nets is not None:
        for ctx in self._native_ctx:       # nothing may still run on the old weights
          torch.cuda.synchronize(self.device)
        for n in self._native_nets[1:]:
          n.close()
      self._native_nets = (ver, native.Net(self.fcgf_model, self.device), native.Net(self.inlier_model, self.device))
    return self._native_nets[1], self._native_nets[2]

  def native_context(self, k=0):
    while len(self._native_ctx) <= k:
      self._native_ctx.append(native.Context(self.device))
    return self._native_ctx[k]

  def _native_ok(self):
    return (self.config.inlier_feature_type == 'ones' and self.safeguard_method == 'correspondence' and
            hasattr(self.fcgf_model, 'CHANNELS'))

  @staticmethod
  def _points(pcd):
    if isinstance(pcd, (np.ndarray, torch.Tensor)):
      return pcd
    if hasattr(pcd, 'points'):            # open3d.geometry.PointCloud
      return np.asarray(pcd.points)
    raise Exception('Unrecognized pcd type')

  def _register_native(self, ctx, xyz0, xyz1):
    """-> (T 4x4 float64, branch, info).  Thread-safe across distinct contexts."""
    fcgf, inl = self.native_networks()
    res = native.pair_register(ctx, fcgf, inl, self._points(xyz0), self._points(xyz1), self.voxel_size,
                               self.clip_weight_thresh, self.use_icp)
    wsum, n0, n1 = float(res[16]), int(res[40]), int(res[41])
    info = dict(wsum=wsum, n0=n0, n1=n1, host_reads=int(res[42]), d2h_bytes=int(res[43]) + 64 * 8)
    T = np.identity(4)
    if wsum >= max(200, n0 * 0.05):
      T[0:3, 0:3] = res[:9].reshape(3, 3)
      T[0:3, 3] = res[9:12]
      branch = 'procrustes'
      info.update(iterations=int(res[12]), loss=float(res[13]), break_count=int(res[14]), n_active=int(res[15]))
      icp = res[17:37] if self.use_icp else None
    else:
      # > Case 1: Safeguard RANSAC + (optional) ICP (reference :302-315), one more host read
      branch = 'safeguard'
      sg = native.pair_safeguard(ctx, 2 * self.voxel_size, self.safeguard_max_iteration, self.safeguard_seed,
                                 self.use_icp)
      T = sg[:16].reshape(4, 4).copy()
      info.update(ransac_fitness=float(sg[16]), ransac_inlier_rmse=float(sg[17]), ransac_hypothesis=int(sg[18]),
                  ransac_inliers=int(sg[19]), host_reads=info['host_reads'] + 1)
      icp = sg[20:40] if self.use_icp else None
    if icp is not None:
      T = icp[:16].reshape(4, 4).copy()
      info.update(icp_fitness=float(icp[16]), icp_inlier_rmse=float(icp[17]), icp_iterations=int(icp[18]))
    info['t_done'] = time.perf_counter()
    return T, branch, info

  def register(self, xyz0, xyz1, inlier_thr=0.00):
    """Main algorithm.  -> 4x4 float64 ndarray mapping cloud 0 into cloud 1's frame
    (core/deep_global_registration.py:238-324)."""
    if not self._native_ok():
      return self.register_stagewise(xyz0, xyz1, inlier_thr)
    self.reg_timer.tic()
    ctx = self.native_context(0)
    T, branch, info = self._register_native(ctx, xyz0, xyz1)
    self.last_branch, self.last_info, self._last_ctx = branch, info, ctx
    wsum_threshold = max(200, info['n0'] * 0.05)
    sign = '>=' if branch == 'procrustes' else '<'
    self._log(f'=> Weighted sum {info["wsum"]:.2f} {sign} threshold {wsum_threshold}')
    t = self.reg_timer.toc()
    self._log(f'=> DGR takes {t:.2} s' if branch == 'procrustes' else f'=> Safeguard takes {t:.2} s')
    return T

  def register_batch(self, pairs, inflight=4):
    """Register independent pairs with `inflight` of them in flight on this GPU (one host thread, stream
    and arena each; SURVEY 8e): the latency-bound stages and host reads of one pair overlap the convolutions
    of the other.  pairs: [(xyz0, xyz1), ...] (arrays, tensors, point clouds, or callables returning such a
    tuple - e.g. file readers).  -> [(T, branch, info), ...] in input order."""
    if not self._native_ok() or inflight <= 1 or len(pairs) <= 1:
      out = []
      for pr in pairs:
        a, b = pr() if callable(pr) else pr
        T = self.register(a, b)
        out.append((T, self.last_branch, dict(self.last_info)))
      return out
    self.native_networks()            # built once, on this thread
    ctxs = [self.native_context(k) for k in range(inflight)]
    results, errors = [None] * len(pairs), []

    def worker(k):
      try:
        torch.cuda.set_device(self.device)
        for i in range(k, len(pairs), inflight):
          a, b = pairs[i]() if callable(pairs[i]) else pairs[i]
          results[i] = self._register_native(ctxs[k], a, b)
      except BaseException as e:   # noqa: BLE001
        errors.append(e)

    threads = [threading.Thread(target=worker, args=(k,), daemon=True) for k in range(inflight)]
    for t in threads:
      t.start()
    for t in threads:
      t.join()
    if errors:
      raise errors[0]
    self.last_branch, self.last_info = results[-1][1], results[-1][2]
    self._last_ctx = ctxs[(len(pairs) - 1) % inflight]
    return results

  def register_stagewise(self, xyz0, xyz1, inlier_thr=0.00):
    """The same algorithm driven stage by stage from Python: the reference's own stage methods, with both
    networks on the native executor.  Every inlier feature type goes through here."""
    self.reg_timer.tic()
    _abi.refresh_stream()
    with torch.no_grad():
      xyz0, coords0, feats0 = self.preprocess(xyz0, 0, _batch=0)
      xyz1, coords1, feats1 = self.preprocess(xyz1, 1, _batch=1)

      self.feat_timer.tic()
      fcgf_feats0, fcgf_feats1 = self.fcgf_feature_extraction_pair(coords0, coords1)
      self.feat_timer.toc()

      idx1 = _abi.knn_top1(fcgf_feats0, fcgf_feats1)              # int32 [N0]
      inlier_coords = _abi.inlier_coords(coords0, coords1, idx1)    # int32 [N0, 7]
      inlier_feats = None                                           # 'ones'
      if self.config.inlier_feature_type != 'ones':
        corres_idx0 = torch.arange(len(idx1), device=self.device)
        inlier_feats = self.inlier_feature_generation(xyz0, xyz1, coords0, coords1, fcgf_feats0,
                                                      fcgf_feats1, corres_idx0, idx1.long())
      # rows are distinct by construction (idx0 = arange over unique voxels)
      logit = self._stage_forward(self.native_networks()[1], inlier_coords, inlier_feats, unique=True)
      weights, wsum_dev = _abi.sigmoid_clip_sum(logit, self.clip_weight_thresh)
      # Procrustes + refinement are launched before the weight-sum gate is known (0.6 ms of GPU
      # time in the rare safeguard case) so that gate and pose come back in ONE host read
      res_dev = _abi.se3_register(xyz0, xyz1, weights.reshape(-1), idx1=idx1,
                                  quantization_size=2 * self.voxel_size, max_iter=1000, max_break_count=20,
                                  break_threshold_ratio=1e-4)
      parts = [res_dev.double(), wsum_dev]
      if self.use_icp:
        # ICP fine-tune (reference :317-322: open3d point-to-point ICP, radius 2 * voxel, initialised
        # with the refined pose), through cloud 1's voxel hash; enqueued before the single readback
        T12 = torch.cat((res_dev[:9].reshape(3, 3), res_dev[9:12].reshape(3, 1)), 1).double().contiguous()
        parts.append(_abi.icp_point_to_point(xyz0, xyz1, coords1._dgr_manager, self.voxel_size,
                                             2 * self.voxel_size, T12, batch=1))
      host = torch.cat(parts).cpu().numpy()
      res, wsum = host[:16], float(host[16])

    wsum_threshold = max(200, len(weights) * 0.05)
    sign = '>=' if wsum >= wsum_threshold else '<'
    self._log(f'=> Weighted sum {wsum:.2f} {sign} threshold {wsum_threshold}')

    T = np.identity(4)
    self.last_info = dict(wsum=wsum, n0=len(weights), n1=len(xyz1))
    if wsum >= wsum_threshold:
      T[0:3, 0:3] = res[:9].reshape(3, 3)
      T[0:3, 3] = res[9:12]
      self.last_branch = 'procrustes'
      self.last_info.update(iterations=int(res[12]), loss=float(res[13]), break_count=int(res[14]),
                            n_active=int(res[15]))
      dgr_time = self.reg_timer.toc()
      self._log(f'=> DGR takes {dgr_time:.2} s')
      icp = host[17:37] if self.use_icp else None
    else:
      # > Case 1: Safeguard RANSAC + (optional) ICP (reference :302-315), one more host read
      self.last_branch = 'safeguard'
      with torch.no_grad():
        ransac_dev = self._safeguard_launch(xyz0, xyz1, None, idx1, 2 * self.voxel_size)
        parts = [ransac_dev]
        if self.use_icp:
          parts.append(_abi.icp_point_to_point(xyz0, xyz1, coords1._dgr_manager, self.voxel_size,
                                               2 * self.voxel_size, ransac_dev[:12].contiguous(), batch=1))
        host = torch.cat(parts).cpu().numpy()
      T = host[:16].reshape(4, 4).copy()
      self.last_info.update(ransac_fitness=float(host[16]), ransac_inlier_rmse=float(host[17]),
                            ransac_hypothesis=int(host[18]), ransac_inliers=int(host[19]))
      icp = host[20:40] if self.use_icp else None
      safeguard_time = self.reg_timer.toc()
      self._log(f'=> Safeguard takes {safeguard_time:.2} s')
    if icp is not None:
      T = icp[:16].reshape(4, 4).copy()
      self.last_info.update(icp_fitness=float(icp[16]), icp_inlier_rmse=float(icp[17]),
                            icp_iterations=int(icp[18]))
    return T
