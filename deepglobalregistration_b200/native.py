"""Python handles of the native executor (csrc/exec.cu): contexts, networks, the one-call pair
registration and its taps.  torch supplies parameter / output memory only.

A `Context` owns a CUDA stream, a grow-only device arena and pinned staging; calls on one context
are serialised by the caller, distinct contexts may be driven from distinct host threads (ctypes
releases the GIL for the duration of a call), which is how two pairs are kept in flight per GPU.
"""
import ctypes as C

import numpy as np
import torch

from . import _abi

TAPS = {'coords': (0, torch.int32), 'xyz': (1, torch.float32), 'features': (2, torch.float32),
        'idx1': (3, torch.int32), 'coords6': (4, torch.int32), 'logit': (5, torch.float32),
        'weights': (6, torch.float32), 'sel': (7, torch.int32)}


class Context:
  def __init__(self, device, stream=None):
    self.device = _abi.require_device(device)
    h = C.c_void_p()
    _abi.call('dgr_ctx_create', self.device.index, stream, C.byref(h))
    self.handle = h

  def close(self):
    if getattr(self, 'handle', None):
      _abi.lib().dgr_ctx_destroy(self.handle)
      self.handle = None

  def __del__(self):
    try:
      self.close()
    except Exception:   # noqa: BLE001
      pass

  @property
  def stream(self):
    return _abi.lib().dgr_ctx_stream(self.handle)

  def stats(self):
    s = (C.c_int64 * 6)()
    _abi.call('dgr_ctx_stats', self.handle, s)
    return dict(host_reads=int(s[0]), d2h_bytes=int(s[1]), h2d_bytes=int(s[2]), arena_high_water=int(s[3]),
                arena_mallocs=int(s[4]), arena_chunks=int(s[5]))

  def profile(self, enable=True):
    _abi.call('dgr_ctx_profile', self.handle, int(bool(enable)))

  def profile_read(self, max_rows=4096):
    """-> float64 [n, 4]: milliseconds, algorithmic flops, gather-scatter-model bytes, kind."""
    buf = np.zeros((max_rows, 4), np.float64)
    n = _abi.lib().dgr_ctx_profile_read(self.handle, _abi.ptr(buf), max_rows)
    return buf[:int(n)].copy()

  STAGES = ('upload+voxelise', 'fcgf_coordinate_phase', 'read1+fcgf_pair_lists', 'fcgf_convolutions', 'feature_knn',
            'inlier_coordinate_phase', 'read2+inlier_pair_lists', 'inlier_convolutions', 'weights+procrustes+refine(+icp)')

  def stage_times(self):
    """{stage: ms} of the last pair registered with profiling on."""
    buf = (C.c_double * 16)()
    n = _abi.lib().dgr_ctx_stage_times(self.handle, buf, 16)
    return {self.STAGES[i]: float(buf[i]) for i in range(min(int(n), len(self.STAGES)))}

  def tap(self, name):
    """Intermediate tensor of the last pair this context registered (a copy, on the device)."""
    which, dtype = TAPS[name]
    rows, cols = C.c_int64(), C.c_int32()
    _abi.call('dgr_pair_tap', self.handle, which, C.byref(rows), C.byref(cols), None)
    out = torch.empty(rows.value, cols.value, dtype=dtype, device=self.device)
    _abi.call('dgr_pair_tap', self.handle, which, None, None, _abi.ptr(out))
    return out[:, 0] if name in ('idx1', 'logit', 'weights', 'sel') else out


def network_parameters(model):
  """The 66 tensors dgr_net_create takes, in execution order, from a ResUNet2-family module (this
  package's model/resunet.py or the reference's own class over the ME shim: same attribute names,
  model/resunet.py:442-596)."""
  out = []

  def conv_bn(conv, norm):
    scale, shift = norm.folded()
    out.extend([conv.kernel.detach().float().contiguous(), scale, shift])

  for l in (1, 2, 3, 4):
    blk = getattr(model, f'block{l}')
    conv_bn(getattr(model, f'conv{l}'), getattr(model, f'norm{l}'))
    conv_bn(blk.conv1, blk.norm1)
    conv_bn(blk.conv2, blk.norm2)
  for l in (4, 3, 2):
    blk = getattr(model, f'block{l}_tr')
    conv_bn(getattr(model, f'conv{l}_tr'), getattr(model, f'norm{l}_tr'))
    conv_bn(blk.conv1, blk.norm1)
    conv_bn(blk.conv2, blk.norm2)
  out.append(model.conv1_tr.kernel.detach().float().contiguous())
  out.append(model.final.kernel.detach().float().contiguous())
  out.append(model.final.bias.detach().float().reshape(-1).contiguous())
  return out


class Net:
  """A ResUNet2-family module as a native layer table.  Parameters are snapshotted at construction
  (eval BatchNorm folded, TF32 slabs packed): rebuild after changing the weights."""

  def __init__(self, model, device):
    self.device = _abi.require_device(device)
    self.params = network_parameters(model)            # kept alive: the library holds raw pointers
    assert all(p.is_cuda and p.dtype == torch.float32 for p in self.params), 'parameters must be CUDA float32'
    self.D = int(model.D)
    self.in_channels = int(model.conv1.in_channels)
    self.out_channels = int(model.final.out_channels)
    ptrs = (C.c_void_p * len(self.params))(*[p.data_ptr() for p in self.params])
    ch = (C.c_int32 * 5)(*[int(c or 0) for c in model.CHANNELS])
    tr = (C.c_int32 * 5)(*[int(c or 0) for c in model.TR_CHANNELS])
    h = C.c_void_p()
    _abi.call('dgr_net_create', self.device.index, self.D, self.in_channels, self.out_channels,
              int(model.conv1.kernel_size), int(bool(model.normalize_feature)), ch, tr, ptrs, len(self.params),
              torch.cuda.current_stream(self.device).cuda_stream, C.byref(h))
    self.handle = h

  def close(self):
    if getattr(self, 'handle', None):
      _abi.lib().dgr_net_destroy(self.handle)
      self.handle = None

  def __del__(self):
    try:
      self.close()
    except Exception:   # noqa: BLE001
      pass

  def forward(self, ctx, coords, feats=None):
    """coords CUDA int32 [n, D+1] (distinct rows), feats [n, in_channels] or None (= ones) -> [n, out]."""
    _abi._chk(coords, torch.int32, 'coords')
    n = coords.shape[0]
    if coords.shape != (n, self.D + 1):
      raise _abi.DgrError(f'coords must be [n, {self.D + 1}], got {list(coords.shape)}')
    if feats is not None:
      _abi._chk(feats, torch.float32, 'feats')
      if feats.shape != (n, self.in_channels):
        raise _abi.DgrError(f'feats must be [{n}, {self.in_channels}], got {list(feats.shape)}')
    out = torch.empty(n, self.out_channels, dtype=torch.float32, device=coords.device)
    # inputs may have been produced on torch's current stream
    torch.cuda.current_stream(coords.device).synchronize()
    _abi.call('dgr_net_forward', ctx.handle, self.handle, _abi.ptr(coords), n, _abi.ptr(feats), _abi.ptr(out))
    torch.cuda.synchronize(coords.device)
    return out


def pair_register(ctx, fcgf, inlier, xyz0, xyz1, voxel, clip, use_icp):
  """One native call for the whole pair.  xyz: numpy float32/float64 [n, 3] (host; uploaded through the
  context's pinned staging) or CUDA tensors.  -> float64 [64] result block (include/dgr_b200.h)."""
  def prep(a):
    if isinstance(a, torch.Tensor):
      if not a.is_cuda:
        a = a.numpy()
      else:
        if a.dtype not in (torch.float32, torch.float64):
          a = a.double()
        a = a.contiguous()
        return a, a.data_ptr(), a.shape[0], int(a.dtype == torch.float64), False
    a = np.ascontiguousarray(a)
    if a.dtype not in (np.float32, np.float64):
      a = a.astype(np.float64)
    return a, a.ctypes.data, a.shape[0], int(a.dtype == np.float64), True

  a, pa, na, fa, ha = prep(xyz0)
  b, pb, nb, fb, hb = prep(xyz1)
  if ha != hb:
    raise _abi.DgrError('both clouds must live on the same side (host arrays or CUDA tensors)')
  if a.ndim != 2 or a.shape[1] != 3 or b.ndim != 2 or b.shape[1] != 3:
    raise _abi.DgrError('point clouds must be [n, 3]')
  if not ha:
    torch.cuda.current_stream(a.device).synchronize()
  res = np.zeros(64, np.float64)
  _abi.call('dgr_pair_register', ctx.handle, fcgf.handle, inlier.handle, pa, na, fa, pb, nb, fb, int(ha),
            float(voxel), float(clip), int(bool(use_icp)), _abi.ptr(res))
  return res


def pair_safeguard(ctx, max_dist, num_hyp, seed, use_icp):
  res = np.zeros(40, np.float64)
  _abi.call('dgr_pair_safeguard', ctx.handle, float(max_dist), int(num_hyp), int(seed) & (2**64 - 1),
            int(bool(use_icp)), _abi.ptr(res))
  return res
