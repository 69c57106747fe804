"""MinkowskiEngine-shaped operator API over libdgr_b200 (forward / inference only).

This is the plugin boundary of the hot path: the reference's models talk to the
sparse-tensor engine exclusively through ``import MinkowskiEngine as ME``
(model/resunet.py:9-10, model/residual_block.py:11-12, model/common.py:8,
core/deep_global_registration.py:16).  The names, argument meaning and error
behaviour below mirror the symbols those files touch (SURVEY.md §8b), accepting
the union of the ME 0.4 and 0.5 keyword spellings the half-migrated reference
uses.  ``deepglobalregistration_b200.shims.install()`` registers this package as
``MinkowskiEngine`` so the reference's model files import unchanged.

Everything computes in the CUDA library; there is no CPU path.
"""
from enum import Enum

import numpy as np
import torch
import torch.nn as nn

from .. import _abi
from .coords import CoordinateManager, CoordinateMapKey
from . import utils  # noqa: F401  (ME.utils.sparse_quantize / batched_coordinates)

__version__ = '0.5.4+dgr_b200'

# Arithmetic of the sparse convolution sub-GEMMs:
#   'tc3'  wgmma 3xTF32 (hi*hi + lo*hi + hi*lo), fp32-accurate - the default
#   'tc1'  wgmma single TF32 product (~1e-3 relative), opt-in fast mode
#   'simt' fp32 FFMA kernel (also the fallback for shapes the tensor-core path rejects)
_CONV_MODE = 'tc3'


def set_conv_mode(mode):
  global _CONV_MODE
  assert mode in ('tc3', 'tc1', 'simt'), mode
  _CONV_MODE = mode


def get_conv_mode():
  return _CONV_MODE


def sparse_conv(feat, conv_mod, km, out):
  """out += gather-GEMM-scatter of `feat` through `km` with conv_mod's kernel."""
  cin, cout = conv_mod.in_channels, conv_mod.out_channels
  if _CONV_MODE != 'simt' and _abi.tc_supported(cin, cout):
    return _abi.spconv_tc_fwd(feat, conv_mod.kernel_transposed(), km, out, passes=3 if _CONV_MODE == 'tc3' else 1)
  return _abi.spconv_fwd(feat, conv_mod.kernel.detach(), km, out)


def needs_grad(*tensors):
  """Training path (SURVEY 8f rank 3): autograd is on and one of the tensors is part of a graph."""
  return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


class SparseConvFunction(torch.autograd.Function):
  """Sparse convolution with a backward pass, for training (core/trainer.py:204-264 calls loss.backward()
  through MinkowskiConvolution / MinkowskiConvolutionTranspose).  Forward: the gather-GEMM-scatter kernels;
  backward: the input gradient is the same kernel on grad_out over the map with its index lists exchanged and
  every W[kappa] transposed, the weight gradient is dgr_spconv_wgrad (per-offset A^T B, deterministic)."""

  @staticmethod
  def forward(ctx, feat, weight, km, n_out):
    feat, weight = feat.contiguous(), weight.contiguous()
    cin, cout = feat.shape[1], weight.shape[-1]
    out = torch.zeros(n_out, cout, dtype=torch.float32, device=feat.device)
    if _CONV_MODE != 'simt' and _abi.tc_supported(cin, cout):
      _abi.spconv_tc_fwd(feat, _abi.pack_weight_tf32(weight.detach(), km.K, cin, cout), km, out,
                         passes=3 if _CONV_MODE == 'tc3' else 1)
    else:
      _abi.spconv_fwd(feat, weight.detach().reshape(km.K, cin, cout), km, out)
    ctx.save_for_backward(feat, weight)
    ctx.km = km
    return out

  @staticmethod
  def backward(ctx, grad_out):
    feat, weight = ctx.saved_tensors
    km = ctx.km
    grad_out = grad_out.contiguous()
    cin, cout = feat.shape[1], grad_out.shape[1]
    w3 = weight.detach().reshape(km.K, cin, cout)
    grad_feat = grad_w = None
    if ctx.needs_input_grad[0]:
      grad_feat = torch.zeros_like(feat)
      _abi.spconv_fwd(grad_out, w3.transpose(1, 2).contiguous(), km.transposed(), grad_feat)
    if ctx.needs_input_grad[1]:
      grad_w = _abi.spconv_wgrad(feat, grad_out, km).reshape(weight.shape)
    return grad_feat, grad_w, None, None


class RegionType(Enum):
  HYPER_CUBE = 0
  HYPER_CROSS = 1
  CUSTOM = 2


class KernelGenerator:
  """ME.KernelGenerator(kernel_size, stride, dilation, is_transpose=, region_type=,
  dimension=) as built by model/residual_block.py:31-36,56-70."""

  def __init__(self, kernel_size=-1, stride=1, dilation=1, is_transpose=False,
               region_type=RegionType.HYPER_CUBE, region_offsets=None, expand_coordinates=False,
               axis_types=None, dimension=-1):
    assert dimension > 0, 'dimension must be a positive integer'
    if region_type is not RegionType.HYPER_CUBE:
      raise NotImplementedError('dgr_b200 builds HYPER_CUBE kernels only (the reference hot path uses '
                                'no other region type)')
    self.kernel_size = _scalar(kernel_size)
    self.stride = _scalar(stride)
    self.dilation = _scalar(dilation)
    if self.dilation != 1:
      raise NotImplementedError('dilation != 1 is not on the DGR hot path')
    self.is_transpose = is_transpose
    self.region_type = region_type
    self.dimension = dimension
    self.kernel_volume = self.kernel_size ** dimension


def _scalar(v):
  if isinstance(v, (list, tuple, np.ndarray, torch.Tensor)):
    vals = {int(a) for a in v}
    assert len(vals) == 1, 'anisotropic kernels/strides are not on the DGR hot path'
    return vals.pop()
  return int(v)


class SparseTensor:
  """ME.SparseTensor: features [N, C] attached to a coordinate map.

  Accepted spellings (0.5 | 0.4): coordinates|coords, coordinate_map_key|coords_key,
  coordinate_manager|coords_manager.  Rows keep the order of the given (unique)
  coordinates, which the reference relies on
  (core/deep_global_registration.py:169,261,283-284)."""

  def __init__(self, features=None, coordinates=None, *, feats=None, coords=None, tensor_stride=1,
               coordinate_map_key=None, coords_key=None, coordinate_manager=None, coords_manager=None,
               device=None, **unused):
    features = features if features is not None else feats
    coordinates = coordinates if coordinates is not None else coords
    key = coordinate_map_key if coordinate_map_key is not None else coords_key
    manager = coordinate_manager if coordinate_manager is not None else coords_manager
    assert isinstance(features, torch.Tensor), 'features must be a torch.Tensor'
    if manager is None:
      _abi.refresh_stream()
      assert coordinates is not None, 'coordinates or a coordinate manager + key must be given'
      if device is None:
        device = features.device if features.is_cuda else coordinates.device
      device = _abi.require_device(device)
      if isinstance(coordinates, np.ndarray):
        coordinates = torch.from_numpy(coordinates)
      manager = getattr(coordinates, '_dgr_manager', None)
      if manager is None or manager.device != device:
        coordinates = coordinates.to(device=device, dtype=torch.int32).contiguous()
        manager = CoordinateManager(coordinates)
      key = manager.origin_key()
    else:
      assert key is not None, 'coordinate_map_key is required with a coordinate manager'
      device = manager.device
    self._F = features.to(device=device, dtype=torch.float32).contiguous()
    self._manager = manager
    self._key = key
    n = manager.num_rows(key)
    if self._F.shape[0] != n:
      raise ValueError(f'features have {self._F.shape[0]} rows but the coordinate map has {n}')

  # -- attributes the reference reads ------------------------------------------------------
  @property
  def F(self):
    return self._F

  @property
  def feats(self):
    return self._F

  @property
  def C(self):
    return self._manager.coordinates(self._key)

  @property
  def coords(self):
    return self.C

  @property
  def D(self):
    return self._manager.D

  @property
  def device(self):
    return self._F.device

  @property
  def dtype(self):
    return self._F.dtype

  @property
  def shape(self):
    return self._F.shape

  @property
  def tensor_stride(self):
    return [self._key.stride] * self.D

  @property
  def coordinate_map_key(self):
    return self._key

  coords_key = coordinate_map_key

  @property
  def coordinate_manager(self):
    return self._manager

  coords_man = coordinate_manager

  def to(self, device):
    if torch.device(device).type != 'cuda':
      raise _abi.DgrError('dgr_b200 SparseTensors live on CUDA only')
    return self

  def __len__(self):
    return self._F.shape[0]

  def _like(self, feats):
    return SparseTensor(feats, coordinate_map_key=self._key, coordinate_manager=self._manager)

  def _check_same_map(self, other):
    if other._manager is not self._manager or other._key != self._key:
      raise ValueError('sparse tensors live on different coordinate maps')

  def __iadd__(self, other):           # out += residual  (model/residual_block.py:131)
    self._check_same_map(other)
    if needs_grad(self._F, other._F):
      self._F = self._F + other._F
    else:
      self._F = _abi.affine_act(self._F, residual=other._F, out=self._F)
    return self

  def __add__(self, other):
    self._check_same_map(other)
    if needs_grad(self._F, other._F):
      return self._like(self._F + other._F)
    return self._like(_abi.affine_act(self._F, residual=other._F))

  def __repr__(self):
    return f'SparseTensor(N={len(self)}, C={self._F.shape[1]}, D={self.D}, stride={self._key.stride})'


def cat(*tensors):
  """ME.cat(a, b): channel concatenation on a shared coordinate map."""
  if len(tensors) == 1 and isinstance(tensors[0], (list, tuple)):
    tensors = tuple(tensors[0])
  out = tensors[0]
  for t in tensors[1:]:
    out._check_same_map(t)
    out = out._like(torch.cat((out.F, t.F), 1) if needs_grad(out.F, t.F) else _abi.cat2(out.F, t.F))
  return out


class MinkowskiNetwork(nn.Module):
  def __init__(self, D):
    super().__init__()
    self.D = D


class _ConvBase(nn.Module):
  IS_TRANSPOSE = False

  def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, bias=False,
               has_bias=None, kernel_generator=None, expand_coordinates=False, dimension=None):
    super().__init__()
    assert dimension is not None and dimension > 0, 'dimension must be a positive integer'
    if has_bias is not None:             # ME 0.4 spelling
      bias = has_bias
    if kernel_generator is None:
      kernel_generator = KernelGenerator(kernel_size, stride, dilation, is_transpose=self.IS_TRANSPOSE,
                                         dimension=dimension)
    self.kernel_generator = kernel_generator
    self.in_channels, self.out_channels = in_channels, out_channels
    self.kernel_size = kernel_generator.kernel_size
    self.stride = _scalar(stride)
    self.dilation = _scalar(dilation)
    self.dimension = dimension
    self.kernel_volume = kernel_generator.kernel_volume
    self.use_mm = self.kernel_volume == 1 and self.stride == 1
    shape = (in_channels, out_channels) if self.kernel_volume == 1 else \
        (self.kernel_volume, in_channels, out_channels)
    self.kernel = nn.Parameter(torch.empty(*shape, dtype=torch.float32))
    self.bias = nn.Parameter(torch.empty(1, out_channels, dtype=torch.float32)) if bias else None
    self.reset_parameters()

  def reset_parameters(self):
    with torch.no_grad():
      n = (self.out_channels if self.IS_TRANSPOSE else self.in_channels) * self.kernel_volume
      stdv = 1.0 / np.sqrt(n)
      self.kernel.uniform_(-stdv, stdv)
      if self.bias is not None:
        self.bias.uniform_(-stdv, stdv)

  def kernel_transposed(self):
    """Packed TF32 hi/lo copy of the kernel for the tensor-core path (dgr_pack_weight_tf32),
    cached per parameter version."""
    k = self.kernel
    ver = (k._version, k.device, k.data_ptr())
    cache = getattr(self, '_wt_cache', None)
    if cache is None or cache[0] != ver:
      wt = _abi.pack_weight_tf32(k.detach().contiguous(), self.kernel_volume, self.in_channels,
                                 self.out_channels)
      self._wt_cache = cache = (ver, wt)
    return cache[1]

  def forward(self, x):
    assert isinstance(x, SparseTensor), 'input must be a SparseTensor'
    assert x.D == self.dimension
    man, key = x.coordinate_manager, x.coordinate_map_key
    # training path: a graph reaches this layer through its input, or the module is in train() mode with
    # trainable parameters; eval-mode inference stays on the forward-only kernels even outside no_grad()
    train = needs_grad(x.F) or (self.training and needs_grad(self.kernel, self.bias))
    if self.use_mm:
      if train:           # 1x1 convolution = a dense layer: torch supplies forward and backward
        out = x.F @ self.kernel
        return x._like(out if self.bias is None else out + self.bias)
      return x._like(_abi.linear_fwd(x.F, self.kernel.detach(), None if self.bias is None
                                     else self.bias.detach()))
    if self.IS_TRANSPOSE:
      out_key, km = man.transpose_kernel_map(key, self.stride, self.kernel_size)
    else:
      out_key, km = man.kernel_map(key, self.stride, self.kernel_size)
    if train:
      out = SparseConvFunction.apply(x.F, self.kernel, km, km.n_out)
      if self.bias is not None:
        out = out + self.bias
      return SparseTensor(out, coordinate_map_key=out_key, coordinate_manager=man)
    w = self.kernel.detach()
    if (not self.IS_TRANSPOSE) and km.nbr is not None and self.in_channels <= 8 and \
        self.out_channels in (16, 32, 64):
      out = _abi.spconv_table_fwd(x.F, w, km, self.out_channels)
    else:
      out = torch.zeros(km.n_out, self.out_channels, dtype=torch.float32, device=x.device)
      sparse_conv(x.F, self, km, out)
    if self.bias is not None:
      out = _abi.affine_act(out, residual=None, scale=torch.ones_like(self.bias).reshape(-1),
                            shift=self.bias.detach().reshape(-1).contiguous(), out=out)
    return SparseTensor(out, coordinate_map_key=out_key, coordinate_manager=man)

  def extra_repr(self):
    return (f'in={self.in_channels}, out={self.out_channels}, kernel_size={self.kernel_size}, '
            f'stride={self.stride}, D={self.dimension}')


class MinkowskiConvolution(_ConvBase):
  """ME.MinkowskiConvolution (model/residual_block.py:38-44, model/resunet.py:589-596)."""


class MinkowskiConvolutionTranspose(_ConvBase):
  """ME.MinkowskiConvolutionTranspose (model/residual_block.py:72-80)."""
  IS_TRANSPOSE = True


class MinkowskiBatchNorm(nn.Module):
  """ME.MinkowskiBatchNorm(C, momentum=) wrapping ``self.bn = nn.BatchNorm1d``
  (model/common.py:13); evaluation mode only."""

  def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
    super().__init__()
    self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                             track_running_stats=track_running_stats)
    self._folded = None

  def folded(self):
    """(scale, shift) fp32 with y = x * scale + shift; cached per parameter version."""
    bn = self.bn
    ver = (bn.weight._version, bn.bias._version, bn.running_mean._version, bn.running_var._version,
           bn.weight.device)
    if self._folded is None or self._folded[0] != ver:
      with torch.no_grad():
        scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
        shift = bn.bias - bn.running_mean * scale
      self._folded = (ver, scale.float().contiguous(), shift.float().contiguous())
    return self._folded[1], self._folded[2]

  def forward(self, x):
    if self.training or needs_grad(x.F):
      # training: batch statistics + running-stat update are nn.BatchNorm1d's, exactly what ME's
      # MinkowskiBatchNorm does (it applies its wrapped BatchNorm1d to the feature matrix)
      return x._like(self.bn(x.F))
    scale, shift = self.folded()
    return x._like(_abi.affine_act(x.F, scale=scale, shift=shift))


class MinkowskiReLU(nn.Module):
  def forward(self, x):
    if needs_grad(x.F):
      return x._like(torch.relu(x.F))
    return x._like(_abi.affine_act(x.F, relu=True))


class _NotOnHotPath(nn.Module):
  def __init__(self, *a, **k):
    super().__init__()
    raise NotImplementedError(f'{type(self).__name__} is not used by the DGR hot path '
                              '(ResUNetBN2C) and is not built')


class MinkowskiSumPooling(_NotOnHotPath):
  pass


class MinkowskiPoolingTranspose(_NotOnHotPath):
  pass


class MinkowskiInstanceNorm(_NotOnHotPath):
  pass


class MinkowskiELU(_NotOnHotPath):
  pass


class MinkowskiGlobalPooling(_NotOnHotPath):
  pass


from . import MinkowskiFunctional  # noqa: E402,F401
