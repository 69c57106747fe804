"""Coordinate maps and kernel maps of one sparse-tensor family (the role of ME's
CoordinateManager), built with the coordinate kernels of libdgr_b200."""
import numpy as np
import torch

from .. import _abi
from .._abi import KEY_MARGIN


class CoordinateMapKey:
  __slots__ = ('stride', 'tag')

  def __init__(self, stride, tag=''):
    self.stride, self.tag = int(stride), tag

  def get_tensor_stride(self):
    return self.stride

  def __eq__(self, o):
    return isinstance(o, CoordinateMapKey) and (self.stride, self.tag) == (o.stride, o.tag)

  def __hash__(self):
    return hash((self.stride, self.tag))

  def __repr__(self):
    return f'CoordinateMapKey(stride={self.stride})'


class _Map:
  __slots__ = ('coords', 'table', 'n')

  def __init__(self, coords, table, n):
    self.coords, self.table, self.n = coords, table, n


def kernel_offsets(kernel_size, D, tensor_stride, device):
  """[K, D] int32 offsets, kappa enumerates axis 0 fastest, centred, scaled by the input
  tensor stride (SURVEY.md §8a frozen semantics (1))."""
  k = int(kernel_size)
  kap = np.arange(k ** D)
  offs = np.stack([((kap // (k ** ax)) % k - k // 2) * tensor_stride for ax in range(D)], 1)
  return torch.from_numpy(offs.astype(np.int32)).to(device)


_OFFSET_CACHE = {}


class CoordinateManager:
  """Holds, per tensor stride, the coordinate matrix [N_s, D+1] and its hash table, plus a
  cache of kernel maps keyed by (in_stride, out_stride, kernel_size)."""

  def __init__(self, coordinates=None, *, _parts=None, assume_unique=False):
    if _parts is not None:
      coords, spec, table = _parts
    elif assume_unique:
      # rows known to be distinct (DGR: first-occurrence voxels, arange-indexed correspondences):
      # no host round trip here; the key-overflow flag is checked with the first kernel-map read
      coords = coordinates
      spec = _abi.keyspec_build(_abi.coords_minmax(coords), coords.shape[1], KEY_MARGIN)
      table, _, _, _ = _abi.unique_first(coords, spec)
    else:
      coords = coordinates
      assert coords.is_cuda and coords.dtype == torch.int32 and coords.dim() == 2
      spec = _abi.keyspec_build(_abi.coords_minmax(coords), coords.shape[1], KEY_MARGIN)
      table, _, _, cnt = _abi.unique_first(coords, spec)
      n_unique = _abi.read_count(cnt)
      if n_unique != coords.shape[0]:
        raise ValueError(f'{coords.shape[0] - n_unique} duplicate coordinates: the DGR hot path feeds '
                         'unique coordinates (sparse_quantize output) and relies on row order')
    # NOTE: callers attach the manager to the very tensor they passed in (`coords._dgr_manager`);
    # holding that same Python object here would close a reference cycle that only the garbage
    # collector can free - hundreds of MB of CUDA memory per pair, a cudaMalloc storm in the caching
    # allocator.  detach() gives an alias (same storage, new object, no back-reference).
    coords = coords.detach()
    self.device = coords.device
    self.D = coords.shape[1] - 1
    self.spec = spec
    self._maps = {1: _Map(coords, table, coords.shape[0])}
    self._kmaps = {}
    self._offsets = {}

  @staticmethod
  def _check_spec(spec):
    if int(spec[1].item()) != 0:
      raise _abi.DgrError('coordinate extent does not fit a 63-bit packed key')

  # -- maps ---------------------------------------------------------------------------------
  def origin_key(self):
    return CoordinateMapKey(1)

  def num_rows(self, key):
    return self._map(key.stride).n

  def coordinates(self, key):
    return self._map(key.stride).coords

  def _map(self, stride):
    """Coordinate map at `stride`, derived from the stride-1 rows with one host read (floor(c / s) * s composes,
    and ranking cells by their first stride-1 row reproduces the cascaded first-occurrence order)."""
    if stride not in self._maps:
      assert stride % 2 == 0 and stride > 1, f'no coordinate map at stride {stride}'
      coords, tables, n_out = _abi.coarse_maps(self._maps[1].coords, self.spec, [stride])
      n, overflow = torch.cat([n_out, self.spec[1:2]]).cpu().tolist()
      _abi.D2H_BYTES += 8
      if overflow:
        raise _abi.DgrError('coordinate extent does not fit a 63-bit packed key')
      self._maps[stride] = _Map(coords[0, :n], tables[0], n)
    return self._maps[stride]

  def _offs(self, kernel_size, stride):
    k = (kernel_size, self.D, stride, self.device)
    if k not in _OFFSET_CACHE:          # process-wide: the offsets depend on nothing else
      _OFFSET_CACHE[k] = kernel_offsets(kernel_size, self.D, stride, self.device)
    return _OFFSET_CACHE[k]

  # -- kernel maps ----------------------------------------------------------------------------
  def kernel_map(self, in_key, conv_stride, kernel_size):
    """Map of a convolution with the given stride on the map `in_key`.
    Returns (out_key, KernelMap)."""
    s_in = in_key.stride
    s_out = s_in * conv_stride
    ck = (s_in, s_out, kernel_size)
    if ck not in self._kmaps:
      m_in, m_out = self._map(s_in), self._map(s_out)
      # the dense neighbour table is kept only where the output-stationary conv1 kernel reads it
      keep = self.D == 3 and conv_stride == 1 and kernel_size > 3
      self._kmaps[ck] = _abi.kernel_map(m_out.coords, self.spec, m_in.table, m_in.n,
                                        self._offs(kernel_size, s_in), keep_table=keep,
                                        mode=_abi.kmap_mode(s_in, s_out, kernel_size), in_coords=m_in.coords,
                                        in_stride=s_in, out_table=m_out.table)
    return CoordinateMapKey(s_out), self._kmaps[ck]

  def transpose_kernel_map(self, in_key, conv_stride, kernel_size):
    """A transposed convolution from stride s to s / conv_stride re-uses the pair lists of
    the matching down-convolution with the roles of input and output exchanged."""
    s_in = in_key.stride
    assert s_in % conv_stride == 0, 'transposed convolution below tensor stride 1'
    s_out = s_in // conv_stride
    if conv_stride == 1:
      return self.kernel_map(in_key, 1, kernel_size)
    ck = (s_out, s_in, kernel_size)
    if ck not in self._kmaps:
      raise NotImplementedError('transposed convolution without a matching strided convolution '
                                '(generating new coordinates) is not on the DGR hot path')
    tk = ('T',) + ck
    if tk not in self._kmaps:
      self._kmaps[tk] = self._kmaps[ck].transposed()
    return CoordinateMapKey(s_out), self._kmaps[tk]
