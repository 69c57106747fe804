"""ctypes binding of libdgr_b200.so (include/dgr_b200.h).

Every entry point's argtypes / restype and the integer DGR_* constants are read from the
header the library is compiled against, so the binding cannot drift from the C ABI.

torch is used here for device memory and the current CUDA stream only; every computation happens inside the
library.  There is no CPU fallback: importing this
module without a built library, or calling into it without an sm_90 device,
raises.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import torch

from .build import INCLUDE

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdgr_b200.so')
HEADER = os.path.join(INCLUDE, 'dgr_b200.h')


class DgrError(RuntimeError):
  pass


# the only C types the binding maps; anything else (int, size_t, a struct by value) is an error, never a guessed width
_SCALARS = {'int32_t': C.c_int32, 'int64_t': C.c_int64, 'uint64_t': C.c_uint64, 'float': C.c_float,
            'double': C.c_double}


def _ctype(decl, c_type, ret=False):
  """ctypes type of the C type `c_type` of declaration `decl`: any pointer is c_void_p (c_char_p for a returned
  const char*)."""
  words = c_type.replace('*', ' * ').split()
  if '*' in words:
    return C.c_char_p if ret and words == ['const', 'char', '*'] else C.c_void_p
  words = [w for w in words if w != 'const']
  if len(words) != 1 or words[0] not in _SCALARS:
    raise DgrError(f'{decl}: no ctypes type for {c_type.strip()!r}')
  return _SCALARS[words[0]]


def read_header(path):
  """-> ({entry point: (restype, [argtypes])}, {DGR_* integer constant: value}) of a dgr_b200.h: every
  `<type> dgr_name(<type> name, ...);` declaration and every `#define DGR_NAME <integer>`."""
  with open(path) as fh:
    src = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', fh.read(), flags=re.S)
  consts = {name: int(v.strip('()')) for name, v in
            re.findall(r'^[ \t]*#[ \t]*define[ \t]+(DGR_\w+)[ \t]+(-?\d+|\(-?\d+\))[ \t]*$', src, re.M)}
  src = re.sub(r'^[ \t]*#.*$', ' ', src, flags=re.M)
  decls = {}
  for ret, name, params in re.findall(r'([\w\s*]*?)\b(dgr_\w+)\s*\(([^;]*?)\)\s*;', src):
    decl = ' '.join(f'{ret} {name}({params})'.split())
    args = [] if params.strip() == 'void' else [_ctype(decl, re.sub(r'\w+\s*$', '', p)) for p in params.split(',')]
    decls[name] = (_ctype(decl, ret, ret=True), args)
  return decls, consts


DECLARATIONS, _DEFINES = read_header(HEADER)

MAX_COLS = _DEFINES['DGR_MAX_COLS']
TILE_ROWS = 128
KEY_MARGIN = 32     # spare cells around the bounding box: covers 7^3 kernels and stride-8 flooring


class KeySpec(C.Structure):
  _fields_ = [('ncols', C.c_int32), ('overflow', C.c_int32), ('lo', C.c_int32 * MAX_COLS),
              ('shift', C.c_int32 * MAX_COLS), ('bits', C.c_int32 * MAX_COLS)]


KEYSPEC_INTS = C.sizeof(KeySpec) // 4

_lib = None


def bind(path, names=None):
  """Load a libdgr_b200.so and set argtypes / restype of the header's entry points (`names`: only these, so that
  another build lacking newer entry points can be bound for comparison)."""
  l = C.CDLL(path)
  for name in DECLARATIONS if names is None else names:
    fn = getattr(l, name)
    fn.restype, fn.argtypes = DECLARATIONS[name]
  return l


def lib():
  """Load the shared library (once).  Fails loudly when it has not been built."""
  global _lib
  if _lib is None:
    if not os.path.exists(LIB_PATH):
      raise DgrError(f'{LIB_PATH} is missing: run `python -m deepglobalregistration_b200.build` '
                     '(there is no CPU fallback)')
    _lib = bind(LIB_PATH)
  return _lib


def _check(status, name):
  if status != 0:
    raise DgrError(f'{name} failed ({status}): {lib().dgr_last_error().decode()}')


_FN = {}

# When set to a list, every ABI call is bracketed by CUDA events on torch's current stream and appends
# (entry point, start event, end event): tools/abi_profile.py turns that into warm, in-context GPU time
# per entry point (ncu's per-launch times are cold-cache and serialised).  None = no overhead.
CALL_PROFILE = None


def call(name, *args):
  fn = _FN.get(name)
  if fn is None:
    fn = _FN[name] = getattr(lib(), name)
  if CALL_PROFILE is not None:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    status = fn(*args)
    e1.record()
    CALL_PROFILE.append((name, e0, e1))
  else:
    status = fn(*args)
  if status != 0:
    _check(status, name)


_checked_devices = set()


def require_device(device):
  device = torch.device(device)
  if device.type != 'cuda':
    raise DgrError(f'libdgr_b200 computes on CUDA (sm_90a) only, got device {device}; there is no '
                   'CPU fallback')
  idx = device.index if device.index is not None else torch.cuda.current_device()
  if idx not in _checked_devices:
    _check(lib().dgr_device_check(idx), 'dgr_device_check')
    _checked_devices.add(idx)
  return torch.device('cuda', idx)


def ptr(t):
  """Address of a tensor's or a host numpy array's data; 0 for None."""
  if t is None:
    return 0
  return t.ctypes.data if isinstance(t, np.ndarray) else t.data_ptr()


_STREAM = None


def stream():
  """Handle of the CUDA stream work is enqueued on.  torch.cuda.current_stream() costs ~12 us per
  call, so the handle is looked up once per public entry point (refresh_stream) and cached."""
  global _STREAM
  if _STREAM is None:
    _STREAM = torch.cuda.current_stream().cuda_stream
  return _STREAM


def refresh_stream():
  global _STREAM
  _STREAM = torch.cuda.current_stream().cuda_stream
  return _STREAM


def _chk(t, dtype, name):
  if t.dtype != dtype or not t.is_cuda or not t.is_contiguous():
    raise DgrError(f'{name}: expected contiguous CUDA {dtype}, got {t.dtype} on {t.device} '
                   f'(contiguous={t.is_contiguous()})')
  return t


def next_pow2(n):
  p = 1
  while p < n:
    p <<= 1
  return p


# --------------------------------------------------------------------------- #
# scratch arena: the big transient workspaces (dense neighbour tables, scan / pack buffers)
# are views of per-(device, stream) buffers that only ever grow, so steady-state calls
# never reach cudaMalloc/cudaFree whatever the cloud sizes are.  Work on one stream is
# ordered, which is what makes the reuse safe.
# --------------------------------------------------------------------------- #
_ARENA = {}


def scratch(name, numel, dtype, device):
  key = (name, dtype, device.index, stream())
  buf = _ARENA.get(key)
  if buf is None or buf.numel() < numel:
    buf = torch.empty(max(int(numel * 1.25), 1024), dtype=dtype, device=device)
    _ARENA[key] = buf
  return buf[:numel]


def workspace(name, dtype, device, query, *args):
  """scratch(name) of the element count the dgr_*_ws_elems entry point `query` gives for args."""
  n = C.c_int64(0)
  call(query, *args, C.byref(n))
  return scratch(name, n.value, dtype, device)


# --------------------------------------------------------------------------- #
# thin typed wrappers (allocate outputs / workspaces with torch, call the ABI)
# --------------------------------------------------------------------------- #
def table_cap(n):
  """Capacity of the table of n keys: a power of two, load factor <= 0.5."""
  return max(1024, next_pow2(2 * max(int(n), 1)))


class HashTable:
  __slots__ = ('keys', 'vals', 'cap')

  def __init__(self, n, device):
    """An empty table for n keys."""
    self.cap = table_cap(n)
    self.keys = torch.empty(self.cap, dtype=torch.int64, device=device)
    self.vals = torch.empty(self.cap, dtype=torch.int32, device=device)
    call('dgr_hash_clear', ptr(self.keys), ptr(self.vals), self.cap, stream())

  @classmethod
  def wrap(cls, keys, vals, cap):
    """A table another call has filled (one level of coarse_maps), not cleared."""
    t = cls.__new__(cls)
    t.keys, t.vals, t.cap = keys, vals, cap
    return t


def quantize_points(xyz, voxel, batch=0):
  """xyz CUDA float64/float32 [n,3] -> (coords int32 [n,4], minmax int32 [8])."""
  assert xyz.is_cuda and xyz.is_contiguous() and xyz.shape[1] == 3
  is64 = {torch.float64: 1, torch.float32: 0}[xyz.dtype]
  n = xyz.shape[0]
  coords = torch.empty(n, 4, dtype=torch.int32, device=xyz.device)
  minmax = torch.empty(8, dtype=torch.int32, device=xyz.device)
  call('dgr_quantize_points', ptr(xyz), is64, n, float(voxel), int(batch), ptr(coords), ptr(minmax),
       stream())
  return coords, minmax


def coords_minmax(coords):
  _chk(coords, torch.int32, 'coords')
  minmax = torch.empty(2 * coords.shape[1], dtype=torch.int32, device=coords.device)
  call('dgr_coords_minmax', ptr(coords), coords.shape[0], coords.shape[1], ptr(minmax), stream())
  return minmax


def keyspec_build(minmax, ncols, margin=KEY_MARGIN):
  spec = torch.empty(KEYSPEC_INTS, dtype=torch.int32, device=minmax.device)
  call('dgr_keyspec_build', ptr(minmax), ncols, margin, ptr(spec), stream())
  return spec


def unique_first(coords, spec):
  """-> (table, sel int32 [n] (first m valid), inverse int32 [n], cnt device int32 [2] =
  (n_unique, key-overflow flag))."""
  _chk(coords, torch.int32, 'coords')
  n, ncols = coords.shape
  dev = coords.device
  table = HashTable(n, dev)
  sel = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
  inverse = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
  cnt = torch.zeros(2, dtype=torch.int32, device=dev)
  slot = scratch('uf_slot', max(n, 1), torch.int32, dev)
  scan = scratch('uf_scan', lib().dgr_scan_ws_elems(n), torch.int32, dev)
  call('dgr_unique_first', ptr(coords), n, ncols, ptr(spec), ptr(table.keys), ptr(table.vals), table.cap,
       ptr(sel), ptr(inverse), ptr(cnt), ptr(slot), ptr(scan), stream())
  return table, sel, inverse, cnt


def read_count(cnt):
  """Host read of unique_first's (count, overflow) pair; raises on key overflow."""
  global D2H_BYTES
  n, overflow = cnt.cpu().tolist()
  D2H_BYTES += 8
  if overflow:
    raise DgrError('coordinates are not finite, or their extent does not fit a 63-bit packed key')
  return n


def voxelise(xyz, voxel, batch=0):
  """The first point of every voxel of xyz CUDA float64/float32 [n, 3]: floor(xyz / voxel) in the input dtype,
  kept rows ascending, one host read.  -> (raw coords int32 [n, 4], spec, table (voxel key -> index into sel),
  sel int32 [m], inverse int32 [n], m); raises on key overflow and on non-finite coordinates."""
  raw, minmax = quantize_points(xyz, voxel, batch)
  spec = keyspec_build(minmax, 4)
  table, sel, inverse, cnt = unique_first(raw, spec)
  n = read_count(cnt)
  return raw, spec, table, sel[:n], inverse, n


CELL_NUDGE_STEPS = _DEFINES['DGR_CELL_NUDGE_STEPS']   # float32 ulps a row may move (dgr_float32_in_cells)


def float32_in_cells(xyz, cells, cell):
  """xyz CUDA float64/float32 [n, 3] as the float32 rows a hash search may read: floor(double(x) / cell) - the cell
  every search kernel computes - equals the row's stored cell `cells` (CUDA int [n, 3]; voxelise's raw coords
  [:, 1:]) in every coordinate.  A table keyed in float64 (or by a float32 division) can hold a row whose float32
  value lies across a cell boundary; such a coordinate is moved toward its cell one float32 ulp at a time, every
  other one is exactly xyz.float().  Without this a search can miss an in-radius row (DESIGN.md §3)."""
  if xyz.dtype not in (torch.float32, torch.float64):
    xyz = xyz.double()
  xyz = xyz.contiguous()
  if cells.dtype != torch.int32 or cells.stride(-1) != 1:
    cells = cells.to(torch.int32).contiguous()
  n = xyz.shape[0]
  if xyz.shape != (n, 3) or cells.shape != (n, 3):
    raise DgrError(f'float32_in_cells: xyz and cells must be [n, 3], got {list(xyz.shape)} and {list(cells.shape)}')
  _chk(xyz, xyz.dtype, 'xyz')
  if not cells.is_cuda or cells.device != xyz.device:
    raise DgrError(f'float32_in_cells: cells must be on {xyz.device}, got {cells.device}')
  out = torch.empty(n, 3, dtype=torch.float32, device=xyz.device)
  call('dgr_float32_in_cells', ptr(xyz), int(xyz.dtype == torch.float64), n, ptr(cells), cells.stride(0),
       float(cell), ptr(out), stream())
  return out


def hash_find(coords, spec, table):
  _chk(coords, torch.int32, 'coords')
  rows = torch.empty(coords.shape[0], dtype=torch.int32, device=coords.device)
  call('dgr_hash_find', ptr(coords), coords.shape[0], coords.shape[1], ptr(spec), ptr(table.keys),
       ptr(table.vals), table.cap, ptr(rows), stream())
  return rows


def gather_rows_i32(src, idx, n):
  out = torch.empty(n, src.shape[1], dtype=torch.int32, device=src.device)
  call('dgr_gather_rows_i32', ptr(src), ptr(idx), n, src.shape[1], ptr(out), stream())
  return out


def coarse_maps(fine, spec, strides):
  """Coordinate maps at up to 4 tensor strides, all derived from the distinct rows `fine` [n, ncols]: level l
  holds floor(c / s) * s of every cell in the order of its first row in `fine`.  -> (coords int32
  [L, max(n, 1), ncols] (first n_out[l] rows of level l valid), tables, n_out device int32 [L])."""
  _chk(fine, torch.int32, 'fine')
  n, ncols = fine.shape
  L, nmx, dev = len(strides), max(n, 1), fine.device
  cap = table_cap(n)               # one capacity for every level: at least 2 n
  keys = torch.empty(L, cap, dtype=torch.int64, device=dev)
  vals = torch.empty(L, cap, dtype=torch.int32, device=dev)
  coords = torch.empty(L, nmx, ncols, dtype=torch.int32, device=dev)
  n_out = torch.empty(L, dtype=torch.int32, device=dev)
  slot = scratch('cm_slot', L * nmx, torch.int32, dev)
  scan = scratch('cm_scan', L * lib().dgr_scan_ws_elems(nmx), torch.int32, dev)
  call('dgr_coarse_maps', ptr(fine), n, None, ncols, ptr(spec), L, (C.c_int32 * L)(*strides), ptr(keys), ptr(vals),
       cap, ptr(coords), ptr(n_out), ptr(slot), ptr(scan), stream())
  return coords, [HashTable.wrap(keys[l], vals[l], cap) for l in range(L)], n_out


class KernelMap:
  """(kappa, j)-sorted pair lists + the gather-GEMM-scatter work list (+ the dense neighbour table when kept)."""
  __slots__ = ('K', 'n_in', 'n_out', 'nbr', 'in_idx', 'out_idx', 'kofs', 'kofs_host', 'n_pairs',
               'tile_k', 'tile_start', 'n_tiles', '_paired')

  def paired_tiles(self):
    """(tile_k, tile_start, n_tiles) with an even tile count per offset (the extra tiles are empty)."""
    if getattr(self, '_paired', None) is None:
      counts = self.kofs_host[1:] - self.kofs_host[:-1]
      per_k = (counts + TILE_ROWS - 1) // TILE_ROWS
      n = int(((per_k + 1) // 2 * 2).sum())
      dev = self.kofs.device
      tk = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
      ts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
      call('dgr_kernel_map_tiles', ptr(self.kofs), self.K, TILE_ROWS, n, 1, ptr(tk), ptr(ts), stream())
      self._paired = (tk, ts, n)
    return self._paired

  def transposed(self):
    t = KernelMap()
    for k in self.__slots__:
      setattr(t, k, getattr(self, k, None))
    t.in_idx, t.out_idx = self.out_idx, self.in_idx
    t.n_in, t.n_out = self.n_out, self.n_in
    t.nbr = None
    return t


KMAP_GENERAL, KMAP_SAME, KMAP_DOWN = (_DEFINES['DGR_KMAP_GENERAL'], _DEFINES['DGR_KMAP_SAME'],
                                     _DEFINES['DGR_KMAP_DOWN'])


def kmap_mode(s_in, s_out, kernel_size):
  """Probe mode of dgr_kmap_probe_mode for the map of a convolution from tensor stride s_in to s_out with the
  centred cube of kernel_offsets: same-stride maps mirror half their offsets, kernel-3 down maps are enumerated
  from their input rows."""
  if s_out == s_in and kernel_size % 2 == 1 and kernel_size > 1:
    return KMAP_SAME
  if s_out == 2 * s_in and kernel_size == 3:
    return KMAP_DOWN
  return KMAP_GENERAL


def kernel_map(out_coords, spec, in_table, n_in, offsets, keep_table=False, mode=KMAP_GENERAL, in_coords=None,
               in_stride=0, out_table=None):
  """offsets: CUDA int32 [K, D] (scaled by the input tensor stride).  Occupancy bits + bucket offsets (and the
  dense neighbour table when kept), then ONE host read of the bucket offsets sizes the pair lists and the work
  list.  mode (kmap_mode): KMAP_SAME needs in_table to be the table of out_coords; KMAP_DOWN reads the input
  rows in_coords at tensor stride in_stride and the table out_table of out_coords."""
  global D2H_BYTES
  _chk(out_coords, torch.int32, 'out_coords')
  _chk(offsets, torch.int32, 'offsets')
  dev = out_coords.device
  n_out, ncols = out_coords.shape
  K = offsets.shape[0]
  nmx = max(n_out, 1)
  bits = scratch('km_bits', K * lib().dgr_kmap_mask_words(nmx), torch.int32, dev)
  cnt = scratch('km_cnt', lib().dgr_kmap_cnt_elems(K, nmx), torch.int32, dev)
  kofs = torch.empty(K + 2, dtype=torch.int32, device=dev)
  meta = scratch('km_meta', 5, torch.int32, dev)          # written by the probe, read by nobody here
  # the miss filter pays off when most probes miss: many offsets per row (6-D, 5^3, 7^3 kernels)
  bloom, n_words = None, 0
  if K > 27 and mode != KMAP_DOWN:
    n_words = lib().dgr_bloom2_words(n_in)
    bloom = scratch('km_bloom', n_words, torch.int32, dev)
    call('dgr_bloom2_build', ptr(in_table.keys), in_table.cap, ptr(bloom), n_words, stream())
  table = (ptr(in_table.keys), ptr(in_table.vals), in_table.cap)
  down = mode == KMAP_DOWN
  call('dgr_kmap_probe_mode', mode, ptr(out_coords), n_out, None, ncols, ptr(spec), *table, ptr(bloom), n_words,
       ptr(offsets), K, ptr(in_coords) if down else None, n_in if down else 0, None, in_stride if down else 0,
       ptr(out_table.keys) if down else None, ptr(out_table.vals) if down else None, out_table.cap if down else 0,
       ptr(bits), ptr(cnt), ptr(kofs), ptr(meta), stream())
  km = KernelMap()
  km.nbr = None
  if keep_table:
    km.nbr = torch.empty(K, nmx, dtype=torch.int32, device=dev)
    call('dgr_kmap_dense', ptr(out_coords), n_out, None, ncols, ptr(spec), *table, ptr(bloom), n_words, ptr(offsets),
         K, ptr(km.nbr), nmx, None, stream())
  kofs_all = kofs.cpu().numpy()
  D2H_BYTES += kofs_all.nbytes
  if kofs_all[K + 1] != 0:
    raise DgrError('coordinate extent does not fit a 63-bit packed key')
  kofs_host = kofs_all[:K + 1]
  P = int(kofs_host[K])
  counts = kofs_host[1:] - kofs_host[:-1]
  n_tiles = int(((counts + TILE_ROWS - 1) // TILE_ROWS).sum())
  km.K, km.n_in, km.n_out = K, n_in, n_out
  km.in_idx = torch.empty(max(P, 1), dtype=torch.int32, device=dev)
  km.out_idx = torch.empty(max(P, 1), dtype=torch.int32, device=dev)
  km.tile_k = torch.empty(max(n_tiles, 1), dtype=torch.int32, device=dev)
  km.tile_start = torch.empty(max(n_tiles, 1), dtype=torch.int32, device=dev)
  if P > 0:
    call('dgr_kmap_fill', ptr(bits), ptr(cnt), K, n_out, ptr(out_coords), ncols, ptr(spec), *table, ptr(offsets),
         ptr(km.in_idx), ptr(km.out_idx), stream())
    call('dgr_kernel_map_tiles', ptr(kofs), K, TILE_ROWS, n_tiles, 0, ptr(km.tile_k), ptr(km.tile_start), stream())
  km.kofs, km.kofs_host, km.n_pairs, km.n_tiles = kofs, kofs_host, P, n_tiles
  km._paired = None
  return km


def spconv_fwd(feat, weight, km, out, relu_in=False):
  """out[km.out_idx] += feat[km.in_idx] @ weight[kappa]; `out` holds the initial value."""
  _chk(feat, torch.float32, 'feat'); _chk(weight, torch.float32, 'weight'); _chk(out, torch.float32, 'out')
  cin, cout = feat.shape[1], out.shape[1]
  assert weight.numel() == km.K * cin * cout, (weight.shape, km.K, cin, cout)
  assert feat.shape[0] == km.n_in and out.shape[0] == km.n_out, (feat.shape, out.shape, km.n_in, km.n_out)
  _conv_profiled('spconv_fwd_kernel', km, cin, cout, lambda: call(
      'dgr_spconv_fwd', ptr(feat), cin, ptr(weight), cout, ptr(km.in_idx), ptr(km.out_idx), ptr(km.kofs),
      ptr(km.tile_k), ptr(km.tile_start), km.n_tiles, TILE_ROWS, int(relu_in), ptr(out), stream()))
  return out


def spconv_wgrad(feat, grad_out, km):
  """Weight gradient [K, cin, cout] of the convolution over `km` (training)."""
  _chk(feat, torch.float32, 'feat'); _chk(grad_out, torch.float32, 'grad_out')
  cin, cout = feat.shape[1], grad_out.shape[1]
  dw = torch.empty(km.K, cin, cout, dtype=torch.float32, device=feat.device)
  call('dgr_spconv_wgrad', ptr(feat), cin, ptr(grad_out), cout, ptr(km.in_idx), ptr(km.out_idx), ptr(km.kofs), km.K,
       ptr(dw), stream())
  return dw


def tc_supported(cin, cout):
  return bool(lib().dgr_spconv_tc_supported(int(cin), int(cout)))


def pack_weight_tf32(weight, K, cin, cout):
  """[K, cin, cout] -> packed TF32 hi/lo slabs [K, cin/32, 2, cout, 32] (shared-memory image
  order) for the tensor-core convolution."""
  _chk(weight, torch.float32, 'weight')
  packed = torch.empty(K, cin // 32, 2, cout, 32, dtype=torch.float32, device=weight.device)
  call('dgr_pack_weight_tf32', ptr(weight), K, cin, cout, ptr(packed), stream())
  return packed


# When set to a list, every sparse-convolution launch appends
# (kernel name, start event, end event, algorithmic flops, gather-scatter-model bytes):
# bench.py's live per-kernel roofline measurement (CUDA events on the launching stream).
CONV_PROFILE = None
D2H_BYTES = 0          # bytes this module has read back to the host (counts, bucket offsets, results)


def _conv_profiled(name, km, cin, cout, fn):
  if CONV_PROFILE is None:
    return fn()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  fn()
  e1.record()
  nonempty = int((km.kofs_host[1:] > km.kofs_host[:-1]).sum())
  flops = 2.0 * km.n_pairs * cin * cout
  # SURVEY.md 8(d): gather read + scatter write + (in, out) index pair + weights of non-empty offsets
  nbytes = km.n_pairs * (cin + cout) * 4.0 + 8.0 * km.n_pairs + nonempty * cin * cout * 4.0
  CONV_PROFILE.append((name, e0, e1, flops, nbytes))


def spconv_tc_fwd(feat, weight_t, km, out, passes=3):
  """Tensor-core gather-GEMM-scatter: out[km.out_idx] += feat[km.in_idx] @ W[kappa]."""
  _chk(feat, torch.float32, 'feat'); _chk(weight_t, torch.float32, 'weight_t'); _chk(out, torch.float32, 'out')
  cin, cout = feat.shape[1], out.shape[1]
  assert weight_t.numel() == 2 * km.K * cin * cout
  assert feat.shape[0] == km.n_in and out.shape[0] == km.n_out
  _conv_profiled('spconv_tc_kernel', km, cin, cout, lambda: call(
      'dgr_spconv_tc_fwd', ptr(feat), cin, ptr(weight_t), cout, ptr(km.in_idx), ptr(km.out_idx),
      ptr(km.kofs), ptr(km.tile_k), ptr(km.tile_start), km.n_tiles, TILE_ROWS, int(passes), ptr(out), stream()))
  return out


def spconv_tc_f16_fwd(feat, weight, km, out, amax=None):
  """3xFP16 tensor-core convolution (weight: the fp32 [K, cin, cout] kernel; packed per call - test helper)."""
  _chk(feat, torch.float32, 'feat'); _chk(weight, torch.float32, 'weight'); _chk(out, torch.float32, 'out')
  cin, cout = feat.shape[1], out.shape[1]
  packed = torch.empty(4 * km.K * cin * cout, dtype=torch.uint8, device=feat.device)
  wscale = torch.empty(2, dtype=torch.float32, device=feat.device)
  call('dgr_pack_weight_f16', ptr(weight), km.K, cin, cout, ptr(packed), ptr(wscale), stream())
  if amax is None:
    amax = torch.empty(1, dtype=torch.float32, device=feat.device)
    call('dgr_absmax_f32', ptr(feat), feat.numel(), ptr(amax), stream())
  call('dgr_spconv_tc_f16_fwd', ptr(feat), cin, ptr(packed), cout, ptr(km.in_idx), ptr(km.out_idx), ptr(km.kofs),
       ptr(km.tile_k), ptr(km.tile_start), km.n_tiles, TILE_ROWS, ptr(amax), ptr(wscale), ptr(out), stream())
  return out


def spconv_table_fwd(feat, weight, km, cout, scale=None, shift=None):
  _chk(feat, torch.float32, 'feat'); _chk(weight, torch.float32, 'weight')
  assert km.nbr is not None
  out = torch.empty(km.n_out, cout, dtype=torch.float32, device=feat.device)
  call('dgr_spconv_table_fwd_strided', ptr(feat), feat.shape[1], ptr(weight), cout, ptr(km.nbr), km.K, km.n_out,
       km.nbr.stride(0), ptr(scale), ptr(shift), ptr(out), stream())
  return out


def linear_fwd(a, weight, bias=None, b=None, relu=False, normalize=False):
  _chk(a, torch.float32, 'a'); _chk(weight, torch.float32, 'weight')
  n, ca = a.shape
  cb = 0 if b is None else b.shape[1]
  cout = weight.numel() // (ca + cb)
  out = torch.empty(n, cout, dtype=torch.float32, device=a.device)
  call('dgr_linear_fwd', ptr(a), ca, ptr(b), cb, n, ptr(weight), cout, ptr(bias), int(relu), int(normalize),
       ptr(out), stream())
  return out


def affine_act(x, scale=None, shift=None, residual=None, relu=False, out=None):
  _chk(x, torch.float32, 'x')
  if out is None:
    out = torch.empty_like(x)
  call('dgr_affine_act', ptr(x), x.shape[0], x.shape[1], ptr(scale), ptr(shift), ptr(residual), int(relu),
       ptr(out), stream())
  return out


def cat2(a, b):
  _chk(a, torch.float32, 'a'); _chk(b, torch.float32, 'b')
  out = torch.empty(a.shape[0], a.shape[1] + b.shape[1], dtype=torch.float32, device=a.device)
  call('dgr_cat2', ptr(a), a.shape[1], ptr(b), b.shape[1], a.shape[0], ptr(out), stream())
  return out


def l2_normalize(x):
  _chk(x, torch.float32, 'x')
  out = torch.empty_like(x)
  call('dgr_l2_normalize', ptr(x), x.shape[0], x.shape[1], ptr(out), stream())
  return out


KNN_MODE = 'tc'      # 'tc': tensor-core pre-filter + exact candidates; 'simt': fp32 brute force


def knn_top1(f0, f1, return_distance=False, mode=None):
  """Top-1 neighbour of every f0 row in f1 (both modes return identical indices)."""
  _chk(f0, torch.float32, 'f0'); _chk(f1, torch.float32, 'f1')
  n0, n1, c = f0.shape[0], f1.shape[0], f0.shape[1]
  mode = mode or KNN_MODE
  ws = scratch('knn_ws', max(n0, 1), torch.int64, f0.device)
  idx = torch.empty(n0, dtype=torch.int32, device=f0.device)
  dist = torch.empty(n0, dtype=torch.float32, device=f0.device) if return_distance else None
  if mode == 'tc' and lib().dgr_knn_tc_supported(c) and n0 > 0:
    fws = scratch('knn_fws', lib().dgr_knn_tc_ws_elems(n0, n1, c), torch.float32, f0.device)
    call('dgr_knn_top1_tc', ptr(f0), n0, ptr(f1), n1, c, ptr(ws), ptr(fws), ptr(idx), ptr(dist), stream())
  else:
    call('dgr_knn_top1', ptr(f0), n0, ptr(f1), n1, c, ptr(ws), ptr(idx), ptr(dist), stream())
  return (idx, dist) if return_distance else idx


def inlier_coords(coords0, coords1, idx1):
  _chk(coords0, torch.int32, 'coords0'); _chk(coords1, torch.int32, 'coords1'); _chk(idx1, torch.int32, 'idx1')
  out = torch.empty(coords0.shape[0], 7, dtype=torch.int32, device=coords0.device)
  call('dgr_inlier_coords', ptr(coords0), ptr(coords1), ptr(idx1), coords0.shape[0], ptr(out), stream())
  return out


def sigmoid_clip_sum(logit, clip):
  _chk(logit, torch.float32, 'logit')
  w = torch.empty_like(logit)
  wsum = torch.empty(1, dtype=torch.float64, device=logit.device)
  call('dgr_sigmoid_clip_sum', ptr(logit), logit.numel(), float(clip), ptr(w), ptr(wsum), stream())
  return w, wsum


def se3_register(x, y, w, idx1=None, quantization_size=1.0, max_iter=1000, max_break_count=20,
                 break_threshold_ratio=1e-4, lr=0.1, gamma=0.999):
  """-> device float32 [16]: R (9), t (3), iterations, loss, break_count, n_active."""
  _chk(x, torch.float32, 'x'); _chk(y, torch.float32, 'y'); _chk(w, torch.float32, 'w')
  n = x.shape[0]
  pack = scratch('se3_pack', 7 * n, torch.float32, x.device)
  cnt = torch.empty(4, dtype=torch.int32, device=x.device)
  res = torch.empty(16, dtype=torch.float32, device=x.device)
  call('dgr_se3_register', ptr(x), ptr(y), ptr(idx1), ptr(w), n, float(quantization_size), int(max_iter),
       int(max_break_count), float(break_threshold_ratio), float(lr), float(gamma), ptr(pack), ptr(cnt),
       ptr(res), stream())
  return res


MAX_NN = 64            # dgr_estimate_normals' bound on the neighbours per point


def _hash_of(manager_or_table):
  """(spec, table) of a CoordinateManager (its stride-1 table) or of a (spec, table) pair."""
  if hasattr(manager_or_table, '_maps'):
    return manager_or_table.spec, manager_or_table._maps[1].table
  spec, table = manager_or_table
  return spec, table


def estimate_normals(xyz, manager_or_table, cell, radius, max_nn, prev=None, return_counts=False, batch=0):
  """Normals of xyz (CUDA float32 [n, 3]) from its neighbours strictly within `radius`, at most `max_nn` (<= 64) of
  them by (d^2, row), searched through the cloud's own voxel hash at `cell` (a CoordinateManager preprocess() built,
  or (spec, table) of a dgr_unique_first table; one point per cell, batch column `batch`).  prev: CUDA float32
  [n, 3] normals to orient against.  -> float32 [n, 3] (and the int32 [n] counts within the radius)."""
  _chk(xyz, torch.float32, 'xyz')
  if prev is not None:
    _chk(prev, torch.float32, 'prev')
    if prev.shape != xyz.shape:
      raise DgrError('prev must hold one normal per point')
  spec, table = _hash_of(manager_or_table)
  n = xyz.shape[0]
  normals = torch.empty(n, 3, dtype=torch.float32, device=xyz.device)
  counts = torch.empty(max(n, 1), dtype=torch.int32, device=xyz.device)[:n]
  call('dgr_estimate_normals', ptr(xyz), n, ptr(spec), ptr(table.keys), ptr(table.vals), table.cap, int(batch),
       float(cell), float(radius), int(max_nn), ptr(prev), ptr(normals), ptr(counts), stream())
  return (normals, counts) if return_counts else normals


def estimate_covariances(xyz, manager_or_table, cell, radius, max_nn, return_counts=False, batch=0):
  """Per-point covariances (open3d's EstimatePerPointCovariances) of xyz (CUDA float32 [n, 3]) over the neighbours
  estimate_normals finds (strictly within `radius`, at most `max_nn` <= 64 by (d^2, row), the cloud's own voxel hash
  at `cell`); the identity below 3 neighbours.  -> float64 [n, 6] (xx, xy, xz, yy, yz, zz) (and the int32 [n] counts
  within the radius, equal to estimate_normals')."""
  _chk(xyz, torch.float32, 'xyz')
  spec, table = _hash_of(manager_or_table)
  n = xyz.shape[0]
  cov = torch.empty(max(n, 1), 6, dtype=torch.float64, device=xyz.device)[:n]
  counts = torch.empty(max(n, 1), dtype=torch.int32, device=xyz.device)[:n]
  call('dgr_estimate_covariances', ptr(xyz), n, ptr(spec), ptr(table.keys), ptr(table.vals), table.cap, int(batch),
       float(cell), float(radius), int(max_nn), ptr(cov), ptr(counts), stream())
  return (cov, counts) if return_counts else cov


def covariances_from_normals(normals, epsilon=1e-3):
  """Generalized-ICP covariances R diag(epsilon, 1, 1) R^T of normals (CUDA float32 [n, 3]; open3d's
  InitializePointCloudForGeneralizedICP).  -> float64 [n, 6] as estimate_covariances."""
  _chk(normals, torch.float32, 'normals')
  n = normals.shape[0]
  cov = torch.empty(max(n, 1), 6, dtype=torch.float64, device=normals.device)[:n]
  call('dgr_covariances_from_normals', ptr(normals), n, float(epsilon), ptr(cov), stream())
  return cov


LOSS_IDS = {name: _DEFINES[f'DGR_LOSS_{name.upper()}'] for name in ('L2', 'L1', 'Huber', 'Cauchy', 'GM', 'Tukey')}


def _loss_id(loss):
  if loss not in LOSS_IDS:
    raise DgrError(f'loss must be one of {sorted(LOSS_IDS)}, got {loss!r}')
  return LOSS_IDS[loss]


def color_gradient(xyz, normals, intensity, manager_or_table, cell, radius, max_nn, return_counts=False, batch=0):
  """Colour gradients (open3d 0.10's InitializePointCloudForColoredICP) of xyz (CUDA float32 [n, 3]) with normals
  (CUDA float32 [n, 3]) and intensities (CUDA float32 [n]) from the neighbours estimate_normals finds (strictly within
  `radius`, at most `max_nn` <= 64 by (d^2, row), the cloud's own voxel hash at `cell`).  -> float32 [n, 3] (and the
  int32 [n] counts within the radius)."""
  _chk(xyz, torch.float32, 'xyz'); _chk(normals, torch.float32, 'normals'); _chk(intensity, torch.float32, 'intensity')
  n = xyz.shape[0]
  if normals.shape != xyz.shape or intensity.shape != (n,):
    raise DgrError('normals and intensity must hold one row per point')
  spec, table = _hash_of(manager_or_table)
  grad = torch.empty(n, 3, dtype=torch.float32, device=xyz.device)
  counts = torch.empty(max(n, 1), dtype=torch.int32, device=xyz.device)[:n]
  call('dgr_color_gradient', ptr(xyz), ptr(normals), ptr(intensity), n, ptr(spec), ptr(table.keys), ptr(table.vals),
       table.cap, int(batch), float(cell), float(radius), int(max_nn), ptr(grad), ptr(counts), stream())
  return (grad, counts) if return_counts else grad


FPFH_MAX_NN = 128      # dgr_compute_fpfh's bound on the neighbours per point (the point itself included)
FPFH_DIM = 33


def compute_fpfh(xyz, normals, manager_or_table, cell, radius, max_nn, batch=0, ld=FPFH_DIM, return_counts=False):
  """FPFH features (open3d 0.10's compute_fpfh_feature) of xyz (CUDA float32 [n, 3]) with normals (CUDA float32
  [n, 3]) from the neighbours strictly within `radius`, at most `max_nn` (<= 128, the point itself included) by
  (d^2, row), searched through the cloud's own voxel hash at `cell` (as estimate_normals; radius <= 6 cells).
  -> float32 [n, ld] (ld >= 33; columns 33 .. ld - 1 are zero, so ld = 64 feeds the tensor-core kNN) (and the int32
  [n] counts within the radius)."""
  _chk(xyz, torch.float32, 'xyz')
  if normals is None:
    raise DgrError('compute_fpfh needs normals: estimate them first')
  _chk(normals, torch.float32, 'normals')
  if normals.shape != xyz.shape:
    raise DgrError('normals must hold one normal per point')
  spec, table = _hash_of(manager_or_table)
  n = xyz.shape[0]
  ws = workspace('fpfh', torch.int64, xyz.device, 'dgr_fpfh_ws_elems', n, int(max_nn))
  out = torch.empty(max(n, 1), max(int(ld), 1), dtype=torch.float32, device=xyz.device)[:n]
  counts = torch.empty(max(n, 1), dtype=torch.int32, device=xyz.device)[:n]
  call('dgr_compute_fpfh', ptr(xyz), ptr(normals), n, ptr(spec), ptr(table.keys), ptr(table.vals), table.cap,
       int(batch), float(cell), float(radius), int(max_nn), int(ld), ptr(ws), ptr(out), ptr(counts), stream())
  return (out, counts) if return_counts else out


def _pose12(T_init, dev):
  if not (isinstance(T_init, torch.Tensor) and T_init.is_cuda and T_init.numel() == 12):
    T_init = torch.as_tensor(T_init, dtype=torch.float64).reshape(4, 4)[:3].contiguous().to(dev)
  return T_init


def _icp(src, tgt, tgt_normals, tgt_manager, voxel, max_dist, T_init, max_iter, rel_fitness, rel_rmse, batch,
         loss=None, loss_k=1.0):
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  if tgt_normals is not None:
    _chk(tgt_normals, torch.float32, 'tgt_normals')
    if tgt_normals.shape != tgt.shape:
      raise DgrError('tgt_normals must hold one normal per target point')
  dev = src.device
  spec, table = _hash_of(tgt_manager)
  T_init = _pose12(T_init, dev)
  ws = workspace('icp', torch.float64, dev, 'dgr_icp_ws_elems', src.shape[0])
  res = torch.empty(20, dtype=torch.float64, device=dev)
  if loss is not None:
    call('dgr_icp_loss', ptr(src), src.shape[0], ptr(tgt), ptr(tgt_normals), ptr(spec), ptr(table.keys),
         ptr(table.vals), table.cap, int(batch), float(voxel), float(max_dist), _loss_id(loss), float(loss_k),
         ptr(T_init), int(max_iter), float(rel_fitness), float(rel_rmse), ptr(ws), ptr(res), stream())
    return res
  # ptr() of an empty tgt_normals is 0, which selects point-to-point; without target points neither update has a
  # correspondence, so both give the same result
  call('dgr_icp', ptr(src), src.shape[0], ptr(tgt), ptr(tgt_normals), ptr(spec), ptr(table.keys), ptr(table.vals),
       table.cap, int(batch), float(voxel), float(max_dist), ptr(T_init), int(max_iter), float(rel_fitness),
       float(rel_rmse), ptr(ws), ptr(res), stream())
  return res


def icp_point_to_point(src, tgt, tgt_manager, voxel, max_dist, T_init, max_iter=30, rel_fitness=1e-6,
                       rel_rmse=1e-6, batch=0):
  """Point-to-point ICP (open3d defaults) of src onto tgt through tgt's voxel hash.
  src / tgt: CUDA float32 [n, 3]; tgt_manager: the CoordinateManager preprocess() built for tgt, or (spec, table)
  of a dgr_unique_first table of tgt at `voxel` (batch column `batch`); T_init: 4x4 (numpy / tensor) or device
  double [12].  -> device double [20] (pose 16, fitness, inlier RMSE, iterations, correspondences)."""
  return _icp(src, tgt, None, tgt_manager, voxel, max_dist, T_init, max_iter, rel_fitness, rel_rmse, batch)


def icp_point_to_plane(src, tgt, tgt_normals, tgt_manager, voxel, max_dist, T_init, max_iter=30, rel_fitness=1e-6,
                       rel_rmse=1e-6, batch=0, loss=None, loss_k=1.0):
  """Point-to-plane ICP (open3d's TransformationEstimationPointToPlane, default criteria) of src onto tgt through
  tgt's voxel hash; arguments as icp_point_to_point plus tgt_normals (CUDA float32 [n_tgt, 3]).  loss: None (the
  plain estimator) or a robust loss of LOSS_IDS with scale loss_k, each row weighted by it (dgr_icp_loss)."""
  if loss is not None and tgt_normals is None:
    raise DgrError('point-to-plane ICP with a loss needs tgt_normals')
  return _icp(src, tgt, tgt_normals, tgt_manager, voxel, max_dist, T_init, max_iter, rel_fitness, rel_rmse, batch,
              loss, loss_k)


def icp_colored(src, src_intensity, tgt, tgt_normals, tgt_intensity, tgt_grad, tgt_manager, voxel, max_dist,
                lambda_geometric, T_init, max_iter=30, rel_fitness=1e-6, rel_rmse=1e-6, batch=0, loss=None,
                loss_k=1.0):
  """Colored ICP (open3d's TransformationEstimationForColoredICP(lambda_geometric), default criteria) of src onto tgt
  through tgt's voxel hash; arguments as icp_point_to_plane plus the intensities (CUDA float32 [n]) of both clouds and
  the target's colour gradients (color_gradient; CUDA float32 [n_tgt, 3]).  loss / loss_k: as icp_point_to_plane,
  each of the two rows weighted on its own scaled residual (dgr_colored_icp_loss).  -> device double [20] as
  icp_point_to_plane."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  for name, a, shape in (('src_intensity', src_intensity, (src.shape[0],)), ('tgt_normals', tgt_normals, tgt.shape),
                         ('tgt_intensity', tgt_intensity, (tgt.shape[0],)), ('tgt_grad', tgt_grad, tgt.shape)):
    _chk(a, torch.float32, name)
    if a.shape != shape:
      raise DgrError(f'{name} must hold one row per point')
  if tgt.shape[0] == 0:
    raise DgrError('colored ICP needs target points')
  dev = src.device
  spec, table = _hash_of(tgt_manager)
  T_init = _pose12(T_init, dev)
  ws = workspace('icp', torch.float64, dev, 'dgr_icp_ws_elems', src.shape[0])
  res = torch.empty(20, dtype=torch.float64, device=dev)
  if loss is not None:
    call('dgr_colored_icp_loss', ptr(src), ptr(src_intensity), src.shape[0], ptr(tgt), ptr(tgt_normals),
         ptr(tgt_intensity), ptr(tgt_grad), ptr(spec), ptr(table.keys), ptr(table.vals), table.cap, int(batch),
         float(voxel), float(max_dist), float(lambda_geometric), _loss_id(loss), float(loss_k), ptr(T_init),
         int(max_iter), float(rel_fitness), float(rel_rmse), ptr(ws), ptr(res), stream())
    return res
  call('dgr_colored_icp', ptr(src), ptr(src_intensity), src.shape[0], ptr(tgt), ptr(tgt_normals), ptr(tgt_intensity),
       ptr(tgt_grad), ptr(spec), ptr(table.keys), ptr(table.vals), table.cap, int(batch), float(voxel), float(max_dist),
       float(lambda_geometric), ptr(T_init), int(max_iter), float(rel_fitness), float(rel_rmse), ptr(ws), ptr(res),
       stream())
  return res


def icp_generalized(src, src_cov, tgt, tgt_cov, tgt_manager, voxel, max_dist, T_init, max_iter=30, rel_fitness=1e-6,
                    rel_rmse=1e-6, batch=0, loss=None, loss_k=1.0):
  """Generalized ICP (open3d's TransformationEstimationForGeneralizedICP, default criteria) of src onto tgt through
  tgt's voxel hash; arguments as icp_point_to_point plus both clouds' covariances (CUDA float64 [n, 6], from
  estimate_covariances or covariances_from_normals) and an optional robust loss as icp_point_to_plane
  (dgr_generalized_icp).  -> device double [20] as icp_point_to_point."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  for name, a, n in (('src_cov', src_cov, src.shape[0]), ('tgt_cov', tgt_cov, tgt.shape[0])):
    _chk(a, torch.float64, name)
    if a.shape != (n, 6):
      raise DgrError(f'{name} must hold one [6] covariance row per point')
  if tgt.shape[0] == 0:
    raise DgrError('generalized ICP needs target points')
  dev = src.device
  spec, table = _hash_of(tgt_manager)
  T_init = _pose12(T_init, dev)
  ws = workspace('icp', torch.float64, dev, 'dgr_icp_ws_elems', src.shape[0])
  res = torch.empty(20, dtype=torch.float64, device=dev)
  call('dgr_generalized_icp', ptr(src), ptr(src_cov), src.shape[0], ptr(tgt), ptr(tgt_cov), ptr(spec), ptr(table.keys),
       ptr(table.vals), table.cap, int(batch), float(voxel), float(max_dist), _loss_id('L2' if loss is None else loss),
       float(loss_k), ptr(T_init), int(max_iter), float(rel_fitness), float(rel_rmse), ptr(ws), ptr(res), stream())
  return res


def information_matrix(src, tgt, tgt_manager, cell, max_dist, T, batch=0):
  """open3d's GetInformationMatrixFromPointClouds: sum of G^T G over the nearest target point q of every transformed
  source point strictly within max_dist (dgr_icp's search through tgt's voxel hash at `cell`; max_dist <= 4 cells).
  src / tgt: CUDA float32 [n, 3]; tgt_manager: a CoordinateManager of tgt or (spec, table) of a dgr_unique_first table
  (batch column `batch`); T: 4x4 mapping src into tgt.  -> device double [37] (6x6 row-major, correspondence count)."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  spec, table = _hash_of(tgt_manager)
  T = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(4, 4))
  ws = workspace('information', torch.float64, src.device, 'dgr_information_matrix_ws_elems', src.shape[0])
  out = torch.empty(37, dtype=torch.float64, device=src.device)
  call('dgr_information_matrix', ptr(src), src.shape[0], ptr(tgt), ptr(spec), ptr(table.keys), ptr(table.vals),
       table.cap, int(batch), float(cell), float(max_dist), ptr(T), ptr(ws), ptr(out), stream())
  return out


POSE_GRAPH_MAX_NODES = _DEFINES['DGR_POSE_GRAPH_MAX_NODES']
POSE_GRAPH_MAX_EDGES = _DEFINES['DGR_POSE_GRAPH_MAX_EDGES']
POSE_GRAPH_STATS = ('iterations', 'iterations_pruned', 'cost', 'pruned', 'status', 'mu', 'mu_pruned', 'cost_start',
                    'cost_first_pass', 'factorisations')


def pose_graph_optimize(poses, ends, T, info, uncertain, confidence, max_correspondence_distance=0.075,
                        edge_prune_threshold=0.25, preference_loop_closure=1.0, reference_node=-1, max_iteration=100,
                        min_relative_increment=1e-6, min_relative_residual_increment=1e-6, min_right_term=1e-6,
                        min_residual=1e-6, max_iteration_lm=20, upper_scale_factor=2 / 3, lower_scale_factor=1 / 3,
                        device='cuda'):
  """open3d's GlobalOptimization with GlobalOptimizationLevenbergMarquardt on the device (one launch, one read).
  poses [N, 4, 4] mapping each fragment into the world; ends [E, 2] (source, target); T [E, 4, 4] mapping source into
  target; info [E, 6, 6]; uncertain [E] bool; confidence [E] (the line process an uncertain edge starts from); host
  arrays.  -> (poses [N, 4, 4], kept [E] bool, line process [E], stats dict)."""
  poses = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(-1, 16))
  n = len(poses)
  ends = np.ascontiguousarray(np.asarray(ends, dtype=np.int32).reshape(-1, 2))
  e = len(ends)
  T = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(e, 16))
  info = np.ascontiguousarray(np.asarray(info, dtype=np.float64).reshape(e, 36))
  unc = np.ascontiguousarray(np.asarray(uncertain, dtype=np.int32).reshape(e))
  conf = np.ascontiguousarray(np.asarray(confidence, dtype=np.float64).reshape(e))
  dev = require_device(device)
  ws = workspace('pose_graph', torch.int64, dev, 'dgr_pose_graph_ws_elems', n, e)
  out = np.zeros((max(n, 1), 16))
  kept = np.zeros(max(e, 1), dtype=np.int32)
  lp = np.zeros(max(e, 1))
  st = np.zeros(16)
  call('dgr_pose_graph_optimize', ptr(poses), n, ptr(ends), ptr(T), ptr(info), ptr(unc), ptr(conf), e,
       float(max_correspondence_distance), float(edge_prune_threshold), float(preference_loop_closure),
       int(reference_node), int(max_iteration), float(min_relative_increment), float(min_relative_residual_increment),
       float(min_right_term), float(min_residual), int(max_iteration_lm), float(upper_scale_factor),
       float(lower_scale_factor), ptr(ws), ptr(out), ptr(kept), ptr(lp), ptr(st), refresh_stream())
  stats = {k: float(st[i]) for i, k in enumerate(POSE_GRAPH_STATS)}
  for k in ('iterations', 'iterations_pruned', 'pruned', 'status', 'factorisations'):
    stats[k] = int(stats[k])
  return out[:n].reshape(n, 4, 4), kept[:e].astype(bool), lp[:e], stats


def ransac_correspondence(x, y, idx0, idx1, max_dist, num_hyp=4000000, seed=0):
  """Safeguard RANSAC over the correspondences (x[idx0[i]], y[idx1[i]]) (an index of None means
  arange).  x / y: CUDA float32 [n, 3]; idx: int32.  -> device double [20] (pose 16, fitness,
  inlier RMSE, winning hypothesis, its inlier count)."""
  _chk(x, torch.float32, 'x'); _chk(y, torch.float32, 'y')
  dev = x.device
  if idx0 is not None: _chk(idx0, torch.int32, 'idx0')
  if idx1 is not None: _chk(idx1, torch.int32, 'idx1')
  n = len(idx0) if idx0 is not None else (len(idx1) if idx1 is not None else x.shape[0])
  if idx0 is not None and idx1 is not None and len(idx0) != len(idx1):
    raise DgrError('idx0 and idx1 differ in length')
  ws = workspace('ransac', torch.int64, dev, 'dgr_ransac_ws_elems', n, int(num_hyp))
  res = torch.empty(20, dtype=torch.float64, device=dev)
  call('dgr_ransac_correspondence', ptr(x), ptr(y), ptr(idx0) if idx0 is not None else None,
       ptr(idx1) if idx1 is not None else None, n, float(max_dist), int(num_hyp), int(seed) & (2**64 - 1),
       ptr(ws), ptr(res), stream())
  return res


def ransac_feature_matching(src, tgt, nn, spec, table, cell, max_dist, edge_ratio=0.0, check_dist=0.0,
                            max_iteration=80000, max_validation=1000, seed=0, batch=0):
  """Feature-matching RANSAC (open3d 0.10 registration_ransac_based_on_feature_matching): hypotheses of 4
  source points src[i] paired with tgt[nn[i]], scored on all of src through tgt's voxel hash (spec / table of
  a dgr_unique_first table at `cell`, one point per cell, rows = rows of tgt, batch column `batch`).
  edge_ratio 0 / check_dist <= 0 turn the edge-length / distance checkers off.  src / tgt: CUDA float32
  [n, 3]; nn: int32 [len(src)].  -> device double [24] (pose 16, fitness, inlier RMSE, winning hypothesis,
  matched points, validated hypotheses scored, hypotheses drawn until the max_validation-th validation)."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt'); _chk(nn, torch.int32, 'nn')
  if nn.numel() != src.shape[0]:
    raise DgrError('nn must hold one target row per source point')
  dev = src.device
  ws = workspace('ransac_fm', torch.int64, dev, 'dgr_ransac_fm_ws_elems', src.shape[0], int(max_iteration),
                 int(max_validation))
  res = torch.empty(24, dtype=torch.float64, device=dev)
  call('dgr_ransac_feature_matching', ptr(src), src.shape[0], ptr(tgt), ptr(nn), ptr(spec), ptr(table.keys),
       ptr(table.vals), table.cap, int(batch), float(cell), float(max_dist), float(edge_ratio), float(check_dist),
       int(max_iteration), int(max_validation), int(seed) & (2**64 - 1), ptr(ws), ptr(res), stream())
  return res


def fgr_feature_matching(src, tgt, nn_st, nn_ts, division_factor=1.4, use_absolute_scale=False, decrease_mu=True,
                         maximum_correspondence_distance=0.025, iteration_number=64, tuple_scale=0.95,
                         maximum_tuple_count=1000, tuple_test=True, seed=0, return_correspondences=False):
  """Fast Global Registration over feature matches (open3d registration_fast_based_on_feature_matching):
  nn_st[i] = nearest target feature of source point i, nn_ts[j] = nearest source feature of target point j
  (knn_top1 both ways).  src / tgt: CUDA float32 [n, 3]; nn: int32.  -> device double [24] (pose 16 mapping src
  into tgt, mutual pairs, correspondences used, tuple trials drawn, final mu, optimiser ran, clouds swapped);
  with return_correspondences also the int32 [n_max, 2] (source, target) buffer whose first res[17] rows are
  the correspondences the optimiser used."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  _chk(nn_st, torch.int32, 'nn_st'); _chk(nn_ts, torch.int32, 'nn_ts')
  n_s, n_t = src.shape[0], tgt.shape[0]
  if nn_st.numel() != n_s or nn_ts.numel() != n_t:
    raise DgrError('nn_st / nn_ts must hold one row per source / target point')
  dev = src.device
  ws = workspace('fgr', torch.int64, dev, 'dgr_fgr_ws_elems', n_s, n_t, int(maximum_tuple_count),
                 int(bool(tuple_test)))
  res = torch.empty(24, dtype=torch.float64, device=dev)
  corres = None
  if return_correspondences:
    n_min = min(n_s, n_t)
    n_max = 3 * min(int(maximum_tuple_count), 100 * n_min) if tuple_test else n_min
    corres = torch.full((max(n_max, 1), 2), -1, dtype=torch.int32, device=dev)
  call('dgr_fgr_feature_matching', ptr(src), n_s, ptr(tgt), n_t, ptr(nn_st), ptr(nn_ts), float(division_factor),
       int(bool(use_absolute_scale)), int(bool(decrease_mu)), float(maximum_correspondence_distance),
       int(iteration_number), float(tuple_scale), int(maximum_tuple_count), int(bool(tuple_test)),
       int(seed) & (2**64 - 1), ptr(ws), ptr(corres), ptr(res), stream())
  return (res, corres) if return_correspondences else res


GOICP_RESULT = ('E', 'lb_min', 'eps', 'K', 'converged', 'rounds', 'children', 'translation_cubes', 'icp_runs',
                'inner_overflows', 'pool_high_water', 'scale', 'host_reads')


def goicp_distance_transform(tgt, dt_size=300, dt_expand=2.0, src=None):
  """Go-ICP's distance transform of tgt (CUDA float32 [n, 3]) normalised together with src (at most 1024 points;
  default: the first 1024 target points).
  -> (int32 [G, G, G] indexed [z, y, x]: squared distance in cells to the nearest occupied cell, s)."""
  src = tgt[:1024] if src is None else src
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  G, dev = int(dt_size), tgt.device
  stat = torch.empty(8, dtype=torch.float64, device=dev)
  y = torch.empty(max(tgt.shape[0], 1), 3, dtype=torch.float32, device=dev)
  dt = torch.empty(max(G, 1) ** 3, dtype=torch.int32, device=dev)
  call('dgr_goicp_dt_build', ptr(src), src.shape[0], ptr(tgt), tgt.shape[0], G, float(dt_expand), ptr(stat), ptr(y),
       ptr(dt), stream())
  st = stat.cpu().numpy()
  s = max(st[3], st[7])
  return dt.reshape(G, G, G), float(s if s > 0 else 1.0)


def goicp(src, tgt, mse_thresh=1e-3, trim_fraction=0.0, dt_size=300, dt_expand=2.0, rot_min=(-math.pi,) * 3,
          rot_width=2 * math.pi, trans_min=(-1.0, -1.0, -1.0), trans_width=2.0, cubes_per_round=64, max_rounds=100000,
          max_rotation_cubes=1 << 20):
  """Go-ICP of src (CUDA float32 [n_s <= 1024, 3]) onto tgt (CUDA float32 [n_t, 3]); domains in the normalised frame
  (both clouds centred, divided by one scale s).  -> device double [32]: 4x4 pose mapping src into tgt, then the
  fields of GOICP_RESULT."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  ws = workspace('goicp', torch.int64, src.device, 'dgr_goicp_ws_elems', src.shape[0], tgt.shape[0], int(dt_size),
                 int(max_rotation_cubes), int(cubes_per_round))
  res = torch.empty(32, dtype=torch.float64, device=src.device)
  rmin, tmin = (C.c_double * 3)(*map(float, rot_min)), (C.c_double * 3)(*map(float, trans_min))
  call('dgr_goicp', ptr(src), src.shape[0], ptr(tgt), tgt.shape[0], float(mse_thresh), float(trim_fraction),
       int(dt_size), float(dt_expand), rmin, float(rot_width), tmin, float(trans_width), int(cubes_per_round),
       int(max_rounds), int(max_rotation_cubes), ptr(ws), ptr(res), stream())
  return res


SUPER4PCS_RESULT = ('lcp_fraction', 'lcp', 'bases', 'valid_bases', 'candidates', 'pairs_dropped',
                    'candidates_dropped', 'best_base', 'best_candidate', 'rounds', 'scale', 'host_reads')
SUPER4PCS_LOG = ('b1', 'b2', 'b3', 'b4', 'valid', 's1', 's2', 'candidates', 'candidates_dropped', 'verified',
                 'best_lcp', 'best_candidate')


def super4pcs(src, tgt, n_sample_tgt=1024, overlap=0.5, delta=0.1, angle_tol=0.0, dt_size=300, dt_expand=2.0,
              max_bases=256, bases_per_round=64, max_pairs=262144, max_candidates=65536, verify_per_base=64,
              terminate_fraction=0.9, seed=0, return_log=False):
  """Super4PCS of src (CUDA float32 [n_s in 4..1024, 3]) onto tgt (CUDA float32 [n_t, 3]); delta in the clouds' units,
  angle_tol in radians (0: 2 delta / min(d1, d2) per base).  -> device double [32]: 4x4 pose mapping src into tgt,
  then the fields of SUPER4PCS_RESULT; with return_log, also the int32 [max_bases, 16] base log (fields
  SUPER4PCS_LOG, then zeros; -1 rows for bases not run)."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  ws = workspace('super4pcs', torch.int64, src.device, 'dgr_super4pcs_ws_elems', src.shape[0], tgt.shape[0],
                 int(n_sample_tgt), int(dt_size), int(bases_per_round), int(max_pairs), int(max_candidates),
                 int(verify_per_base))
  res = torch.empty(32, dtype=torch.float64, device=src.device)
  log = torch.empty(max(int(max_bases), 1), 16, dtype=torch.int32, device=src.device) if return_log else None
  call('dgr_super4pcs', ptr(src), src.shape[0], ptr(tgt), tgt.shape[0], int(n_sample_tgt), float(overlap),
       float(delta), float(angle_tol), int(dt_size), float(dt_expand), int(max_bases), int(bases_per_round),
       int(max_pairs), int(max_candidates), int(verify_per_base), float(terminate_fraction),
       int(seed) & (2**64 - 1), ptr(ws), ptr(log) if return_log else None, ptr(res), stream())
  return (res, log) if return_log else res


POINTNET_PARAMS = _DEFINES['DGR_POINTNET_PARAMS']
POINTNET_PACKED_BYTES = _DEFINES['DGR_POINTNET_PACKED_BYTES']
POINTNETLK_RESULT = ('iterations', 'last_dx', 'last_r', 'status', 'n_src', 'n_tgt', 'host_reads')
POINTNETLK_LOG = ('g00', 'g01', 'g02', 'g03', 'g10', 'g11', 'g12', 'g13', 'g20', 'g21', 'g22', 'g23', 'dx_norm',
                  'r_norm')


def pointnet_pack(params):
  """PointNetLK feature network parameters (CUDA float64 [POINTNET_PARAMS], core/pointnetlk.load_pointnet_weights'
  order) -> the packed device image (uint8 [POINTNET_PACKED_BYTES]): BatchNorm folded, TF32 hi / lo tiles."""
  _chk(params, torch.float64, 'params')
  if params.numel() != POINTNET_PARAMS:
    raise DgrError(f'params: expected {POINTNET_PARAMS} values, got {params.numel()}')
  packed = torch.empty(POINTNET_PACKED_BYTES, dtype=torch.uint8, device=params.device)
  call('dgr_pointnet_pack', ptr(params), ptr(packed), stream())
  return packed


def _chk_packed(packed, device):
  """packed must be pointnet_pack's image: uint8 [POINTNET_PACKED_BYTES] on `device`, 16-byte aligned (bulk copies)."""
  _chk(packed, torch.uint8, 'packed')
  if packed.numel() != POINTNET_PACKED_BYTES or packed.device != device or packed.data_ptr() % 16:
    raise DgrError(f'packed: expected pointnet_pack\'s {POINTNET_PACKED_BYTES} bytes on {device}, 16-byte aligned; got '
                   f'{packed.numel()} bytes on {packed.device} at offset {packed.data_ptr() % 16}')


def pointnet_forward(points, poses, packed, centre=None):
  """Max-pooled PointNet features of points (CUDA float32 [n, 3]) under each pose (CUDA float64 [B, 3, 4] or
  [B, 4, 4]) about centre (CUDA float64 [3]; None: the origin) -> CUDA float32 [B, 1024]."""
  _chk(points, torch.float32, 'points')
  if points.dim() != 2 or points.shape[1] != 3:
    raise DgrError(f'points: expected [n, 3], got {tuple(points.shape)}')
  if poses.dim() != 3 or tuple(poses.shape[1:]) not in ((3, 4), (4, 4)):
    raise DgrError(f'poses: expected [B, 3, 4] or [B, 4, 4], got {tuple(poses.shape)}')
  poses = poses[:, :3, :].contiguous()
  _chk(poses, torch.float64, 'poses')
  if centre is not None:
    _chk(centre, torch.float64, 'centre')
    if centre.numel() != 3:
      raise DgrError(f'centre: expected 3 values, got {centre.numel()}')
  _chk_packed(packed, points.device)
  out = torch.empty(poses.shape[0], 1024, dtype=torch.float32, device=points.device)
  call('dgr_pointnet_forward', ptr(points), points.shape[0], ptr(centre), ptr(poses), poses.shape[0], ptr(packed),
       ptr(out), stream())
  return out


def pointnetlk(src, tgt, packed, delta=1e-2, max_iter=10, xtol=1e-7, return_jacobian=False, return_log=False):
  """PointNetLK of src onto tgt (CUDA float32 [n, 3] each) with the packed network of pointnet_pack.
  -> device double [32]: 4x4 pose mapping src into tgt, then the fields of POINTNETLK_RESULT; with return_jacobian,
  also J (double [1024, 6]); with return_log, also the double [max_iter, 16] iteration log (POINTNETLK_LOG, then
  zeros; NaN rows for iterations not run)."""
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  for name, t in (('src', src), ('tgt', tgt)):
    if t.dim() != 2 or t.shape[1] != 3:
      raise DgrError(f'{name}: expected [n, 3], got {tuple(t.shape)}')
  _chk_packed(packed, src.device)
  ws = workspace('pointnetlk', torch.int64, src.device, 'dgr_pointnetlk_ws_elems', src.shape[0], tgt.shape[0],
                 int(max_iter))
  res = torch.empty(32, dtype=torch.float64, device=src.device)
  jac = torch.empty(1024, 6, dtype=torch.float64, device=src.device) if return_jacobian else None
  log = torch.full((max(int(max_iter), 1), 16), float('nan'), dtype=torch.float64, device=src.device) \
      if return_log else None
  call('dgr_pointnetlk', ptr(src), src.shape[0], ptr(tgt), tgt.shape[0], ptr(packed), float(delta), int(max_iter),
       float(xtol), ptr(ws), ptr(jac), ptr(log), ptr(res), stream())
  out = (res,) + ((jac,) if return_jacobian else ()) + ((log,) if return_log else ())
  return out if len(out) > 1 else res


# --------------------------------------------------------------------------- #
# RGB-D fusion (csrc/tsdf.cu): the device half of o3d_integration.ScalableTSDFVolume
# --------------------------------------------------------------------------- #
TSDF_RES = _DEFINES['DGR_TSDF_RES']
TSDF_RAYCAST_MAX_STEPS = _DEFINES['DGR_TSDF_RAYCAST_MAX_STEPS']


def _host_f64(a, n, name):
  a = np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1))
  if a.size != n:
    raise DgrError(f'{name}: expected {n} values, got {a.size}')
  return a


def tsdf_touch_ws(width, height, stride, voxel_length, sdf_trunc):
  """-> (candidate units per frame, workspace words) of dgr_tsdf_touch."""
  n_cand, words = C.c_int64(0), C.c_int64(0)
  call('dgr_tsdf_touch_ws_elems', int(width), int(height), int(stride), float(voxel_length), float(sdf_trunc),
       C.byref(n_cand), C.byref(words))
  return n_cand.value, words.value


def tsdf_touch(depth, intr, pose, voxel_length, sdf_trunc, stride, keys, vals, unit_keys, n_total, touched, counts,
               ws):
  """Units touched by the CUDA float32 depth [H, W] from camera_pose `pose` (4x4 host); new ones are appended to the
  volume (table keys / vals, unit_keys [cap, 3]).  touched / counts (int32 [3]) are written; no host read."""
  _chk(depth, torch.float32, 'depth')
  intr = _host_f64(intr, 4, 'intr')
  pose = _host_f64(np.asarray(pose, dtype=np.float64).reshape(4, 4)[:3], 12, 'pose')
  call('dgr_tsdf_touch', ptr(depth), depth.shape[1], depth.shape[0], ptr(intr), ptr(pose), float(voxel_length),
       float(sdf_trunc), TSDF_RES, int(stride), ptr(keys), ptr(vals), keys.numel(), ptr(unit_keys), unit_keys.shape[0],
       int(n_total), ptr(touched), ptr(counts), ptr(ws), stream())


def tsdf_rehash(unit_keys, n_total, keys, vals):
  call('dgr_tsdf_rehash', ptr(unit_keys), int(n_total), ptr(keys), ptr(vals), keys.numel(), stream())


def tsdf_integrate(depth, color, intr, extrinsic, voxel_length, sdf_trunc, unit_keys, touched, n_touched, tsdf,
                   weight, rgb):
  """Integrate one frame (depth CUDA float32 [H, W], color CUDA uint8 [H, W, 3] or None) into the touched units."""
  _chk(depth, torch.float32, 'depth')
  if color is not None:
    _chk(color, torch.uint8, 'color')
    if tuple(color.shape) != (depth.shape[0], depth.shape[1], 3):
      raise DgrError(f'color: expected {(depth.shape[0], depth.shape[1], 3)}, got {tuple(color.shape)}')
  intr = _host_f64(intr, 4, 'intr')
  ext = _host_f64(np.asarray(extrinsic, dtype=np.float64).reshape(4, 4)[:3], 12, 'extrinsic')
  call('dgr_tsdf_integrate', ptr(depth), ptr(color), depth.shape[1], depth.shape[0], ptr(intr), ptr(ext),
       float(voxel_length), float(sdf_trunc), TSDF_RES, ptr(unit_keys), ptr(touched), int(n_touched), ptr(tsdf),
       ptr(weight), ptr(rgb), tsdf.shape[0], stream())


def tsdf_extract(unit_keys, n_units, keys, vals, tsdf, weight, rgb, voxel_length):
  """Marching cubes over the first n_units slots (one host read).  -> (vertices [nv, 3] f64, colours [nv, 3] f64 or
  None, triangles [nt, 3] int32), CUDA tensors in canonical order."""
  dev = tsdf.device
  words = C.c_int64(0)
  call('dgr_tsdf_extract_ws_elems', int(n_units), C.byref(words))
  ws = torch.empty(max(words.value, 1), dtype=torch.int64, device=dev)
  totals = torch.empty(2, dtype=torch.int32, device=dev)
  call('dgr_tsdf_extract_count', ptr(unit_keys), int(n_units), ptr(keys), ptr(vals), keys.numel(), ptr(tsdf),
       ptr(weight), TSDF_RES, ptr(ws), ptr(totals), stream())
  nv, nt = (int(v) for v in totals.cpu())
  verts = torch.empty(nv, 3, dtype=torch.float64, device=dev)
  cols = torch.empty(nv, 3, dtype=torch.float64, device=dev) if rgb is not None else None
  tris = torch.empty(nt, 3, dtype=torch.int32, device=dev)
  call('dgr_tsdf_extract_write', ptr(unit_keys), int(n_units), ptr(tsdf), ptr(rgb), float(voxel_length), ptr(ws),
       ptr(verts), ptr(cols), ptr(tris), stream())
  return verts, cols, tris


def tsdf_raycast(keys, vals, tsdf, weight, rgb, width, height, intr, pose, voxel_length, sdf_trunc, depth_min,
                 depth_max, weight_threshold, depth, intensity=None, colour=None):
  """Render one camera from the volume (dgr_tsdf_raycast, one launch, no host read): pose is camera_pose = inv(extrinsic)
  (4x4 host); keys / vals None for an empty volume.  Writes the CUDA float32 outputs depth [H, W] and, for an RGB8
  volume (rgb not None), intensity [H, W] and colour [H, W, 3] when given."""
  for name, t, shape in (('depth', depth, (height, width)), ('intensity', intensity, (height, width)),
                         ('colour', colour, (height, width, 3))):
    if t is not None:
      _chk(t, torch.float32, name)
      if tuple(t.shape) != shape:
        raise DgrError(f'{name}: expected {shape}, got {tuple(t.shape)}')
  intr = _host_f64(intr, 4, 'intr')
  pose = _host_f64(np.asarray(pose, dtype=np.float64).reshape(4, 4)[:3], 12, 'pose')
  call('dgr_tsdf_raycast', ptr(keys), ptr(vals), 0 if keys is None else keys.numel(), ptr(tsdf), ptr(weight),
       ptr(rgb), int(width), int(height), ptr(intr), ptr(pose), float(voxel_length), float(sdf_trunc), TSDF_RES,
       float(depth_min), float(depth_max), float(weight_threshold), ptr(depth), ptr(intensity), ptr(colour), stream())


def tsdf_mc_tables():
  """-> (edge_table [256], tri_table [256, 16]) int32 numpy: the library's marching-cubes tables."""
  edge = np.zeros(256, np.int32)
  tri = np.zeros((256, 16), np.int32)
  call('dgr_tsdf_mc_tables', ptr(edge), ptr(tri))
  return edge, tri


ODOMETRY_MAX_LEVELS = _DEFINES['DGR_ODOMETRY_MAX_LEVELS']
ODOMETRY_MAX_ITERATIONS = _DEFINES['DGR_ODOMETRY_MAX_ITERATIONS']
ODOMETRY_RESULT = _DEFINES['DGR_ODOMETRY_RESULT']
ODOMETRY_RESULT_HEAD = _DEFINES['DGR_ODOMETRY_RESULT_HEAD']
ODOMETRY_JACOBIANS = {'hybrid': _DEFINES['DGR_ODOMETRY_JACOBIAN_HYBRID'], 'color': _DEFINES['DGR_ODOMETRY_JACOBIAN_COLOR']}


def rgbd_odometry_ws_layout(width, height, levels):
  """Word offsets of the images dgr_rgbd_odometry leaves in its workspace (dgr_b200.h)."""
  off = np.zeros(8 * int(levels) + 3, dtype=np.int64)
  call('dgr_rgbd_odometry_ws_layout', int(width), int(height), int(levels), ptr(off))
  return off


def rgbd_odometry(src_intensity, src_depth, tgt_intensity, tgt_depth, intrinsic, odo_init, jacobian='hybrid',
                  iterations=(20, 10, 5), max_depth_diff=0.03, min_depth=0.0, max_depth=4.0, ws=None, result=None):
  """open3d's legacy compute_rgbd_odometry (dgr_rgbd_odometry), enqueued without a host read.  Images: CUDA float32
  [H, W] intensity and metric depth of both frames; intrinsic: (fx, fy, cx, cy); odo_init: 4x4 mapping the source
  camera into the target camera; iterations: per level, coarsest first.  ws: a uint64 workspace of
  dgr_rgbd_odometry_ws_elems words (an arena buffer by default); result: a CUDA float64 [ODOMETRY_RESULT] to write.
  -> result (pose 16, success, steps, info 36, its count, per-step counts)."""
  H, W = src_depth.shape if src_depth.dim() == 2 else (0, 0)
  for name, a in (('src_intensity', src_intensity), ('src_depth', src_depth), ('tgt_intensity', tgt_intensity),
                  ('tgt_depth', tgt_depth)):
    _chk(a, torch.float32, name)
    if a.shape != (H, W):
      raise DgrError(f'{name} must be [H, W] = [{H}, {W}], got {tuple(a.shape)}')
  if jacobian not in ODOMETRY_JACOBIANS:
    raise DgrError(f'jacobian must be one of {sorted(ODOMETRY_JACOBIANS)}, got {jacobian!r}')
  dev = src_depth.device
  intr = np.ascontiguousarray(np.asarray(intrinsic, dtype=np.float64).reshape(4))
  init = np.ascontiguousarray(np.asarray(odo_init, dtype=np.float64).reshape(4, 4))
  its = np.ascontiguousarray(np.asarray(iterations, dtype=np.int32).reshape(-1))
  L = len(its)
  if ws is None:
    n = C.c_int64(0)
    call('dgr_rgbd_odometry_ws_elems', int(W), int(H), L, C.byref(n))
    ws = scratch('rgbd_odometry', n.value, torch.int64, dev)
  if result is None:
    result = torch.empty(ODOMETRY_RESULT, dtype=torch.float64, device=dev)
  call('dgr_rgbd_odometry', ptr(src_intensity), ptr(src_depth), ptr(tgt_intensity), ptr(tgt_depth), int(W), int(H),
       ptr(intr), ptr(init), ODOMETRY_JACOBIANS[jacobian], ptr(its), L, float(max_depth_diff), float(min_depth),
       float(max_depth), ptr(ws), ptr(result), stream())
  return result
