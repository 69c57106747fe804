"""ctypes binding of libdgr_b200.so (include/dgr_b200.h).

torch is used here for device memory and the current CUDA stream only; every
computation happens inside the library.  There is no CPU fallback: importing this
module without a built library, or calling into it without an sm_90 device,
raises.
"""
import ctypes as C
import math
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdgr_b200.so')

MAX_COLS = 8
TILE_ROWS = 128


class KeySpec(C.Structure):
  _fields_ = [('ncols', C.c_int32), ('overflow', C.c_int32), ('lo', C.c_int32 * MAX_COLS),
              ('shift', C.c_int32 * MAX_COLS), ('bits', C.c_int32 * MAX_COLS)]


KEYSPEC_INTS = C.sizeof(KeySpec) // 4

_p, _i32, _i64, _f32, _f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double

# name -> argtypes; every function returns int32 status unless listed in _RESTYPES
SIGNATURES = {
    'dgr_version': [],
    'dgr_last_error': [],
    'dgr_launch_count': [],
    'dgr_device_check': [_i32],
    'dgr_quantize_points': [_p, _i32, _i64, _f64, _i32, _p, _p, _p],
    'dgr_coords_minmax': [_p, _i64, _i32, _p, _p],
    'dgr_keyspec_build': [_p, _i32, _i32, _p, _p],
    'dgr_hash_clear': [_p, _p, _i64, _p],
    'dgr_unique_first': [_p, _i64, _i32, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _p],
    'dgr_scan_ws_elems': [_i64],
    'dgr_hash_find': [_p, _i64, _i32, _p, _p, _p, _i64, _p, _p],
    'dgr_gather_rows_i32': [_p, _p, _i64, _i32, _p, _p],
    'dgr_spconv_fwd': [_p, _i32, _p, _i32, _p, _p, _p, _p, _p, _i32, _i32, _i32, _p, _p],
    'dgr_spconv_tc_supported': [_i32, _i32],
    'dgr_pack_weight_tf32': [_p, _i32, _i32, _i32, _p, _p],
    'dgr_spconv_tc_fwd': [_p, _i32, _p, _i32, _p, _p, _p, _p, _p, _i32, _i32, _i32, _p, _p],
    'dgr_linear_fwd': [_p, _i32, _p, _i32, _i64, _p, _i32, _p, _i32, _i32, _p, _p],
    'dgr_affine_act': [_p, _i64, _i32, _p, _p, _p, _i32, _p, _p],
    'dgr_cat2': [_p, _i32, _p, _i32, _i64, _p, _p],
    'dgr_l2_normalize': [_p, _i64, _i32, _p, _p],
    'dgr_knn_top1': [_p, _i64, _p, _i64, _i32, _p, _p, _p, _p],
    'dgr_knn_tc_supported': [_i32],
    'dgr_knn_tc_ws_elems': [_i64, _i64, _i32],
    'dgr_knn_top1_tc': [_p, _i64, _p, _i64, _i32, _p, _p, _p, _p, _p],
    'dgr_inlier_coords': [_p, _p, _p, _i64, _p, _p],
    'dgr_sigmoid_clip_sum': [_p, _i64, _f32, _p, _p, _p],
    'dgr_estimate_normals': [_p, _i64, _p, _p, _p, _i64, _i32, _f64, _f64, _i32, _p, _p, _p, _p],
    'dgr_icp_ws_elems': [_i64, _p],
    'dgr_icp': [_p, _i64, _p, _p, _p, _p, _p, _i64, _i32, _f64, _f64, _p, _i32, _f64, _f64, _p, _p, _p],
    'dgr_ransac_ws_elems': [_i64, _i64, _p],
    'dgr_ransac_correspondence': [_p, _p, _p, _p, _i64, _f64, _i64, C.c_uint64, _p, _p, _p],
    'dgr_ransac_fm_ws_elems': [_i64, _i64, _i64, _p],
    'dgr_ransac_feature_matching': [_p, _i64, _p, _p, _p, _p, _p, _i64, _i32, _f64, _f64, _f64, _f64, _i64, _i64,
                                    C.c_uint64, _p, _p, _p],
    'dgr_fgr_ws_elems': [_i64, _i64, _i64, _i32, _p],
    'dgr_fgr_feature_matching': [_p, _i64, _p, _i64, _p, _p, _f64, _i32, _i32, _f64, _i32, _f64, _i64, _i32, C.c_uint64,
                                 _p, _p, _p, _p],
    'dgr_goicp_dt_build': [_p, _i64, _p, _i64, _i32, _f64, _p, _p, _p, _p],
    'dgr_goicp_ws_elems': [_i64, _i64, _i32, _i64, _i32, _p],
    'dgr_goicp': [_p, _i64, _p, _i64, _f64, _f64, _i32, _f64, _p, _f64, _p, _f64, _i32, _i32, _i64, _p, _p, _p],
    'dgr_super4pcs_ws_elems': [_i64, _i64, _i64, _i32, _i32, _i64, _i64, _i32, _p],
    'dgr_super4pcs': [_p, _i64, _p, _i64, _i64, _f64, _f64, _f64, _i32, _f64, _i32, _i32, _i64, _i64, _i32, _f64,
                      C.c_uint64, _p, _p, _p, _p],
    'dgr_pointnet_pack': [_p, _p, _p],
    'dgr_pointnet_forward': [_p, _i64, _p, _p, _i32, _p, _p, _p],
    'dgr_pointnetlk_ws_elems': [_i64, _i64, _i32, _p],
    'dgr_pointnetlk': [_p, _i64, _p, _i64, _p, _f64, _i32, _f64, _p, _p, _p, _p, _p],
    'dgr_se3_register': [_p, _p, _p, _p, _i64, _f32, _i32, _i32, _f32, _f32, _f32, _p, _p, _p, _p],
    # ---- round 2: coordinate planning with device-side counts (csrc/coordplan.cu) ----
    'dgr_spconv_table_fwd_strided': [_p, _i32, _p, _i32, _p, _i32, _i64, _i64, _p, _p, _p, _p],
    'dgr_compact_voxel_pair': [_p, _p, _p, _i64, _i64, _p, _i32, _p, _i32, _p, _p, _p, _p],
    'dgr_table_build_unique': [_p, _i64, _p, _i32, _p, _p, _p, _i64, _p],
    'dgr_coarse_scan_elems': [_i64],
    'dgr_coarse_maps': [_p, _i64, _p, _i32, _p, _i32, _p, _p, _p, _i64, _p, _p, _p, _p, _p],
    'dgr_bloom2_build': [_p, _i64, _p, _i64, _p],
    'dgr_bloom2_words': [_i64],
    'dgr_kmap_mask_words': [_i64],
    'dgr_kmap_cnt_elems': [_i32, _i64],
    'dgr_kmap_probe': [_p, _i64, _p, _i32, _p, _p, _p, _i64, _p, _i64, _p, _i32, _p, _p, _p, _p, _p],
    'dgr_kmap_fill': [_p, _p, _i32, _i64, _p, _i32, _p, _p, _p, _i64, _p, _p, _p, _p],
    'dgr_kernel_map_tiles': [_p, _i32, _i32, _i32, _i32, _p, _p, _p],
    'dgr_kmap_dense': [_p, _i64, _p, _i32, _p, _p, _p, _i64, _p, _i64, _p, _i32, _p, _i64, _p, _p],
    'dgr_spconv_ones_bits_fwd': [_p, _i32, _p, _i64, _i32, _i64, _p, _p, _p, _p],
    'dgr_spconv_wgrad': [_p, _i32, _p, _i32, _p, _p, _p, _i32, _p, _p],
    'dgr_affine_act_amax': [_p, _i64, _i32, _p, _p, _p, _i32, _p, _p, _p],
    'dgr_absmax_f32': [_p, _i64, _p, _p],
    'dgr_spconv_tc_f16_supported': [_i32, _i32],
    'dgr_pack_weight_f16': [_p, _i32, _i32, _i32, _p, _p, _p],
    'dgr_spconv_tc_f16_fwd': [_p, _i32, _p, _i32, _p, _p, _p, _p, _p, _i32, _i32, _p, _p, _p, _p],
    # ---- round 2: native executor (csrc/exec.cu) ----
    'dgr_ctx_create': [_i32, _p, _p],
    'dgr_ctx_destroy': [_p],
    'dgr_ctx_stream': [_p],
    'dgr_ctx_stats': [_p, _p],
    'dgr_ctx_profile': [_p, _i32],
    'dgr_ctx_profile_read': [_p, _p, _i64],
    'dgr_ctx_stage_times': [_p, _p, _i32],
    'dgr_net_create': [_i32, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _i32, _p, _p],
    'dgr_net_destroy': [_p],
    'dgr_net_forward': [_p, _p, _p, _i64, _p, _p],
    'dgr_pair_register': [_p, _p, _p, _p, _i64, _i32, _p, _i64, _i32, _i32, _f64, _f32, _i32, _p],
    'dgr_pair_safeguard': [_p, _f64, _i64, C.c_uint64, _i32, _p],
    'dgr_pair_tap': [_p, _i32, _p, _p, _p],
}
_RESTYPES = {'dgr_coarse_scan_elems': _i64, 'dgr_kmap_mask_words': _i64, 'dgr_kmap_cnt_elems': _i64, 'dgr_ctx_stream': C.c_void_p,
             'dgr_ctx_profile_read': _i64, 'dgr_last_error': C.c_char_p, 'dgr_knn_tc_ws_elems': _i64, 'dgr_launch_count': _i64, 'dgr_spconv_tc_supported': _i32, 'dgr_scan_ws_elems': _i64, 'dgr_bloom2_words': _i64}

_lib = None


class DgrError(RuntimeError):
  pass


def lib():
  """Load the shared library (once).  Fails loudly when it has not been built."""
  global _lib
  if _lib is None:
    if not os.path.exists(LIB_PATH):
      raise DgrError(f'{LIB_PATH} is missing: run `python -m deepglobalregistration_b200.build` '
                     '(there is no CPU fallback)')
    l = C.CDLL(LIB_PATH)
    for name, args in SIGNATURES.items():
      fn = getattr(l, name)
      fn.argtypes = args
      fn.restype = _RESTYPES.get(name, _i32)
    _lib = l
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
  return 0 if t is None else t.data_ptr()


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


def keyspec_build(minmax, ncols, margin=32):
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
  rank = scratch('uf_rank', max(n, 1), torch.int32, dev)
  scan = scratch('uf_scan', lib().dgr_scan_ws_elems(n), torch.int32, dev)
  call('dgr_unique_first', ptr(coords), n, ncols, ptr(spec), ptr(table.keys), ptr(table.vals), table.cap,
       ptr(sel), ptr(inverse), ptr(cnt), ptr(slot), ptr(rank), ptr(scan), stream())
  return table, sel, inverse, cnt


def read_count(cnt):
  """Host read of unique_first's (count, overflow) pair; raises on key overflow."""
  global D2H_BYTES
  n, overflow = cnt.cpu().tolist()
  D2H_BYTES += 8
  if overflow:
    raise DgrError('coordinate extent does not fit a 63-bit packed key')
  return n


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
  scan = scratch('cm_scan', L * lib().dgr_coarse_scan_elems(nmx), torch.int32, dev)
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


def kernel_map(out_coords, spec, in_table, n_in, offsets, keep_table=False):
  """offsets: CUDA int32 [K, D] (scaled by the input tensor stride).  Occupancy bits + bucket offsets (and the
  dense neighbour table when kept), then ONE host read of the bucket offsets sizes the pair lists and the work
  list."""
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
  if K > 27:
    n_words = lib().dgr_bloom2_words(n_in)
    bloom = scratch('km_bloom', n_words, torch.int32, dev)
    call('dgr_bloom2_build', ptr(in_table.keys), in_table.cap, ptr(bloom), n_words, stream())
  table = (ptr(in_table.keys), ptr(in_table.vals), in_table.cap)
  call('dgr_kmap_probe', ptr(out_coords), n_out, None, ncols, ptr(spec), *table, ptr(bloom), n_words, ptr(offsets), K,
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


def _icp(src, tgt, tgt_normals, tgt_manager, voxel, max_dist, T_init, max_iter, rel_fitness, rel_rmse, batch):
  _chk(src, torch.float32, 'src'); _chk(tgt, torch.float32, 'tgt')
  if tgt_normals is not None:
    _chk(tgt_normals, torch.float32, 'tgt_normals')
    if tgt_normals.shape != tgt.shape:
      raise DgrError('tgt_normals must hold one normal per target point')
  dev = src.device
  spec, table = _hash_of(tgt_manager)
  if not (isinstance(T_init, torch.Tensor) and T_init.is_cuda and T_init.numel() == 12):
    T_init = torch.as_tensor(T_init, dtype=torch.float64).reshape(4, 4)[:3].contiguous().to(dev)
  words = C.c_int64(0)
  call('dgr_icp_ws_elems', src.shape[0], C.byref(words))
  ws = scratch('icp', words.value, torch.float64, dev)
  res = torch.empty(20, dtype=torch.float64, device=dev)
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
                       rel_rmse=1e-6, batch=0):
  """Point-to-plane ICP (open3d's TransformationEstimationPointToPlane, default criteria) of src onto tgt through
  tgt's voxel hash; arguments as icp_point_to_point plus tgt_normals (CUDA float32 [n_tgt, 3])."""
  return _icp(src, tgt, tgt_normals, tgt_manager, voxel, max_dist, T_init, max_iter, rel_fitness, rel_rmse, batch)


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
  words = C.c_int64(0)
  call('dgr_ransac_ws_elems', n, int(num_hyp), C.byref(words))
  ws = scratch('ransac', words.value, torch.int64, dev)
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
  words = C.c_int64(0)
  call('dgr_ransac_fm_ws_elems', src.shape[0], int(max_iteration), int(max_validation), C.byref(words))
  ws = scratch('ransac_fm', words.value, torch.int64, dev)
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
  words = C.c_int64(0)
  call('dgr_fgr_ws_elems', n_s, n_t, int(maximum_tuple_count), int(bool(tuple_test)), C.byref(words))
  ws = scratch('fgr', words.value, torch.int64, dev)
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
  args = (src.shape[0], tgt.shape[0], int(dt_size), int(max_rotation_cubes), int(cubes_per_round))
  words = C.c_int64(0)
  call('dgr_goicp_ws_elems', *args, C.byref(words))
  ws = scratch('goicp', words.value, torch.int64, src.device)
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
  words = C.c_int64(0)
  call('dgr_super4pcs_ws_elems', src.shape[0], tgt.shape[0], int(n_sample_tgt), int(dt_size), int(bases_per_round),
       int(max_pairs), int(max_candidates), int(verify_per_base), C.byref(words))
  ws = scratch('super4pcs', words.value, torch.int64, src.device)
  res = torch.empty(32, dtype=torch.float64, device=src.device)
  log = torch.empty(max(int(max_bases), 1), 16, dtype=torch.int32, device=src.device) if return_log else None
  call('dgr_super4pcs', ptr(src), src.shape[0], ptr(tgt), tgt.shape[0], int(n_sample_tgt), float(overlap),
       float(delta), float(angle_tol), int(dt_size), float(dt_expand), int(max_bases), int(bases_per_round),
       int(max_pairs), int(max_candidates), int(verify_per_base), float(terminate_fraction),
       int(seed) & (2**64 - 1), ptr(ws), ptr(log) if return_log else None, ptr(res), stream())
  return (res, log) if return_log else res


POINTNET_PARAMS = 154368              # DGR_POINTNET_PARAMS
POINTNET_PACKED_BYTES = 1185792       # DGR_POINTNET_PACKED_BYTES
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
  words = C.c_int64(0)
  call('dgr_pointnetlk_ws_elems', src.shape[0], tgt.shape[0], int(max_iter), C.byref(words))
  ws = scratch('pointnetlk', words.value, torch.int64, src.device)
  res = torch.empty(32, dtype=torch.float64, device=src.device)
  jac = torch.empty(1024, 6, dtype=torch.float64, device=src.device) if return_jacobian else None
  log = torch.full((max(int(max_iter), 1), 16), float('nan'), dtype=torch.float64, device=src.device) \
      if return_log else None
  call('dgr_pointnetlk', ptr(src), src.shape[0], ptr(tgt), tgt.shape[0], ptr(packed), float(delta), int(max_iter),
       float(xtol), ptr(ws), ptr(jac), ptr(log), ptr(res), stream())
  out = (res,) + ((jac,) if return_jacobian else ()) + ((log,) if return_log else ())
  return out if len(out) > 1 else res
