"""CPU-side checks: the C-ABI library builds, loads and exports every symbol declared in
include/dgr_b200.h (no compute calls without a GPU); the ME-shaped host API has the
surface the reference touches; product code fails loudly without CUDA."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def built():
  from deepglobalregistration_b200 import build
  return build.build()


def test_library_exports_and_binds_every_declared_symbol(built):
  header = open(os.path.join(ROOT, 'include', 'dgr_b200.h')).read()
  declared = set(re.findall(r'\b(dgr_[a-z0-9_]+)\s*\(', header))
  declared -= {'dgr_keyspec_t'}
  assert len(declared) >= 25
  lib = ctypes.CDLL(built)
  missing = [s for s in sorted(declared) if not hasattr(lib, s)]
  assert not missing, missing
  from deepglobalregistration_b200 import _abi
  bound = _abi.bind(built)
  assert {s for s in declared if getattr(bound, s).argtypes is not None} == declared
  assert set(_abi.DECLARATIONS) == declared, set(_abi.DECLARATIONS) ^ declared
  assert _abi.lib().dgr_version() == 100
  assert ctypes.sizeof(_abi.KeySpec) == 4 * (2 + 3 * 8)


def test_header_binding_types(tmp_path):
  """The argtypes / restypes and constants read from include/dgr_b200.h, pinned for a few declarations; a C type
  without a fixed-width ctypes equivalent is rejected, not guessed."""
  from deepglobalregistration_b200 import _abi
  p, i32, i64, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64
  f32, f64 = ctypes.c_float, ctypes.c_double
  D = _abi.DECLARATIONS
  assert D['dgr_pose_graph_optimize'] == (i32, [p, i64, p, p, p, p, p, i64, f64, f64, f64, i32, i32, f64, f64, f64,
                                                f64, i32, f64, f64, p, p, p, p, p, p])
  assert D['dgr_ransac_correspondence'] == (i32, [p, p, p, p, i64, f64, i64, u64, p, p, p])
  assert D['dgr_sigmoid_clip_sum'] == (i32, [p, i64, f32, p, p, p])
  assert D['dgr_version'] == (i32, [])
  assert D['dgr_last_error'] == (ctypes.c_char_p, [])
  assert D['dgr_ctx_stream'] == (p, [p])
  assert D['dgr_kmap_mask_words'] == (i64, [i64])
  assert _abi.POINTNET_PACKED_BYTES == 1185792 and _abi.POSE_GRAPH_MAX_EDGES == 32640
  assert _abi.read_header(_abi.HEADER)[1]['DGR_TSDF_COORD_MIN'] == -1048576
  bad = tmp_path / 'bad.h'
  bad.write_text('#include <stddef.h>\nint32_t dgr_bad(const float* x, size_t n, void* stream);\n')
  with pytest.raises(_abi.DgrError, match='dgr_bad.*size_t'):
    _abi.read_header(str(bad))


def test_sm90a_sass_present(built):
  out = os.popen(f'cuobjdump -lelf {built} 2>/dev/null').read()
  assert 'sm_90a' in out


def test_no_cpu_fallback():
  from deepglobalregistration_b200 import _abi
  with pytest.raises(_abi.DgrError):
    _abi.require_device('cpu')
  if not torch.cuda.is_available():
    from deepglobalregistration_b200 import me as ME
    with pytest.raises(Exception):
      ME.SparseTensor(torch.ones(2, 1), coordinates=torch.zeros(2, 4, dtype=torch.int32))


def test_product_never_imports_oracle():
  pkg = os.path.join(ROOT, 'deepglobalregistration_b200')
  for dp, _, files in os.walk(pkg):
    for f in files:
      if f.endswith('.py'):
        src = open(os.path.join(dp, f)).read()
        assert not re.search(r'^\s*(from|import)\s+oracle\b', src, re.M), os.path.join(dp, f)


def test_me_surface_and_state_dict_layout():
  from deepglobalregistration_b200 import shims, synthetic as syn
  ME = shims.install()
  import MinkowskiEngine
  import MinkowskiEngine.MinkowskiFunctional as MEF
  assert MinkowskiEngine is ME and callable(MEF.relu)
  for name in ('SparseTensor', 'MinkowskiNetwork', 'MinkowskiConvolution', 'MinkowskiConvolutionTranspose',
               'KernelGenerator', 'RegionType', 'MinkowskiBatchNorm', 'cat', 'MinkowskiSumPooling',
               'MinkowskiPoolingTranspose', 'MinkowskiInstanceNorm', 'MinkowskiReLU', 'MinkowskiELU'):
    assert hasattr(ME, name), name
  assert callable(ME.utils.sparse_quantize) and callable(ME.utils.batched_coordinates)
  conv = ME.MinkowskiConvolution(3, 8, kernel_size=3, stride=2, has_bias=True, dimension=3)   # 0.4 spelling
  assert conv.kernel.shape == (27, 3, 8) and conv.bias.shape == (1, 8)
  assert ME.MinkowskiConvolution(3, 8, kernel_size=1, dimension=6).kernel.shape == (3, 8)
  assert ME.MinkowskiConvolutionTranspose(4, 2, kernel_size=3, stride=2, dimension=6).kernel.shape == (729, 4, 2)
  bn = ME.MinkowskiBatchNorm(8, momentum=0.05)
  assert set(bn.state_dict()) == {'bn.weight', 'bn.bias', 'bn.running_mean', 'bn.running_var',
                                  'bn.num_batches_tracked'}
  with pytest.raises(NotImplementedError):
    ME.MinkowskiInstanceNorm(8)
  bc = ME.utils.batched_coordinates([torch.zeros(3, 3).int(), torch.ones(2, 3).int()])
  assert bc.shape == (5, 4) and bc[:, 0].tolist() == [0, 0, 0, 1, 1] and bc.dtype == torch.int32
  from deepglobalregistration_b200.model import load_model
  assert load_model('NoSuchNet') is None
  for D, cin, cout, k in ((3, 1, 32, 7), (6, 1, 1, 3)):
    m = load_model('ResUNetBN2C')(cin, cout, conv1_kernel_size=k, D=D)
    sd = syn.resunet_state_dict(0, cin, cout, k, D) if D == 3 else None
    if sd is not None:
      assert m.load_state_dict(sd).missing_keys == []
    n_par = sum(p.numel() for p in m.parameters())
    assert n_par == (8_760_384 if D == 3 else 235_926_689), n_par


def test_kernel_offsets_match_oracle():
  from deepglobalregistration_b200.me.coords import kernel_offsets
  from oracle import sparse_ops as so
  for k, D, s in ((3, 3, 1), (7, 3, 1), (5, 3, 2), (3, 6, 4)):
    assert np.array_equal(kernel_offsets(k, D, s, 'cpu').numpy(), so.kernel_offsets(k, D, s))


def test_native_layer_table_parameter_order():
  """native.network_parameters lists the 66 tensors dgr_net_create documents, in execution order, for this
  package's ResUNetBN2C (the reference's attribute names, model/resunet.py:442-596)."""
  from deepglobalregistration_b200 import native, synthetic as syn
  from deepglobalregistration_b200.model import load_model
  models = [load_model('ResUNetBN2C')(1, 32, bn_momentum=0.05, conv1_kernel_size=7, normalize_feature=True, D=3)]
  C, T = [None, 32, 64, 128, 256], [None, 64, 64, 64, 128]
  for m in models:
    m.load_state_dict(syn.resunet_state_dict(0, 1, 32, 7, 3))
    m.eval()
    ps = native.network_parameters(m)
    assert len(ps) == 66 and all(p.dtype == torch.float32 and p.is_contiguous() for p in ps)
    assert tuple(ps[0].shape) == (343, 1, 32) and tuple(ps[1].shape) == (32,) and tuple(ps[2].shape) == (32,)
    assert tuple(ps[3].shape) == (27, 32, 32)                       # block1.conv1
    assert tuple(ps[9].shape) == (27, C[1], C[2])                   # conv2 (stride 2)
    assert tuple(ps[36].shape) == (27, C[4], T[4])                  # conv4_tr
    assert tuple(ps[45].shape) == (27, C[3] + T[4], T[3])           # conv3_tr reads cat(decoder, skip)
    assert tuple(ps[63].shape) == (C[1] + T[2], T[1]) and tuple(ps[64].shape) == (T[1], 32) and tuple(ps[65].shape) == (32,)
    # folded BatchNorm: scale = weight / sqrt(var + eps)
    bn = m.norm1.bn
    assert torch.allclose(ps[1], bn.weight / torch.sqrt(bn.running_var + bn.eps))


# The argument check every voxel-hash search shares (dgr_check_hash_search), host-only: each call also breaks one
# argument checked after it (max_nn 0, max_iter -1, a non-finite pose, edge_ratio -1), so that no call launches.
HASH_SEARCHES = {'dgr_estimate_normals': (4, 'max_nn'), 'dgr_color_gradient': (4, 'max_nn'),
                 'dgr_compute_fpfh': (6, 'max_nn'), 'dgr_icp': (4, 'bad ICP parameters'),
                 'dgr_colored_icp': (4, 'bad ICP parameters'), 'dgr_information_matrix': (4, 'must be finite'),
                 'dgr_ransac_feature_matching': (4, 'edge_ratio')}
HASH_REFUSALS = ('capacity must be a power of two', 'must be positive', 'search radius above')


def hash_search_refusal(name, cap, cell, radius):
  """Which dgr_check_hash_search refusal entry point `name` gives for (cap, cell, radius); None when it passes."""
  from deepglobalregistration_b200 import _abi
  keep = [(ctypes.c_double * 16)(*[math.nan] * 16)]
  nz = ctypes.addressof(keep[0])                      # a host address where only null is checked
  args = {
      'dgr_estimate_normals': (None, 0, None, None, None, cap, 0, cell, radius, 0, None, None, None, None),
      'dgr_color_gradient': (None, None, None, 0, None, None, None, cap, 0, cell, radius, 0, None, None, None),
      'dgr_compute_fpfh': (None, nz, 0, None, None, None, cap, 0, cell, radius, 0, 33, None, None, None, None),
      'dgr_icp': (None, 0, None, None, nz, nz, nz, cap, 0, cell, radius, nz, -1, 1e-6, 1e-6, nz, nz, None),
      'dgr_colored_icp': (None, None, 0, nz, nz, nz, nz, nz, nz, nz, cap, 0, cell, radius, 0.968, nz, -1, 1e-6, 1e-6,
                          nz, nz, None),
      'dgr_information_matrix': (None, 0, None, nz, nz, nz, cap, 0, cell, radius, nz, nz, nz, None),
      'dgr_ransac_feature_matching': (nz, 1, nz, nz, nz, nz, nz, cap, 0, cell, radius, -1.0, 0.0, 1, 1, 0, nz, nz,
                                      None),
  }[name]
  assert getattr(_abi.lib(), name)(*args) == _abi._DEFINES['DGR_ERR_ARG']
  msg = _abi.lib().dgr_last_error().decode()
  hit = [m for m in HASH_REFUSALS if m in msg]
  assert hit or HASH_SEARCHES[name][1] in msg, msg
  return hit[0] if hit else None


def largest_radius(reach, cell):
  """The largest double radius with ceil(radius / cell) <= reach."""
  r = reach * cell
  while math.ceil(r / cell) > reach:
    r = float(np.nextafter(r, 0.0))
  while math.ceil(float(np.nextafter(r, math.inf)) / cell) <= reach:
    r = float(np.nextafter(r, math.inf))
  return r


@pytest.mark.parametrize('name', sorted(HASH_SEARCHES))
def test_hash_search_argument_boundaries(built, name):
  reach = HASH_SEARCHES[name][0]
  for cell in (0.0625, 0.05, 0.3, 0.07, 1e-3):
    r = largest_radius(reach, cell)
    assert hash_search_refusal(name, 1024, cell, r) is None, (cell, r)
    assert hash_search_refusal(name, 1024, cell, float(np.nextafter(r, math.inf))) == 'search radius above'
    assert hash_search_refusal(name, 1024, cell, 0.5 * cell) is None
  assert hash_search_refusal(name, 1024, 0.0625, reach * 0.0625) is None          # an exact ratio at the reach
  assert hash_search_refusal(name, 1024, 0.0625, (reach + 1) * 0.0625) == 'search radius above'
  for bad in (math.nan, math.inf, -math.inf, 0.0, -0.0, -0.05, 5e-324 * -1):
    assert hash_search_refusal(name, 1024, bad, 0.1) == 'must be positive', bad
    if bad != math.inf:
      assert hash_search_refusal(name, 1024, 0.05, bad) == 'must be positive', bad
  assert hash_search_refusal(name, 1024, 0.05, math.inf) == 'search radius above'
  for cap in (0, 3, 6, 1000, -8, 2 ** 62 + 2 ** 61):
    assert hash_search_refusal(name, cap, 0.05, 0.1) == 'capacity must be a power of two', cap
  for cap in (1, 2, 2 ** 20, 2 ** 62):
    assert hash_search_refusal(name, cap, 0.05, 0.1) is None, cap


def ordered(x32):
  """float32 bits as integers in value order (-0.0 and +0.0 both 0): differences count ulps."""
  b = np.asarray(x32, np.float32).view(np.int32).astype(np.int64)
  return np.where(b < 0, -(b & 0x7FFFFFFF), b)


def test_float32_in_cells_argument_checks(built):
  """dgr_float32_in_cells refuses a NaN, infinite, zero or negative cell and null pointers before any launch; an
  empty call is a no-op."""
  from deepglobalregistration_b200 import _abi
  lib = _abi.lib()
  keep = (ctypes.c_double * 16)()
  nz = ctypes.addressof(keep)                         # a host address where only null is checked
  launches = lib.dgr_launch_count()

  def refusal(xyz, n, cells, stride, cell, out):
    assert lib.dgr_float32_in_cells(xyz, 1, n, cells, stride, cell, out, None) == _abi._DEFINES['DGR_ERR_ARG']
    return lib.dgr_last_error().decode()

  for bad in (math.nan, math.inf, -math.inf, 0.0, -0.0, -0.05, -5e-324):
    assert 'cell must be positive and finite' in refusal(nz, 4, nz, 3, bad, nz), bad
  for xyz, cells, out in ((None, nz, nz), (nz, None, nz), (nz, nz, None)):
    assert 'null argument' in refusal(xyz, 4, cells, 3, 0.05, out)
  assert 'at least 3 ints' in refusal(nz, 4, nz, 2, 0.05, nz)
  assert 'row count' in refusal(nz, -1, nz, 3, 0.05, nz)
  assert lib.dgr_float32_in_cells(None, 1, 0, None, 3, 0.05, None, None) == 0
  assert lib.dgr_launch_count() == launches
  assert _abi.CELL_NUDGE_STEPS == 4
